/*
 * vibevoice_b200.h -- C ABI of libvibevoice_b200.so (hand-written sm_90a kernels + native runtime).
 *
 * The reference (vibevoice-community/VibeVoice) is 100% Python/PyTorch and has no FFI layer; its
 * boundary for this path is the Python surface of
 *   vibevoice/modular/modeling_vibevoice_inference.py:68   VibeVoiceForConditionalGenerationInference
 * This header is the boundary a drop-in replacement binds instead (via ctypes, see INTEGRATION.md):
 * every entry point below names the reference code it replaces (file:line in vibevoice-community/VibeVoice).
 *
 * Conventions
 *   - plain C: opaque handle, raw pointers, sizes; no torch / C++ types.
 *   - every compute call is asynchronous on the `stream` argument (a cudaStream_t passed as void*),
 *     never allocates, never synchronises the host; device pointers are owned by the caller unless
 *     stated otherwise.
 *   - return 0 on success, negative vv_status otherwise; vv_last_error() gives the message of the
 *     last failure on the calling thread.
 *   - row r of the LM batch: r in [0,B) = positive (conditional) stream of sample r,
 *     r in [B,2B) = negative (CFG-unconditional) stream of sample r-B
 *     (modeling_vibevoice_inference.py:379-386, 576-589).
 */
#ifndef VIBEVOICE_B200_H_
#define VIBEVOICE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VV_ABI_VERSION 1

typedef struct vv_ctx vv_ctx;

typedef enum {
  VV_OK = 0,
  VV_ERR_INVALID = -1,   /* bad argument / shape mismatch / unknown tensor name */
  VV_ERR_CUDA = -2,      /* CUDA runtime error (message has the cudaGetErrorString) */
  VV_ERR_STATE = -3,     /* call order violated (e.g. compute before vv_finalize_weights) */
  VV_ERR_NOMEM = -4      /* KV page pool exhausted / allocation failed */
} vv_status;

typedef enum { VV_DT_BF16 = 0, VV_DT_F32 = 1, VV_DT_F16 = 2 } vv_dtype;

/* Architecture numbers; mirrors vibevoice/modular/configuration_vibevoice.py:13-241 and
 * vibevoice/configs/qwen2.5_1.5b_64k.json.  Arrays follow the JSON order. */
typedef struct {
  /* decoder_config (Qwen2) */
  int32_t hidden_size, intermediate_size, num_layers, num_q_heads, num_kv_heads, head_dim, vocab_size;
  int32_t max_position_embeddings, tie_word_embeddings;
  float rms_norm_eps, rope_theta;
  /* diffusion_head_config */
  int32_t head_layers, head_ffn_dim, latent_size;
  float head_rms_eps;
  /* acoustic tokenizer decoder + semantic tokenizer encoder (7.5 Hz streaming codec) */
  int32_t n_stages;                 /* len(depths) == len(ratios)+1, <= 8 */
  int32_t dec_ratios[8];            /* decoder_ratios, e.g. 8,5,5,4,2,2 */
  int32_t dec_depths[8];            /* reversed encoder depths, e.g. 8,3,3,3,3,3,3 */
  int32_t dec_n_filters;
  int32_t enc_ratios[8];            /* semantic encoder_ratios as listed in the JSON (8,5,5,4,2,2) */
  int32_t enc_depths[8];            /* 3,3,3,3,3,3,8 */
  int32_t enc_n_filters;
  int32_t acoustic_vae_dim, semantic_vae_dim;
  float codec_eps;
  /* special token ids (modular_vibevoice_text_tokenizer.py:163-181); valid_ids are the only logits
   * that survive VibeVoiceTokenConstraintProcessor (modeling_vibevoice_inference.py:53-66, 405-419),
   * sorted ascending so ties resolve like a full-vocab argmax. */
  int32_t n_valid_ids;
  int32_t valid_ids[8];
  /* runtime sizing */
  int32_t max_batch;                /* B: samples resident on this GPU */
  int32_t max_diffusion_steps;      /* upper bound for vv_set_diffusion_steps */
} vv_model_desc;

/* ---- lifetime ------------------------------------------------------------------------------- */
int vv_abi_version(void);
const char* vv_last_error(void);
int vv_create(const vv_model_desc* desc, int device, vv_ctx** out);
void vv_destroy(vv_ctx* ctx);

/* ---- weights: same tensor names as the HF checkpoint (modeling_vibevoice.py:119-142) --------- *
 * `data` may be a host or device pointer (cudaMemcpyDefault).  Matrices are stored as bf16,
 * vectors (bias / norm / gamma) as fp32; layouts are repacked for the kernels in
 * vv_finalize_weights (qkv concat, gate/up interleave, conv -> window-GEMV form).
 * Unknown names return VV_ERR_INVALID; names not needed by this path (e.g. acoustic encoder) are
 * accepted and ignored (returns 1). */
int vv_load_tensor(vv_ctx* ctx, const char* name, const void* data, int dtype, const int64_t* shape, int ndim);
int vv_set_speech_factors(vv_ctx* ctx, float scaling_factor, float bias_factor); /* modeling_vibevoice.py:131-132 */
int vv_finalize_weights(vv_ctx* ctx);     /* fails with the list of missing tensors */
int64_t vv_weight_bytes(vv_ctx* ctx, int which); /* 0 lm, 1 head-per-step, 2 cond_proj, 3 decoder, 4 semantic, 5 connectors */

/* ---- paged KV cache (replaces HF DynamicCache, modeling_vibevoice_inference.py:303, 556-562) -- *
 * 2B sequences share one pool of pages (64 tokens each, all layers); pages return to the pool when vv_kv_set_len shrinks a sequence. */
int vv_kv_init(vv_ctx* ctx, int64_t n_pages);   /* calling it again re-sizes the pool: every sequence is dropped, LM graphs re-captured */
int vv_kv_reserve(vv_ctx* ctx, int seq, int64_t n_tokens, void* stream); /* make positions < n_tokens addressable */
int vv_kv_set_len(vv_ctx* ctx, int seq, int64_t len, void* stream);      /* e.g. 0 = negative-stream refresh (:549-565) */
int vv_kv_write(vv_ctx* ctx, int seq, int layer, int64_t pos0, int64_t n_tokens,
                const void* k_bf16, const void* v_bf16, void* stream);   /* prefill hand-off: [n_tokens, kv_heads, head_dim] */
int vv_kv_delete_slot(vv_ctx* ctx, int seq, int64_t pos, void* stream);  /* forget ONE older entry: the last entry moves into its place (order is
                                                                           * irrelevant to attention); refresh_negative=False bookkeeping, :599-624 */
int64_t vv_kv_pages_free(vv_ctx* ctx);
int64_t vv_kv_pages_total(vv_ctx* ctx);

/* ---- a-3: LLM decode step for pos+neg rows in ONE weight pass ---------------------------------- *
 * replaces self(**model_inputs) at :480-482 and the negative forward at :583-585.
 * embeds [2B,H] fp32 (row r<B positive, r>=B negative).  Every row with row_mode 1 (default: all)
 * runs and writes its K/V at position kv_len[r]; the length itself only moves in vv_kv_commit, so a
 * speculative negative-stream step that the host state machine rejects costs nothing to undo
 * (the reference shifts whole caches instead, :594-624).
 * Outputs: hidden [2B,H] fp32 (final norm applied), logits [B, n_valid_ids] fp32 for the positive
 * rows, tokens [B] int32 = constrained argmax (valid_ids[argmax]).                                */
int vv_set_rope_inv_freq(vv_ctx* ctx, const float* inv_freq_host, int n); /* Qwen2RotaryEmbedding.inv_freq, n = head_dim/2 */
int vv_set_row_mode(vv_ctx* ctx, const int32_t* row_mode_host, void* stream);  /* [2B] 0 = skip row */
int vv_lm_decode(vv_ctx* ctx, const float* embeds, float* hidden, float* logits, int32_t* tokens, void* stream);
int vv_lm_head(vv_ctx* ctx, const float* hidden /*[B,H] final-normed*/, float* logits, int32_t* tokens, void* stream);
/* full-vocabulary logits [B, vocab] fp32 of the positive rows (outputs.logits[:, -1, :] at :488); used only when the caller passes its own
 * LogitsProcessor objects or top-k / top-p warpers, which act on the whole vocabulary before the token constraint (:310-319, :490). */
int vv_lm_logits_full(vv_ctx* ctx, const float* hidden /*[B,H] final-normed*/, float* logits_out, void* stream);
/* Streaming-0.5B variant (modeling_vibevoice_streaming_inference.py:178-318): decoder layers [layer_begin, layer_end) only, for the
 * rows enabled by vv_set_row_mode; K/V appended speculatively at kv_len exactly as in vv_lm_decode.  hidden [2B,H] receives the
 * residual stream, passed through the model's final RMSNorm iff final_norm != 0 (the lower text stack has none, :143-146). */
int vv_lm_decode_range(vv_ctx* ctx, const float* embeds, int layer_begin, int layer_end, int final_norm, float* hidden, void* stream); /* :242 + :488-498 */
/* advance sequence lengths after the host state machine decided which rows keep their new entry
 * (negative stream advances only on diffusion tokens, :594-624).  advance[r] in {0,1}, r < 2B. */
int vv_kv_commit(vv_ctx* ctx, const int32_t* advance_host, void* stream);
int64_t vv_kv_len(vv_ctx* ctx, int seq);
int vv_embed_tokens(vv_ctx* ctx, const int32_t* tokens_host, int n, float* out /*[n,H] fp32*/, void* stream); /* :569 */

/* ---- a-4: CFG diffusion sampler (sample_speech_tokens :697-710 + dpm_solver.py) ---------------- */
/* set_ddpm_inference_steps (:146) + scheduler.set_timesteps: the host computes the DPM-Solver++ scalar
 * tables (vibevoice_b200/schedule.py mirrors dpm_solver.py:321-423) and hands them over:
 * timesteps[n] (as float), coef[n][6] = {a0, s0, ks, kx, rinv, order}.  The sample-independent
 * timestep embeddings t_embedder(t_i) are computed here once. */
int vv_set_diffusion_steps(vv_ctx* ctx, int n_steps, const float* timesteps, const float* coef, void* stream);
/* `algorithm_type='sde-dpmsolver++'` (the Gradio demo's scheduler, demo/gradio_demo.py:141-146; dpm_solver.py:680-686, 785-793):
 * coef7[n][7] = {a0, s0, ks, kx, rinv, order, kn}; the update adds kn * step_noise[step].  The reference draws that noise with
 * randn_tensor(model_output.shape) once per step on the model's device (dpm_solver.py:993-997); the caller provides the rows it
 * needs as step_noise [n_steps][B][64] fp32 (device, persistent) through vv_set_step_noise before vv_diffusion_sample/vv_frame_tail. */
int vv_set_diffusion_steps_sde(vv_ctx* ctx, int n_steps, const float* timesteps, const float* coef7, void* stream);
int vv_set_step_noise(vv_ctx* ctx, const float* step_noise);
/* cond [2B,H] fp32 = LM hidden (rows as above); noise [B,64] fp32 = rows [0:n] of the reference's CPU
 * draw scattered to their sample slots; active[B] int32 (device) marks rows in diffusion mode.
 * latent_out [B,64] fp32 (the *scaled* latent, i.e. what acoustic_connector consumes, :667). */
int vv_diffusion_sample(vv_ctx* ctx, const float* cond, const float* noise, const int32_t* active, float cfg_scale,
                        float* latent_out, void* stream);

/* ---- a-5/a-6/a-7/a-8: codec frame, semantic frame, connectors, streaming state ----------------- */
int vv_codec_decode_frame(vv_ctx* ctx, const float* latent, const int32_t* active, float* audio_out /*[B,3200]*/, void* stream);
int vv_semantic_encode_frame(vv_ctx* ctx, const float* audio /*[B,3200]*/, const int32_t* active, float* feat_out /*[B,128]*/, void* stream);
int vv_connect(vv_ctx* ctx, const float* latent /*[B,64]*/, const float* sem /*[B,128]*/, const int32_t* active,
               float* embeds_inout /*[2B,H]: rows r<B overwritten where active*/, void* stream);
int vv_codec_state_zero(vv_ctx* ctx, const int32_t* rows_host, int n, void* stream);   /* <speech_end>, :542-546 */
int vv_codec_state_reset(vv_ctx* ctx, void* stream);                                    /* new generate() call */

/* ---- fused frame tail: sampler -> decoder -> semantic -> connectors in one enqueue ------------- *
 * (:626-672).  Also copies the positive rows' next embeddings into the negative rows of `embeds_inout`
 * so the following vv_lm_decode feeds both streams the same input (:579-581). */
int vv_frame_tail(vv_ctx* ctx, const float* hidden, const float* noise, const int32_t* active, float cfg_scale,
                  float* latent_out, float* audio_out, float* embeds_inout, void* stream);

/* ---- introspection for tests / bench ----------------------------------------------------------- */
int64_t vv_launch_count(vv_ctx* ctx);     /* kernels launched by this ctx so far */
int vv_debug_gemv(vv_ctx* ctx, const void* w_bf16, const float* bias, const float* x, float* y, int M, int N, int K,
                  int prologue, const float* pro_w, float eps, int epilogue, void* stream);

int vv_debug_barrier_bench(vv_ctx* ctx, int iters, int ctas_per_sm, float* ms_out);
/* one linear through the persistent weight-stream kernel (wgmma + TMA, csrc/vv_stream.cuh): y = [y +] alpha * (W pro(x) + bias).
 * prologue: 0 none, 1 RMSNorm(pro_w, eps), 3 SwiGLU pairs (x is [M][2K]), 4 GELU, 6 SiLU; alpha_kind: 0 one, 2 gamma[n]. Synchronises. */
int vv_debug_stream_gemv(vv_ctx* ctx, const void* w_bf16, const float* bias, const float* x, float* y, int M, int N, int K, int prologue,
                         const float* pro_w, float eps, int alpha_kind, const float* alpha, int accumulate, void* stream);
int vv_stream_trace_read2(vv_ctx* ctx, long long* out /*[max_ops][sm_count][2]*/, int max_ops);  /* every CTA's barrier arrival / release (globaltimer ns); returns sm_count */
int vv_stream_trace_read(vv_ctx* ctx, long long* out /*[max_ops][12]*/, int* out_meta /*[max_ops][4]*/, int max_ops, const char* program_prefix);
                                                   /* VV_STREAM_TRACE=<cta>: per-stage clock stamps of one CTA of the last traced launch */
int vv_stream_diag(vv_ctx* ctx, unsigned* out6);   /* watchdog record of a trapped stream kernel: code, cta, thread, stage, iteration, extra */

#ifdef __cplusplus
}
#endif
#endif /* VIBEVOICE_B200_H_ */
