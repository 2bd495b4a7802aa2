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
 * Unknown names return VV_ERR_INVALID; names not needed by this path (fix_std, rotary_emb, a tied lm_head) are
 * accepted and ignored (returns 1).  The acoustic tokenizer encoder is optional: vv_finalize_weights packs it for
 * vv_voice_encode when all of its tensors were loaded and fails, naming the missing ones, when only some were. */
int vv_load_tensor(vv_ctx* ctx, const char* name, const void* data, int dtype, const int64_t* shape, int ndim);
int vv_set_speech_factors(vv_ctx* ctx, float scaling_factor, float bias_factor); /* modeling_vibevoice.py:131-132 */
int vv_finalize_weights(vv_ctx* ctx);     /* fails with the list of missing tensors */
int64_t vv_weight_bytes(vv_ctx* ctx, int which); /* 0 lm, 1 head-per-step, 2 cond_proj, 3 decoder, 4 semantic, 5 connectors,
                                                    6 streaming heads (0 when the checkpoint has none) */

/* ---- paged KV cache (replaces HF DynamicCache, modeling_vibevoice_inference.py:303, 556-562) -- *
 * 2B sequences share one pool of pages (64 tokens each, all layers); pages return to the pool when vv_kv_set_len shrinks a sequence. */
int vv_kv_init(vv_ctx* ctx, int64_t n_pages);   /* calling it again re-sizes the pool: every sequence is dropped, LM graphs re-captured */
int vv_kv_reserve(vv_ctx* ctx, int seq, int64_t n_tokens, void* stream); /* make positions < n_tokens addressable; pages it adds
                                                                            arrive with K and V zero in every layer */
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

/* ---- a-9: voice prompts (modeling_vibevoice_inference.py:149-163, 216-224) ---------------------- *
 * Non-streaming acoustic tokenizer encoder (modular_vibevoice_tokenizer.py:384-418, 776-813) over n voices of T samples each (the padded
 * speech_tensors as given), F = ceil(T / 3200) frames per voice; x = mean + sigma[v] * eps; feat = (x + speech_bias) * speech_scale;
 * acoustic_connector.  sigma is one scale per voice whatever std_dist_type is (gaussian: std_n[v] * fix_std / 0.8, fix: fix_std, none: 0;
 * eps may then be NULL).  Needs the encoder weights (else VV_ERR_STATE) and at least vv_voice_encode_workspace bytes of 256-byte aligned
 * device workspace (else VV_ERR_INVALID, nothing launched); a larger workspace processes more voices / rows per pass with the same result.
 * Outputs: mean_out [n,F,vae_dim] fp32 (optional), embeds_out [n,F,H] fp32. */
int64_t vv_voice_encode_workspace(vv_ctx* ctx, int n_voices, int64_t n_samples);   /* minimum workspace bytes of the call below */
int vv_voice_encode(vv_ctx* ctx, const float* wavs /*[n,T] fp32*/, int n, int64_t T, const float* sigma /*[n]*/, const float* eps /*[n,F,vae_dim]*/,
                    float* mean_out /*[n,F,vae_dim] or NULL*/, float* embeds_out /*[n,F,H] fp32*/, void* workspace, int64_t workspace_bytes,
                    void* stream);

/* ---- f-2: native prompt prefill (modeling_vibevoice_inference.py:467-482, the prompt half of step 0) ---------------------------- *
 * All decoder layers over n_tokens prompt rows of ONE sequence at positions [pos0, pos0 + n) on wgmma GEMMs and causal flash attention
 * (csrc/vv_prefill.cuh).  embeds [n,H] fp32 (device); the rotated K/V are written as bf16 straight into the paged pool (the layout
 * vv_kv_write uses); attention is causal over everything the sequence holds below pos0 + n, so pos0 > 0 continues a sequence.  Like
 * vv_kv_write it does not move kv_len (call vv_kv_set_len).  hidden_last [H] fp32 = final-norm hidden state of the last row.
 * Arithmetic: bf16 GEMM operands, bf16 Q / K / V / P, fp32 accumulators, residual stream and softmax statistics.  Tokens run in chunks of a
 * multiple of 64 rows sized from the workspace; results are bit-identical for every workspace size.
 * Errors: workspace below vv_lm_prefill_workspace or not 256-byte aligned -> VV_ERR_INVALID with nothing launched; bad seq, n < 1 or
 * pos0 + n > max_position_embeddings -> VV_ERR_INVALID; pages cannot be reserved -> VV_ERR_NOMEM; before vv_finalize_weights / vv_kv_init
 * -> VV_ERR_STATE. */
int64_t vv_lm_prefill_workspace(vv_ctx* ctx, int64_t n_tokens);          /* minimum workspace bytes of the call below */
int vv_lm_prefill(vv_ctx* ctx, int seq, int64_t pos0, int64_t n_tokens, const float* embeds, float* hidden_last, void* workspace,
                  int64_t workspace_bytes, void* stream);
/* embedding rows of DEVICE token ids (any count; vv_embed_tokens takes at most 16 host ids): out [n,H] fp32; ids outside [0, vocab) give
 * zero rows. */
int vv_embed_gather(vv_ctx* ctx, const int32_t* ids_dev, int64_t n, float* out, void* stream);

/* ---- streaming-0.5B per-token modules (modeling_vibevoice_streaming.py:42-53, 124-131) ------------------------------------------ *
 * Optional weights: model.tts_input_types.weight [2,H], tts_eos_classifier.fc1.{weight [H,H], bias [H]}, fc2.{weight [1,H], bias [1]},
 * all five or none (else vv_finalize_weights fails), kept in fp32 whatever dtype they arrive in; without them both calls return
 * VV_ERR_STATE and vv_weight_bytes(ctx, 6) is 0.
 * vv_tts_type_embed: dst[rows[i]] = src + tts_input_types[type_id] for i < n (n <= 16 host row indices, rows of H fp32 floats; src may be
 * one of them).  One fp32 add per element.
 * vv_eos_prob: prob_out[0] = sigmoid(fc2 . relu(fc1 . hidden + b1) + b2), logit_out[0] (may be NULL) = the logit; hidden [H] fp32, all
 * device pointers.  One launch, fp32 accumulation in a fixed order (results are bit-identical from call to call); calls on one ctx must
 * not overlap (they share a workspace). */
int vv_tts_type_embed(vv_ctx* ctx, const float* src, int type_id, const int32_t* rows_host, int n, float* dst, void* stream);
int vv_eos_prob(vv_ctx* ctx, const float* hidden, float* prob_out, float* logit_out, void* stream);

/* ---- introspection for tests / bench ----------------------------------------------------------- */
/* the inverse of vv_kv_write: K / V [n][kv_heads][head_dim] bf16 of positions [pos0, pos0 + n) of (seq, layer); either output may be NULL */
int vv_debug_kv_read(vv_ctx* ctx, int seq, int layer, int64_t pos0, int64_t n, void* k_out, void* v_out, void* stream);
int64_t vv_launch_count(vv_ctx* ctx);     /* kernels launched by this ctx so far */
int vv_debug_gemv(vv_ctx* ctx, const void* w_bf16, const float* bias, const float* x, float* y, int M, int N, int K,
                  int prologue, const float* pro_w, float eps, int epilogue, void* stream);
/* the same dispatch (GEMV, tensor-core GEMMs, wgmma) with every feature the codec passes use: y[m][n] = epi(W pro(x_m) + bias[n]).
 * Row m = (b, t) = (m / map_T, m % map_T) of x starts at x + b * map_bs + t * ldx floats (map_T = 0: dense rows ldx apart); rows may
 * overlap, which is how a convolution reads its window.  prologue: 0 none, 1 RMSNorm(pro_w, eps), 3 SiLU.  epilogue: 0 none, 2 + res,
 * 3 res + epi_a[m][n] (rows epi_lda apart) *, 4 res + epi_a[n] *, 6 GELU, 7 SiLU; res rows ldres apart; res == y with ldres == ldy runs
 * in place, and on grids smaller than the GPU the tensor-core GEMMs then split K and add into y with fp32 atomics.  info[2] = {kernel,
 * split-K factor}: kernel 0 GEMV, 1..7 gemm_mma_ring_kernel <1,GELU> <1,NONE> <0,GAMMA_RESID> <0,NONE> <0,GELU> <0,RESID> <-1,-1>,
 * 8 gemm_mma_kernel, 9 split_bf16_kernel + gemm_wgmma_kernel.  Needs vv_finalize_weights (VV_ERR_STATE).  Synchronises. */
int vv_debug_gemv2(vv_ctx* ctx, const void* w_bf16, const float* bias, const float* x, int64_t ldx, int map_T, int64_t map_bs, float* y,
                   int64_t ldy, const float* res, int64_t ldres, int M, int N, int K, int prologue, const float* pro_w, float eps,
                   int epilogue, const float* epi_a, int64_t epi_lda, int32_t* info, void* stream);
/* One acoustic-decoder (which = 0: latent [B,64] -> audio [B,3200]) or semantic-encoder (which = 1: audio [B,3200] -> features
 * [B,semantic_vae_dim]) pass over the current streaming state, launched directly (no graph), with the input of every stage boundary
 * copied out: after every convolution and every Block1D of the kernel-per-stage path, at the hand-off between the weight-stream program
 * and that path, and the pass output.  Tap i is [B][T_i][C_i] fp32 (time-major, like the kernels' activations) at float offset
 * B * sum_{j<i} T_j * C_j of `taps`.  meta (optional) [n_taps][5] = {kind: 0 conv, 1 block, 2 stream hand-off, 3 pass output; stage;
 * index in stage; T; C}: conv (i, 0) = output of stage i's convolution, block (i, j) = output of block j of stage i, hand-off (s, 0) =
 * input of stage s, output (n_stages, 0).  Which stages run in the stream program depends on max_batch; meta describes the split that
 * runs.  Commits the history of `active` rows exactly like vv_codec_decode_frame / vv_semantic_encode_frame (same state, so both may be
 * interleaved on one context).  taps == NULL: fills meta and returns n_taps, nothing launched.  Too little tap space or a bad `which`:
 * VV_ERR_INVALID with nothing launched; before vv_finalize_weights: VV_ERR_STATE.  Returns n_taps.  Synchronises. */
int vv_debug_codec_taps(vv_ctx* ctx, int which, const float* in, const int32_t* active, float* out, float* taps, int64_t taps_floats,
                        int32_t* meta, void* stream);
/* vv_diffusion_sample launched directly (no graph) with every solver block's result copied out.  The preamble is the production one
 * (cond_proj, the conditioning kernel, the all-steps modulation GEMM); the sampler program then runs as one launch per block, each built by
 * the production builder and checked stage by stage (kernel variant, K split) against the production program: proj(-1), then per step i
 * head layer li = 0 .. L-1, the final layer and proj(i) (CFG + DPM-Solver++ update of step i, then noisy_images_proj).  SDE step noise
 * and the device-held CFG scale are used as in production.  Tap j is [rows_j][cols_j] fp32 at float offset sum_{k<j} rows_k * cols_k of
 * `taps`; meta (optional) [n_taps][7] = {kind, step, layer, rows, cols, kernel, split}, in this order:
 *   kind 0: silu(t_embedder.mlp.0(t)) [N][H]      1: t embedding temb [N][H]  (both as left by vv_set_diffusion_steps)
 *   kind 2: cond_proj(cond) [2B][H]               3: AdaLN modulation of every step [N * 2B][(3L+2)H]
 *   then kind 6 z_0 (= noise), 7 x0 (zeros), 8 x [2B][H] for step -1, and per step i: kind 4 residual stream after head layer `layer`
 *   [2B][H], 5 head output v [2B][64], 6 z_{i+1} [B][64], 7 x0_i [B][64], 8 x = noisy_images_proj(z_{i+1}) [2B][H]; last, kind 9 latent_out.
 * kernel / split: kinds 0-3 = the {kernel, split-K factor} linear() ran (numbering as vv_debug_gemv2); block taps = the stream-kernel variant
 * and the number of stages (after the K split) of the block that wrote them.  taps == NULL: fills meta (kernel -1) and returns n_taps,
 * nothing launched.  Too little tap space: VV_ERR_INVALID with nothing launched; before vv_set_diffusion_steps (or SDE without step noise):
 * VV_ERR_STATE.  Returns n_taps.  Synchronises. */
int vv_debug_sampler_taps(vv_ctx* ctx, const float* cond, const float* noise, float cfg_scale, float* latent_out, float* taps,
                          int64_t taps_floats, int32_t* meta, void* stream);
/* Decoder layer `layer` of vv_lm_prefill alone, over n rows of sequence `seq` at positions [pos0, pos0 + n), from the fp32 residual input
 * x_in [n][H] (device), with what each of its kernels left copied out.  It runs the kernels vv_lm_prefill runs for that layer, in the same
 * chunks of the same workspace rule, reserves the same pages and writes the layer's K/V into the pool.  hidden_last (optional, [H] fp32):
 * the final-norm hidden state of the last output row, as vv_lm_prefill computes it.  Tap k is [n][cols_k] at byte offset
 * sum_{j<k} n * cols_j * bytes_j of `taps`; meta (optional) [7][3] = {kind, bytes per element, cols}, kinds in this order:
 *   0 norm1 bf16 [n][H]   1 Q after bias and RoPE bf16 [n][nq]   2 attention output bf16 [n][nq]   3 residual after the o-projection
 *   fp32 [n][H]   4 norm2 bf16 [n][H]   5 silu(gate) * up bf16 [n][I]   6 layer output fp32 [n][H].
 * taps == NULL: fills meta and returns 7, nothing launched.  Errors: those of vv_lm_prefill, a bad layer -> VV_ERR_INVALID, too little tap
 * space -> VV_ERR_INVALID, all with nothing launched.  Returns 7.  Synchronises. */
int vv_debug_prefill_taps(vv_ctx* ctx, int seq, int64_t pos0, int64_t n, int layer, const float* x_in, float* hidden_last, void* workspace,
                          int64_t workspace_bytes, void* taps, int64_t taps_bytes, int32_t* meta, void* stream);

/* vv_voice_encode with every stage boundary copied out: it runs the same kernels in the same order, with the same voice groups and GEMM
 * row chunks for the given workspace.  Tap k is [n][T_k][C_k] fp32 (time-major) at float offset n * sum_{j<k} T_j * C_j of `taps`; a
 * group of voices writes its rows at its first voice's offset, so the layout does not depend on the workspace.  meta (optional)
 * [n_taps][5] = {kind, stage, index, T, C}, in run order: kind 0 (i, 0) = output of stage i's convolution, (n_stages, 0) = the head conv
 * (the latent mean [F][vae_dim]); 1 (i, j) = the mixer half x + gamma * dwconv7(RMSNorm(x)) of block j of stage i; 2 (i, j) = the output
 * of that block; 3 (n_stages, 0) = the connector's fc1 output [F][H] before its RMSNorm; 4 (n_stages, 0) = the embeddings [F][H] (also
 * written to embeds_out).  taps == NULL: fills meta and returns n_taps, nothing launched.  Errors: those of vv_voice_encode, and too
 * little tap space -> VV_ERR_INVALID, all with nothing launched.  Returns n_taps.  Synchronises. */
int vv_debug_voice_taps(vv_ctx* ctx, const float* wavs, int n, int64_t T, const float* sigma, const float* eps, float* embeds_out,
                        void* workspace, int64_t workspace_bytes, float* taps, int64_t taps_floats, int32_t* meta, void* stream);

int vv_debug_barrier_bench(vv_ctx* ctx, int iters, int ctas_per_sm, float* ms_out);
/* one linear through the persistent weight-stream kernel (wgmma + TMA, csrc/vv_stream.cuh): y = [y +] alpha * (W pro(x) + bias).
 * prologue: 0 none, 1 RMSNorm(pro_w, eps), 3 SwiGLU pairs (x is [M][2K]), 4 GELU, 6 SiLU; alpha_kind: 0 one, 2 gamma[n]. Synchronises. */
int vv_debug_stream_gemv(vv_ctx* ctx, const void* w_bf16, const float* bias, const float* x, float* y, int M, int N, int K, int prologue,
                         const float* pro_w, float eps, int alpha_kind, const float* alpha, int accumulate, void* stream);
/* the same linear with every stage feature exposed: y[m][n] = (store ? 0 : y[m][n]) + alpha * (W pro(x[m]) + bias[n]), rows of x / y
 * ldx / ldy floats apart (SwiGLU: x rows hold 2K interleaved gate / up sums).  prologue 2 = AdaLN: RMSNorm(pro_w or 1, eps) * (1 + scale) +
 * shift with scale / shift rows pro_ld floats apart; alpha_kind 1 = gate alpha[m][n] (row stride lda), 2 = gamma alpha[n].  store needs
 * K <= 64.  operand_cap > 0 caps the activation-operand bytes of the stage, so that smaller shapes run through the K split as well.
 * Synchronises; returns the number of stages the linear ran as (> 1: split along K). */
int vv_debug_stream_gemv2(vv_ctx* ctx, const void* w_bf16, const float* bias, const float* x, int64_t ldx, float* y, int64_t ldy, int M, int N,
                          int K, int prologue, const float* pro_w, float eps, const float* pro_shift, const float* pro_scale, int64_t pro_ld,
                          int alpha_kind, const float* alpha, int64_t lda, int store, int64_t operand_cap, void* stream);
int vv_stream_trace_read2(vv_ctx* ctx, long long* out /*[max_ops][sm_count][2]*/, int max_ops);  /* every CTA's barrier arrival / release (globaltimer ns); returns sm_count */
int vv_stream_trace_read(vv_ctx* ctx, long long* out /*[max_ops][12]*/, int* out_meta /*[max_ops][4]*/, int max_ops, const char* program_prefix);
                                                   /* VV_STREAM_TRACE=<cta>: per-stage clock stamps of one CTA of the last traced launch */
int vv_stream_diag(vv_ctx* ctx, unsigned* out6);   /* watchdog record of a trapped stream kernel: code, cta, thread, stage, iteration, extra */

#ifdef __cplusplus
}
#endif
#endif /* VIBEVOICE_B200_H_ */
