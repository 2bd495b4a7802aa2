// vv_stream.cuh -- persistent weight-stream kernel: every M <= 8..64-row linear of the generation loop as a warpgroup MMA (wgmma) whose
// weight tiles arrive by TMA (cp.async.bulk.tensor, 128-byte swizzle) through a deep shared-memory ring that keeps running ACROSS the
// grid-wide dependencies between stages.
//
// Why this shape (DESIGN 7): one speech frame is a chain of ~450 dependent skinny linears (28 LM layers x 4, 30 diffusion steps x 9,
// codec front).  As one kernel per stage each of them pays launch + cold pipeline + drain (~5 us) around a 1-9 us weight stream, and HBM
// idles in between.  Here ONE cooperative grid (one CTA per SM) runs a whole program of stages:
//
//   warps 0-3 workers   (one warpgroup) grid barrier -> prologue: activations from L2, RMSNorm / AdaLN / SwiGLU / GELU / solver update
//                       applied, split into bf16 hi + lo (x = hi + lo to 2^-17) and written as the MMA's B operand in the canonical K-major
//                       SWIZZLE_128B layout (rows [0, nB/2) = hi, [nB/2, nB) = lo, so ONE MMA yields both partial products) -> per weight
//                       tile 2 x 4 wgmma.mma_async m64 x nB x 16 (the tile's two 64-row halves, N = 16..64 activation rows), fp32
//                       accumulators in registers, the ring slot handed back to the producer once its MMAs retired -> epilogue per
//                       (row tile, k range) segment straight from the accumulators: hi + lo, bias / gate / gamma scaling, fp32 atomics
//                       (red.global.add) into the output.
//   warp 4   producer   walks the program's static schedule and issues the TMA loads of this CTA's weight tiles (128 rows x 64 k, bf16,
//                       16 KB) into an S-stage ring.  Weights never depend on activations, so it runs ahead of the grid barriers: while
//                       the workers synchronise / stage activations for stage i, the ring already fills with tiles of stage i, i+1...
//
// Work split ("stream-K"): a stage with R = ceil(N/128) row tiles and KB = ceil(K/64) k-blocks has U = R*KB tile units, dealt out as
// contiguous ranges [c*U/G, (c+1)*U/G) to the G CTAs in row-tile-major order: every SM streams the same number of bytes (+-1 tile) for
// ANY shape, a CTA owns <= 3 (row tile, k range) segments, each accumulated and written out in turn, and partial sums meet in the output through
// atomics.  That is why epilogues are linear (bias, scaling, residual) and the non-linearities (SwiGLU, GELU) live in the NEXT stage's
// prologue.
//
// Attention stages (SK_ATTN) run in the same kernel: K / V pages of the paged cache arrive through the same ring, scores and P V by mma.sync,
// RoPE / KV append fused, split-KV partials merged in the o-projection's prologue.  Codec stages add a causal-window gather prologue and a
// distributed mixer stage (SK_MIX).
//
// The kernel is bound by the chain of ~520 dependent grid-wide stages per frame, and INSIDE a stage by instruction fetch: every stage runs
// its worker path once, straight-line.  Hence one instantiation per program family (stream_kernel<FEAT, TRACE>), compile-time head_dim / operand
// height where a program allows it, descriptor fields in registers, descriptor-only arithmetic between barrier arrival and barrier wait, and
// uniform early exits instead of predicated-off rows.
//
// Reference arithmetic: the linear stages are the same linears as the stand-alone kernels in vv_kernels.cuh (see the anchors there);
// attention and the solver update cite theirs at SAtt and SDpm.
#pragma once
#include "vv_kernels.cuh"

namespace vv {

// ---------------------------------------------------------------------------------------------------------------------------------
// grid-wide synchronisation
// ---------------------------------------------------------------------------------------------------------------------------------
struct GridBar { unsigned count; unsigned pad0[31]; unsigned gen; unsigned pad1[31]; };   // arrival counter and generation on separate 128 B lines

VV_DEVINL unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
VV_DEVINL unsigned ld_relaxed_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
VV_DEVINL void st_release_u32(unsigned* p, unsigned v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
VV_DEVINL void st_relaxed_u32(unsigned* p, unsigned v) { asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
VV_DEVINL unsigned atom_add_acqrel_u32(unsigned* p, unsigned v) {
  unsigned r;
  asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(r) : "l"(p), "r"(v) : "memory");
  return r;
}
VV_DEVINL void red_add_release_u32(unsigned* p, unsigned v) { asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// sense-free generation barrier across all CTAs of a cooperative launch (used by barrier_bench_kernel)
VV_DEVINL void grid_barrier(GridBar* gb, unsigned nctas) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned gen = ld_relaxed_u32(&gb->gen);
    const unsigned prev = atom_add_acqrel_u32(&gb->count, 1u);
    if (prev == nctas - 1) {
      st_relaxed_u32(&gb->count, 0u);
      st_release_u32(&gb->gen, gen + 1);
    } else {
      while (ld_acquire_u32(&gb->gen) == gen) { }
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256) barrier_bench_kernel(GridBar* gb, int iters, float* sink) {
  float acc = 0.f;
  for (int i = 0; i < iters; ++i) {
    grid_barrier(gb, gridDim.x);
    acc += 1.f;
  }
  if (threadIdx.x == 0 && blockIdx.x == 0) *sink = acc;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// program representation (built on the host in vv_runtime.cu, read-only on the device)
// ---------------------------------------------------------------------------------------------------------------------------------
constexpr int ST_THREADS = 160;          // warps 0..3 workers (one warpgroup: wgmma), warp 4 producer
constexpr int ST_WORKERS = 128;
constexpr int ST_TILE = 16384;           // one weight tile: 128 rows x 64 bf16
constexpr int ST_MAXSEG = 8;             // (row tile, k range) segments a CTA may own in one stage
constexpr int ST_MAX_STAGES = 12;
constexpr int ST_BAR_REP = 0;

enum SKind { SK_GEMV = 0, SK_NOP = 1, SK_ATTN = 2, SK_MIX = 3 };
enum SPro { SP_NONE = 0, SP_RMSNORM = 1, SP_ADALN = 2, SP_SWIGLU = 3, SP_GELU = 4, SP_DPM = 5, SP_SILU = 6, SP_COMBINE = 7, SP_WINDOW = 8, SP_MIXER = 9 };
enum SAlpha { SA_ONE = 0, SA_GATE = 1 /* alpha[m][n], row stride lda */, SA_GAMMA = 2 /* alpha[n] */ };

// CFG + DPM-Solver++(2M) update of step `step`, evaluated in the prologue of the stage that projects the new latent (noisy_images_proj):
// B-operand row m = z'[m mod B].  Rows b (conditional) and B+b (unconditional) of the head output v give
//   v = v_u + s (v_c - v_u); x0 = a0 z - s0 v; z' = ks z - kx x0 [- 0.5 kx rinv (x0 - x0_prev)] [+ kn * step_noise[step]]
// (modeling_vibevoice_inference.py:703-709 + schedule/dpm_solver.py:581-584, 669-677, 738-764; sde-dpmsolver++, dpm_solver.py:680-686 /
// 785-793: same two forms with other ks / kx plus the variance-noise term; step_noise is [n_steps][B][64], nullptr until
// vv_set_step_noise binds it).  step = -1: z' = the initial noise.
// s and the coefficients are per sample: cfg_p is cfg[B] and the coefficients of sample b come from rows[step][b]; a row with fewer steps
// than the program runs identity steps (ks = 1, kx = 0, kn = 0) first (vv_set_row_sampler).
struct SDpm {
  const float* z_in; float* z_out; const float* x0_in; float* x0_out; const float* v; const float* noise;
  const float* cfg_p; const float* step_noise; float* latent_out;
  int step, B;
  const DpmCoef* rows;      // [n_steps][B] device table
  unsigned char pad_[24];   // keeps SOp at its size: a smaller descriptor changes ptxas' register allocation of every kernel variant
};

// Decode attention as a stage of the stream (SK_ATTN), and its split-partial merge as the prologue of the o-projection (SP_COMBINE).
// Units = (row m, kv head g, 64-token page t) in that order, dealt out to the CTAs as contiguous ranges like the weight tiles; the K and V
// page of a unit are two 16 KB ring slots filled by TMA (each page is contiguous in the pool: [64 tokens][128] bf16 -> two 64 x 64 boxes,
// SWIZZLE_128B), so the KV cache streams through the same ring, prefetched across the grid barriers like the weights.
// A CTA's run of units inside one (m, g) is a segment: one online-softmax partial (max, sum, acc[G heads][128]) written to slot
// `cta - first_cta(m, g)` of part_acc / part_ml; SP_COMBINE merges the partials of a head while it stages the o-projection's activations.
// Reference: transformers Qwen2Attention (modeling_qwen2.py:116-174).
struct SAtt {
  const float* qkv;            // [M][(q_heads + 2 kv_heads) * 128] fp32, bias added, not rotated
  KvView kv;                   // this layer's pool pointers (new K/V rows are written here), page table, kv_len, row_mode
  float* part_acc;             // [M][kv_heads][gridDim][8][128]
  float* part_ml;              // [M][kv_heads][gridDim][8][2]
  const float* inv_freq;
  float scale;
  unsigned long long tmap_k, tmap_v;   // tensor maps over the WHOLE K / V pool: [layers * pages * kv_heads * 64 rows][128] bf16, box 64 x 64
  unsigned row_base;           // first row of this layer in those maps
  int hd;                      // head_dim: 128 (a K / V page = two 64-column boxes) or 64 (one box, 8 KB of the slot used)
  float* rope_cs;              // [M][64][2] cos / sin of (kv_len[m] * inv_freq[d]): written by the QKV stage, read here (accurate sincosf of
                               // positions up to 64K is too slow to recompute in every CTA)
};

// Streaming-codec prologues (modular_vibevoice_tokenizer.py:327-382, 620-684; same arithmetic as assemble_window / dwconv_res / rows_norm):
//  SP_WINDOW  activation row (b, t) = rows [t*stride, t*stride + k) of the causal window [hist[b] (ctx rows) ; alpha*src[b]+beta (T_in rows)],
//             each row `cin` wide, flattened (K = k * cin): strided / transposed convolutions as window GEMVs.  The CTA that owns unit 0
//             writes the next history (the window's last ctx rows) into `next`.
//  SK_MIX     (a stage of its own, no linear) the first half of a Block1D for rows (b, t), t < T, C = K channels, channels dealt out to CTAs:
//             xn = RMSNorm(x) * norm_w;  x1 = x + gamma * (dw_b + sum_j dw_w[j] * win[t + j]),  win = [hist[b] (6 normalised rows) ; xn];
//             writes x1 (the residual base both FFN linears work on) and the next history (last 6 rows of the window).
//             (As the prologue of the FFN linear every CTA would recompute the whole block's mixer.)
struct SCodec {
  const float* hist; float* next;        // [B][ctx][cin] / [B][6][C]
  const float* src;                      // SP_WINDOW: [B][T_in][cin]
  int ctx, T_in, T_out, stride, cin;     // SP_WINDOW geometry (T_out rows per sample); SP_MIXER: T_out = T
  float alpha, beta;
  const float* norm_w; const float* dw_w; const float* dw_b; const float* gamma; const float* ffn_norm_w;   // SP_MIXER
  float* x1_out;                         // SP_MIXER: [M][C]
  float eps;
};

struct alignas(16) SOp {
  int kind;
  int sync_before;          // wait until every CTA has finished the previous stage (grid barrier) before touching activations
  int M, N, K;              // activation rows, weight rows (outputs), reduction length (K % 8 == 0)
  int nB;                   // MMA N: 16, 32 or 64 (rows [0,nB/2) = hi, [nB/2,nB) = lo)
  int k0, krow;             // K-split slice: this stage reduces over columns [k0, k0 + K) of rows krow long (x, pro_w, pro_scale / shift,
                            // SP_COMBINE heads are addressed at k0 + k; RMSNorm / AdaLN statistics always cover the whole krow-long row)
  unsigned long long tmap;  // device address of the CUtensorMap of the TILE-MAJOR copy of W: [R*KB tiles][128 rows][64 k] bf16, zero padded
                            // (seen as a 2-D tensor [R*KB*128][64]; box 64 x 128 = one contiguous 16 KB tile, SWIZZLE_128B)
  int pro;
  const float* x; long long ldx;         // activations, row stride in floats (SP_SWIGLU: interleaved gate/up sums, row length 2K)
  const float* pro_w; float pro_eps;     // norm weight [K] (may be null for SP_ADALN)
  const float* pro_shift; const float* pro_scale; long long pro_ld;
  SDpm dpm;                              // SP_DPM only
  SAtt att;                              // SK_ATTN, SP_COMBINE
  SCodec cod;                            // SP_WINDOW, SP_MIXER
  float* y; long long ldy;               // y[m][n] += alpha * (acc + bias[n] if the segment starts at k = 0);  store != 0: y = ... (KB == 1 only)
  const float* bias;
  int alpha_kind; const float* alpha; long long lda;
  int store;
  float* init_dst; long long init_n;     // optional: zero-fill jobs (buffers a LATER stage accumulates into), spread over the grid
  float* init2_dst; long long init2_n;
  int rope_rows;                         // > 0: this stage also fills att.rope_cs for rows [0, rope_rows) (CTA m computes row m)
};

struct SParams {
  const SOp* ops; int n_ops;
  unsigned* bar_count;      // arrival counter of the grid barrier, zeroed by the host before every launch
  unsigned* diag;           // host-mapped: [0] = error code, [1..7] = where (watchdog)
  int n_stages;             // ring depth
  int b_bytes;              // bytes of the activation-operand region
  int max_inflight;         // TMA tiles a CTA may have in flight (<= n_stages)
  const int* kv_len; const int* row_mode; int n_seq, kv_heads;   // sequence state for attention stages (null / 0 when the program has none)
  long long* trace;         // optional [n_ops][ST_TRACE] clock64 stamps of CTA `trace_cta` (tools/stream_trace.py), else null
  int trace_cta;
  long long* trace2;        // optional [n_ops][G][2] globaltimer (ns) of every CTA: arrival at / release from the grid barrier
};
constexpr int ST_TRACE = 12;   // 0 op start, 1 barrier passed, 2 row stats done, 3 B operand staged, 4 accumulators complete, 5 epilogue issued,
                               // 6 MMA loop entered, 7 MMA saw the last tile, 8 last MMA retired, 9 producer issued the last tile of the stage

// W [N][K] row-major -> tile-major [R][KB][128][64], zero padded.  TMA boxes cut out of the row-major matrix (128 rows x 128 B, kilobytes
// apart) make every row its own DRAM burst, so the kernel reads tiles that are contiguous in HBM instead; units of a stage are consecutive tiles, i.e. every CTA reads ONE contiguous byte range per stage.
// A K-split slice packs columns [k0, k0 + K) of a W whose rows are ldw long.
__global__ void tile_pack_kernel(const bf16* __restrict__ W, bf16* __restrict__ T, int N, int K, int KB, long long ldw, int k0, long long n_chunks) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_chunks; i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i & 7), r = (int)((i >> 3) & 127);
    const long long tile = i >> 10;
    const int kb = (int)(tile % KB), rt = (int)(tile / KB);
    const int n = rt * 128 + r, k = kb * 64 + ch * 8;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (n < N && k < K) v = *reinterpret_cast<const uint4*>(W + (size_t)n * ldw + k0 + k);   // K % 8 == 0: a chunk never straddles K
    *reinterpret_cast<uint4*>(T + i * 8) = v;
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------------------------------------------
VV_DEVINL void st_die(unsigned* diag, unsigned code, unsigned a, unsigned b, unsigned c) {
  if (diag) {
    diag[1] = blockIdx.x; diag[2] = threadIdx.x; diag[3] = a; diag[4] = b; diag[5] = c;
    __threadfence_system();
    diag[0] = code;
    __threadfence_system();
  }
  __trap();
}
// bounded mbarrier wait: a lost arrival must end in a diagnosable trap, never in a hung GPU
VV_DEVINL void mbar_wait_wd(unsigned long long* bar, unsigned parity, unsigned* diag, unsigned code, unsigned a, unsigned b) {
  const unsigned addr = smem_u32(bar);
  unsigned ok = 0;
  long long t0 = 0;
  for (unsigned spins = 0;; ++spins) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
    if (ok) return;
    if ((spins & 1023u) == 1023u) {
      const long long t = clock64();
      if (t0 == 0) t0 = t;
      else if (t - t0 > 6000000000ll) st_die(diag, code, a, b, parity);
    }
  }
}
VV_DEVINL void tma_load_2d(void* smem_dst, unsigned long long tmap, int c0, int c1, unsigned long long* bar, unsigned long long policy) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], [%4], %5;"
               ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "l"(policy) : "memory");
}
VV_DEVINL long long gtime_ns() { long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
VV_DEVINL float ldcg1(const float* p) { return __ldcg(p); }
VV_DEVINL float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
VV_DEVINL void red_add_f32(float* p, float v) { asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }
VV_DEVINL void worker_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// attention units of row m: kv_heads * pages(m) (0 for rows that are switched off); returns the total, fills this CTA's range
// kv_len / row_mode are constant during a launch; the kernel keeps a copy in shared memory (SeqView) -- read from global memory at the start
// of every attention stage they were 4 dependent L2 round trips on the critical path
struct SeqView { const int* kv_len; const int* row_mode; int kv_heads; };
VV_DEVINL unsigned att_tiles(const SeqView& q, int m) { return q.row_mode[m] ? (unsigned)((q.kv_len[m] + 1 + KV_PAGE - 1) / KV_PAGE) : 0u; }
// Work split of an attention stage.  Every (row m, kv head g) group with pages contributes nt + ST_ATT_SEGW VIRTUAL units: the first
// ST_ATT_SEGW stand for the fixed cost of a segment (Q staging, warp merge, partial write ~ 4 pages), the rest are its pages in
// order.  CTAs take contiguous ranges of virtual units, so a CTA that also gets the few pages of a short (CFG-negative) row gets
// correspondingly fewer pages of the long one (otherwise the CTA owning both short groups arrives late at every layer's barrier).
constexpr unsigned ST_ATT_SEGW = 4;
VV_DEVINL unsigned att_vtotal(const SeqView& q, int M) {
  unsigned V = 0;
  for (int m = 0; m < M; ++m) { const unsigned nt = att_tiles(q, m); if (nt) V += (nt + ST_ATT_SEGW) * (unsigned)q.kv_heads; }
  return V;
}
VV_DEVINL unsigned cta_of_unit(unsigned u, unsigned U, unsigned G) { return ((u + 1u) * G - 1u) / U; }     // inverse of u0 = U c / G
struct AttSeg { int m, g, t0, t1; unsigned nt, vf; };     // pages [t0, t1) of group (m, g); vf = first virtual unit of the group
struct AttIter { unsigned v0, v1, vf; int gi; };          // this CTA's virtual range, walking the groups in order
VV_DEVINL void att_begin(const SeqView& q, int M, AttIter& it) {
  const unsigned V = att_vtotal(q, M);
  it.v0 = V * blockIdx.x / gridDim.x; it.v1 = V * (blockIdx.x + 1u) / gridDim.x; it.vf = 0; it.gi = 0;
}
VV_DEVINL bool att_next(const SeqView& q, int M, AttIter& it, AttSeg& sg) {
  while (it.gi < M * q.kv_heads && it.vf < it.v1) {
    const int m = it.gi / q.kv_heads, g = it.gi - m * q.kv_heads;
    const unsigned nt = att_tiles(q, m);
    ++it.gi;
    if (nt == 0) continue;
    const unsigned vf = it.vf, len = nt + ST_ATT_SEGW;
    it.vf += len;
    const unsigned a = it.v0 > vf ? it.v0 : vf, b = it.v1 < vf + len ? it.v1 : vf + len;
    if (b <= a) continue;
    const unsigned t0 = a - vf > ST_ATT_SEGW ? a - vf - ST_ATT_SEGW : 0u, t1 = b - vf > ST_ATT_SEGW ? b - vf - ST_ATT_SEGW : 0u;
    if (t1 <= t0) continue;
    sg.m = m; sg.g = g; sg.t0 = (int)t0; sg.t1 = (int)t1; sg.nt = nt; sg.vf = vf;
    return true;
  }
  return false;
}
// byte offset of element (token row, d) inside a K / V ring slot: two 64-column halves of 8 KB, 128-byte rows, 16-byte chunks XOR-swizzled
VV_DEVINL unsigned kv_off(int tok, int d) { return (unsigned)(((d >> 6) << 13) + tok * 128 + ((((d & 63) >> 3) ^ (tok & 7)) << 4) + (d & 7) * 2); }

// this CTA's unit range of a stage: units are (row tile, k-block) pairs in row-tile-major order
// (32-bit arithmetic: U * gridDim < 2^32 is checked on the host; 64-bit divisions here would sit on the critical path of every stage)
VV_DEVINL void st_part(const SOp& op, unsigned& u0, unsigned& u1, int& KB) {
  KB = (op.K + 63) >> 6;
  const unsigned U = (unsigned)((op.N + 127) >> 7) * (unsigned)KB;
  u0 = U * blockIdx.x / gridDim.x;
  u1 = U * (blockIdx.x + 1u) / gridDim.x;
}

// epilogue operands of a linear stage: y[m][n] (+)= alpha * (acc + bias[n] if the segment starts at k = 0)
struct StEpi { const float* bias; const float* alpha; float* y; long long lda, ldy; bool gate, gamma, store; };

template <int NB> VV_DEVINL void wgmma_nb(float (&d)[NB / 2], unsigned long long a, unsigned long long b) {
  if constexpr (NB == 16) wgmma_m64n16(d, a, b, 1);
  else if constexpr (NB == 32) wgmma_m64n32(d, a, b, 1);
  else wgmma_m64n64(d, a, b, 1);
}

// The worker warpgroup's MMA + epilogue of one linear stage: units [u0, u1) = (row tile, k-block) pairs whose weight tiles sit in the ring
// from slot `slot` (phase `ph`) on, B operand of k-block j (relative to the first one) at breg + j * NB * 128.  The units form <= 3
// (row tile, k range) segments.  Per segment: the epilogue operands (bias, gamma, gate) are requested first, so they arrive while the MMAs
// run; per tile the two 64-row halves of the weight tile times the NB-row operand, 4 k-steps each, the MMAs of a tile running while the
// next tile's are issued and its ring slot released once they retired; then the accumulators go out through the epilogue.
template <int NB>
VV_DEVINL void st_mma_epilogue(unsigned char* ring, unsigned char* breg, unsigned long long* full_bar, unsigned long long* empty_bar, int NS,
                               unsigned slot, unsigned ph, unsigned u0, unsigned u1, int KB, int M, int N, const StEpi& ep, unsigned* diag,
                               int oi, long long* trs) {
  constexpr int R = NB / 2;                  // accumulator registers per 64-row half; operand rows [0, NB/2) = hi, [NB/2, NB) = lo
  constexpr int HG = NB / 16;                // 8-column groups of the hi half
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned long long da0 = wgmma_desc_sw128(smem_u32(ring)), db0 = wgmma_desc_sw128(smem_u32(breg));
  const unsigned bstep = (unsigned)(NB * 128) >> 4;          // descriptor start-address units (16 B) per k-block of the B operand
  const int rt_first = (int)(u0 / (unsigned)KB), kb_first = (int)(u0 - (unsigned)rt_first * (unsigned)KB);
  if (trs) trs[6] = clock64();
  unsigned jloc = 0;
  int rt = rt_first, kb = kb_first;
  for (unsigned u = u0; u < u1; ++rt, kb = 0) {
    const unsigned seg_end = min(u1, u + (unsigned)(KB - kb));
    // ---------------- epilogue operands of row tile rt: requested now, consumed after the MMAs ----------------
    const bool from0 = kb == 0;                               // this segment holds k-block 0 of its row tile -> it adds the bias
    float e_bias[2][2], e_gam[2][2], e_gate[2][2][HG][2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = rt * 128 + h * 64 + warp * 16 + (lane >> 2) + 8 * e;
        const bool live = n < N;
        e_bias[h][e] = (live && from0 && ep.bias) ? ep.bias[n] : 0.f;
        e_gam[h][e] = (live && ep.gamma) ? ep.alpha[n] : 1.f;
#pragma unroll
        for (int j = 0; j < HG; ++j)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int m = 8 * j + 2 * (lane & 3) + c;
            e_gate[h][e][j][c] = (live && ep.gate && m < M) ? ldcg1(ep.alpha + (long long)m * ep.lda + n) : 1.f;
          }
      }
    // ---------------- MMAs of the segment ----------------
    float acc[2][R];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < R; ++i) acc[h][i] = 0.f;
    unsigned prev = 0;
    for (unsigned v = u; v < seg_end; ++v) {
      mbar_wait_wd(&full_bar[slot], ph, diag, 3u, (unsigned)oi, v - u0);
      __syncwarp();                                           // reconverge after the per-thread spin: wgmma is warpgroup-collective
      if (trs && v + 1 == u1) trs[7] = clock64();
      const unsigned long long da = da0 + (unsigned long long)(slot * (unsigned)(ST_TILE >> 4));
      const unsigned long long db = db0 + (unsigned long long)(jloc * bstep);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        wgmma_nb<NB>(acc[0], da + 2 * k, db + 2 * k);
        wgmma_nb<NB>(acc[1], da + 512 + 2 * k, db + 2 * k);
      }
      wgmma_commit();
      wgmma_wait<1>();                                        // this warp's MMAs of the previous tile retired: hand its slot back
      if (v > u && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = slot;
      if (++slot == (unsigned)NS) { slot = 0; ph ^= 1u; }
      if (++jloc == (unsigned)KB) jloc = 0;                   // (only when the CTA holds >= KB units: B region = all k-blocks)
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty_bar[prev]);
    if (trs && seg_end == u1) { trs[4] = clock64(); trs[8] = trs[4]; }
    u = seg_end;
    // ---------------- epilogue of row tile rt ----------------
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = rt * 128 + h * 64 + warp * 16 + (lane >> 2) + 8 * e;
        if (n >= N) continue;
#pragma unroll
        for (int j = 0; j < HG; ++j)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int m = 8 * j + 2 * (lane & 3) + c;
            if (m < M) {
              const float val = (acc[h][4 * j + 2 * e + c] + acc[h][4 * (j + HG) + 2 * e + c] + e_bias[h][e]) * e_gam[h][e] * e_gate[h][e][j][c];
              float* yp = ep.y + (long long)m * ep.ldy + n;
              if (ep.store) *yp = val; else red_add_f32(yp, val);
            }
          }
      }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------------------------------------------------------------
// FEAT = the stage kinds / prologues / epilogue scalings a program may use (bit SP_x, bit 16 + SK_x, bit 24 + SA_x).  One instantiation per
// program family: the all-features kernel is 224 KB of SASS and every stage runs its path exactly once, so the instruction cache misses
// on most of it: code a program never executes costs time (compare instantiations with tools/ab_run.sh).
// TRACE = per-stage clock stamps compiled in (tools/stream_trace.py); the production instantiations carry none of that code.
template <unsigned FEAT, bool TRACE>
__global__ void __launch_bounds__(ST_THREADS, 1) stream_kernel(SParams P) {
#define PRO_IS(x) (((FEAT >> (x)) & 1u) != 0u && pro == (x))
#define KIND_IS(x) (((FEAT >> (16 + (x))) & 1u) != 0u && op.kind == (x))
#define ALPHA_IS(x) (((FEAT >> (24 + (x))) & 1u) != 0u && op.alpha_kind == (x))
// bit 30: every attention stage of the program has head_dim 128 -> compile-time loop bounds (the run-time-bounded loops of the 64 / 128
// generalisation cost the LM stack 13 % when they were introduced)
#define ATT_HD(a) ((((FEAT >> 30) & 1u) != 0u) ? 128 : (a).hd)
// bit 29: every linear stage of the program has a 16-row activation operand (M <= 8 rows: one prompt per GPU) -> compile-time nB
#define OP_NB(o) ((((FEAT >> 29) & 1u) != 0u) ? 16 : (o).nB)
  extern __shared__ unsigned char st_raw[];
  __shared__ unsigned long long full_bar[ST_MAX_STAGES], empty_bar[ST_MAX_STAGES];
  __shared__ float s_red[4][8];
  __shared__ float s_inv[64];
  // z' of every sample (SP_DPM); the 16-row-operand variants run B <= 4 samples and keep the smaller table
  __shared__ float s_z[(((FEAT >> 29) & 1u) != 0u ? 8 : MAX_BATCH) * 64];
  __shared__ __align__(16) unsigned char s_opbuf[2][sizeof(SOp)];
  __shared__ int s_pinfo[128];
  const unsigned raw_addr = smem_u32(st_raw);
  unsigned char* sm = st_raw + ((1024u - (raw_addr & 1023u)) & 1023u);      // 1024 B aligned (swizzle atom)
  unsigned char* ring = sm;
  unsigned char* breg = sm + (size_t)P.n_stages * ST_TILE;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NS = P.n_stages;
  const unsigned G = gridDim.x;
  // sequence state: only programs with attention stages read it (the RoPE table is a job of the LM program's QKV stage).  The other
  // families keep 16 entries, so their static shared memory -- which sets the ring depth of every codec and sampler program -- stays put.
  constexpr int NSEQ = ((FEAT >> (16 + SK_ATTN)) & 1u) != 0u ? MAX_SEQ : 16;
  __shared__ int s_kvlen[NSEQ], s_rmode[NSEQ];
  if (tid < NSEQ) {
    s_kvlen[tid] = (P.kv_len && tid < P.n_seq) ? P.kv_len[tid] : 0;
    s_rmode[tid] = (P.row_mode && tid < P.n_seq) ? P.row_mode[tid] : 0;
  }
  SeqView seq; seq.kv_len = s_kvlen; seq.row_mode = s_rmode; seq.kv_heads = P.kv_heads;

  if (tid == 0) {
    // a ring slot is free again when each of the four worker warps has seen its MMAs retire (or its attention reads end): 4 arrivals
    for (int i = 0; i < NS; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], ST_WORKERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == ST_WORKERS / 32) {
    // =============================== producer: weights only, never waits on activations ===============================
    if (lane == 0) {
      unsigned long long policy;
      asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
      unsigned it = 0, done = 0;
      const unsigned cap = (unsigned)P.max_inflight;
      auto acquire_slot = [&](int oi, unsigned bytes) -> unsigned {    // next ring slot, respecting the in-flight cap; arms its full barrier
        const unsigned slot = it % (unsigned)NS, ph = (it / (unsigned)NS) & 1u;
        while (it - done >= cap) {
          mbar_wait_wd(&full_bar[done % (unsigned)NS], (done / (unsigned)NS) & 1u, P.diag, 6u, (unsigned)oi, done);
          ++done;
        }
        mbar_wait_wd(&empty_bar[slot], ph ^ 1u, P.diag, 1u, (unsigned)oi, it);
        mbar_expect_tx(&full_bar[slot], bytes);
        ++it;
        return slot;
      };
      unsigned long long policy_kv;
      asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy_kv));
      for (int oi = 0; oi < P.n_ops; ++oi) {
        const SOp& op = P.ops[oi];
        if (KIND_IS(SK_ATTN)) {
          // K page then V page of every unit: two 64 x 64 boxes each (d 0..63, d 64..127) into one 16 KB slot
          const SAtt& a = op.att;
          AttIter ai; AttSeg sg;
          att_begin(seq, op.M, ai);
          while (att_next(seq, op.M, ai, sg)) {
            for (int t = sg.t0; t < sg.t1; ++t) {
              const int page = a.kv.page_table[(size_t)sg.m * a.kv.max_pages + t];
              const int row0 = (int)(a.row_base + (unsigned)((page * a.kv.kv_heads + sg.g) * KV_PAGE));
              const unsigned pbytes = (unsigned)(KV_PAGE * ATT_HD(a) * 2);
              unsigned slot = acquire_slot(oi, pbytes);
              tma_load_2d(ring + (size_t)slot * ST_TILE, a.tmap_k, 0, row0, &full_bar[slot], policy_kv);
              if (ATT_HD(a) > 64) tma_load_2d(ring + (size_t)slot * ST_TILE + 8192, a.tmap_k, 64, row0, &full_bar[slot], policy_kv);
              slot = acquire_slot(oi, pbytes);
              tma_load_2d(ring + (size_t)slot * ST_TILE, a.tmap_v, 0, row0, &full_bar[slot], policy_kv);
              if (ATT_HD(a) > 64) tma_load_2d(ring + (size_t)slot * ST_TILE + 8192, a.tmap_v, 64, row0, &full_bar[slot], policy_kv);
            }
          }
          continue;
        }
        if (op.kind != SK_GEMV) continue;
        unsigned u0, u1; int KB;
        st_part(op, u0, u1, KB);
        const unsigned long long tmap = op.tmap;
        for (unsigned u = u0; u < u1; ++u, ++it) {
          const unsigned slot = it % (unsigned)NS, ph = (it / (unsigned)NS) & 1u;
          // at most `cap` tiles of this CTA are in flight: the ring may be deep (it buffers ARRIVED tiles across the barriers), but every
          // request queued in the memory system delays the latency-critical activation loads and barrier traffic of the other warps
          while (it - done >= cap) {
            mbar_wait_wd(&full_bar[done % (unsigned)NS], (done / (unsigned)NS) & 1u, P.diag, 6u, (unsigned)oi, done);
            ++done;
          }
          mbar_wait_wd(&empty_bar[slot], ph ^ 1u, P.diag, 1u, (unsigned)oi, it);
          mbar_expect_tx(&full_bar[slot], (unsigned)ST_TILE);
          // tile-major weights: unit u = (row tile, k-block) is the contiguous 16 KB block u, so a CTA streams one contiguous range
          tma_load_2d(ring + (size_t)slot * ST_TILE, tmap, 0, (int)(u * 128), &full_bar[slot], policy);
        }
        if (TRACE && P.trace && (int)blockIdx.x == P.trace_cta) P.trace[(size_t)oi * ST_TRACE + 9] = clock64();
      }
    }
  } else if (warp < ST_WORKERS / 32) {
    // =============================== workers: barrier, prologue (B operand), MMA, epilogue ===============================
    const int wt = tid;                       // 0..127
    const int ww = warp;
    unsigned bar_target = 0;
    unsigned wslot = 0, wph = 0;              // ring position (the workers read K/V pages from the ring; weight tiles are only counted)
    auto ring_advance = [&](unsigned n) { const unsigned adv = wslot + n; wph ^= (adv / (unsigned)NS) & 1u; wslot = adv % (unsigned)NS; };
    // stage descriptors are copied into shared memory ONE STAGE AHEAD (cp.async): read straight from global memory, each first touch of a
    // descriptor field would be an L2/DRAM round trip on the critical path
    constexpr int OPCH = (int)(sizeof(SOp) / 16);
    if (wt < OPCH) cp_async16(s_opbuf[0] + wt * 16, reinterpret_cast<const unsigned char*>(P.ops) + wt * 16, 16);
    cp_async_commit();
    cp_async_wait<0>();
    worker_sync();
    for (int oi = 0; oi < P.n_ops; ++oi) {
      const SOp& op = *reinterpret_cast<const SOp*>(s_opbuf[oi & 1]);
      if (oi + 1 < P.n_ops && wt < OPCH)
        cp_async16(s_opbuf[(oi + 1) & 1] + wt * 16, reinterpret_cast<const unsigned char*>(P.ops + oi + 1) + wt * 16, 16);
      cp_async_commit();
      const bool tr = TRACE && P.trace && (int)blockIdx.x == P.trace_cta && wt == 0;
      if (tr) P.trace[(size_t)oi * ST_TRACE + 0] = clock64();
      // the grid barrier sits as LATE as possible inside every stage: everything that only depends on the descriptor (unit range, chunk
      // coordinates and addresses: a dozen integer divisions, ~0.6 us) is computed by the waiting workers BEFORE it
      // (arrival first: every worker's global writes of the previous stage were issued before the sync that ended it)
      if (op.sync_before) {
        bar_target += G;
        if (wt == 0) {
          if (TRACE && P.trace2) P.trace2[((size_t)oi * G + blockIdx.x) * 2] = gtime_ns();
          red_add_release_u32(P.bar_count, 1u);
        }
      }
      auto grid_barrier = [&]() {
        if (op.sync_before) {
          if (wt == 0) {
            // arrival = one fire-and-forget release reduction, then poll the counter: under the weight stream every dependent L2 round
            // trip is expensive, so the form with the fewest of them wins.
            long long t0 = 0;
            for (unsigned spins = 0; ld_acquire_u32(P.bar_count) < bar_target; ++spins) {
              if ((spins & 255u) == 255u) {
                const long long t = clock64();
                if (t0 == 0) t0 = t;
                else if (t - t0 > 6000000000ll) st_die(P.diag, 4u, (unsigned)oi, bar_target, ld_acquire_u32(P.bar_count));
              }
            }
            if (TRACE && P.trace2) P.trace2[((size_t)oi * G + blockIdx.x) * 2 + 1] = gtime_ns();
          }
          worker_sync();
        }
        if (tr) P.trace[(size_t)oi * ST_TRACE + 1] = clock64();
      };
      // zero-fill jobs for later stages and the RoPE table: anywhere between this stage's barrier and the next one
      auto side_jobs = [&]() {
        if (op.init_dst) {
          for (long long i = (long long)blockIdx.x * ST_WORKERS + wt; i < op.init_n; i += (long long)G * ST_WORKERS) op.init_dst[i] = 0.f;
        }
        if (op.init2_dst) {
          for (long long i = (long long)blockIdx.x * ST_WORKERS + wt; i < op.init2_n; i += (long long)G * ST_WORKERS) op.init2_dst[i] = 0.f;
        }
        if (op.rope_rows > 0 && (int)blockIdx.x < op.rope_rows && wt < ATT_HD(op.att) / 2) {
          const int m = blockIdx.x;
          float sn, cs;
          sincosf((float)s_kvlen[m] * op.att.inv_freq[wt], &sn, &cs);
          *reinterpret_cast<float2*>(op.att.rope_cs + ((size_t)m * (HD / 2) + wt) * 2) = make_float2(cs, sn);
        }
      };
      do {
      if (op.kind != SK_GEMV && !KIND_IS(SK_ATTN)) { grid_barrier(); side_jobs(); }
      if (KIND_IS(SK_MIX)) {
        const SCodec& w = op.cod;
        const int C = op.K, M = op.M, T = w.T_out, Bn = M / T;
        // full-row statistics of x: rows in pairs, <= 16 float4 per thread in flight
        const int K4 = C >> 2;
        for (int m0 = 0; m0 < M; m0 += 2) {
          float4 sv[2][8];
#pragma unroll
          for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int q = wt + i * ST_WORKERS;
              sv[r][i] = (m0 + r < M && q < K4) ? ldcg4(op.x + (long long)(m0 + r) * op.ldx + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
          float ss[2] = {0.f, 0.f};
#pragma unroll
          for (int r = 0; r < 2; ++r) {
#pragma unroll
            for (int i = 0; i < 8; ++i) ss[r] += sv[r][i].x * sv[r][i].x + sv[r][i].y * sv[r][i].y + sv[r][i].z * sv[r][i].z + sv[r][i].w * sv[r][i].w;
            ss[r] = warp_sum(ss[r]);
            if (lane == 0) s_red[ww][(m0 & 6) + r] = ss[r];
          }
          if (((m0 & 6) == 6) || m0 + 2 >= M) {
            worker_sync();
            const int base = m0 & ~7;
            if (wt < 8 && base + wt < M) s_inv[base + wt] = rsqrtf((s_red[0][wt] + s_red[1][wt] + s_red[2][wt] + s_red[3][wt]) / (float)C + w.eps);
            worker_sync();
          }
        }
        // this CTA's channels, one (sample, channel) item per thread: every operand requested before the first is used
        const int c0 = (int)((unsigned)C * blockIdx.x / G), c1 = (int)((unsigned)C * (blockIdx.x + 1u) / G), nc = c1 - c0;
        for (int it = wt; it < nc * Bn; it += ST_WORKERS) {
          const int b = it / nc, c = c0 + (it - b * nc);
          float hv[6], tap[7], xr[8];
#pragma unroll
          for (int j = 0; j < 6; ++j) hv[j] = ldcg1(w.hist + ((size_t)b * 6 + j) * C + c);
#pragma unroll
          for (int t = 0; t < 8; ++t) xr[t] = t < T ? ldcg1(op.x + (long long)(b * T + t) * op.ldx + c) : 0.f;
#pragma unroll
          for (int j = 0; j < 7; ++j) tap[j] = w.dw_w[(size_t)j * C + c];
          const float nw = w.norm_w[c], gm = w.gamma[c], db = w.dw_b[c];
          float win[14];                                   // [hist (6) ; xn (T <= 8)]
#pragma unroll
          for (int j = 0; j < 6; ++j) win[j] = hv[j];
#pragma unroll
          for (int t = 0; t < 8; ++t) win[6 + t] = t < T ? xr[t] * s_inv[b * T + t] * nw : 0.f;
#pragma unroll
          for (int r = 0; r < 6; ++r) {                      // next history = window rows T .. T+5
            float val = 0.f;
#pragma unroll
            for (int q = 0; q < 14; ++q) if (q == T + r) val = win[q];
            w.next[((size_t)b * 6 + r) * C + c] = val;
          }
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            if (t < T) {
              float acc = db;
#pragma unroll
              for (int j = 0; j < 7; ++j) acc = fmaf(tap[j], win[t + j], acc);
              w.x1_out[(size_t)(b * T + t) * C + c] = xr[t] + gm * acc;
            }
          }
        }
        break;
      }
      if (KIND_IS(SK_ATTN)) {
        // =========================== decode attention over the ring (see SAtt) ===========================
        const SAtt& a = op.att;
        const unsigned U = att_vtotal(seq, op.M);
        const int Gq = a.kv.q_heads / a.kv.kv_heads, nkv = a.kv.kv_heads;
        const int hd = ATT_HD(a), hh2 = hd >> 1, nks = hd >> 4;                         // head_dim, RoPE half, 16-wide k / d steps
        bf16 (*Qs)[AT2_LD] = reinterpret_cast<bf16 (*)[AT2_LD]>(breg);              // [16][136]: rows 0..7 hi, 8..15 lo of the G query heads
        bf16* knew = reinterpret_cast<bf16*>(breg + 16 * AT2_LD * 2);
        bf16* vnew = knew + HD;
        float* mo = reinterpret_cast<float*>(breg + 8192);                          // [4 warps][8 heads][128]
        float* mlw = mo + 4 * 8 * HD;                                               // [4][8][2]
        AttIter ai; AttSeg sg;
        att_begin(seq, op.M, ai);
        bool have = att_next(seq, op.M, ai, sg);                                    // partition arithmetic: ahead of the barrier
        { int hv_ = have; asm volatile("" : "+r"(hv_), "+r"(sg.m), "+r"(sg.g), "+r"(sg.t0), "+r"(sg.t1), "+r"(sg.nt), "+r"(sg.vf)); have = hv_ != 0; }
        grid_barrier();
        side_jobs();
        bool first_seg = true;
        for (; have; have = att_next(seq, op.M, ai, sg)) {
          const int m = sg.m, g = sg.g, t = sg.t0, t_end = sg.t1;
          const unsigned nt = sg.nt;
          const int pos = s_kvlen[m], L = pos + 1;
          const bool owner = (t_end == (int)nt);                                    // this CTA holds the page of the newest token
          const float* row = a.qkv + (size_t)m * (a.kv.q_heads + 2 * nkv) * hd;
          for (int i = wt; i < 8 * hh2; i += ST_WORKERS) {
            const int h = i / hh2, d = i - h * hh2;
            float o1 = 0.f, o2 = 0.f;
            if (h < Gq) {
              const float2 csn = __ldcg(reinterpret_cast<const float2*>(a.rope_cs + ((size_t)m * (HD / 2) + d) * 2));
              const float cs = csn.x, sn = csn.y;
              const float x1 = ldcg1(row + (g * Gq + h) * hd + d), x2 = ldcg1(row + (g * Gq + h) * hd + d + hh2);
              o1 = (x1 * cs - x2 * sn) * a.scale;
              o2 = (x2 * cs + x1 * sn) * a.scale;
            }
            const bf16 h1 = __float2bfloat16_rn(o1), h2 = __float2bfloat16_rn(o2);
            Qs[h][d] = h1; Qs[h][d + hh2] = h2;
            Qs[h + 8][d] = __float2bfloat16_rn(o1 - __bfloat162float(h1));
            Qs[h + 8][d + hh2] = __float2bfloat16_rn(o2 - __bfloat162float(h2));
          }
          if (owner) {                                                              // rotate k, round K / V to bf16, append to the pool
            const int page = a.kv.page_table[(size_t)m * a.kv.max_pages + pos / KV_PAGE];
            const size_t oo = (((size_t)page * nkv + g) * KV_PAGE + (pos % KV_PAGE)) * hd;
            if (wt < hh2) {
              const int d = wt;
              const float2 csn = __ldcg(reinterpret_cast<const float2*>(a.rope_cs + ((size_t)m * (HD / 2) + d) * 2));
              const float cs = csn.x, sn = csn.y;
              const float x1 = ldcg1(row + (a.kv.q_heads + g) * hd + d), x2 = ldcg1(row + (a.kv.q_heads + g) * hd + d + hh2);
              const bf16 k1 = __float2bfloat16_rn(x1 * cs - x2 * sn), k2 = __float2bfloat16_rn(x2 * cs + x1 * sn);
              knew[d] = k1; knew[d + hh2] = k2;
              a.kv.kpool[oo + d] = k1; a.kv.kpool[oo + d + hh2] = k2;
            } else {
              for (int d = wt - hh2; d < hd; d += ST_WORKERS - hh2) {
                const bf16 vv_ = __float2bfloat16_rn(ldcg1(row + (a.kv.q_heads + nkv + g) * hd + d));
                vnew[d] = vv_;
                a.kv.vpool[oo + d] = vv_;
              }
            }
          }
          worker_sync();
          if (tr && first_seg) P.trace[(size_t)oi * ST_TRACE + 2] = clock64();
          unsigned qa[8][4];
#pragma unroll
          for (int ks = 0; ks < 8; ++ks) if (ks < nks) ldmatrix_x4(qa[ks], &Qs[lane & 15][ks * 16 + (lane >> 4) * 8]);
          float o[16][4];
#pragma unroll
          for (int i = 0; i < 16; ++i) { o[i][0] = 0.f; o[i][1] = 0.f; o[i][2] = 0.f; o[i][3] = 0.f; }
          float m_run = -INFINITY, l_run = 0.f;
          for (int tt = t; tt < t_end; ++tt) {
            const int tok0 = tt * KV_PAGE;
            const unsigned slotK = wslot, phK = wph;
            ring_advance(1);
            const unsigned slotV = wslot, phV = wph;
            ring_advance(1);
            unsigned char* Ks = ring + (size_t)slotK * ST_TILE;
            unsigned char* Vs = ring + (size_t)slotV * ST_TILE;
            mbar_wait_wd(&full_bar[slotK], phK, P.diag, 7u, (unsigned)oi, (unsigned)tt);
            const bool splice = owner && tt == (int)nt - 1;
            if (splice) {                          // the page was fetched before (or while) the new row was written: patch it in shared memory
              mbar_wait_wd(&full_bar[slotV], phV, P.diag, 7u, (unsigned)oi, (unsigned)tt);
              if (wt < hd) {
                *reinterpret_cast<bf16*>(Ks + kv_off(pos - tok0, wt)) = knew[wt];
                *reinterpret_cast<bf16*>(Vs + kv_off(pos - tok0, wt)) = vnew[wt];
              }
              worker_sync();
            }
            float sa[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
              if (ks < nks) {
                unsigned kb[4];
                ldmatrix_x4(kb, Ks + kv_off(ww * 16 + (lane & 7) + ((lane >> 4) << 3), ks * 16 + ((lane >> 3) & 1) * 8));
                mma_bf16_16816(sa[0], qa[ks], kb[0], kb[1]);
                mma_bf16_16816(sa[1], qa[ks], kb[2], kb[3]);
              }
            }
            const int tb = tok0 + ww * 16 + (lane & 3) * 2;
            float sv[4] = {sa[0][0] + sa[0][2], sa[0][1] + sa[0][3], sa[1][0] + sa[1][2], sa[1][1] + sa[1][3]};
            if (tb >= L) sv[0] = -INFINITY;
            if (tb + 1 >= L) sv[1] = -INFINITY;
            if (tb + 8 >= L) sv[2] = -INFINITY;
            if (tb + 9 >= L) sv[3] = -INFINITY;
            float mt = fmaxf(fmaxf(sv[0], sv[1]), fmaxf(sv[2], sv[3]));
            mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
            mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
            const float mn = fmaxf(m_run, mt);
            const float msafe = (mn == -INFINITY) ? 0.f : mn;
            float pv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) pv[i] = __expf(sv[i] - msafe);
            const float corr = __expf(m_run - msafe);
            float rs = pv[0] + pv[1] + pv[2] + pv[3];
            rs += __shfl_xor_sync(0xffffffffu, rs, 1);
            rs += __shfl_xor_sync(0xffffffffu, rs, 2);
            l_run = l_run * corr + rs;
            m_run = mn;
#pragma unroll
            for (int i = 0; i < 16; ++i) { o[i][0] *= corr; o[i][1] *= corr; o[i][2] *= corr; o[i][3] *= corr; }
            float ph_[4], pl_[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { ph_[i] = __bfloat162float(__float2bfloat16_rn(pv[i])); pl_[i] = pv[i] - ph_[i]; }
            unsigned pa[4] = {pack_bf16(ph_[0], ph_[1]), pack_bf16(pl_[0], pl_[1]), pack_bf16(ph_[2], ph_[3]), pack_bf16(pl_[2], pl_[3])};
            if (!splice) mbar_wait_wd(&full_bar[slotV], phV, P.diag, 7u, (unsigned)oi, (unsigned)tt);
#pragma unroll
            for (int np = 0; np < 8; ++np) {
              if (np < nks) {
                unsigned vb[4];
                ldmatrix_x4_trans(vb, Vs + kv_off(ww * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, np * 16 + (lane >> 4) * 8));
                mma_bf16_16816(o[2 * np], pa, vb[0], vb[1]);
                mma_bf16_16816(o[2 * np + 1], pa, vb[2], vb[3]);
              }
            }
            if (splice) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            worker_sync();                         // all four warps are done with both pages
            if (lane == 0) { mbar_arrive(&empty_bar[slotK]); mbar_arrive(&empty_bar[slotV]); }
          }
          if (tr && first_seg) P.trace[(size_t)oi * ST_TRACE + 3] = clock64();
          // merge the 4 warps' (m, l, O) and publish this segment's partial
          const int h = lane >> 2;
#pragma unroll
          for (int ntl = 0; ntl < 16; ++ntl) {
            if (ntl < 2 * nks) {
              const int d = ntl * 8 + (lane & 3) * 2;
              mo[(ww * 8 + h) * HD + d] = o[ntl][0] + o[ntl][2];
              mo[(ww * 8 + h) * HD + d + 1] = o[ntl][1] + o[ntl][3];
            }
          }
          if ((lane & 3) == 0) { mlw[(ww * 8 + h) * 2] = m_run; mlw[(ww * 8 + h) * 2 + 1] = l_run; }
          worker_sync();
          const unsigned pslot = blockIdx.x - cta_of_unit(sg.vf + ST_ATT_SEGW, U, G);      // first CTA that holds pages of this group
          const size_t pbase = (((size_t)m * nkv + g) * G + pslot) * 8;
          for (int hh = 0; hh < Gq; ++hh) {
            float mx = -INFINITY;
#pragma unroll
            for (int w = 0; w < 4; ++w) mx = fmaxf(mx, mlw[(w * 8 + hh) * 2]);
            float num = 0.f, den = 0.f;
#pragma unroll
            for (int w = 0; w < 4; ++w) {
              const float mw = mlw[(w * 8 + hh) * 2];
              const float wgt = (mw == -INFINITY) ? 0.f : __expf(mw - mx);
              num = fmaf(wgt, mo[(w * 8 + hh) * HD + wt], num);
              den = fmaf(wgt, mlw[(w * 8 + hh) * 2 + 1], den);
            }
            if (wt < hd) a.part_acc[(pbase + hh) * HD + wt] = num;
            if (wt == 0) { a.part_ml[(pbase + hh) * 2] = mx; a.part_ml[(pbase + hh) * 2 + 1] = den; }
          }
          worker_sync();
          if (tr && first_seg) P.trace[(size_t)oi * ST_TRACE + 4] = clock64();
          first_seg = false;
        }
        if (tr) P.trace[(size_t)oi * ST_TRACE + 5] = clock64();
        break;
      }
      if (op.kind != SK_GEMV) break;
      unsigned u0, u1; int KB;
      st_part(op, u0, u1, KB);
      const unsigned mslot = wslot, mph = wph;          // ring position of this stage's first weight tile
      ring_advance(u1 - u0);
      if (u0 == u1) { grid_barrier(); side_jobs(); break; }
      const int M = op.M, K = op.K, N = op.N, nB = OP_NB(op), half = nB >> 1;
      const int units = (int)(u1 - u0);
      const int count = units < KB ? units : KB;          // k-blocks of activations this CTA needs (contiguous mod KB from kb_first)
      const int rt_first = (int)(u0 / (unsigned)KB), kb_first = (int)(u0 - (unsigned)rt_first * (unsigned)KB);
      const int pro = op.pro;
      // ---------------- prologue: ONE batch of L2 loads (row statistics + the first activation chunks), then compute ----------------
      // (a statistics loop followed by a staging loop would cost one L2 round trip per loop iteration; every load below is issued before
      //  the first value is consumed)
      const int total = M * count * 8;                     // 16-byte chunks (8 consecutive k of one activation row) to stage
      const bool norm = (PRO_IS(SP_RMSNORM) || PRO_IS(SP_ADALN));
      // SP_COMBINE scratch behind the B operand: [M][NH][G] merge weights w_p / sum_p w_p l_p | group partial sums | merged[M][count][64]
      const int cmb_base = (count * nB * 128 + 1023) & ~1023;
      float* s_w = reinterpret_cast<float*>(breg + cmb_base);
      const int cmb_kbh = (PRO_IS(SP_COMBINE) ? ATT_HD(op.att) : 128) >> 6;     // k-blocks per head (head_dim 128: two, 64: one)
      const int cmb_nh = ((kb_first % cmb_kbh) + count - 1) / cmb_kbh + 1;   // distinct heads among this CTA's k-blocks
      const int cmb_off = cmb_base + ((M * cmb_nh * (int)G * 4 + 15) & ~15);
      const int cmb_part = (M * count * 256 > 2048) ? M * count * 256 : 2048;     // bytes of the group partial sums (npg * out4 float4)
      struct ChunkRef { const float* xr; const float* pw; const float* psc; const float* psh; int m, jloc, ch, k; bool valid, live, fresh; };
      auto chunk_ref = [&](int c) -> ChunkRef {             // coordinates + source address of chunk c: descriptor-only arithmetic
        ChunkRef r;
        r.m = c / (count * 8);
        const int q = c - r.m * (count * 8);
        r.jloc = q >> 3; r.ch = q & 7;
        int kb = kb_first + r.jloc; if (kb >= KB) kb -= KB;
        r.k = kb * 64 + r.ch * 8;
        r.valid = c < total;
        r.live = r.valid && r.k < K && !PRO_IS(SP_DPM) && !PRO_IS(SP_COMBINE);
        r.fresh = false;
        r.xr = op.x; r.pw = nullptr; r.psc = nullptr; r.psh = nullptr;
        if (!r.live) return r;
        const int ka = r.k + op.k0;                          // column of the full row (r.k: column of this stage's slice)
        if (PRO_IS(SP_WINDOW)) {
          const SCodec& w = op.cod;
          const int b = r.m / w.T_out, t = r.m - b * w.T_out, j = ka / w.cin, ci = ka - j * w.cin, rr = t * w.stride + j;
          r.fresh = rr >= w.ctx;
          r.xr = rr < w.ctx ? w.hist + ((size_t)b * w.ctx + rr) * w.cin + ci : w.src + ((size_t)b * w.T_in + (rr - w.ctx)) * w.cin + ci;
        } else if (PRO_IS(SP_SWIGLU)) {
          r.xr = op.x + (long long)r.m * op.ldx + 2 * ka;
        } else {
          r.xr = op.x + (long long)r.m * op.ldx + ka;
          if (norm && op.pro_w) r.pw = op.pro_w + ka;
          if (PRO_IS(SP_ADALN)) {
            const long long o = (long long)r.m * op.pro_ld + ka;
            r.psc = op.pro_scale + o; r.psh = op.pro_shift + o;
          }
        }
        return r;
      };
      auto chunk_load = [&](const ChunkRef& r, float4* in) {            // raw operands of one chunk (nothing is consumed here)
        if (!r.live) return;
        const float* xr = r.xr;
        const int m = r.m, k = r.k;
        if (PRO_IS(SP_WINDOW)) {
          in[0] = ldcg4(xr); in[1] = ldcg4(xr + 4);
          return;
        }
        if (PRO_IS(SP_SWIGLU)) {
          in[0] = ldcg4(xr); in[1] = ldcg4(xr + 4); in[2] = ldcg4(xr + 8); in[3] = ldcg4(xr + 12);
          return;
        }
        in[0] = ldcg4(xr); in[1] = ldcg4(xr + 4);
        if (norm) {
          if (r.pw) { in[2] = *reinterpret_cast<const float4*>(r.pw); in[3] = *reinterpret_cast<const float4*>(r.pw + 4); }
          else { in[2] = make_float4(1.f, 1.f, 1.f, 1.f); in[3] = in[2]; }
        }
        if (PRO_IS(SP_ADALN)) {
          in[4] = ldcg4(r.psc); in[5] = ldcg4(r.psc + 4);
          in[6] = ldcg4(r.psh); in[7] = ldcg4(r.psh + 4);
        }
      };
      auto chunk_store = [&](const ChunkRef& r, const float4* in) {
        if (!r.valid) return;
        const int m = r.m, jloc = r.jloc, ch = r.ch, k = r.k;
        float v[8];
        if (k >= K) {
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = 0.f;          // k >= K: the weight tile is zero there, keep 0 * x finite
        } else if (PRO_IS(SP_SWIGLU)) {
          v[0] = silu_f(in[0].x) * in[0].y; v[1] = silu_f(in[0].z) * in[0].w; v[2] = silu_f(in[1].x) * in[1].y; v[3] = silu_f(in[1].z) * in[1].w;
          v[4] = silu_f(in[2].x) * in[2].y; v[5] = silu_f(in[2].z) * in[2].w; v[6] = silu_f(in[3].x) * in[3].y; v[7] = silu_f(in[3].z) * in[3].w;
        } else if (PRO_IS(SP_DPM)) {
          const float* zr = s_z + (m % op.dpm.B) * 64 + k;
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = zr[j];
        } else if (PRO_IS(SP_WINDOW)) {
          const SCodec& w = op.cod;
          v[0] = in[0].x; v[1] = in[0].y; v[2] = in[0].z; v[3] = in[0].w; v[4] = in[1].x; v[5] = in[1].y; v[6] = in[1].z; v[7] = in[1].w;
          if (r.fresh) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) v[jj] = v[jj] * w.alpha + w.beta;
          }
        } else if (PRO_IS(SP_COMBINE)) {
          const float* cv = reinterpret_cast<const float*>(breg + cmb_off + cmb_part) + ((size_t)(m * count + jloc) * 64 + ch * 8);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = cv[j];
        } else {
          v[0] = in[0].x; v[1] = in[0].y; v[2] = in[0].z; v[3] = in[0].w; v[4] = in[1].x; v[5] = in[1].y; v[6] = in[1].z; v[7] = in[1].w;
          if (norm) {
            const float inv = s_inv[m];
            const float w[8] = {in[2].x, in[2].y, in[2].z, in[2].w, in[3].x, in[3].y, in[3].z, in[3].w};
            if (PRO_IS(SP_RMSNORM)) {
#pragma unroll
              for (int j = 0; j < 8; ++j) v[j] *= inv * w[j];
            } else {
              const float sc[8] = {in[4].x, in[4].y, in[4].z, in[4].w, in[5].x, in[5].y, in[5].z, in[5].w};
              const float sh[8] = {in[6].x, in[6].y, in[6].z, in[6].w, in[7].x, in[7].y, in[7].z, in[7].w};
#pragma unroll
              for (int j = 0; j < 8; ++j) v[j] = v[j] * inv * w[j] * (1.f + sc[j]) + sh[j];
            }
          } else if (PRO_IS(SP_GELU)) {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = gelu_erf_f(v[j]);
          } else if (PRO_IS(SP_SILU)) {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = silu_f(v[j]);
          }
        }
        float h[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] = __bfloat162float(__float2bfloat16_rn(v[j]));
        const uint4 hv = make_uint4(pack_bf16(h[0], h[1]), pack_bf16(h[2], h[3]), pack_bf16(h[4], h[5]), pack_bf16(h[6], h[7]));
        const uint4 lv = make_uint4(pack_bf16(v[0] - h[0], v[1] - h[1]), pack_bf16(v[2] - h[2], v[3] - h[3]),
                                    pack_bf16(v[4] - h[4], v[5] - h[5]), pack_bf16(v[6] - h[6], v[7] - h[7]));
        unsigned char* blk = breg + (size_t)jloc * (size_t)(nB * 128);
        const int rl = half + m;
        *reinterpret_cast<uint4*>(blk + (m >> 3) * 1024 + (m & 7) * 128 + ((ch ^ (m & 7)) << 4)) = hv;
        *reinterpret_cast<uint4*>(blk + (rl >> 3) * 1024 + (rl & 7) * 128 + ((ch ^ (rl & 7)) << 4)) = lv;
      };
      ChunkRef r0 = chunk_ref(wt), r1 = chunk_ref(wt + ST_WORKERS);
      const int K4 = op.krow >> 2;                          // row statistics: the whole row, also in a K-split slice
      int rot = (int)((blockIdx.x * 67u) % (unsigned)(K4 > 0 ? K4 : 1));     // statistics loads: every CTA starts at a different column
      // materialise the descriptor-only values HERE, ahead of the barrier (the compiler would otherwise sink them to their first use)
      asm volatile("" : "+l"(r0.xr), "+r"(r0.m), "+r"(r0.k), "+r"(r0.jloc), "+l"(r1.xr), "+r"(r1.m), "+r"(r1.k), "+r"(r1.jloc), "+r"(rot));
      if (norm) asm volatile("" : "+l"(r0.pw), "+l"(r0.psc), "+l"(r0.psh), "+l"(r1.pw), "+l"(r1.psc), "+l"(r1.psh));
      // attention merge: the (row, head) a warp merges first and the first accumulator item of every thread, again descriptor-only
      const bool cmb = PRO_IS(SP_COMBINE);
      const unsigned Ua = cmb ? att_vtotal(seq, M) : 1u;
      const int cmb_Gq = cmb ? op.att.kv.q_heads / op.att.kv.kv_heads : 1, cmb_nkv = cmb ? op.att.kv.kv_heads : 1;
      // a K-split slice covers whole heads [h0, h0 + KB / cmb_kbh); a CTA's k-blocks wrap around inside the slice
      const int cmb_h0 = op.k0 / (cmb_kbh * 64), cmb_hs = KB / cmb_kbh;
      struct CmbPrep { const float* ml; unsigned c_first; int Pn; };
      auto cmb_prep = [&](int pi) -> CmbPrep {
        const SAtt& a = op.att;
        const int m = pi / cmb_nh, hid = pi - m * cmb_nh;
        const int h = cmb_h0 + ((kb_first / cmb_kbh) + hid) % cmb_hs, g = h / cmb_Gq, hh = h - g * cmb_Gq;
        unsigned pre = 0;
        for (int mm = 0; mm < m; ++mm) { const unsigned n2 = att_tiles(seq, mm); if (n2) pre += (n2 + ST_ATT_SEGW) * (unsigned)cmb_nkv; }
        const unsigned nt = att_tiles(seq, m);
        CmbPrep r; r.ml = a.part_ml; r.c_first = 0; r.Pn = 0;
        if (nt) {
          const unsigned first = pre + (unsigned)g * (nt + ST_ATT_SEGW) + ST_ATT_SEGW;      // virtual unit of page 0 of this group
          r.c_first = cta_of_unit(first, Ua, G);
          r.Pn = (int)(cta_of_unit(first + nt - 1u, Ua, G) - r.c_first) + 1;
          r.ml = a.part_ml + ((((size_t)m * cmb_nkv + g) * G) * 8 + hh) * 2;                 // slot stride 16 floats
        }
        return r;
      };
      struct CmbItem { const float* ap; int o4, pg, pi; };
      const int out4 = M * count * 16;
      int npg = 1;
      while (npg * 2 * out4 <= ST_WORKERS && npg < 8) npg *= 2;
      auto cmb_item = [&](int w0) -> CmbItem {
        const SAtt& a = op.att;
        CmbItem r;
        r.o4 = w0 % out4; r.pg = w0 / out4;
        const int m = r.o4 / (count * 16), q = r.o4 - m * (count * 16), jloc = q >> 4, q4 = q & 15;
        int kb = kb_first + jloc; if (kb >= KB) kb -= KB;
        const int k = op.k0 + kb * 64 + q4 * 4, h = k / ATT_HD(a), d = k - h * ATT_HD(a), g = h / cmb_Gq, hh = h - g * cmb_Gq;
        r.pi = m * cmb_nh + ((kb_first % cmb_kbh) + jloc) / cmb_kbh;
        r.ap = a.part_acc + ((((size_t)m * cmb_nkv + g) * G) * 8 + hh) * HD + d;             // slot stride 8 * 128 floats
        return r;
      };
      CmbPrep cp0; cp0.ml = nullptr; cp0.c_first = 0; cp0.Pn = 0;
      CmbItem ci0; ci0.ap = nullptr; ci0.o4 = 0; ci0.pg = 0; ci0.pi = 0;
      if (cmb) {
        if (ww < M * cmb_nh) cp0 = cmb_prep(ww);
        if (wt < out4 * npg) ci0 = cmb_item(wt);
        asm volatile("" : "+l"(cp0.ml), "+r"(cp0.c_first), "+r"(cp0.Pn), "+l"(ci0.ap), "+r"(ci0.o4), "+r"(ci0.pg), "+r"(ci0.pi));
      }
      grid_barrier();
      if (cmb) {
        const bool all_live = Ua >= G;                                        // every CTA owns at least one attention unit (long contexts)
        for (int pi = ww; pi < M * cmb_nh; pi += 4) {                     // one warp per (row, head)
          const CmbPrep cp = (pi == ww) ? cp0 : cmb_prep(pi);
          const int Pn = cp.Pn;
          float* wrow = s_w + (size_t)pi * G;
          if (Pn) {
            const unsigned c_first = cp.c_first;
            const float* ml = cp.ml;
            float2 mlv[8];                                                                // (max, sum) of slots lane, lane + 32, ...: ONE round trip
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int pq = lane + 32 * i;
              // slots of CTAs whose unit range is empty (fewer units than CTAs: short contexts) are never written: skip them
              const unsigned cc = c_first + (unsigned)pq;
              const bool live = pq < Pn && (all_live || (Ua * cc / G != Ua * (cc + 1u) / G));
              mlv[i] = live ? __ldcg(reinterpret_cast<const float2*>(ml + (size_t)pq * 16)) : make_float2(-INFINITY, 0.f);
            }
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < 8; ++i) mx = fmaxf(mx, mlv[i].x);
            mx = warp_max(mx);
            float den = 0.f, wv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              wv[i] = (mlv[i].x == -INFINITY) ? 0.f : __expf(mlv[i].x - mx);
              den = fmaf(wv[i], mlv[i].y, den);
            }
            den = warp_sum(den);
            const float rden = 1.f / den;
#pragma unroll
            for (int i = 0; i < 8; ++i) { const int pq = lane + 32 * i; if (pq < Pn) wrow[pq] = wv[i] * rden; }
          }
          if (lane == 0) s_pinfo[pi] = Pn;
        }
        worker_sync();
        // merged[m][jloc][64] = sum_p w_p acc_p: work items (output float4, partial group) over all 128 threads, <= 16 loads in flight each
        float4* s_cpart = reinterpret_cast<float4*>(breg + cmb_off);       // [npg][out4], npg * out4 <= 128
        for (int w0 = wt; w0 < out4 * npg; w0 += ST_WORKERS) {
          const CmbItem ci = (w0 == wt) ? ci0 : cmb_item(w0);
          const int o4 = ci.o4, pg = ci.pg, pi = ci.pi;
          const int Pn = s_pinfo[pi];
          const float* wrow = s_w + (size_t)pi * G;
          const float* ap = ci.ap;
          float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int p0 = pg; p0 < Pn; p0 += 16 * npg) {
            float4 v[16];
            float wv[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const int pq = p0 + i * npg;
              wv[i] = pq < Pn ? wrow[pq] : 0.f;                 // weight 0 = absent / empty slot: its accumulator is never read
              v[i] = wv[i] != 0.f ? ldcg4(ap + (size_t)pq * (8 * HD)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const float w = wv[i];
              acc.x = fmaf(w, v[i].x, acc.x); acc.y = fmaf(w, v[i].y, acc.y); acc.z = fmaf(w, v[i].z, acc.z); acc.w = fmaf(w, v[i].w, acc.w);
            }
          }
          s_cpart[pg * out4 + o4] = acc;
        }
        worker_sync();
        float4* s_comb = reinterpret_cast<float4*>(breg + cmb_off + cmb_part);  // [M][count][16] float4
        for (int o4 = wt; o4 < out4; o4 += ST_WORKERS) {
          float4 acc = s_cpart[o4];
          for (int pg = 1; pg < npg; ++pg) { const float4 t4 = s_cpart[pg * out4 + o4]; acc.x += t4.x; acc.y += t4.y; acc.z += t4.z; acc.w += t4.w; }
          s_comb[o4] = acc;
        }
        worker_sync();
      }
      if (PRO_IS(SP_WINDOW) && u0 == 0) {                               // owner: next history = last ctx rows of every sample's window
        const SCodec& w = op.cod;
        const int per = w.ctx * w.cin, nrow = w.ctx + w.T_in;
        for (int i = wt; i < (M / w.T_out) * per; i += ST_WORKERS) {
          const int b = i / per, q = i - b * per, rr = q / w.cin, ci = q - rr * w.cin, r = nrow - w.ctx + rr;
          w.next[i] = r < w.ctx ? ldcg1(w.hist + ((size_t)b * w.ctx + r) * w.cin + ci)
                                : ldcg1(w.src + ((size_t)b * w.T_in + (r - w.ctx)) * w.cin + ci) * w.alpha + w.beta;
        }
      }
      float4 in0[8], in1[8];
      chunk_load(r0, in0);                                  // first chunks of this thread: in flight during the statistics
      chunk_load(r1, in1);
      if (tr) P.trace[(size_t)oi * ST_TRACE + 10] = clock64();
      if (norm) {
        // sum of squares of every full row: rows in pairs, <= 16 float4 per thread in flight (K <= 4096), further columns looped
        // (rot: every CTA starts at a different column -- all SMs read the same rows at the same moment, in phase they queue on the
        //  same L2 lines)
        const float* const sx = op.x; const long long sldx = op.ldx;
        for (int m0 = 0; m0 < M; m0 += 2) {
          float4 sv[2][8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int q = wt + i * ST_WORKERS;
            int qr = q + rot; if (qr >= K4) qr -= K4;
            const float* sp = sx + (long long)m0 * sldx + 4 * qr;
            sv[0][i] = q < K4 ? ldcg4(sp) : make_float4(0.f, 0.f, 0.f, 0.f);
            sv[1][i] = (m0 + 1 < M && q < K4) ? ldcg4(sp + sldx) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
          float ss[2] = {0.f, 0.f};
#pragma unroll
          for (int r = 0; r < 2; ++r) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              ss[r] += sv[r][i].x * sv[r][i].x + sv[r][i].y * sv[r][i].y + sv[r][i].z * sv[r][i].z + sv[r][i].w * sv[r][i].w;
            }
            if (m0 + r < M)
              for (int q = wt + 8 * ST_WORKERS; q < K4; q += ST_WORKERS) {
                int qr = q + rot; if (qr >= K4) qr -= K4;
                const float4 v = ldcg4(sx + (long long)(m0 + r) * sldx + 4 * qr);
                ss[r] += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
              }
            ss[r] = warp_sum(ss[r]);
            if (lane == 0) s_red[ww][(m0 & 6) + r] = ss[r];
          }
          if (tr && m0 == 0) P.trace[(size_t)oi * ST_TRACE + 11] = clock64();
          if (((m0 & 6) == 6) || m0 + 2 >= M) {             // flush every 8 rows (s_red holds 8 rows)
            worker_sync();
            const int base = m0 & ~7;
            if (wt < 8 && base + wt < M) s_inv[base + wt] = rsqrtf((s_red[0][wt] + s_red[1][wt] + s_red[2][wt] + s_red[3][wt]) / (float)op.krow + op.pro_eps);
            worker_sync();
          }
        }
      } else if (PRO_IS(SP_DPM)) {
        // z' for every sample (formula at SDpm); every CTA with work recomputes it, the owner of unit 0 publishes
        const SDpm& d = op.dpm;
        for (int i = wt; i < d.B * 64; i += ST_WORKERS) {
          const int b = i >> 6, e = i & 63;
          float zn, x0 = 0.f;
          if (d.step < 0) {
            zn = ldcg1(d.noise + i);
          } else {
            const DpmCoef c = d.rows[(size_t)d.step * d.B + b];
            const float cfg = ldcg1(d.cfg_p + b);
            const float vc = ldcg1(d.v + (size_t)b * 64 + e), vu = ldcg1(d.v + (size_t)(d.B + b) * 64 + e);
            const float vv_ = vu + cfg * (vc - vu);
            const float zo = ldcg1(d.z_in + i);
            x0 = c.a0 * zo - c.s0 * vv_;
            zn = c.ks * zo - c.kx * x0;
            if (c.order == 2) zn -= 0.5f * c.kx * (c.rinv * (x0 - ldcg1(d.x0_in + i)));
            if (d.step_noise) zn += c.kn * ldcg1(d.step_noise + ((size_t)d.step * d.B + b) * 64 + e);
          }
          s_z[i] = zn;
          if (u0 == 0) {                       // exactly one CTA owns unit 0 of the stage
            d.z_out[i] = zn; d.x0_out[i] = x0;
            if (d.latent_out) d.latent_out[i] = zn;
          }
        }
        worker_sync();
      }
      if (tr) P.trace[(size_t)oi * ST_TRACE + 2] = clock64();
      chunk_store(r0, in0);
      chunk_store(r1, in1);
#pragma unroll 1
      for (int c = wt + 2 * ST_WORKERS; c < total; c += 2 * ST_WORKERS) {
        r0 = chunk_ref(c); r1 = chunk_ref(c + ST_WORKERS);
        chunk_load(r0, in0);
        chunk_load(r1, in1);
        chunk_store(r0, in0);
        chunk_store(r1, in1);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy smem writes -> visible to the tensor core
      worker_sync();
      if (tr) P.trace[(size_t)oi * ST_TRACE + 3] = clock64();
      side_jobs();
      {
        StEpi ep;
        ep.bias = op.bias; ep.alpha = op.alpha; ep.y = op.y; ep.lda = op.lda; ep.ldy = op.ldy;
        ep.gate = ALPHA_IS(SA_GATE); ep.gamma = ALPHA_IS(SA_GAMMA); ep.store = op.store != 0;
        long long* const trs = tr ? P.trace + (size_t)oi * ST_TRACE : nullptr;
        if (nB == 16) st_mma_epilogue<16>(ring, breg, full_bar, empty_bar, NS, mslot, mph, u0, u1, KB, M, N, ep, P.diag, oi, trs);
        else if (nB == 32) st_mma_epilogue<32>(ring, breg, full_bar, empty_bar, NS, mslot, mph, u0, u1, KB, M, N, ep, P.diag, oi, trs);
        else st_mma_epilogue<64>(ring, breg, full_bar, empty_bar, NS, mslot, mph, u0, u1, KB, M, N, ep, P.diag, oi, trs);
      }
      if (tr) P.trace[(size_t)oi * ST_TRACE + 5] = clock64();
      } while (0);
      cp_async_wait<0>();                      // next stage's descriptor has landed ...
      worker_sync();                           // ... for every worker; also: all workers' global writes of this stage are issued
    }
  }
}
#undef PRO_IS
#undef KIND_IS
#undef ALPHA_IS
#undef ATT_HD
#undef OP_NB


}  // namespace vv
