// vv_runtime.cu -- native runtime behind include/vibevoice_b200.h: weight registry + repacker,
// paged KV allocator, streaming-codec state slab, per-frame kernel programs (CUDA-graph cached).
//
// The reference owns none of this (it is eager PyTorch + HF DynamicCache + python dict caches:
// modeling_vibevoice_inference.py:367-695, modular_vibevoice_tokenizer.py:193-256); SURVEY 8b
// sketches the C ABI this file implements.
#include "../../include/vibevoice_b200.h"
#include "vv_kernels.cuh"
#include "vv_stream.cuh"
#include "vv_voice.cuh"
#include "vv_prefill.cuh"

#include <cuda.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <initializer_list>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <tuple>
#include <vector>

using namespace vv;

static thread_local std::string g_err;
static int fail(int code, const char* fmt, ...) {
  char buf[2048];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define CK(expr)                                                                                     \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    if (_e != cudaSuccess) return fail(VV_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
  } while (0)
#define CKL() CK(cudaGetLastError())
#define RET(expr)            \
  do {                       \
    int _r = (expr);         \
    if (_r < 0) return _r;   \
  } while (0)

struct RawTensor {
  void* p = nullptr;
  std::vector<int64_t> shape;
  bool is_f32 = false;
  size_t numel = 0;
};

struct Block {            // Block1D (tokenizer.py:620-684)
  int C = 0;
  float *norm_w = nullptr, *dw_w = nullptr, *dw_b = nullptr, *gamma = nullptr, *ffn_norm_w = nullptr, *b1 = nullptr, *b2 = nullptr,
        *ffn_gamma = nullptr;
  bf16 *w1 = nullptr, *w2 = nullptr;
  float *hist = nullptr, *next = nullptr;   // [B][6][C]
};
struct ConvL {             // stem / downsample / upsample / head conv in window-GEMV form
  int Cin = 0, Cout = 0, k = 0, stride = 1, ctx = 0, N = 0, K = 0;
  bf16* w = nullptr; float* wf = nullptr; float* bias = nullptr;
  float *hist = nullptr, *next = nullptr;   // [B][ctx][Cin]
};
struct Codec {
  std::vector<ConvL> convs;                  // index i = layer before stage i ; last = head
  std::vector<std::vector<Block>> stages;
  std::vector<int> T;                        // frames per stage (per 1 latent frame)
  std::vector<int> C;
  StateSeg* segs_dev = nullptr; int n_segs = 0;
  int64_t weight_bytes = 0;
};
struct VoiceEnc {           // non-streaming acoustic encoder for voice prompts (a-9); present iff the checkpoint has its tensors
  bool present = false;
  std::vector<ConvL> convs;                  // stem, downsample i (before stage i), head: bf16 [Cout][K] tap-major, K = k*Cin rounded up to 8
  std::vector<std::vector<Block>> stages;    // no streaming state (hist / next stay null)
  std::vector<int> C;
  int64_t weight_bytes = 0;
};
struct LmLayer { bf16 *wqkv, *wo, *wgu, *wdown; float *bqkv, *ln1, *ln2; };
struct HeadLayer { bf16 *wgu, *wdown; float* norm; };

struct GraphEntry { cudaGraphExec_t exec = nullptr; int64_t launches = 0; };

struct vv_ctx {
  vv_model_desc d;
  int device = 0;
  bool finalized = false;
  bool use_graphs = true;
  bool use_pdl = true;
  bf16* s_planes = nullptr; size_t planes_elems = 0;
  int use_wgmma = 1;        // warpgroup (wgmma) GEMM: 0 off, 1 auto (wide GEMMs), 2 every M > 8 GEMM (VV_WGMMA)
  int wr_tasks_min = 296;
  int wr_force = 0;
  int gemv_grid_cap = 0;
  int sm_count = 132;
  std::map<std::string, RawTensor> raw;
  std::set<std::string> expected;
  std::set<std::string> voice_expected;      // acoustic encoder tensors: all or none
  std::vector<void*> allocs;
  float speech_scale = NAN, speech_bias = NAN;
  // LM
  std::vector<LmLayer> lm;
  float* lm_norm = nullptr; bf16* embed = nullptr; const bf16* lm_head_w = nullptr; bf16* head_valid = nullptr; int* valid_ids_dev = nullptr; float* inv_freq = nullptr;
  int Nqkv = 0;
  // head
  bf16 *h_noisy = nullptr, *h_cond = nullptr, *h_t0 = nullptr, *h_t2 = nullptr, *h_mod = nullptr, *h_final = nullptr;
  std::vector<HeadLayer> head;
  int n_steps = 0; float* temb = nullptr; float* tfreqs = nullptr;
  int32_t temb_info[2][2] = {{-1, 0}, {-1, 0}};   // {kernel, split-K} linear() ran for t_embedder.mlp.0 / .2 (vv_debug_sampler_taps)
  std::vector<DpmCoef> coef_host; int coef_version = 0;
  bool sde = false; const float* step_noise = nullptr;   // sde-dpmsolver++: per-step variance noise [n_steps][B][64] (vv_set_step_noise)
  // connectors
  bf16 *ca_fc1 = nullptr, *ca_fc2 = nullptr, *cs_fc1 = nullptr, *cs_fc2 = nullptr;
  float *ca_b1 = nullptr, *ca_b2 = nullptr, *ca_n = nullptr, *cs_b1 = nullptr, *cs_b2 = nullptr, *cs_n = nullptr;
  Codec dec, enc;
  VoiceEnc venc;
  int64_t wbytes[6] = {0, 0, 0, 0, 0, 0};
  // KV
  int64_t n_pages = 0; int max_pages = 0; bf16 *kpool = nullptr, *vpool = nullptr;
  int* page_table_dev = nullptr; int* kv_len_dev = nullptr; int* row_mode_dev = nullptr;
  std::vector<int64_t> kv_len_host; std::vector<std::vector<int>> seq_pages; std::vector<int> free_pages;
  // scratch
  float* s_lgu = nullptr;   // LM gate/up raw sums [2B][2I] (weight-stream path)
  float *s_h = nullptr, *s_qkv = nullptr;
  float *s_condp = nullptr, *s_call = nullptr, *s_mod = nullptr, *s_hx = nullptr, *s_v = nullptr, *s_z = nullptr,
        *s_x0 = nullptr, *s_tfeat = nullptr, *s_t1 = nullptr, *s_hgu = nullptr;
  float *s_xa = nullptr, *s_xb = nullptr, *s_u = nullptr, *s_win = nullptr, *s_xn = nullptr;
  float *s_e = nullptr, *s_c1 = nullptr, *s_feat = nullptr, *s_audio = nullptr, *s_latent = nullptr;
  int* s_tok = nullptr;
  std::map<std::string, GraphEntry> graphs;
  GridBar* gridbar = nullptr;
  // weight-stream programs (vv_stream.cuh)
  struct StreamProg {
    SOp* ops = nullptr; int n_ops = 0; CUtensorMap* tmaps = nullptr; int n_stages = 0; int b_bytes = 0; int smem = 0; int gemv_ops = 0; int variant = 0;
  };
  std::map<std::string, StreamProg> sprogs;
  unsigned* st_bar = nullptr;            // grid-barrier counter of the stream kernel
  unsigned* st_diag_host = nullptr; unsigned* st_diag_dev = nullptr;   // host-mapped watchdog record
  int st_inflight = 4;                   // VV_STREAM_INFLIGHT: TMA tiles (16 KB) a CTA keeps in flight
  float* dec_front_x = nullptr;                  // where the streamed decoder front leaves its rows (same for every program: fixed structure)
  float *s_cx = nullptr, *s_cu = nullptr;        // codec rows / FFN hidden sums of the stream path (two buffers each)
  float* s_rope = nullptr;                        // [2B][64][2] cos / sin of the current positions
  float *s_pacc2 = nullptr, *s_pml2 = nullptr;   // attention partials of the stream path: [2B][kv_heads][SMs][8][128] / [..][8][2]
  std::map<std::tuple<const bf16*, int, int>, bf16*> tiled; size_t tiled_bytes = 0;   // tile-major copies of the weights the stream kernel reads,
                                                                                         // per (weight, first column, columns)
  long long* st_trace2 = nullptr;
  long long* st_trace = nullptr; int st_trace_ops = 0; int st_trace_cta = 0; int st_trace_last_ops = 0;   // VV_STREAM_TRACE=<cta>: per-stage clock stamps of one CTA
  float* cfg_dev = nullptr; float cfg_last = NAN;   // CFG scale lives in device memory so captured graphs do not depend on its value
  int64_t launches = 0;
  std::map<long long, int> occ_cache;
};

struct L {  // launcher
  vv_ctx* c; cudaStream_t s;
};

constexpr int MMA_MIN_ROWS = 9;   // M >= this -> tensor-core GEMM (all prologues/epilogues), below -> weight-streaming GEMV (at M = 8 the GEMV streams weights faster)

// every hot-path kernel goes through here: programmatic dependent launch (PDL) lets kernel N+1 be scheduled and run its
// weight-only prologue while kernel N drains; inside CUDA-graph capture these become programmatic dependency edges.
template <typename... KArgs, typename... Args>
static cudaError_t launch_k(const L& l, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = l.s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = l.c->use_pdl ? 1 : 0;
  l.c->launches++;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// ------------------------------------------------------------------------------------------------
template <class T>
static int dmalloc(vv_ctx* c, T** p, size_t n, bool zero = true) {
  void* q = nullptr;
  cudaError_t e = cudaMalloc(&q, std::max<size_t>(n, 1) * sizeof(T));
  if (e != cudaSuccess) return fail(VV_ERR_NOMEM, "cudaMalloc(%zu bytes): %s", n * sizeof(T), cudaGetErrorString(e));
  if (zero) cudaMemset(q, 0, std::max<size_t>(n, 1) * sizeof(T));
  c->allocs.push_back(q);
  *p = (T*)q;
  return 0;
}

static int gemv_smem_bytes(int MB, int K) { int Kp = (K + 255) & ~255; return (MB * Kp + 2 * 8 * 4 * MB) * 4; }

template <int MB>
static int launch_gemv_t(const L& l, GemvP& p, int grid, int smem) {
  static bool attr_set[8] = {false, false, false, false, false, false, false, false};
  (void)attr_set;
  CK(cudaFuncSetAttribute(gemv_kernel<MB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  CK(launch_k(l, gemv_kernel<MB>, dim3(grid), dim3(256), smem, p));
  return 0;
}

template <int MB>
static int gemv_occupancy(vv_ctx* c, int smem) {
  long long key = ((long long)MB << 32) | (unsigned)smem;
  auto it = c->occ_cache.find(key);
  if (it != c->occ_cache.end()) return it->second;
  int occ = 1;
  cudaFuncSetAttribute(gemv_kernel<MB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gemv_kernel<MB>, 256, smem) != cudaSuccess || occ < 1) occ = 1;
  c->occ_cache[key] = occ;
  return occ;
}

// which kernel linear() ran (vv_debug_gemv2)
enum {
  LIN_GEMV = 0, LIN_RING_RMS_GELU, LIN_RING_RMS_NONE, LIN_RING_GAMMA_RESID, LIN_RING_NONE, LIN_RING_GELU, LIN_RING_RESID, LIN_RING_GENERIC,
  LIN_MMA, LIN_WGMMA
};

// y = epi(W * pro(x) + bias); dispatches GEMV (M <= 16) or the tiled GEMM.  info (optional): {LIN_* kernel, split-K factor}.
static int linear(const L& l, GemvP p, int32_t* info = nullptr) {
  if (p.K % 8 != 0) return fail(VV_ERR_INVALID, "linear: K=%d not a multiple of 8", p.K);
  if (((uintptr_t)p.x & 15) || (p.xmap.rs & 3) || (p.xmap.bs & 3)) return fail(VV_ERR_INVALID, "linear: activation rows must be 16-byte aligned");
  // wgmma path: wide GEMMs that fill the chip with 128-row weight tiles (the all-steps AdaLN modulation GEMM:
  // [N_steps*2B, H] x [(3L+2)H, H]^T = 168 CTAs on 1.5B); mode 2 forces it for every M > 8 GEMM (tests)
  const int wg_ctas = ((p.N + WG_BM - 1) / WG_BM) * ((p.M + WG_BN - 1) / WG_BN);
  if (l.c->use_wgmma && p.M > 8 && p.pro == PRO_NONE && p.epi != EPI_SWIGLU && (l.c->use_wgmma == 2 || wg_ctas >= 96)) {
    if ((size_t)p.M * p.K > l.c->planes_elems) return fail(VV_ERR_INVALID, "wgmma: activation planes scratch too small (%d x %d)", p.M, p.K);
    bf16* hi = l.c->s_planes;
    bf16* lo = l.c->s_planes + l.c->planes_elems;
    const long long n4 = (long long)p.M * (p.K >> 2);
    CK(launch_k(l, split_bf16_kernel, dim3((unsigned)std::min<long long>((n4 + 255) / 256, 1184)), dim3(256), 0, p.x, p.xmap, hi, lo, p.M, p.K));
    CK(cudaFuncSetAttribute(gemm_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM));
    CK(launch_k(l, gemm_wgmma_kernel, dim3((p.N + WG_BM - 1) / WG_BM, (p.M + WG_BN - 1) / WG_BN), dim3(128), (size_t)WG_SMEM, p, (const bf16*)hi, (const bf16*)lo));
    if (info) { info[0] = LIN_WGMMA; info[1] = 1; }
    return 0;
  }
  if (p.M >= MMA_MIN_ROWS) {
    dim3 grid((p.N + MM_BN - 1) / MM_BN, (p.M + MM_BM - 1) / MM_BM);
    const bool inplace_res = (p.epi == EPI_RESID || p.epi == EPI_GAMMA_RESID || p.epi == EPI_GATED_RESID) && p.res == p.y && p.ldres == p.ldy;
    const int nk = (p.K + MM_BK - 1) / MM_BK;
    if (inplace_res && nk >= 8 && (int)(grid.x * grid.y) < l.c->sm_count) {
      int z = std::min(std::min(nk / 2, 16), (2 * l.c->sm_count) / (int)(grid.x * grid.y));
      grid.z = std::max(z, 1);
    }
    const bool ring_rms = p.pro == PRO_RMSNORM && grid.z == 1 && p.K <= MR_MAXK_NORM && p.K % 4 == 0;
    if ((p.pro == PRO_NONE || ring_rms) && p.epi != EPI_SWIGLU) {
      // the combinations the codec passes use get their own instantiation (FFN1: folded RMSNorm + GELU; FFN2 / transposed convs: plain or
      // gamma-residual, split-K or not); anything else runs the run-time-switched one
      void (*fn)(GemvP) = gemm_mma_ring_kernel<-1, -1>;
      int which = LIN_RING_GENERIC;
      if (ring_rms && p.epi == EPI_GELU) fn = gemm_mma_ring_kernel<1, EPI_GELU>, which = LIN_RING_RMS_GELU;
      else if (ring_rms && p.epi == EPI_NONE) fn = gemm_mma_ring_kernel<1, EPI_NONE>, which = LIN_RING_RMS_NONE;
      else if (!ring_rms && p.epi == EPI_GAMMA_RESID) fn = gemm_mma_ring_kernel<0, EPI_GAMMA_RESID>, which = LIN_RING_GAMMA_RESID;
      else if (!ring_rms && p.epi == EPI_NONE) fn = gemm_mma_ring_kernel<0, EPI_NONE>, which = LIN_RING_NONE;
      else if (!ring_rms && p.epi == EPI_GELU) fn = gemm_mma_ring_kernel<0, EPI_GELU>, which = LIN_RING_GELU;
      else if (!ring_rms && p.epi == EPI_RESID) fn = gemm_mma_ring_kernel<0, EPI_RESID>, which = LIN_RING_RESID;
      CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, MR_SMEM_NORM));
      CK(launch_k(l, fn, dim3(grid), dim3(128), (size_t)(ring_rms ? MR_SMEM_NORM : MR_SMEM), p));
      if (info) { info[0] = which; info[1] = (int32_t)grid.z; }
      return 0;
    }
    CK(launch_k(l, gemm_mma_kernel, dim3(grid), dim3(128), 0, p));
    if (info) { info[0] = LIN_MMA; info[1] = (int32_t)grid.z; }
    return 0;
  }
  int MB = p.M <= 1 ? 1 : (p.M <= 2 ? 2 : (p.M <= 4 ? 4 : 8));
  while (MB > 1 && gemv_smem_bytes(MB, p.K) > 200 * 1024) MB >>= 1;
  if (gemv_smem_bytes(MB, p.K) > 200 * 1024) return fail(VV_ERR_INVALID, "gemv: K=%d too large", p.K);
  int WR = 8;
  while (WR > 1 && (p.N + 4 * WR - 1) / (4 * WR) < l.c->wr_tasks_min) WR >>= 1;
  const int nchunks = (p.K + 255) / 256;
  while (WR < 8 && 8 / WR > nchunks) WR <<= 1;      // never more k-split warps than 256-element chunks
  if (l.c->wr_force) WR = l.c->wr_force;
  p.WK = 8 / WR;
  const int ntasks = (p.N + 4 * WR - 1) / (4 * WR);
  const int smem = gemv_smem_bytes(MB, p.K);
  int occ = MB == 1 ? gemv_occupancy<1>(l.c, smem) : MB == 2 ? gemv_occupancy<2>(l.c, smem) : MB == 4 ? gemv_occupancy<4>(l.c, smem)
                                                                                                          : gemv_occupancy<8>(l.c, smem);
  int grid = std::min(ntasks, l.c->sm_count * occ);
  if (l.c->gemv_grid_cap) grid = std::min(grid, l.c->gemv_grid_cap);
  if (info) { info[0] = LIN_GEMV; info[1] = 1; }
  switch (MB) {
    case 1: return launch_gemv_t<1>(l, p, grid, smem);
    case 2: return launch_gemv_t<2>(l, p, grid, smem);
    case 4: return launch_gemv_t<4>(l, p, grid, smem);
    default: return launch_gemv_t<8>(l, p, grid, smem);
  }
}

static GemvP mk(const bf16* W, const float* bias, const float* x, long long ldx, float* y, int ldy, int M, int N, int K) {
  GemvP p;
  memset(&p, 0, sizeof p);
  p.W = W; p.bias = bias; p.x = x; p.xmap = dense_rows(ldx); p.y = y; p.ldy = ldy; p.M = M; p.N = N; p.K = K;
  p.pro = PRO_NONE; p.epi = EPI_NONE; p.WK = 1;
  return p;
}

// ------------------------------------------------------------------------------------------------
// weight-stream programs (vv_stream.cuh): host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
  }
  return fn;
}
// tile-major weight copy [n_tiles][128][64] bf16 -> 2-D tensor map over [n_tiles*128][64], box = one 16 KB tile, 128-byte swizzle
static int make_weight_tmap(const bf16* T, long long n_tiles, CUtensorMap* out) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return fail(VV_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
  const int N = (int)n_tiles, K = 64;
  const cuuint64_t dims[2] = {64, (cuuint64_t)n_tiles * 128};
  const cuuint64_t strides[1] = {128};
  const cuuint32_t box[2] = {64, 128};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)T, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VV_ERR_CUDA, "cuTensorMapEncodeTiled([%d tiles x %d]) failed with %d", N, K, (int)r);
  return 0;
}
// tile-major copy of columns [k0, k0 + K) of W [N][ldw] (cached per weight pointer and column range; `fresh` = never cache: the caller's
// buffer may be re-used with other contents)
static int tiled_weight(vv_ctx* c, const bf16* W, long long ldw, int N, int K, int k0, bool fresh, bf16** out, long long* n_tiles) {
  if (K % 8 || k0 % 8 || ldw % 8 || ((uintptr_t)W & 15))
    return fail(VV_ERR_INVALID, "stream: weight [%d x %d] must have K %% 8 == 0 and a 16-byte aligned base", N, K);
  const long long KB = (K + 63) / 64, R = (N + 127) / 128;
  *n_tiles = R * KB;
  const auto key = std::make_tuple(W, k0, K);
  if (!fresh) {
    auto it = c->tiled.find(key);
    if (it != c->tiled.end()) { *out = it->second; return 0; }
  }
  bf16* T = nullptr;
  RET(dmalloc(c, &T, (size_t)(*n_tiles) * 8192, false));
  const long long n_chunks = *n_tiles * 1024;
  tile_pack_kernel<<<(unsigned)std::min<long long>((n_chunks + 255) / 256, (long long)c->sm_count * 32), 256>>>(W, T, N, K, (int)KB, ldw, k0, n_chunks);
  CKL();
  CK(cudaDeviceSynchronize());
  if (!fresh) c->tiled[key] = T;
  c->tiled_bytes += (size_t)(*n_tiles) * 16384;
  *out = T;
  return 0;
}

struct StreamBuilder {
  vv_ctx* c;
  std::vector<SOp> ops;
  std::vector<CUtensorMap> tmaps;
  std::vector<const bf16*> wsrc;   // op -> weight [N][K] of a linear stage (else null); sliced, packed and mapped by finish_stream
  explicit StreamBuilder(vv_ctx* c_) : c(c_) {}
  SOp& push(int kind, bool sync) {
    SOp o;
    memset(&o, 0, sizeof o);
    o.kind = kind; o.sync_before = sync ? 1 : 0; o.nB = 16;
    ops.push_back(o); wsrc.push_back(nullptr);
    return ops.back();
  }
  // y[m][n] (+)= alpha * (W x'[m] + bias); x' = pro(x)
  bool fresh_weights = false;
  std::vector<bf16*> owned;         // tile-major copies made with fresh_weights (freed by the caller)
  long long operand_cap = 0;        // > 0: bytes a linear stage's operand region may take before it is split along K (default: what leaves
                                    // ST_MIN_RING ring slots)
  int kv_tmap = -1;                 // index of the K-pool tensor map (V-pool map follows) for SK_ATTN stages
  std::vector<int> needs_kv;        // ops whose att.tmap_k / tmap_v must be patched
  int use_kv_pool() {
    if (kv_tmap >= 0) return 0;
    const auto& d = c->d;
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) return fail(VV_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    const cuuint64_t rows = (cuuint64_t)d.num_layers * c->n_pages * d.num_kv_heads * KV_PAGE;
    const cuuint64_t dims[2] = {(cuuint64_t)d.head_dim, rows};
    const cuuint64_t strides[1] = {(cuuint64_t)d.head_dim * 2};
    const cuuint32_t box[2] = {64, KV_PAGE};
    const cuuint32_t estr[2] = {1, 1};
    for (bf16* pool : {c->kpool, c->vpool}) {
      CUtensorMap tm;
      CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)pool, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return fail(VV_ERR_CUDA, "cuTensorMapEncodeTiled(KV pool) failed with %d", (int)r);
      tmaps.push_back(tm);
    }
    kv_tmap = (int)tmaps.size() - 2;
    return 0;
  }
  void fill_att(SAtt* a, int layer) {
    const auto& d = c->d;
    const size_t per_layer = (size_t)c->n_pages * d.num_kv_heads * KV_PAGE * d.head_dim;
    memset(a, 0, sizeof *a);
    a->hd = d.head_dim;
    a->qkv = c->s_qkv;
    a->kv.kpool = c->kpool + per_layer * layer; a->kv.vpool = c->vpool + per_layer * layer;
    a->kv.page_table = c->page_table_dev; a->kv.max_pages = c->max_pages; a->kv.kv_len = c->kv_len_dev; a->kv.row_mode = c->row_mode_dev;
    a->kv.kv_heads = d.num_kv_heads; a->kv.q_heads = d.num_q_heads;
    a->part_acc = c->s_pacc2; a->part_ml = c->s_pml2; a->inv_freq = c->inv_freq; a->scale = 1.0f / sqrtf((float)d.head_dim);
    a->row_base = (unsigned)((size_t)layer * c->n_pages * d.num_kv_heads * KV_PAGE);
    a->rope_cs = c->s_rope;
  }
  int attn(int layer, int M) {
    RET(use_kv_pool());
    SOp& o = push(SK_ATTN, true);
    o.M = M;
    fill_att(&o.att, layer);
    needs_kv.push_back((int)ops.size() - 1);
    return 0;
  }
  int gemv(const bf16* W, const float* bias, const float* x, long long ldx, float* y, long long ldy, int M, int N, int K, bool sync, SOp** out) {
    if (M < 1 || M > 32) return fail(VV_ERR_INVALID, "stream gemv: M=%d outside [1,32]", M);
    if (N < 1 || K < 8 || K % 8 || ((uintptr_t)W & 15))
      return fail(VV_ERR_INVALID, "stream: weight [%d x %d] must have K %% 8 == 0 and a 16-byte aligned base", N, K);
    SOp& o = push(SK_GEMV, sync);
    o.M = M; o.N = N; o.K = K; o.krow = K; o.nB = M <= 8 ? 16 : (M <= 16 ? 32 : 64);
    o.x = x; o.ldx = ldx; o.y = y; o.ldy = ldy; o.bias = bias; o.pro = SP_NONE; o.alpha_kind = SA_ONE;
    wsrc.back() = W;
    *out = &ops.back();
    return 0;
  }
  void nop(bool sync, float* init_dst, long long init_n) {
    SOp& o = push(SK_NOP, sync);
    o.init_dst = init_dst; o.init_n = init_n;
  }
};

// stream_kernel instantiations: one per program family, each compiled with only the stage kinds / prologues / scalings the family uses
// (instruction-cache footprint, see the template's comment); a program runs on the first variant whose feature set covers it.
constexpr unsigned sfeat(std::initializer_list<int> pros, std::initializer_list<int> kinds, std::initializer_list<int> alphas) {
  unsigned f = 0;
  for (int x : pros) f |= 1u << x;
  for (int x : kinds) f |= 1u << (16 + x);
  for (int x : alphas) f |= 1u << (24 + x);
  return f;
}
constexpr unsigned SF_SAMP = sfeat({SP_NONE, SP_ADALN, SP_SWIGLU, SP_DPM}, {SK_GEMV, SK_NOP}, {SA_ONE, SA_GATE});
constexpr unsigned SF_LM = sfeat({SP_NONE, SP_RMSNORM, SP_SWIGLU, SP_COMBINE}, {SK_GEMV, SK_NOP, SK_ATTN}, {SA_ONE});
constexpr unsigned SF_CODEC = sfeat({SP_NONE, SP_WINDOW, SP_RMSNORM, SP_GELU}, {SK_GEMV, SK_NOP, SK_MIX}, {SA_ONE, SA_GAMMA});
constexpr unsigned SF_HD128 = 1u << 30;          // every attention stage has head_dim 128 (compile-time loop bounds)
constexpr unsigned SF_LM128 = SF_LM | SF_HD128;
constexpr unsigned SF_NB16 = 1u << 29;           // every linear stage has a 16-row activation operand (compile-time nB)
constexpr unsigned SF_ALL = 0xffffffffu & ~SF_HD128 & ~SF_NB16;
typedef void (*StreamFn)(SParams);
static const struct { unsigned feat; StreamFn fn; StreamFn fn_trace; const char* name; } STREAM_VARIANTS[] = {
#define SVAR(f, name) {f, stream_kernel<f, false>, stream_kernel<f, true>, name}
  SVAR(SF_SAMP | SF_NB16, "sampler (16-row operand)"), SVAR(SF_SAMP, "sampler"),
  SVAR(SF_LM128 | SF_NB16, "lm (head_dim 128, 16-row operand)"), SVAR(SF_LM128, "lm (head_dim 128)"), SVAR(SF_LM, "lm"),
  SVAR(SF_CODEC | SF_NB16, "codec (16-row operand)"), SVAR(SF_CODEC, "codec"), SVAR(SF_ALL, "all")};
#undef SVAR
constexpr int N_STREAM_VARIANTS = 8;

constexpr int ST_MIN_RING = 3;    // ring slots a program must keep: a linear stage whose operand region leaves fewer is split along K

// Bytes of the operand region a linear stage needs when it reduces over KBs k-blocks: the B operand of every k-block a CTA touches (+ the
// attention-merge scratch of SP_COMBINE: merge weights, group partial sums, merged rows).  *heads = distinct heads per CTA (SP_COMBINE).
static long long stage_operand_bytes(const vv_ctx* c, const SOp& o, long long KBs, long long* heads) {
  const int G = c->sm_count;
  const long long R = (o.N + 127) / 128, per = (R * KBs + G - 1) / G, count = std::min(per, KBs);
  long long bytes = count * o.nB * 128;
  *heads = 0;
  if (o.pro == SP_COMBINE) {
    const long long kbh = c->d.head_dim / 64, nh = (count + kbh - 2) / kbh + 2;
    *heads = nh;
    bytes = ((bytes + 1023) & ~1023ll) + o.M * nh * G * 4 + 16 + std::max<long long>(2048, o.M * count * 256) + o.M * count * 256;
  }
  return bytes;
}

// K split: y += alpha * W pro(x) is a sum over k-blocks and the epilogue is an atomic sum, so a stage whose operand region is too large
// for the ring runs as consecutive slices over k-block ranges (SP_COMBINE: whole heads).  The first slice keeps the grid barrier, bias,
// zero-fill jobs and RoPE rows; the others follow without a barrier.  Every slice has its own tile-major weight copy and tensor map.
static int split_and_map(StreamBuilder& b, long long cap, std::vector<int>* tmap_of) {
  vv_ctx* c = b.c;
  std::vector<SOp> ops;
  std::vector<int> first(b.ops.size() + 1, 0);     // stage i of the builder -> its first stage after the split (first[n] = stage count)
  tmap_of->clear();
  for (size_t i = 0; i < b.ops.size(); ++i) {
    first[i] = (int)ops.size();
    const SOp& o = b.ops[i];
    if (o.kind != SK_GEMV) { ops.push_back(o); tmap_of->push_back(-1); continue; }
    const long long KB = (o.K + 63) / 64;
    const long long gran = o.pro == SP_COMBINE ? c->d.head_dim / 64 : 1;
    const bool can_split = o.pro != SP_DPM && o.pro != SP_WINDOW && !o.store;
    auto fits = [&](long long kbs) {
      long long nh;
      const long long bytes = stage_operand_bytes(c, o, kbs, &nh);
      return bytes <= cap && o.M * nh <= 128;
    };
    long long kbs = KB;
    if (can_split && !fits(KB))
      for (long long s = 2; s <= KB; ++s) {
        kbs = ((KB + s - 1) / s + gran - 1) / gran * gran;
        if (fits(kbs) || kbs <= gran) break;
      }
    for (long long kb0 = 0; kb0 < KB; kb0 += kbs) {
      SOp so = o;
      so.k0 = (int)(kb0 * 64);
      so.K = (int)std::min<long long>(kbs * 64, o.K - so.k0);
      if (kb0 > 0) {
        so.sync_before = 0; so.bias = nullptr; so.rope_rows = 0;
        so.init_dst = nullptr; so.init_n = 0; so.init2_dst = nullptr; so.init2_n = 0;
      }
      bf16* T; long long n_tiles;
      RET(tiled_weight(c, b.wsrc[i], o.K, o.N, so.K, so.k0, b.fresh_weights, &T, &n_tiles));
      if (b.fresh_weights) b.owned.push_back(T);
      CUtensorMap tm;
      RET(make_weight_tmap(T, n_tiles, &tm));
      b.tmaps.push_back(tm);
      ops.push_back(so); tmap_of->push_back((int)b.tmaps.size() - 1);
    }
  }
  first[b.ops.size()] = (int)ops.size();
  std::vector<int> needs_kv;
  for (int i : b.needs_kv)
    for (int j = first[i]; j < first[i + 1]; ++j) needs_kv.push_back(j);
  if (getenv("VV_VERBOSE") && ops.size() != b.ops.size())
    fprintf(stderr, "[vv] stream program: %zu stages after the K split of %zu\n", ops.size(), b.ops.size());
  b.ops.swap(ops);
  b.needs_kv.swap(needs_kv);
  b.wsrc.assign(b.ops.size(), nullptr);
  return 0;
}

static int finish_stream(StreamBuilder& b, vv_ctx::StreamProg* pr) {
  vv_ctx* c = b.c;
  const int G = c->sm_count;
  unsigned feat = 0;
  bool hd128 = true, nb16 = true;
  for (const SOp& o : b.ops) {
    if (o.kind == SK_GEMV && o.nB != 16) nb16 = false;
    feat |= (1u << o.pro) | (1u << (16 + o.kind)) | (1u << (24 + o.alpha_kind));
    if ((o.kind == SK_ATTN || o.pro == SP_COMBINE || o.rope_rows > 0) && o.att.hd != 128) hd128 = false;
  }
  pr->variant = N_STREAM_VARIANTS - 1;
  if (!getenv("VV_STREAM_GENERIC"))
    for (int v = 0; v < N_STREAM_VARIANTS; ++v)
      if ((feat & ~STREAM_VARIANTS[v].feat) == 0 && (hd128 || !(STREAM_VARIANTS[v].feat & SF_HD128)) && (nb16 || !(STREAM_VARIANTS[v].feat & SF_NB16)) &&
          !(getenv("VV_STREAM_NO_NB16") && (STREAM_VARIANTS[v].feat & SF_NB16))) { pr->variant = v; break; }
  if (getenv("VV_VERBOSE")) fprintf(stderr, "[vv] stream program: %zu stages, features %08x -> kernel variant '%s'\n", b.ops.size(), feat, STREAM_VARIANTS[pr->variant].name);
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, STREAM_VARIANTS[pr->variant].fn));
  const int max_dyn = 232448 - (int)fa.sharedSizeBytes - 256;
  std::vector<int> tmap_of;
  RET(split_and_map(b, b.operand_cap > 0 ? b.operand_cap : (long long)max_dyn - 1024 - (long long)ST_MIN_RING * ST_TILE, &tmap_of));
  int b_bytes = 2048;
  for (const SOp& o : b.ops) {
    if (o.kind == SK_MIX && (o.cod.T_out > 8 || o.K % 4 || o.K > 4096)) return fail(VV_ERR_INVALID, "stream: mixer stage handles T <= 8, C <= 4096");
    if (o.kind == SK_ATTN) b_bytes = std::max(b_bytes, 32768);        // Q tile, new K/V row and the warp-merge buffers live in the operand region
    if (o.kind != SK_GEMV) continue;
    const long long KB = (o.K + 63) / 64, R = (o.N + 127) / 128, U = R * KB;
    const long long per = (U + G - 1) / G;
    long long nh;
    b_bytes = std::max<long long>(b_bytes, stage_operand_bytes(c, o, KB, &nh));
    const long long segs = (per + KB - 1) / KB + 1;
    if (segs > ST_MAXSEG) return fail(VV_ERR_INVALID, "stream: stage [%d x %d] needs %lld accumulators per CTA", o.N, o.K, segs);
    if (o.store && KB != 1) return fail(VV_ERR_INVALID, "stream: store epilogue needs K <= 64");
    if (o.pro == SP_WINDOW && (o.cod.cin % 8)) return fail(VV_ERR_INVALID, "stream: window prologue needs a channel count that is a multiple of 8");
    if (o.pro == SP_COMBINE) {
      const int hd = c->d.head_dim;
      if ((long long)o.M * nh > 128 || o.k0 % hd || o.K % hd || o.k0 + o.K > hd * c->d.num_q_heads)
        return fail(VV_ERR_INVALID, "stream: attention-merge prologue does not fit (M=%d, heads %d..%d, %lld per CTA)", o.M, o.k0 / hd,
                    (o.k0 + o.K) / hd, nh);
    }
    if (U * (G + 1) >= (1ll << 32)) return fail(VV_ERR_INVALID, "stream: stage [%d x %d] has too many tiles for 32-bit scheduling", o.N, o.K);
  }
  int ns = (max_dyn - 1024 - b_bytes) / ST_TILE;
  ns = std::min(ns, ST_MAX_STAGES);
  if (getenv("VV_STREAM_STAGES")) ns = std::min(ns, atoi(getenv("VV_STREAM_STAGES")));
  if (ns < 2) return fail(VV_ERR_INVALID, "stream: activation operand of %d bytes leaves no room for the weight ring", b_bytes);
  pr->n_stages = ns; pr->b_bytes = b_bytes; pr->smem = ns * ST_TILE + b_bytes + 1024;
  pr->n_ops = (int)b.ops.size();
  RET(dmalloc(c, &pr->tmaps, std::max<size_t>(b.tmaps.size(), 1), false));
  RET(dmalloc(c, &pr->ops, b.ops.size(), false));
  for (int i : b.needs_kv) {
    b.ops[i].att.tmap_k = (unsigned long long)(uintptr_t)(pr->tmaps + b.kv_tmap);
    b.ops[i].att.tmap_v = (unsigned long long)(uintptr_t)(pr->tmaps + b.kv_tmap + 1);
  }
  for (size_t i = 0; i < b.ops.size(); ++i) {
    if (tmap_of[i] >= 0) b.ops[i].tmap = (unsigned long long)(uintptr_t)(pr->tmaps + tmap_of[i]);
    pr->gemv_ops += b.ops[i].kind == SK_GEMV;
  }
  if (!b.tmaps.empty()) CK(cudaMemcpy(pr->tmaps, b.tmaps.data(), b.tmaps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(pr->ops, b.ops.data(), b.ops.size() * sizeof(SOp), cudaMemcpyHostToDevice));
  CK(cudaFuncSetAttribute(STREAM_VARIANTS[pr->variant].fn, cudaFuncAttributeMaxDynamicSharedMemorySize, max_dyn));
  CK(cudaFuncSetAttribute(STREAM_VARIANTS[pr->variant].fn_trace, cudaFuncAttributeMaxDynamicSharedMemorySize, max_dyn));
  return 0;
}

static int launch_stream(const L& l, const vv_ctx::StreamProg& pr) {
  vv_ctx* c = l.c;
  CK(cudaMemsetAsync(c->st_bar, 0, sizeof(unsigned), l.s));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = dim3(c->sm_count); cfg.blockDim = dim3(ST_THREADS); cfg.dynamicSmemBytes = pr.smem; cfg.stream = l.s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;      // all CTAs must be co-resident: they synchronise through a grid barrier
  attr[0].val.cooperative = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  SParams P;
  P.ops = pr.ops; P.n_ops = pr.n_ops; P.bar_count = c->st_bar; P.diag = c->st_diag_dev; P.n_stages = pr.n_stages; P.b_bytes = pr.b_bytes;
  P.max_inflight = std::max(1, std::min(pr.n_stages, c->st_inflight));
  P.kv_len = c->kv_len_dev; P.row_mode = c->row_mode_dev; P.n_seq = 2 * c->d.max_batch; P.kv_heads = c->d.num_kv_heads;
  P.trace = (c->st_trace && pr.n_ops <= c->st_trace_ops) ? c->st_trace : nullptr; P.trace_cta = c->st_trace_cta;
  P.trace2 = P.trace ? c->st_trace2 : nullptr;
  if (P.trace) c->st_trace_last_ops = pr.n_ops;
  c->launches++;
  CK(cudaLaunchKernelEx(&cfg, P.trace ? STREAM_VARIANTS[pr.variant].fn_trace : STREAM_VARIANTS[pr.variant].fn, P));
  return 0;
}

// ------------------------------------------------------------------------------------------------
// expected tensor names (same as vibevoice_b200/synth.py::param_specs, i.e. the HF checkpoint keys)
// ------------------------------------------------------------------------------------------------
static std::string S(const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  return buf;
}
static void block_names(std::set<std::string>& e, const std::string& p) {
  for (const char* s : {"norm.weight", "mixer.conv.conv.conv.weight", "mixer.conv.conv.conv.bias", "gamma", "ffn_norm.weight",
                        "ffn.linear1.weight", "ffn.linear1.bias", "ffn.linear2.weight", "ffn.linear2.bias", "ffn_gamma"})
    e.insert(p + "." + s);
}
static void build_expected(vv_ctx* c) {
  auto& e = c->expected;
  const auto& d = c->d;
  const std::string lm = "model.language_model";
  e.insert(lm + ".embed_tokens.weight");
  e.insert(lm + ".norm.weight");
  for (int l = 0; l < d.num_layers; ++l) {
    std::string q = S("%s.layers.%d", lm.c_str(), l);
    for (const char* s : {"self_attn.q_proj.weight", "self_attn.q_proj.bias", "self_attn.k_proj.weight", "self_attn.k_proj.bias",
                          "self_attn.v_proj.weight", "self_attn.v_proj.bias", "self_attn.o_proj.weight", "mlp.gate_proj.weight",
                          "mlp.up_proj.weight", "mlp.down_proj.weight", "input_layernorm.weight", "post_attention_layernorm.weight"})
      e.insert(q + "." + s);
  }
  if (!d.tie_word_embeddings) e.insert("lm_head.weight");
  const std::string h = "model.prediction_head";
  for (const char* s : {"noisy_images_proj.weight", "cond_proj.weight", "t_embedder.mlp.0.weight", "t_embedder.mlp.2.weight",
                        "final_layer.linear.weight", "final_layer.adaLN_modulation.1.weight"})
    e.insert(h + "." + s);
  for (int l = 0; l < d.head_layers; ++l)
    for (const char* s : {"ffn.gate_proj.weight", "ffn.up_proj.weight", "ffn.down_proj.weight", "norm.weight", "adaLN_modulation.1.weight"})
      e.insert(S("%s.layers.%d.%s", h.c_str(), l, s));
  for (const char* cn : {"model.acoustic_connector", "model.semantic_connector"})
    for (const char* s : {"fc1.weight", "fc1.bias", "norm.weight", "fc2.weight", "fc2.bias"}) e.insert(std::string(cn) + "." + s);
  const std::string dp = "model.acoustic_tokenizer.decoder", ep = "model.semantic_tokenizer.encoder";
  for (int i = 0; i < d.n_stages; ++i) {
    if (i == 0) { e.insert(dp + ".upsample_layers.0.0.conv.conv.weight"); e.insert(dp + ".upsample_layers.0.0.conv.conv.bias"); }
    else { e.insert(S("%s.upsample_layers.%d.0.convtr.convtr.weight", dp.c_str(), i)); e.insert(S("%s.upsample_layers.%d.0.convtr.convtr.bias", dp.c_str(), i)); }
    for (int j = 0; j < d.dec_depths[i]; ++j) block_names(e, S("%s.stages.%d.%d", dp.c_str(), i, j));
    e.insert(S("%s.downsample_layers.%d.0.conv.conv.weight", ep.c_str(), i));
    e.insert(S("%s.downsample_layers.%d.0.conv.conv.bias", ep.c_str(), i));
    for (int j = 0; j < d.enc_depths[i]; ++j) block_names(e, S("%s.stages.%d.%d", ep.c_str(), i, j));
  }
  for (const char* s : {"head.conv.conv.weight", "head.conv.conv.bias"}) { e.insert(dp + "." + s); e.insert(ep + "." + s); }
  // the acoustic encoder has the semantic encoder's structure (enc_ratios / enc_depths / enc_n_filters); only its vae_dim differs
  const std::string ap = "model.acoustic_tokenizer.encoder";
  auto& v = c->voice_expected;
  for (int i = 0; i < d.n_stages; ++i) {
    v.insert(S("%s.downsample_layers.%d.0.conv.conv.weight", ap.c_str(), i));
    v.insert(S("%s.downsample_layers.%d.0.conv.conv.bias", ap.c_str(), i));
    for (int j = 0; j < d.enc_depths[i]; ++j) block_names(v, S("%s.stages.%d.%d", ap.c_str(), i, j));
  }
  for (const char* s : {"head.conv.conv.weight", "head.conv.conv.bias"}) v.insert(ap + "." + s);
}

// ------------------------------------------------------------------------------------------------
extern "C" int vv_abi_version(void) { return VV_ABI_VERSION; }
extern "C" const char* vv_last_error(void) { return g_err.c_str(); }

extern "C" int vv_create(const vv_model_desc* desc, int device, vv_ctx** out) {
  if (!desc || !out) return fail(VV_ERR_INVALID, "vv_create: null argument");
  if (desc->head_dim != 128 && desc->head_dim != 64) return fail(VV_ERR_INVALID, "head_dim %d unsupported (64 or 128)", desc->head_dim);
  if (desc->max_batch < 1 || desc->max_batch > 8) return fail(VV_ERR_INVALID, "max_batch must be in [1,8]");
  if (desc->n_stages < 2 || desc->n_stages > 8) return fail(VV_ERR_INVALID, "n_stages out of range");
  if (desc->num_q_heads % desc->num_kv_heads || desc->num_q_heads / desc->num_kv_heads > ATT_MAXG)
    return fail(VV_ERR_INVALID, "GQA group size unsupported");
  if (desc->latent_size != 64 || desc->acoustic_vae_dim != 64) return fail(VV_ERR_INVALID, "latent size must be 64");
  if (desc->n_valid_ids < 1 || desc->n_valid_ids > 8) return fail(VV_ERR_INVALID, "n_valid_ids out of range");
  CK(cudaSetDevice(device));
  vv_ctx* c = new vv_ctx();
  c->d = *desc;
  c->device = device;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  c->sm_count = prop.multiProcessorCount;
  const char* ng = getenv("VV_NO_GRAPH");
  c->use_graphs = !(ng && ng[0] == '1');
  c->wr_tasks_min = c->sm_count;      // one task per SM (tools/bench_gemv.py compares geometries)
  if (getenv("VV_WR_TASKS_MIN")) c->wr_tasks_min = atoi(getenv("VV_WR_TASKS_MIN"));
  if (getenv("VV_WR_FORCE")) c->wr_force = atoi(getenv("VV_WR_FORCE"));
  if (getenv("VV_GEMV_GRID_CAP")) c->gemv_grid_cap = atoi(getenv("VV_GEMV_GRID_CAP"));
  if (getenv("VV_STREAM_INFLIGHT")) c->st_inflight = atoi(getenv("VV_STREAM_INFLIGHT"));
  if (getenv("VV_WGMMA")) c->use_wgmma = atoi(getenv("VV_WGMMA"));
  const char* np = getenv("VV_NO_PDL");
  c->use_pdl = !(np && np[0] == '1');
  build_expected(c);
  *out = c;
  return 0;
}

extern "C" void vv_destroy(vv_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  for (auto& g : c->graphs) if (g.second.exec) cudaGraphExecDestroy(g.second.exec);
  for (auto& r : c->raw) if (r.second.p) cudaFree(r.second.p);
  for (void* p : c->allocs) cudaFree(p);
  if (c->st_diag_host) cudaFreeHost(c->st_diag_host);
  delete c;
}

static bool stored_as_f32(const std::string& name, const int64_t* shape, int ndim) {
  if (ndim <= 1) return true;
  if (name.find("mixer.conv.conv.conv.weight") != std::string::npos) return true;                 // depthwise [C,1,7]
  if (ndim == 3 && (shape[0] == 1 || shape[1] == 1)) return true;                                  // 1->32 stem, 32->1 head
  return false;
}

extern "C" int vv_load_tensor(vv_ctx* c, const char* name_, const void* data, int dtype, const int64_t* shape, int ndim) {
  if (!c || !name_ || !data) return fail(VV_ERR_INVALID, "vv_load_tensor: null argument");
  if (c->finalized) return fail(VV_ERR_STATE, "vv_load_tensor after vv_finalize_weights");
  std::string name(name_);
  CK(cudaSetDevice(c->device));
  if (name == "model.speech_scaling_factor" || name == "model.speech_bias_factor") {
    float v; char tmp[4];
    CK(cudaMemcpy(tmp, data, dtype == VV_DT_F32 ? 4 : 2, cudaMemcpyDefault));
    if (dtype == VV_DT_F32) memcpy(&v, tmp, 4);
    else if (dtype == VV_DT_BF16) { unsigned u = ((unsigned)(*(unsigned short*)tmp)) << 16; memcpy(&v, &u, 4); }
    else v = __half2float(*(__half*)tmp);
    (name == "model.speech_scaling_factor" ? c->speech_scale : c->speech_bias) = v;
    return 0;
  }
  if (!c->expected.count(name) && !c->voice_expected.count(name)) {
    if (name.find("fix_std") != std::string::npos ||
        name.find("rotary_emb") != std::string::npos || (name == "lm_head.weight" && c->d.tie_word_embeddings))
      return 1;   // not on this path
    return fail(VV_ERR_INVALID, "vv_load_tensor: unknown tensor '%s'", name.c_str());
  }
  size_t n = 1;
  for (int i = 0; i < ndim; ++i) n *= (size_t)shape[i];
  RawTensor t;
  t.shape.assign(shape, shape + ndim);
  t.numel = n;
  t.is_f32 = stored_as_f32(name, shape, ndim);
  const size_t esz = dtype == VV_DT_F32 ? 4 : 2;
  void* dst = nullptr;
  CK(cudaMalloc(&dst, n * (t.is_f32 ? 4 : 2)));
  t.p = dst;
  const bool same = (t.is_f32 && dtype == VV_DT_F32) || (!t.is_f32 && dtype == VV_DT_BF16);
  if (same) {
    CK(cudaMemcpy(dst, data, n * esz, cudaMemcpyDefault));
  } else {
    void* tmp = nullptr;
    CK(cudaMalloc(&tmp, n * esz));
    CK(cudaMemcpy(tmp, data, n * esz, cudaMemcpyDefault));
    const int grid = (int)std::min<size_t>((n + 255) / 256, 65535);
    if (t.is_f32 && dtype == VV_DT_BF16) cvt_bf16_to_f32_kernel<<<grid, 256>>>((const bf16*)tmp, (float*)dst, n);
    else if (t.is_f32 && dtype == VV_DT_F16) cvt_f16_to_f32_kernel<<<grid, 256>>>((const __half*)tmp, (float*)dst, n);
    else if (!t.is_f32 && dtype == VV_DT_F32) cvt_f32_to_bf16_kernel<<<grid, 256>>>((const float*)tmp, (bf16*)dst, n);
    else cvt_f16_to_bf16_kernel<<<grid, 256>>>((const __half*)tmp, (bf16*)dst, n);
    CKL();
    CK(cudaDeviceSynchronize());
    cudaFree(tmp);
  }
  auto it = c->raw.find(name);
  if (it != c->raw.end() && it->second.p) cudaFree(it->second.p);
  c->raw[name] = t;
  return 0;
}

extern "C" int vv_set_speech_factors(vv_ctx* c, float s, float b) {
  if (!c) return fail(VV_ERR_INVALID, "null ctx");
  c->speech_scale = s; c->speech_bias = b;
  return 0;
}

// ---- repack helpers ------------------------------------------------------------------------------
static int need(vv_ctx* c, const std::string& name, RawTensor** t, std::vector<int64_t> shape) {
  auto it = c->raw.find(name);
  if (it == c->raw.end()) return fail(VV_ERR_STATE, "missing tensor %s", name.c_str());
  if (it->second.shape != shape) {
    std::string a, b;
    for (auto v : it->second.shape) a += std::to_string(v) + ",";
    for (auto v : shape) b += std::to_string(v) + ",";
    return fail(VV_ERR_INVALID, "tensor %s has shape [%s] expected [%s]", name.c_str(), a.c_str(), b.c_str());
  }
  *t = &it->second;
  return 0;
}
static int take_bf16(vv_ctx* c, const std::string& name, std::vector<int64_t> shape, bf16** out, int64_t* bytes) {
  RawTensor* t;
  RET(need(c, name, &t, shape));
  if (t->is_f32) return fail(VV_ERR_INVALID, "%s stored as f32, expected bf16", name.c_str());
  *out = (bf16*)t->p;
  c->allocs.push_back(t->p);
  t->p = nullptr;
  if (bytes) *bytes += (int64_t)t->numel * 2;
  return 0;
}
static int take_f32(vv_ctx* c, const std::string& name, std::vector<int64_t> shape, float** out, int64_t* bytes) {
  RawTensor* t;
  RET(need(c, name, &t, shape));
  if (!t->is_f32) return fail(VV_ERR_INVALID, "%s stored as bf16, expected f32", name.c_str());
  *out = (float*)t->p;
  c->allocs.push_back(t->p);
  t->p = nullptr;
  if (bytes) *bytes += (int64_t)t->numel * 2;   // algorithmic bytes are quoted at bf16 (SURVEY 8d)
  return 0;
}
static void drop(vv_ctx* c, const std::string& name) {
  auto it = c->raw.find(name);
  if (it != c->raw.end() && it->second.p) { cudaFree(it->second.p); it->second.p = nullptr; }
}

static int build_block(vv_ctx* c, const std::string& p, int C, Block* b, int64_t* bytes, std::vector<StateSeg>* segs) {
  b->C = C;
  RET(take_f32(c, p + ".norm.weight", {C}, &b->norm_w, bytes));
  RawTensor* t;
  RET(need(c, p + ".mixer.conv.conv.conv.weight", &t, {C, 1, 7}));
  RET(dmalloc(c, &b->dw_w, (size_t)7 * C));
  repack_dw_kernel<<<(C * 7 + 255) / 256, 256>>>((const float*)t->p, b->dw_w, C);
  CKL();
  *bytes += (int64_t)C * 7 * 2;
  RET(take_f32(c, p + ".mixer.conv.conv.conv.bias", {C}, &b->dw_b, bytes));
  RET(take_f32(c, p + ".gamma", {C}, &b->gamma, bytes));
  RET(take_f32(c, p + ".ffn_norm.weight", {C}, &b->ffn_norm_w, bytes));
  RET(take_bf16(c, p + ".ffn.linear1.weight", {4 * C, C}, &b->w1, bytes));
  RET(take_f32(c, p + ".ffn.linear1.bias", {4 * C}, &b->b1, bytes));
  RET(take_bf16(c, p + ".ffn.linear2.weight", {C, 4 * C}, &b->w2, bytes));
  RET(take_f32(c, p + ".ffn.linear2.bias", {C}, &b->b2, bytes));
  RET(take_f32(c, p + ".ffn_gamma", {C}, &b->ffn_gamma, bytes));
  if (!segs) return 0;      // non-streaming use: no conv state
  const int B = c->d.max_batch;
  RET(dmalloc(c, &b->hist, (size_t)B * 6 * C));
  RET(dmalloc(c, &b->next, (size_t)B * 6 * C));
  segs->push_back({b->hist, b->next, 6 * C});
  return 0;
}

// Conv1d [Co][Ci][k] -> window GEMV weight [Co][k*Ci]
static int build_conv(vv_ctx* c, const std::string& p, int Ci, int Co, int k, int stride, ConvL* L_, int64_t* bytes,
                      std::vector<StateSeg>* segs) {
  L_->Cin = Ci; L_->Cout = Co; L_->k = k; L_->stride = stride; L_->ctx = (k - 1) - (stride - 1); L_->N = Co; L_->K = k * Ci;
  RawTensor* t;
  RET(need(c, p + ".weight", &t, {Co, Ci, k}));
  const size_t n = (size_t)Co * Ci * k;
  if (t->is_f32) {
    RET(dmalloc(c, &L_->wf, n));
    repack_conv_f32_kernel<<<(int)((n + 255) / 256), 256>>>((const float*)t->p, L_->wf, Co, Ci, k);
  } else {
    RET(dmalloc(c, &L_->w, n));
    repack_conv_kernel<<<(int)std::min<size_t>((n + 255) / 256, 65535), 256>>>((const bf16*)t->p, L_->w, Co, Ci, k);
  }
  CKL();
  *bytes += (int64_t)n * 2;
  RET(take_f32(c, p + ".bias", {Co}, &L_->bias, bytes));
  const int B = c->d.max_batch;
  RET(dmalloc(c, &L_->hist, (size_t)B * L_->ctx * Ci));
  RET(dmalloc(c, &L_->next, (size_t)B * L_->ctx * Ci));
  segs->push_back({L_->hist, L_->next, L_->ctx * Ci});
  return 0;
}
// ConvTranspose1d [Ci][Co][2s] -> [(j,co)][(half,ci)], bias tiled over j
static int build_convtr(vv_ctx* c, const std::string& p, int Ci, int Co, int s, ConvL* L_, int64_t* bytes, std::vector<StateSeg>* segs) {
  L_->Cin = Ci; L_->Cout = Co; L_->k = 2 * s; L_->stride = s; L_->ctx = 1; L_->N = s * Co; L_->K = 2 * Ci;
  RawTensor* t;
  RET(need(c, p + ".weight", &t, {Ci, Co, 2 * s}));
  if (t->is_f32) return fail(VV_ERR_INVALID, "%s: unexpected f32 convtr weight", p.c_str());
  const size_t n = (size_t)Ci * Co * 2 * s;
  RET(dmalloc(c, &L_->w, n));
  repack_convtr_kernel<<<(int)std::min<size_t>((n + 255) / 256, 65535), 256>>>((const bf16*)t->p, L_->w, Ci, Co, s);
  CKL();
  *bytes += (int64_t)n * 2;
  RawTensor* bt;
  RET(need(c, p + ".bias", &bt, {Co}));
  RET(dmalloc(c, &L_->bias, (size_t)s * Co));
  tile_bias_kernel<<<(s * Co + 255) / 256, 256>>>((const float*)bt->p, L_->bias, Co, s);
  CKL();
  *bytes += (int64_t)Co * 2;
  const int B = c->d.max_batch;
  RET(dmalloc(c, &L_->hist, (size_t)B * Ci));
  RET(dmalloc(c, &L_->next, (size_t)B * Ci));
  segs->push_back({L_->hist, L_->next, Ci});
  return 0;
}

// Conv1d [Co][Ci][k] (fp32 or bf16) -> bf16 window-GEMM weight [Co][K], K = k*Ci rounded up to a multiple of 8 with zero columns
static int build_conv_gemm(vv_ctx* c, const std::string& p, int Ci, int Co, int k, int stride, ConvL* L_, int64_t* bytes) {
  L_->Cin = Ci; L_->Cout = Co; L_->k = k; L_->stride = stride; L_->ctx = k - stride; L_->N = Co; L_->K = (k * Ci + 7) & ~7;
  RawTensor* t;
  RET(need(c, p + ".weight", &t, {Co, Ci, k}));
  const long long n = (long long)Co * L_->K;
  RET(dmalloc(c, &L_->w, (size_t)n, false));
  const unsigned grid = (unsigned)std::min<long long>((n + 255) / 256, 65535);
  if (t->is_f32) repack_conv_pad_kernel<float><<<grid, 256>>>((const float*)t->p, L_->w, Co, Ci, k, L_->K);
  else repack_conv_pad_kernel<bf16><<<grid, 256>>>((const bf16*)t->p, L_->w, Co, Ci, k, L_->K);
  CKL();
  *bytes += (int64_t)Co * Ci * k * 2;
  RET(take_f32(c, p + ".bias", {Co}, &L_->bias, bytes));
  return 0;
}

// acoustic tokenizer encoder (tokenizer.py:694-774) for vv_voice_encode: packed iff the checkpoint has its tensors, all of them
static int build_voice_encoder(vv_ctx* c) {
  const auto& d = c->d;
  std::string missing;
  int nm = 0;
  for (auto& n : c->voice_expected) if (!c->raw.count(n)) { if (nm < 8) missing += n + " "; ++nm; }
  if (nm == (int)c->voice_expected.size()) return 0;
  if (nm) return fail(VV_ERR_STATE, "acoustic encoder: %d of %zu tensors missing, e.g. %s", nm, c->voice_expected.size(), missing.c_str());
  if (d.enc_n_filters % 8 || d.hidden_size % 8) return fail(VV_ERR_INVALID, "acoustic encoder: n_filters and hidden size must be multiples of 8");
  VoiceEnc& v = c->venc;
  const std::string p = "model.acoustic_tokenizer.encoder";
  const int ns = d.n_stages, nf = d.enc_n_filters;
  v.convs.resize(ns + 1); v.stages.resize(ns); v.C.resize(ns);
  for (int i = 0; i < ns; ++i) {
    const int C = nf << i;
    if (i == 0) RET(build_conv_gemm(c, p + ".downsample_layers.0.0.conv.conv", 1, C, 7, 1, &v.convs[0], &v.weight_bytes));
    else {
      const int r = d.enc_ratios[ns - 1 - i];     // TokenizerEncoder reverses the ratio list (tokenizer.py:701)
      RET(build_conv_gemm(c, S("%s.downsample_layers.%d.0.conv.conv", p.c_str(), i), C / 2, C, 2 * r, r, &v.convs[i], &v.weight_bytes));
    }
    v.C[i] = C;
    v.stages[i].resize(d.enc_depths[i]);
    for (int j = 0; j < d.enc_depths[i]; ++j) RET(build_block(c, S("%s.stages.%d.%d", p.c_str(), i, j), C, &v.stages[i][j], &v.weight_bytes, nullptr));
  }
  RET(build_conv_gemm(c, p + ".head.conv.conv", nf << (ns - 1), d.acoustic_vae_dim, 7, 1, &v.convs[ns], &v.weight_bytes));
  v.present = true;
  return 0;
}

static int upload_segs(vv_ctx* c, Codec* k, const std::vector<StateSeg>& segs) {
  k->n_segs = (int)segs.size();
  RET(dmalloc(c, &k->segs_dev, segs.size()));
  CK(cudaMemcpy(k->segs_dev, segs.data(), segs.size() * sizeof(StateSeg), cudaMemcpyHostToDevice));
  return 0;
}

extern "C" int vv_finalize_weights(vv_ctx* c) {
  if (!c) return fail(VV_ERR_INVALID, "null ctx");
  if (c->finalized) return fail(VV_ERR_STATE, "already finalized");
  CK(cudaSetDevice(c->device));
  {
    std::string missing; int nm = 0;
    for (auto& n : c->expected) if (!c->raw.count(n)) { if (nm < 8) missing += n + " "; ++nm; }
    if (nm) return fail(VV_ERR_STATE, "%d tensors missing, e.g. %s", nm, missing.c_str());
    if (std::isnan(c->speech_scale) || std::isnan(c->speech_bias))
      return fail(VV_ERR_STATE, "speech_scaling_factor / speech_bias_factor are NaN (random-init checkpoints: call vv_set_speech_factors)");
  }
  const auto& d = c->d;
  const int H = d.hidden_size, I = d.intermediate_size, nq = d.num_q_heads * d.head_dim, nkv = d.num_kv_heads * d.head_dim, B = d.max_batch;
  const int M2 = 2 * B;
  // ---------------- LM ----------------
  const std::string lm = "model.language_model";
  c->Nqkv = nq + 2 * nkv;
  c->lm.resize(d.num_layers);
  int64_t* wb = &c->wbytes[0];
  for (int l = 0; l < d.num_layers; ++l) {
    LmLayer& y = c->lm[l];
    std::string q = S("%s.layers.%d", lm.c_str(), l);
    RawTensor *tq, *tk, *tv, *bq, *bk, *bv, *tg, *tu;
    RET(need(c, q + ".self_attn.q_proj.weight", &tq, {nq, H}));
    RET(need(c, q + ".self_attn.k_proj.weight", &tk, {nkv, H}));
    RET(need(c, q + ".self_attn.v_proj.weight", &tv, {nkv, H}));
    RET(need(c, q + ".self_attn.q_proj.bias", &bq, {nq}));
    RET(need(c, q + ".self_attn.k_proj.bias", &bk, {nkv}));
    RET(need(c, q + ".self_attn.v_proj.bias", &bv, {nkv}));
    RET(dmalloc(c, &y.wqkv, (size_t)c->Nqkv * H, false));
    RET(dmalloc(c, &y.bqkv, (size_t)c->Nqkv, false));
    CK(cudaMemcpy(y.wqkv, tq->p, (size_t)nq * H * 2, cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(y.wqkv + (size_t)nq * H, tk->p, (size_t)nkv * H * 2, cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(y.wqkv + (size_t)(nq + nkv) * H, tv->p, (size_t)nkv * H * 2, cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(y.bqkv, bq->p, (size_t)nq * 4, cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(y.bqkv + nq, bk->p, (size_t)nkv * 4, cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(y.bqkv + nq + nkv, bv->p, (size_t)nkv * 4, cudaMemcpyDeviceToDevice));
    *wb += (int64_t)c->Nqkv * H * 2 + (int64_t)c->Nqkv * 2;
    for (const char* s : {"q", "k", "v"}) { drop(c, q + ".self_attn." + s + "_proj.weight"); drop(c, q + ".self_attn." + s + "_proj.bias"); }
    RET(take_bf16(c, q + ".self_attn.o_proj.weight", {H, nq}, &y.wo, wb));
    RET(need(c, q + ".mlp.gate_proj.weight", &tg, {I, H}));
    RET(need(c, q + ".mlp.up_proj.weight", &tu, {I, H}));
    RET(dmalloc(c, &y.wgu, (size_t)2 * I * H, false));
    interleave_rows_kernel<<<4096, 256>>>((const bf16*)tg->p, (const bf16*)tu->p, y.wgu, (size_t)I, (size_t)H);
    CKL();
    CK(cudaDeviceSynchronize());
    *wb += (int64_t)2 * I * H * 2;
    drop(c, q + ".mlp.gate_proj.weight"); drop(c, q + ".mlp.up_proj.weight");
    RET(take_bf16(c, q + ".mlp.down_proj.weight", {H, I}, &y.wdown, wb));
    RET(take_f32(c, q + ".input_layernorm.weight", {H}, &y.ln1, wb));
    RET(take_f32(c, q + ".post_attention_layernorm.weight", {H}, &y.ln2, wb));
  }
  RET(take_f32(c, lm + ".norm.weight", {H}, &c->lm_norm, wb));
  RET(take_bf16(c, lm + ".embed_tokens.weight", {d.vocab_size, H}, &c->embed, nullptr));
  {
    RET(dmalloc(c, &c->valid_ids_dev, 8));
    CK(cudaMemcpy(c->valid_ids_dev, d.valid_ids, sizeof(int) * d.n_valid_ids, cudaMemcpyHostToDevice));
    RET(dmalloc(c, &c->head_valid, (size_t)8 * H));
    const bf16* table = c->embed;
    if (!d.tie_word_embeddings) {
      bf16* lmh;
      RET(take_bf16(c, "lm_head.weight", {d.vocab_size, H}, &lmh, nullptr));
      table = lmh;
    }
    c->lm_head_w = table;
    gather_rows_kernel<<<d.n_valid_ids, 256>>>(table, c->valid_ids_dev, c->head_valid, H);
    CKL();
    *wb += (int64_t)d.n_valid_ids * H * 2;
    const int hd = d.head_dim;
    RET(dmalloc(c, &c->inv_freq, hd / 2));
    std::vector<float> f(hd / 2);
    for (int i = 0; i < hd / 2; ++i) f[i] = 1.0f / powf(d.rope_theta, (float)(2 * i) / (float)hd);
    CK(cudaMemcpy(c->inv_freq, f.data(), sizeof(float) * (hd / 2), cudaMemcpyHostToDevice));
  }
  // ---------------- diffusion head ----------------
  {
    const std::string h = "model.prediction_head";
    const int F = d.head_ffn_dim, LH = d.head_layers;
    int64_t* hb = &c->wbytes[1];
    RET(take_bf16(c, h + ".noisy_images_proj.weight", {H, 64}, &c->h_noisy, hb));
    RET(take_bf16(c, h + ".cond_proj.weight", {H, H}, &c->h_cond, &c->wbytes[2]));
    RET(take_bf16(c, h + ".t_embedder.mlp.0.weight", {H, 256}, &c->h_t0, nullptr));
    RET(take_bf16(c, h + ".t_embedder.mlp.2.weight", {H, H}, &c->h_t2, nullptr));
    RET(take_bf16(c, h + ".final_layer.linear.weight", {64, H}, &c->h_final, hb));
    const size_t modrows = (size_t)(3 * LH + 2) * H;
    RET(dmalloc(c, &c->h_mod, modrows * H, false));
    c->head.resize(LH);
    // the per-step weights of all head layers live in one slab: per layer interleaved gate/up [2F][H], then down [H][F]
    // (the sampler program packs its tile-major copies from here)
    const size_t per_layer_el = (size_t)3 * F * H;
    bf16* slab;
    RET(dmalloc(c, &slab, per_layer_el * LH, false));
    for (int l = 0; l < LH; ++l) {
      std::string q = S("%s.layers.%d", h.c_str(), l);
      RawTensor *tg, *tu, *tm, *td;
      RET(need(c, q + ".ffn.gate_proj.weight", &tg, {F, H}));
      RET(need(c, q + ".ffn.up_proj.weight", &tu, {F, H}));
      c->head[l].wgu = slab + per_layer_el * l;
      c->head[l].wdown = c->head[l].wgu + (size_t)2 * F * H;
      interleave_rows_kernel<<<4096, 256>>>((const bf16*)tg->p, (const bf16*)tu->p, c->head[l].wgu, (size_t)F, (size_t)H);
      CKL();
      CK(cudaDeviceSynchronize());
      *hb += (int64_t)2 * F * H * 2;
      drop(c, q + ".ffn.gate_proj.weight"); drop(c, q + ".ffn.up_proj.weight");
      RET(need(c, q + ".ffn.down_proj.weight", &td, {H, F}));
      CK(cudaMemcpy(c->head[l].wdown, td->p, (size_t)H * F * 2, cudaMemcpyDeviceToDevice));
      *hb += (int64_t)H * F * 2;
      drop(c, q + ".ffn.down_proj.weight");
      RET(take_f32(c, q + ".norm.weight", {H}, &c->head[l].norm, hb));
      RET(need(c, q + ".adaLN_modulation.1.weight", &tm, {3 * H, H}));
      CK(cudaMemcpy(c->h_mod + (size_t)l * 3 * H * H, tm->p, (size_t)3 * H * H * 2, cudaMemcpyDeviceToDevice));
      *hb += (int64_t)3 * H * H * 2;
      drop(c, q + ".adaLN_modulation.1.weight");
    }
    RawTensor* tm;
    RET(need(c, h + ".final_layer.adaLN_modulation.1.weight", &tm, {2 * H, H}));
    CK(cudaMemcpy(c->h_mod + (size_t)LH * 3 * H * H, tm->p, (size_t)2 * H * H * 2, cudaMemcpyDeviceToDevice));
    *hb += (int64_t)2 * H * H * 2;
    drop(c, h + ".final_layer.adaLN_modulation.1.weight");
    const int NS = std::max(d.max_diffusion_steps, 1);
    RET(dmalloc(c, &c->temb, (size_t)NS * H));
    RET(dmalloc(c, &c->tfreqs, 128));
    std::vector<float> fr(128);
    for (int j = 0; j < 128; ++j) fr[j] = expf((-9.210340371976184f * (float)j) / 128.0f);
    CK(cudaMemcpy(c->tfreqs, fr.data(), 128 * 4, cudaMemcpyHostToDevice));
    RET(dmalloc(c, &c->s_tfeat, (size_t)NS * 256));
    RET(dmalloc(c, &c->s_t1, (size_t)NS * H));
    RET(dmalloc(c, &c->s_condp, (size_t)M2 * H));
    RET(dmalloc(c, &c->s_call, (size_t)NS * M2 * H));
    RET(dmalloc(c, &c->s_mod, (size_t)NS * M2 * modrows));
    RET(dmalloc(c, &c->cfg_dev, 4));
    RET(dmalloc(c, &c->gridbar, 2));
    RET(dmalloc(c, &c->st_bar, 32));
    if (getenv("VV_STREAM_TRACE")) {
      c->st_trace_cta = atoi(getenv("VV_STREAM_TRACE"));
      c->st_trace_ops = 4096;
      RET(dmalloc(c, &c->st_trace, (size_t)c->st_trace_ops * ST_TRACE));
      RET(dmalloc(c, &c->st_trace2, (size_t)c->st_trace_ops * c->sm_count * 2));
    }
    CK(cudaHostAlloc((void**)&c->st_diag_host, 64, cudaHostAllocMapped));
    memset(c->st_diag_host, 0, 64);
    CK(cudaHostGetDevicePointer((void**)&c->st_diag_dev, c->st_diag_host, 0));
    RET(dmalloc(c, &c->s_hx, (size_t)M2 * H));
    RET(dmalloc(c, &c->s_hgu, (size_t)2 * M2 * 2 * F));
    RET(dmalloc(c, &c->s_v, (size_t)M2 * 64));
    RET(dmalloc(c, &c->s_z, (size_t)2 * B * 64));
    RET(dmalloc(c, &c->s_x0, (size_t)2 * B * 64));
  }
  // ---------------- connectors ----------------
  {
    int64_t* cb = &c->wbytes[5];
    const std::string a = "model.acoustic_connector", s = "model.semantic_connector";
    RET(take_bf16(c, a + ".fc1.weight", {H, d.acoustic_vae_dim}, &c->ca_fc1, cb));
    RET(take_f32(c, a + ".fc1.bias", {H}, &c->ca_b1, cb));
    RET(take_f32(c, a + ".norm.weight", {H}, &c->ca_n, cb));
    RET(take_bf16(c, a + ".fc2.weight", {H, H}, &c->ca_fc2, cb));
    RET(take_f32(c, a + ".fc2.bias", {H}, &c->ca_b2, cb));
    RET(take_bf16(c, s + ".fc1.weight", {H, d.semantic_vae_dim}, &c->cs_fc1, cb));
    RET(take_f32(c, s + ".fc1.bias", {H}, &c->cs_b1, cb));
    RET(take_f32(c, s + ".norm.weight", {H}, &c->cs_n, cb));
    RET(take_bf16(c, s + ".fc2.weight", {H, H}, &c->cs_fc2, cb));
    RET(take_f32(c, s + ".fc2.bias", {H}, &c->cs_b2, cb));
    RET(dmalloc(c, &c->s_e, (size_t)B * H));
    RET(dmalloc(c, &c->s_c1, (size_t)B * H));
    RET(dmalloc(c, &c->s_feat, (size_t)B * d.semantic_vae_dim));
    RET(dmalloc(c, &c->s_audio, (size_t)B * 3200 * 4));
    RET(dmalloc(c, &c->s_latent, (size_t)B * 64));
  }
  // ---------------- codec decoder (tokenizer.py:823-912) ----------------
  int hop = 1;
  for (int i = 0; i < d.n_stages - 1; ++i) hop *= d.dec_ratios[i];
  size_t max_tc = 0, max_win = 0;
  {
    Codec& k = c->dec;
    int64_t* kb = &c->wbytes[3];
    std::vector<StateSeg> segs;
    const std::string p = "model.acoustic_tokenizer.decoder";
    const int ns = d.n_stages, nf = d.dec_n_filters;
    k.convs.resize(ns + 1); k.stages.resize(ns); k.T.resize(ns); k.C.resize(ns);
    int T = 1;
    for (int i = 0; i < ns; ++i) {
      const int C = nf << (ns - 1 - i);
      if (i == 0) RET(build_conv(c, p + ".upsample_layers.0.0.conv.conv", d.acoustic_vae_dim, C, 7, 1, &k.convs[0], kb, &segs));
      else { RET(build_convtr(c, S("%s.upsample_layers.%d.0.convtr.convtr", p.c_str(), i), C * 2, C, d.dec_ratios[i - 1], &k.convs[i], kb, &segs)); T *= d.dec_ratios[i - 1]; }
      k.T[i] = T; k.C[i] = C;
      max_tc = std::max(max_tc, (size_t)T * C);
      max_win = std::max(max_win, (size_t)(T + 8) * C * 2);
      k.stages[i].resize(d.dec_depths[i]);
      for (int j = 0; j < d.dec_depths[i]; ++j) RET(build_block(c, S("%s.stages.%d.%d", p.c_str(), i, j), C, &k.stages[i][j], kb, &segs));
    }
    RET(build_conv(c, p + ".head.conv.conv", nf, 1, 7, 1, &k.convs[ns], kb, &segs));
    if (T != hop) return fail(VV_ERR_INVALID, "decoder hop mismatch");
    RET(upload_segs(c, &k, segs));
    k.weight_bytes = *kb;
  }
  // ---------------- semantic encoder (tokenizer.py:694-774) ----------------
  {
    Codec& k = c->enc;
    int64_t* kb = &c->wbytes[4];
    std::vector<StateSeg> segs;
    const std::string p = "model.semantic_tokenizer.encoder";
    const int ns = d.n_stages, nf = d.enc_n_filters;
    k.convs.resize(ns + 1); k.stages.resize(ns); k.T.resize(ns); k.C.resize(ns);
    int T = hop;
    for (int i = 0; i < ns; ++i) {
      const int C = nf << i;
      if (i == 0) RET(build_conv(c, p + ".downsample_layers.0.0.conv.conv", 1, C, 7, 1, &k.convs[0], kb, &segs));
      else {
        const int r = d.enc_ratios[ns - 1 - i];     // TokenizerEncoder reverses the ratio list (tokenizer.py:701)
        RET(build_conv(c, S("%s.downsample_layers.%d.0.conv.conv", p.c_str(), i), C / 2, C, 2 * r, r, &k.convs[i], kb, &segs));
        if (T % r) return fail(VV_ERR_INVALID, "encoder ratio mismatch");
        T /= r;
      }
      k.T[i] = T; k.C[i] = C;
      max_tc = std::max(max_tc, (size_t)T * C);
      max_win = std::max(max_win, (size_t)(T + 16) * C * 2);
      k.stages[i].resize(d.enc_depths[i]);
      for (int j = 0; j < d.enc_depths[i]; ++j) RET(build_block(c, S("%s.stages.%d.%d", p.c_str(), i, j), C, &k.stages[i][j], kb, &segs));
    }
    if (T != 1) return fail(VV_ERR_INVALID, "encoder hop mismatch");
    RET(build_conv(c, p + ".head.conv.conv", nf << (ns - 1), d.semantic_vae_dim, 7, 1, &k.convs[ns], kb, &segs));
    RET(upload_segs(c, &k, segs));
    k.weight_bytes = *kb;
  }
  RET(build_voice_encoder(c));
  max_win = std::max(max_win, (size_t)(hop + 8) * 64);
  RET(dmalloc(c, &c->s_xa, (size_t)B * max_tc));
  RET(dmalloc(c, &c->s_xb, (size_t)B * max_tc));
  RET(dmalloc(c, &c->s_xn, (size_t)B * max_tc));
  RET(dmalloc(c, &c->s_u, (size_t)B * max_tc * 4));
  RET(dmalloc(c, &c->s_win, (size_t)B * max_win));
  c->planes_elems = std::max<size_t>((size_t)B * max_tc * 4, (size_t)std::max(d.max_diffusion_steps, 1) * M2 * H);
  RET(dmalloc(c, &c->s_planes, 2 * c->planes_elems));
  // ---------------- LM scratch ----------------
  RET(dmalloc(c, &c->s_h, (size_t)M2 * H));
  RET(dmalloc(c, &c->s_qkv, (size_t)M2 * c->Nqkv));
  RET(dmalloc(c, &c->s_lgu, (size_t)M2 * 2 * I));
  RET(dmalloc(c, &c->s_rope, (size_t)M2 * HD));
  RET(dmalloc(c, &c->s_cx, (size_t)2 * B * 8192));
  RET(dmalloc(c, &c->s_cu, (size_t)2 * B * 32768));
  RET(dmalloc(c, &c->s_pacc2, (size_t)M2 * d.num_kv_heads * c->sm_count * 8 * HD));
  RET(dmalloc(c, &c->s_pml2, (size_t)M2 * d.num_kv_heads * c->sm_count * 8 * 2));
  RET(dmalloc(c, &c->s_tok, 64));
  RET(dmalloc(c, &c->kv_len_dev, 16));
  RET(dmalloc(c, &c->row_mode_dev, 16));
  {
    int ones[16];
    for (int i = 0; i < 16; ++i) ones[i] = 1;
    CK(cudaMemcpy(c->row_mode_dev, ones, sizeof ones, cudaMemcpyHostToDevice));
  }
  c->kv_len_host.assign(M2, 0);
  c->seq_pages.assign(M2, {});
  for (auto& r : c->raw) if (r.second.p) { cudaFree(r.second.p); r.second.p = nullptr; }
  CK(cudaDeviceSynchronize());
  c->finalized = true;
  return 0;
}

extern "C" int64_t vv_weight_bytes(vv_ctx* c, int which) { return (c && which >= 0 && which < 6) ? c->wbytes[which] : -1; }
extern "C" int64_t vv_launch_count(vv_ctx* c) { return c ? c->launches : -1; }

// ------------------------------------------------------------------------------------------------
// graph cache: every per-frame program is captured once per distinct argument tuple and replayed
// ------------------------------------------------------------------------------------------------
template <class F>
static int run_cached(vv_ctx* c, const std::string& key, cudaStream_t s, F&& enqueue) {
  if (!c->use_graphs || s == nullptr) { L l{c, s}; return enqueue(l); }
  auto it = c->graphs.find(key);
  if (it == c->graphs.end()) {
    const int64_t before = c->launches;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    L l{c, s};
    int r = enqueue(l);
    cudaGraph_t g = nullptr;
    cudaError_t e = cudaStreamEndCapture(s, &g);
    if (r < 0) { if (g) cudaGraphDestroy(g); return r; }
    if (e != cudaSuccess) return fail(VV_ERR_CUDA, "graph capture failed (%s): %s", key.c_str(), cudaGetErrorString(e));
    GraphEntry ge;
    ge.launches = c->launches - before;
    c->launches = before;
    e = cudaGraphInstantiate(&ge.exec, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) return fail(VV_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(e));
    it = c->graphs.emplace(key, ge).first;
  }
  CK(cudaGraphLaunch(it->second.exec, s));
  c->launches += it->second.launches;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// KV pages
// ------------------------------------------------------------------------------------------------
template <class T>
static void dfree(vv_ctx* c, T** p) {
  if (!*p) return;
  auto it = std::find(c->allocs.begin(), c->allocs.end(), (void*)*p);
  if (it != c->allocs.end()) c->allocs.erase(it);
  cudaFree(*p);
  *p = nullptr;
}
static void drop_graphs(vv_ctx* c, std::initializer_list<const char*> prefixes) {
  for (auto it = c->graphs.begin(); it != c->graphs.end();) {
    bool hit = false;
    for (const char* pre : prefixes) hit = hit || it->first.rfind(pre, 0) == 0;
    if (hit) { cudaGraphExecDestroy(it->second.exec); it = c->graphs.erase(it); }
    else ++it;
  }
}

// (Re-)size the page pool.  Calling it again drops every sequence (lengths 0, all pages free) and re-allocates the pool, so a
// long-lived service can grow the cache between generate() calls; captured LM graphs bake the pool pointers and are re-captured.
extern "C" int vv_kv_init(vv_ctx* c, int64_t n_pages) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "vv_kv_init before vv_finalize_weights");
  if (n_pages < 2 * c->d.max_batch) return fail(VV_ERR_INVALID, "vv_kv_init: need at least one page per sequence (%d)", 2 * c->d.max_batch);
  CK(cudaSetDevice(c->device));
  if (c->kpool) {
    CK(cudaDeviceSynchronize());
    dfree(c, &c->kpool); dfree(c, &c->vpool); dfree(c, &c->page_table_dev);
    drop_graphs(c, {"lm:", "lmr:", "frame:"});
    for (auto it = c->sprogs.begin(); it != c->sprogs.end();) {
      if (it->first.rfind("lmf:", 0) == 0) { dfree(c, &it->second.ops); dfree(c, &it->second.tmaps); it = c->sprogs.erase(it); }
      else ++it;
    }
    std::fill(c->kv_len_host.begin(), c->kv_len_host.end(), 0);
    for (auto& pg : c->seq_pages) pg.clear();
  }
  const auto& d = c->d;
  const size_t per_layer = (size_t)n_pages * d.num_kv_heads * KV_PAGE * d.head_dim;
  RET(dmalloc(c, &c->kpool, per_layer * d.num_layers));
  RET(dmalloc(c, &c->vpool, per_layer * d.num_layers));
  c->n_pages = n_pages;
  c->max_pages = (int)n_pages;
  const size_t nt = (size_t)2 * d.max_batch * c->max_pages;
  RET(dmalloc(c, &c->page_table_dev, nt));
  c->free_pages.clear();
  for (int i = (int)n_pages - 1; i >= 0; --i) c->free_pages.push_back(i);
  return 0;
}
extern "C" int64_t vv_kv_pages_free(vv_ctx* c) { return c ? (int64_t)c->free_pages.size() : -1; }
extern "C" int64_t vv_kv_pages_total(vv_ctx* c) { return c ? c->n_pages : -1; }
extern "C" int64_t vv_kv_len(vv_ctx* c, int seq) { return (c && seq >= 0 && seq < (int)c->kv_len_host.size()) ? c->kv_len_host[seq] : -1; }

// page-table entries travel BY VALUE in the launch arguments: pages return to the free list when a sequence shrinks, so an entry can be
// rewritten while copies of its previous value are still queued on the stream -- an asynchronous copy out of a host mirror would race
struct PageVals { int v[32]; };
// block (i, layer) zeroes the K and V rows of page pv.v[i] in that layer; block (0, 0) also writes the page-table entries.  A page handed out
// again can hold a previous owner's entries, non-finite ones included, in the slots past the new owner's length: attention masks their
// scores, but its P V product would still take 0 * NaN = NaN from them.  Zeroing here, once per page grant, keeps that off the decode step.
__global__ void page_grant_kernel(int* dst, PageVals pv, int n, bf16* kpool, bf16* vpool, size_t per_layer, size_t page_elems) {
  if (blockIdx.x == 0 && blockIdx.y == 0 && (int)threadIdx.x < n) dst[threadIdx.x] = pv.v[threadIdx.x];
  const size_t o = per_layer * blockIdx.y + (size_t)pv.v[blockIdx.x] * page_elems;
  uint4* k = reinterpret_cast<uint4*>(kpool + o);
  uint4* v = reinterpret_cast<uint4*>(vpool + o);
  for (size_t i = threadIdx.x; i < page_elems / 8; i += blockDim.x) { k[i] = make_uint4(0u, 0u, 0u, 0u); v[i] = make_uint4(0u, 0u, 0u, 0u); }
}

extern "C" int vv_kv_reserve(vv_ctx* c, int seq, int64_t n_tokens, void* stream) {
  if (!c || !c->kpool) return fail(VV_ERR_STATE, "KV pool not initialised");
  if (seq < 0 || seq >= 2 * c->d.max_batch) return fail(VV_ERR_INVALID, "bad seq %d", seq);
  auto& pg = c->seq_pages[seq];
  const int64_t needp = (n_tokens + KV_PAGE - 1) / KV_PAGE;
  if (needp > c->max_pages) return fail(VV_ERR_NOMEM, "KV page pool too small (seq %d needs %lld pages of %d)", seq, (long long)needp, c->max_pages);
  size_t first = pg.size();
  while ((int64_t)pg.size() < needp) {
    if (c->free_pages.empty()) return fail(VV_ERR_NOMEM, "KV page pool exhausted (seq %d needs %lld pages)", seq, (long long)needp);
    pg.push_back(c->free_pages.back());
    c->free_pages.pop_back();
  }
  while (first < pg.size()) {
    PageVals pv;
    const int n = (int)std::min<size_t>(32, pg.size() - first);
    for (int i = 0; i < 32; ++i) pv.v[i] = i < n ? pg[first + i] : 0;
    const auto& d = c->d;
    const size_t page_elems = (size_t)d.num_kv_heads * KV_PAGE * d.head_dim;
    page_grant_kernel<<<dim3(n, d.num_layers), 256, 0, (cudaStream_t)stream>>>(c->page_table_dev + (size_t)seq * c->max_pages + first, pv, n,
                                                                                 c->kpool, c->vpool, (size_t)c->n_pages * page_elems, page_elems);
    CKL();
    c->launches++;
    first += n;
  }
  return 0;
}
// pages beyond the new length go back to the free list (a negative stream restarts at every <speech_start>; a server reuses rows)
static void release_pages(vv_ctx* c, int seq, int64_t len) {
  auto& pg = c->seq_pages[seq];
  const size_t keep = (size_t)((len + KV_PAGE - 1) / KV_PAGE);
  while (pg.size() > keep) { c->free_pages.push_back(pg.back()); pg.pop_back(); }
}

struct Lens { int v[16]; };
__global__ void kv_set_all_kernel(int* kv_len, Lens l, int n) { if (threadIdx.x < n) kv_len[threadIdx.x] = l.v[threadIdx.x]; }

static int push_lens(vv_ctx* c, cudaStream_t s) {
  Lens l;
  const int n = 2 * c->d.max_batch;
  for (int i = 0; i < 16; ++i) l.v[i] = i < n ? (int)c->kv_len_host[i] : 0;
  kv_set_all_kernel<<<1, 32, 0, s>>>(c->kv_len_dev, l, n);
  CKL();
  c->launches++;
  return 0;
}
extern "C" int vv_kv_set_len(vv_ctx* c, int seq, int64_t len, void* stream) {
  if (!c || !c->kpool) return fail(VV_ERR_STATE, "KV pool not initialised");
  if (seq < 0 || seq >= 2 * c->d.max_batch) return fail(VV_ERR_INVALID, "bad seq %d", seq);
  if (len < 0 || len > (int64_t)c->seq_pages[seq].size() * KV_PAGE) return fail(VV_ERR_INVALID, "vv_kv_set_len: %lld outside the reserved range of seq %d", (long long)len, seq);
  c->kv_len_host[seq] = len;
  release_pages(c, seq, len);
  return push_lens(c, (cudaStream_t)stream);
}
extern "C" int vv_kv_commit(vv_ctx* c, const int32_t* adv, void* stream) {
  if (!c || !c->kpool) return fail(VV_ERR_STATE, "KV pool not initialised");
  for (int i = 0; i < 2 * c->d.max_batch; ++i) c->kv_len_host[i] += adv[i] ? 1 : 0;
  return push_lens(c, (cudaStream_t)stream);
}
// drop the entry at position `pos` of a sequence: the last committed entry moves into its place (all layers), the length shrinks by one.
// Attention does not depend on the order of the cached entries (keys are stored rotated), so this is how a sequence forgets an OLDER entry --
// the reference's cache shifting with refresh_negative=False hides one (modeling_vibevoice_inference.py:599-624).
__global__ void kv_move_kernel(bf16* kpool, bf16* vpool, const int* page_row, int kv_heads, int hd, size_t per_layer, int src, int dst) {
  const int layer = blockIdx.x;
  const int sp = page_row[src / KV_PAGE], dp = page_row[dst / KV_PAGE];
  for (int i = threadIdx.x; i < kv_heads * hd; i += blockDim.x) {
    const int h = i / hd, d = i % hd;
    const size_t so = per_layer * layer + (((size_t)sp * kv_heads + h) * KV_PAGE + (src % KV_PAGE)) * hd + d;
    const size_t dofs = per_layer * layer + (((size_t)dp * kv_heads + h) * KV_PAGE + (dst % KV_PAGE)) * hd + d;
    kpool[dofs] = kpool[so];
    vpool[dofs] = vpool[so];
  }
}
extern "C" int vv_kv_delete_slot(vv_ctx* c, int seq, int64_t pos, void* stream) {
  if (!c || !c->kpool) return fail(VV_ERR_STATE, "KV pool not initialised");
  if (seq < 0 || seq >= 2 * c->d.max_batch) return fail(VV_ERR_INVALID, "bad seq %d", seq);
  const int64_t len = c->kv_len_host[seq];
  if (pos < 0 || pos >= len) return fail(VV_ERR_INVALID, "vv_kv_delete_slot: position %lld outside [0,%lld)", (long long)pos, (long long)len);
  const auto& d = c->d;
  if (pos != len - 1) {
    const size_t per_layer = (size_t)c->n_pages * d.num_kv_heads * KV_PAGE * d.head_dim;
    kv_move_kernel<<<d.num_layers, 256, 0, (cudaStream_t)stream>>>(c->kpool, c->vpool, c->page_table_dev + (size_t)seq * c->max_pages, d.num_kv_heads, d.head_dim, per_layer,
                                                                  (int)(len - 1), (int)pos);
    CKL();
    c->launches++;
  }
  c->kv_len_host[seq] = len - 1;
  release_pages(c, seq, len - 1 + 1);     // keep the page of the next speculative entry
  return push_lens(c, (cudaStream_t)stream);
}
extern "C" int vv_set_row_mode(vv_ctx* c, const int32_t* rm, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  Lens l;
  for (int i = 0; i < 16; ++i) l.v[i] = i < 2 * c->d.max_batch ? rm[i] : 0;
  kv_set_all_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(c->row_mode_dev, l, 2 * c->d.max_batch);
  CKL();
  c->launches++;
  return 0;
}
extern "C" int vv_set_rope_inv_freq(vv_ctx* c, const float* f, int n) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  if (n != c->d.head_dim / 2) return fail(VV_ERR_INVALID, "inv_freq must have %d entries", c->d.head_dim / 2);
  CK(cudaMemcpy(c->inv_freq, f, sizeof(float) * n, cudaMemcpyHostToDevice));
  return 0;
}
extern "C" int vv_kv_write(vv_ctx* c, int seq, int layer, int64_t pos0, int64_t n_tokens, const void* k, const void* v, void* stream) {
  if (!c || !c->kpool) return fail(VV_ERR_STATE, "KV pool not initialised");
  RET(vv_kv_reserve(c, seq, pos0 + n_tokens, stream));
  const auto& d = c->d;
  const size_t per_layer = (size_t)c->n_pages * d.num_kv_heads * KV_PAGE * d.head_dim;
  kv_write_kernel<<<(unsigned)n_tokens, 128, 0, (cudaStream_t)stream>>>((const bf16*)k, (const bf16*)v, c->kpool + per_layer * layer,
                                                                      c->vpool + per_layer * layer,
                                                                      c->page_table_dev + (size_t)seq * c->max_pages, d.num_kv_heads, d.head_dim, pos0, n_tokens);
  CKL();
  c->launches++;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// a-3: LM decode
// ------------------------------------------------------------------------------------------------
static int enqueue_lm_head(const L& l, const float* hidden, float* logits, int32_t* tokens) {
  vv_ctx* c = l.c;
  CK(launch_k(l, lm_head_argmax_kernel, dim3(c->d.max_batch), dim3(256), 0, hidden, c->head_valid, c->valid_ids_dev, c->d.n_valid_ids, c->d.hidden_size, logits, tokens));
  return 0;
}

// All of decoder layers [li0, li1) as ONE weight-stream program over the residual stream s_h (rows = 2B sequences; rows with row_mode 0
// neither read nor append KV): per layer QKV -> attention (K/V pages through the ring) -> O (prologue merges the attention partials) ->
// gate/up -> down.  5 grid barriers per layer, no kernel boundary inside the stack.
static int lm_stream_prog_full(vv_ctx* c, int li0, int li1, const vv_ctx::StreamProg** out) {
  char key[64];
  snprintf(key, sizeof key, "lmf:%d:%d", li0, li1);
  auto it = c->sprogs.find(key);
  if (it != c->sprogs.end()) { *out = &it->second; return 0; }
  const auto& d = c->d;
  const int H = d.hidden_size, I = d.intermediate_size, M = 2 * d.max_batch, nq = d.num_q_heads * d.head_dim;
  StreamBuilder b(c);
  b.nop(false, c->s_qkv, (long long)M * c->Nqkv);
  for (int li = li0; li < li1; ++li) {
    const LmLayer& y = c->lm[li];
    SOp* o;
    RET(b.gemv(y.wqkv, y.bqkv, c->s_h, H, c->s_qkv, c->Nqkv, M, c->Nqkv, H, true, &o));
    o->pro = SP_RMSNORM; o->pro_w = y.ln1; o->pro_eps = d.rms_norm_eps;
    if (li == li0) { b.fill_att(&o->att, li); o->rope_rows = M; }        // positions are the same for every layer of this call
    RET(b.attn(li, M));
    RET(b.gemv(y.wo, nullptr, nullptr, 0, c->s_h, H, M, H, nq, true, &o));
    o->pro = SP_COMBINE;
    b.fill_att(&o->att, li);
    b.needs_kv.push_back((int)b.ops.size() - 1);
    o->init_dst = c->s_qkv; o->init_n = (long long)M * c->Nqkv;
    o->init2_dst = c->s_lgu; o->init2_n = (long long)M * 2 * I;
    RET(b.gemv(y.wgu, nullptr, c->s_h, H, c->s_lgu, 2 * I, M, 2 * I, H, true, &o));
    o->pro = SP_RMSNORM; o->pro_w = y.ln2; o->pro_eps = d.rms_norm_eps;
    RET(b.gemv(y.wdown, nullptr, c->s_lgu, 2 * I, c->s_h, H, M, H, I, true, &o));
    o->pro = SP_SWIGLU;
  }
  vv_ctx::StreamProg pr;
  RET(finish_stream(b, &pr));
  it = c->sprogs.emplace(key, pr).first;
  *out = &it->second;
  return 0;
}

static int enqueue_final_norm(const L& l, float* hidden) {
  vv_ctx* c = l.c;
  const auto& d = c->d;
  const int H = d.hidden_size, M = 2 * d.max_batch;
  if (H >= 512) CK(launch_k(l, rows_norm_block_kernel, dim3(M), dim3(256), 0, c->s_h, c->lm_norm, hidden, H, d.rms_norm_eps));
  else CK(launch_k(l, rows_norm_kernel, dim3((M + 7) / 8), dim3(256), 0, c->s_h, c->lm_norm, hidden, M, H, d.rms_norm_eps));
  return 0;
}

static int enqueue_lm_decode(const L& l, const float* embeds, float* hidden, float* logits, int32_t* tokens, const vv_ctx::StreamProg& sprog) {
  vv_ctx* c = l.c;
  const int H = c->d.hidden_size, M = 2 * c->d.max_batch;
  CK(cudaMemcpyAsync(c->s_h, embeds, (size_t)M * H * 4, cudaMemcpyDeviceToDevice, l.s));
  RET(launch_stream(l, sprog));
  RET(enqueue_final_norm(l, hidden));
  return enqueue_lm_head(l, hidden, logits, tokens);
}

// streaming-0.5B (SURVEY 8f-1): the Qwen2 stack is split into a lower text-only stack without final norm and an upper "TTS LM" stack
// (modeling_vibevoice_streaming.py:134-146); each stack keeps its own KV sequences (lengths differ: the upper stack also sees the speech
// positions).  One call runs layers [begin, end) for the rows enabled by vv_set_row_mode, appends their K/V speculatively at kv_len (commit
// with vv_kv_commit as for vv_lm_decode) and returns the residual stream -- normalised with the model's final norm iff final_norm != 0.
static int enqueue_lm_range(const L& l, const float* embeds, int final_norm, float* hidden, const vv_ctx::StreamProg& sprog) {
  vv_ctx* c = l.c;
  const int H = c->d.hidden_size, M = 2 * c->d.max_batch;
  CK(cudaMemcpyAsync(c->s_h, embeds, (size_t)M * H * 4, cudaMemcpyDeviceToDevice, l.s));
  RET(launch_stream(l, sprog));
  if (final_norm) return enqueue_final_norm(l, hidden);
  CK(cudaMemcpyAsync(hidden, c->s_h, (size_t)M * H * 4, cudaMemcpyDeviceToDevice, l.s));
  return 0;
}

extern "C" int vv_lm_decode(vv_ctx* c, const float* embeds, float* hidden, float* logits, int32_t* tokens, void* stream) {
  if (!c || !c->kpool) return fail(VV_ERR_STATE, "vv_lm_decode: KV pool not initialised");
  CK(cudaSetDevice(c->device));
  for (int s = 0; s < 2 * c->d.max_batch; ++s) RET(vv_kv_reserve(c, s, c->kv_len_host[s] + 1, stream));
  char key[256];
  snprintf(key, sizeof key, "lm:%p:%p:%p:%p", (const void*)embeds, (void*)hidden, (void*)logits, (void*)tokens);
  const vv_ctx::StreamProg* sprog;      // built outside stream capture
  RET(lm_stream_prog_full(c, 0, c->d.num_layers, &sprog));
  return run_cached(c, key, (cudaStream_t)stream, [&](const L& l) { return enqueue_lm_decode(l, embeds, hidden, logits, tokens, *sprog); });
}
extern "C" int vv_lm_head(vv_ctx* c, const float* hidden, float* logits, int32_t* tokens, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  L l{c, (cudaStream_t)stream};
  return enqueue_lm_head(l, hidden, logits, tokens);
}
// Full-vocabulary logits for the positive rows: only needed when the caller installs its own LogitsProcessor objects or samples with
// top-k / top-p warpers, which rank the whole vocabulary BEFORE the token constraint (modeling_vibevoice_inference.py:310-319, 488-490).
// One GEMV over the (tied) embedding / lm_head matrix; the default path never calls this (it computes the <= 5 surviving logits only).
extern "C" int vv_lm_logits_full(vv_ctx* c, const float* hidden, float* logits_out, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  CK(cudaSetDevice(c->device));
  L l{c, (cudaStream_t)stream};
  GemvP p = mk(c->lm_head_w, nullptr, hidden, c->d.hidden_size, logits_out, c->d.vocab_size, c->d.max_batch, c->d.vocab_size, c->d.hidden_size);
  return linear(l, p);
}
struct Toks { int v[16]; };
__global__ void embed_gather_val_kernel(const bf16* __restrict__ table, Toks t, float* __restrict__ out, int H) {
  const bf16* row = table + (size_t)t.v[blockIdx.x] * H;
  for (int k = threadIdx.x; k < H; k += blockDim.x) out[(size_t)blockIdx.x * H + k] = __bfloat162float(row[k]);
}
extern "C" int vv_lm_decode_range(vv_ctx* c, const float* embeds, int layer_begin, int layer_end, int final_norm, float* hidden, void* stream) {
  if (!c || !c->kpool) return fail(VV_ERR_STATE, "vv_lm_decode_range: KV pool not initialised");
  if (layer_begin < 0 || layer_end > c->d.num_layers || layer_begin >= layer_end) return fail(VV_ERR_INVALID, "bad layer range [%d,%d)", layer_begin, layer_end);
  CK(cudaSetDevice(c->device));
  for (int s = 0; s < 2 * c->d.max_batch; ++s) RET(vv_kv_reserve(c, s, c->kv_len_host[s] + 1, stream));
  char key[256];
  snprintf(key, sizeof key, "lmr:%p:%p:%d:%d:%d", (const void*)embeds, (void*)hidden, layer_begin, layer_end, final_norm);
  const vv_ctx::StreamProg* sprog;
  RET(lm_stream_prog_full(c, layer_begin, layer_end, &sprog));
  return run_cached(c, key, (cudaStream_t)stream, [&](const L& l) { return enqueue_lm_range(l, embeds, final_norm, hidden, *sprog); });
}

extern "C" int vv_embed_tokens(vv_ctx* c, const int32_t* tokens_host, int n, float* out, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  if (n < 1 || n > 16) return fail(VV_ERR_INVALID, "vv_embed_tokens: n must be in [1,16]");
  Toks t;
  for (int i = 0; i < 16; ++i) {
    t.v[i] = i < n ? tokens_host[i] : 0;
    if (t.v[i] < 0 || t.v[i] >= c->d.vocab_size) return fail(VV_ERR_INVALID, "token id %d out of range", t.v[i]);
  }
  embed_gather_val_kernel<<<n, 256, 0, (cudaStream_t)stream>>>(c->embed, t, out, c->d.hidden_size);
  CKL();
  c->launches++;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// a-4: diffusion sampler
// ------------------------------------------------------------------------------------------------
static int set_diffusion_steps(vv_ctx* c, int n_steps, const float* timesteps, const float* coef, int ncol, void* stream);
extern "C" int vv_set_diffusion_steps(vv_ctx* c, int n_steps, const float* timesteps, const float* coef, void* stream) {
  return set_diffusion_steps(c, n_steps, timesteps, coef, 6, stream);
}
extern "C" int vv_set_diffusion_steps_sde(vv_ctx* c, int n_steps, const float* timesteps, const float* coef7, void* stream) {
  return set_diffusion_steps(c, n_steps, timesteps, coef7, 7, stream);
}
extern "C" int vv_set_step_noise(vv_ctx* c, const float* step_noise) {
  if (!c) return fail(VV_ERR_INVALID, "null ctx");
  if (c->step_noise != step_noise) {            // captured graphs hold the old pointer
    drop_graphs(c, {"tail:", "diff:", "frame:"});
  }
  c->step_noise = step_noise;
  return 0;
}
static int set_diffusion_steps(vv_ctx* c, int n_steps, const float* timesteps, const float* coef, int ncol, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  if (n_steps < 1 || n_steps > c->d.max_diffusion_steps) return fail(VV_ERR_INVALID, "n_steps %d outside [1,%d]", n_steps, c->d.max_diffusion_steps);
  CK(cudaSetDevice(c->device));
  cudaStream_t s = (cudaStream_t)stream;
  const int H = c->d.hidden_size;
  std::vector<DpmCoef> cf(n_steps);
  for (int i = 0; i < n_steps; ++i) {
    cf[i].a0 = coef[i * ncol + 0]; cf[i].s0 = coef[i * ncol + 1]; cf[i].ks = coef[i * ncol + 2]; cf[i].kx = coef[i * ncol + 3];
    cf[i].rinv = coef[i * ncol + 4]; cf[i].order = (int)coef[i * ncol + 5]; cf[i].kn = ncol == 7 ? coef[i * ncol + 6] : 0.f;
  }
  c->sde = (ncol == 7);
  c->coef_host = cf;
  c->coef_version++;
  CK(cudaStreamSynchronize(s));
  float* tdev = c->s_t1;   // reuse as staging for the timesteps (n floats) before it is overwritten below
  CK(cudaMemcpy(tdev, timesteps, sizeof(float) * n_steps, cudaMemcpyHostToDevice));
  timestep_feat_kernel<<<n_steps, 256, 0, s>>>(tdev, c->tfreqs, c->s_tfeat, n_steps);
  CKL();
  CK(cudaStreamSynchronize(s));
  L l{c, s};
  GemvP p = mk(c->h_t0, nullptr, c->s_tfeat, 256, c->s_t1, H, n_steps, H, 256);
  p.epi = EPI_SILU;
  RET(linear(l, p, c->temb_info[0]));
  p = mk(c->h_t2, nullptr, c->s_t1, H, c->temb, H, n_steps, H, H);
  RET(linear(l, p, c->temb_info[1]));
  CK(cudaStreamSynchronize(s));
  c->n_steps = n_steps;
  // programs captured with another step count are stale
  drop_graphs(c, {"tail:", "diff:", "frame:"});
  return 0;
}

__global__ void set_float_kernel(float* p, float v) { *p = v; }
// the CFG scale is read from device memory by the solver kernels, so one captured graph serves every value (a service with a
// user-controlled cfg_scale would otherwise capture and keep one frame-tail graph per distinct float)
static int set_cfg(vv_ctx* c, float cfg, cudaStream_t s) {
  if (memcmp(&cfg, &c->cfg_last, sizeof(float)) == 0) return 0;
  set_float_kernel<<<1, 1, 0, s>>>(c->cfg_dev, cfg);
  CKL();
  c->launches++;
  c->cfg_last = cfg;
  return 0;
}

// The N-step sampler as ONE weight-stream program (vv_stream.cuh): per step 4 x (gate/up with AdaLN prologue -> raw sums; down with SwiGLU
// prologue, gated-residual epilogue) + final layer + noisy_images_proj whose prologue is the CFG / DPM-Solver++ update.  10 grid barriers
// per step instead of 10 kernels, and the TMA ring keeps streaming head weights across all of them.
// The program is a sequence of blocks: block 0 = proj(-1) (x = noisy_images_proj(initial noise)); then per step i, from block
// 1 + i (L + 2): head layer li = 0 .. L-1 (gate/up + down), the final layer, proj(i).  sampler_build emits blocks [blk0, blk1) only.  Every
// value one block hands to the next lives in global memory (s_hx, the gu double buffer, s_v, the s_z / s_x0 parity buffers, s_mod) and the
// zero-fill jobs ride on earlier stages, so the blocks launched one after another compute what the whole program does (vv_debug_sampler_taps).
static int sampler_blocks(const vv_ctx* c) { return 1 + c->n_steps * (c->d.head_layers + 2); }
static int sampler_build(StreamBuilder& b, const float* noise, float* latent_out, int blk0, int blk1) {
  vv_ctx* c = b.c;
  const auto& d = c->d;
  const int H = d.hidden_size, F = d.head_ffn_dim, B = d.max_batch, M = 2 * B, LH = d.head_layers, N = c->n_steps;
  const long long modld = (long long)(3 * LH + 2) * H;
  auto in = [&](int blk) { return blk >= blk0 && blk < blk1; };
  auto dpm = [&](int i) {
    SDpm o;
    memset(&o, 0, sizeof o);
    if (i < 0) { o.z_in = c->s_z + B * 64; o.z_out = c->s_z; o.x0_in = c->s_x0 + B * 64; o.x0_out = c->s_x0; }
    else {
      o.z_in = c->s_z + (size_t)(i & 1) * B * 64; o.z_out = c->s_z + (size_t)((i + 1) & 1) * B * 64;
      o.x0_in = c->s_x0 + (size_t)(i & 1) * B * 64; o.x0_out = c->s_x0 + (size_t)((i + 1) & 1) * B * 64;
    }
    o.v = c->s_v; o.noise = noise; o.cfg_p = c->cfg_dev; o.step_noise = c->sde ? c->step_noise : nullptr;
    o.latent_out = (i == N - 1) ? latent_out : nullptr; o.step = i; o.B = B;
    if (i >= 0) o.c = c->coef_host[i];
    return o;
  };
  auto proj = [&](int i, bool sync) -> int {       // x = noisy_images_proj(z'), z' = solver update of step i (i = -1: the initial noise)
    SOp* o;
    RET(b.gemv(c->h_noisy, nullptr, nullptr, 0, c->s_hx, H, M, H, 64, sync, &o));
    o->pro = SP_DPM; o->store = 1; o->dpm = dpm(i);
    return 0;
  };
  float* gu[2] = {c->s_hgu, c->s_hgu + (size_t)M * 2 * F};
  if (in(0)) {
    RET(proj(-1, false));
    b.ops.back().init_dst = gu[0]; b.ops.back().init_n = (long long)M * 2 * F;
  }
  for (int i = 0; i < N; ++i) {
    const float* mod = c->s_mod + (size_t)i * M * modld;
    const int base = 1 + i * (LH + 2);
    for (int li = 0; li < LH; ++li) {
      if (!in(base + li)) continue;
      const HeadLayer& hl = c->head[li];
      SOp* o;
      RET(b.gemv(hl.wgu, nullptr, c->s_hx, H, gu[li & 1], 2 * F, M, 2 * F, H, true, &o));
      o->pro = SP_ADALN; o->pro_w = hl.norm; o->pro_eps = d.head_rms_eps;
      o->pro_shift = mod + (size_t)li * 3 * H; o->pro_scale = mod + (size_t)li * 3 * H + H; o->pro_ld = modld;
      o->init_dst = gu[(li + 1) & 1]; o->init_n = (long long)M * 2 * F;           // the other buffer: its reader (down of li-1) is done
      RET(b.gemv(hl.wdown, nullptr, gu[li & 1], 2 * F, c->s_hx, H, M, H, F, true, &o));
      o->pro = SP_SWIGLU; o->alpha_kind = SA_GATE; o->alpha = mod + (size_t)li * 3 * H + 2 * H; o->lda = modld;
      if (li == 0) { o->init_dst = c->s_v; o->init_n = (long long)M * 64; }        // final layer of this step accumulates into s_v
    }
    if (in(base + LH)) {
      SOp* o;
      RET(b.gemv(c->h_final, nullptr, c->s_hx, H, c->s_v, 64, M, 64, H, true, &o));
      o->pro = SP_ADALN; o->pro_w = nullptr; o->pro_eps = d.head_rms_eps;
      o->pro_shift = mod + (size_t)LH * 3 * H; o->pro_scale = mod + (size_t)LH * 3 * H + H; o->pro_ld = modld;
    }
    if (in(base + LH + 1)) RET(proj(i, true));
  }
  if (!b.ops.empty()) b.ops.front().sync_before = 0;     // the first stage of a launch waits for nothing
  return 0;
}
static int sampler_stream_prog(vv_ctx* c, const float* noise, float* latent_out, const vv_ctx::StreamProg** out) {
  char key[256];
  snprintf(key, sizeof key, "samp:%p:%p:%d:%d:%p:%d", (const void*)noise, (void*)latent_out, c->n_steps, (int)c->sde, (const void*)c->step_noise,
           c->coef_version);       // solver coefficients are baked into the program
  auto it = c->sprogs.find(key);
  if (it != c->sprogs.end()) { *out = &it->second; return 0; }
  StreamBuilder b(c);
  RET(sampler_build(b, noise, latent_out, 0, sampler_blocks(c)));
  vv_ctx::StreamProg pr;
  RET(finish_stream(b, &pr));
  it = c->sprogs.emplace(key, pr).first;
  *out = &it->second;
  return 0;
}

// Everything the samp: program reads besides its inputs: cond_proj, the conditioning kernel and the all-steps AdaLN modulation GEMM.
// info_cond / info_mod (optional): {kernel, split-K} linear() ran for cond_proj / the modulation GEMM.
static int diffusion_preamble(const L& l, const float* cond, int32_t* info_cond = nullptr, int32_t* info_mod = nullptr) {
  vv_ctx* c = l.c;
  const auto& d = c->d;
  const int H = d.hidden_size, M = 2 * d.max_batch, LH = d.head_layers, N = c->n_steps;
  if (N < 1) return fail(VV_ERR_STATE, "vv_set_diffusion_steps not called");
  const int modld = (3 * LH + 2) * H;
  if (c->sde && !c->step_noise) return fail(VV_ERR_STATE, "sde-dpmsolver++ needs vv_set_step_noise before sampling");
  GemvP p = mk(c->h_cond, nullptr, cond, H, c->s_condp, H, M, H, H);
  RET(linear(l, p, info_cond));
  {
    const long long n = (long long)N * M * H;
    CK(launch_k(l, head_cond_prep_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, c->s_condp, c->temb, c->s_call, N, M, H));
  }
  // AdaLN modulation of ALL steps and layers in one tensor-core GEMM: c_all [N*M, H] x W_mod^T -> [N*M, (3L+2)H].
  // (the reference recomputes Linear(silu(c)) inside every head call, diffusion_head.py:159, 185; c depends only on (cond, t_i))
  p = mk(c->h_mod, nullptr, c->s_call, H, c->s_mod, modld, N * M, modld, H);
  RET(linear(l, p, info_mod));
  return 0;
}

static int enqueue_diffusion(const L& l, const float* cond, const vv_ctx::StreamProg& sprog) {
  RET(diffusion_preamble(l, cond));
  return launch_stream(l, sprog);
}

extern "C" int vv_diffusion_sample(vv_ctx* c, const float* cond, const float* noise, const int32_t* active, float cfg, float* latent_out,
                                   void* stream) {
  (void)active;   // rows are independent; inactive rows are computed and ignored (static shapes keep the program graph-replayable)
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  CK(cudaSetDevice(c->device));
  RET(set_cfg(c, cfg, (cudaStream_t)stream));
  char key[256];
  snprintf(key, sizeof key, "diff:%p:%p:%p", (const void*)cond, (const void*)noise, (void*)latent_out);
  const vv_ctx::StreamProg* sprog;      // built outside stream capture (it allocates and copies)
  RET(sampler_stream_prog(c, noise, latent_out, &sprog));
  return run_cached(c, key, (cudaStream_t)stream, [&](const L& l) { return enqueue_diffusion(l, cond, *sprog); });
}

// ---- solver-step taps of the sampler (vv_debug_sampler_taps): the preamble's outputs, then what every block of the samp: program leaves
// behind, copied out in order.  block = the sampler block after which the tap is copied (-1: before the first).
enum { STAP_THID = 0, STAP_TEMB, STAP_COND, STAP_MOD, STAP_LAYER, STAP_V, STAP_Z, STAP_X0, STAP_HX, STAP_LATENT };
struct SampTap { int kind, step, layer, rows, cols; const float* src; int block; };
static void sampler_tap_plan(const vv_ctx* c, float* latent_out, std::vector<SampTap>* plan) {
  const auto& d = c->d;
  const int H = d.hidden_size, B = d.max_batch, M = 2 * B, LH = d.head_layers, N = c->n_steps, modld = (3 * LH + 2) * H;
  plan->clear();
  plan->push_back({STAP_THID, -1, -1, N, H, c->s_t1, -1});
  plan->push_back({STAP_TEMB, -1, -1, N, H, c->temb, -1});
  plan->push_back({STAP_COND, -1, -1, M, H, c->s_condp, -1});
  plan->push_back({STAP_MOD, -1, -1, N * M, modld, c->s_mod, -1});
  auto proj = [&](int i, int blk) {             // proj(i) writes z_{i+1} and x0_i into parity slot (i + 1) & 1 (i = -1: slot 0)
    const size_t slot = (size_t)((i + 1) & 1) * B * 64;
    plan->push_back({STAP_Z, i, -1, B, 64, c->s_z + slot, blk});
    plan->push_back({STAP_X0, i, -1, B, 64, c->s_x0 + slot, blk});
    plan->push_back({STAP_HX, i, -1, M, H, c->s_hx, blk});
  };
  proj(-1, 0);
  for (int i = 0; i < N; ++i) {
    const int base = 1 + i * (LH + 2);
    for (int li = 0; li < LH; ++li) plan->push_back({STAP_LAYER, i, li, M, H, c->s_hx, base + li});
    plan->push_back({STAP_V, i, -1, M, 64, c->s_v, base + LH});
    proj(i, base + LH + 1);
  }
  plan->push_back({STAP_LATENT, N - 1, -1, B, 64, latent_out, sampler_blocks(c) - 1});
}
// the fields that make two stages compute the same thing (the tensor-map and op-array addresses differ between programs)
static bool same_stage(const SOp& a, const SOp& b) {
  return a.kind == b.kind && a.M == b.M && a.N == b.N && a.K == b.K && a.nB == b.nB && a.k0 == b.k0 && a.krow == b.krow && a.pro == b.pro &&
         a.x == b.x && a.ldx == b.ldx && a.pro_w == b.pro_w && a.pro_shift == b.pro_shift && a.pro_scale == b.pro_scale && a.y == b.y &&
         a.ldy == b.ldy && a.alpha_kind == b.alpha_kind && a.alpha == b.alpha && a.store == b.store && a.init_dst == b.init_dst &&
         a.init_n == b.init_n && a.dpm.z_in == b.dpm.z_in && a.dpm.z_out == b.dpm.z_out && a.dpm.x0_in == b.dpm.x0_in &&
         a.dpm.x0_out == b.dpm.x0_out && a.dpm.v == b.dpm.v && a.dpm.noise == b.dpm.noise && a.dpm.step_noise == b.dpm.step_noise &&
         a.dpm.latent_out == b.dpm.latent_out && a.dpm.step == b.dpm.step && memcmp(&a.dpm.c, &b.dpm.c, sizeof a.dpm.c) == 0;
}
extern "C" int vv_debug_sampler_taps(vv_ctx* c, const float* cond, const float* noise, float cfg, float* latent_out, float* taps,
                                     int64_t taps_floats, int32_t* meta, void* stream) {
  if (!c) return fail(VV_ERR_INVALID, "null ctx");
  if (!c->finalized) return fail(VV_ERR_STATE, "vv_debug_sampler_taps: not finalized");
  if (c->n_steps < 1) return fail(VV_ERR_STATE, "vv_debug_sampler_taps: vv_set_diffusion_steps not called");
  std::vector<SampTap> plan;
  sampler_tap_plan(c, latent_out, &plan);
  const int n = (int)plan.size();
  long long need = 0;
  for (int i = 0; i < n; ++i) {
    const SampTap& t = plan[i];
    need += (long long)t.rows * t.cols;
    if (meta) { int32_t* m = meta + 7 * i; m[0] = t.kind; m[1] = t.step; m[2] = t.layer; m[3] = t.rows; m[4] = t.cols; m[5] = -1; m[6] = 0; }
  }
  if (!taps) return n;
  if (taps_floats < need) return fail(VV_ERR_INVALID, "vv_debug_sampler_taps: %lld floats of tap space, the sampler needs %lld", (long long)taps_floats, need);
  if (!cond || !noise || !latent_out) return fail(VV_ERR_INVALID, "vv_debug_sampler_taps: null condition, noise or latent");
  if (c->sde && !c->step_noise) return fail(VV_ERR_STATE, "sde-dpmsolver++ needs vv_set_step_noise before sampling");
  CK(cudaSetDevice(c->device));
  cudaStream_t s = (cudaStream_t)stream;
  // production's own program (cached under its production key, as vv_diffusion_sample would): every block must run on its kernel variant
  // and be exactly its stages, K split included
  const vv_ctx::StreamProg* full;
  RET(sampler_stream_prog(c, noise, latent_out, &full));
  std::vector<SOp> full_ops(full->n_ops);
  CK(cudaMemcpy(full_ops.data(), full->ops, full_ops.size() * sizeof(SOp), cudaMemcpyDeviceToHost));
  const int nb = sampler_blocks(c);
  std::vector<vv_ctx::StreamProg> progs(nb);
  auto release = [&]() { for (auto& p : progs) { if (p.ops) dfree(c, &p.ops); if (p.tmaps) dfree(c, &p.tmaps); } };
  int rc = 0, at = 0;
  for (int k = 0; k < nb && rc == 0; ++k) {
    StreamBuilder b(c);
    rc = sampler_build(b, noise, latent_out, k, k + 1);
    if (rc == 0) rc = finish_stream(b, &progs[k]);
    if (rc == 0 && progs[k].variant != full->variant)
      rc = fail(VV_ERR_STATE, "vv_debug_sampler_taps: block %d runs on kernel variant %d, the program on %d", k, progs[k].variant, full->variant);
    for (int j = 0; rc == 0 && j < (int)b.ops.size(); ++j, ++at)
      if (at >= full->n_ops || !same_stage(b.ops[j], full_ops[at]) || (j > 0 && b.ops[j].sync_before != full_ops[at].sync_before))
        rc = fail(VV_ERR_STATE, "vv_debug_sampler_taps: stage %d of block %d is not stage %d of the program", j, k, at);
  }
  if (rc == 0 && at != full->n_ops) rc = fail(VV_ERR_STATE, "vv_debug_sampler_taps: the blocks have %d stages, the program %d", at, full->n_ops);
  if (rc < 0) { release(); return rc; }
  int32_t info[2][2] = {{-1, 0}, {-1, 0}};      // cond_proj, modulation GEMM
  L l{c, s};
  size_t t = 0;
  long long off = 0;
  auto put = [&](int blk) -> int {
    for (; t < plan.size() && plan[t].block == blk; ++t) {
      const long long cnt = (long long)plan[t].rows * plan[t].cols;
      CK(cudaMemcpyAsync(taps + off, plan[t].src, (size_t)cnt * sizeof(float), cudaMemcpyDeviceToDevice, s));
      off += cnt;
    }
    return 0;
  };
  rc = set_cfg(c, cfg, s);
  if (rc == 0) rc = diffusion_preamble(l, cond, info[0], info[1]);
  if (rc == 0) rc = put(-1);
  for (int k = 0; k < nb && rc == 0; ++k) {
    rc = launch_stream(l, progs[k]);
    if (rc == 0) rc = put(k);
  }
  if (rc == 0 && cudaStreamSynchronize(s) != cudaSuccess) rc = fail(VV_ERR_CUDA, "vv_debug_sampler_taps: %s", cudaGetErrorString(cudaGetLastError()));
  release();
  if (rc < 0) return rc;
  if (c->st_diag_host[0]) return fail(VV_ERR_CUDA, "stream kernel watchdog: code %u cta %u thread %u a %u b %u c %u", c->st_diag_host[0], c->st_diag_host[1],
                                      c->st_diag_host[2], c->st_diag_host[3], c->st_diag_host[4], c->st_diag_host[5]);
  if (t != plan.size()) return fail(VV_ERR_STATE, "vv_debug_sampler_taps: copied %zu of %d taps", t, n);
  if (meta)
    for (int i = 0; i < n; ++i) {
      int32_t* m = meta + 7 * i;
      const SampTap& p = plan[i];
      const int32_t* ki = p.kind == STAP_THID ? c->temb_info[0] : p.kind == STAP_TEMB ? c->temb_info[1] : p.kind == STAP_COND ? info[0]
                        : p.kind == STAP_MOD ? info[1] : nullptr;
      if (ki) { m[5] = ki[0]; m[6] = ki[1]; }
      else { m[5] = progs[p.block].variant; m[6] = progs[p.block].n_ops; }    // progs' fields outlive release(): only the device arrays go
    }
  return n;
}

// ------------------------------------------------------------------------------------------------
// a-5 / a-6: streaming codec
// ------------------------------------------------------------------------------------------------
static int assemble(const L& l, const float* src, const float* hist, float* win, float* next, int B, int T, int ctx, int C,
                    const float* norm_w, float eps, float alpha, float beta) {
  const int rows = B * (ctx + T);
  if (C >= 512) CK(launch_k(l, assemble_window_block_kernel, dim3(rows), dim3(256), 0, src, hist, win, next, B, T, ctx, C, norm_w, eps, alpha, beta));
  else CK(launch_k(l, assemble_window_kernel, dim3((rows + 7) / 8), dim3(256), 0, src, hist, win, next, B, T, ctx, C, norm_w, eps, alpha, beta));
  return 0;
}

// one Block1D over x [B,T,C] (in `xin`), result in `xout` (may not alias xin)
static int enqueue_block(const L& l, const Block& b, const float* xin, float* xout, int B, int T, float eps) {
  vv_ctx* c = l.c;
  const int C = b.C, M = B * T;
  RET(assemble(l, xin, b.hist, c->s_win, b.next, B, T, 6, C, b.norm_w, eps, 1.f, 0.f));
  {
    const long long n = (long long)M * C;
    CK(launch_k(l, dwconv_res_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, xin, c->s_win, b.dw_w, b.dw_b, b.gamma, xout, B, T, C));
  }
  GemvP p;
  if (M < MMA_MIN_ROWS || (C <= MR_MAXK_NORM && c->use_wgmma != 2)) {
    p = mk(b.w1, b.b1, xout, C, c->s_u, 4 * C, M, 4 * C, C);
    p.pro = PRO_RMSNORM; p.pro_w = b.ffn_norm_w; p.pro_eps = eps; p.epi = EPI_GELU;
    RET(linear(l, p));
  } else {
    if (C >= 512) CK(launch_k(l, rows_norm_block_kernel, dim3(M), dim3(256), 0, xout, b.ffn_norm_w, c->s_xn, C, eps));
    else CK(launch_k(l, rows_norm_kernel, dim3((M + 7) / 8), dim3(256), 0, xout, b.ffn_norm_w, c->s_xn, M, C, eps));
    p = mk(b.w1, b.b1, c->s_xn, C, c->s_u, 4 * C, M, 4 * C, C);
    p.epi = EPI_GELU;
    RET(linear(l, p));
  }
  p = mk(b.w2, b.b2, c->s_u, 4 * C, xout, C, M, C, 4 * C);
  p.epi = EPI_GAMMA_RESID; p.epi_a = b.ffn_gamma; p.res = xout; p.ldres = C;
  return linear(l, p);
}

static int conv_apply(const L& l, const ConvL& cv, const float* win, float* y, int B, int T_out, int T_in) {
  // rows (b,t) read window rows [t*stride, t*stride + k) of a [ctx+T_in, Cin] window
  RowMap xm; xm.T = T_out; xm.bs = (long long)(cv.ctx + T_in) * cv.Cin; xm.rs = (long long)cv.stride * cv.Cin;
  const int M = B * T_out;
  if (cv.wf) {
    const long long n = (long long)M * cv.N;
    if (cv.K >= 64) CK(launch_k(l, conv_warp_kernel, dim3((unsigned)((n + 7) / 8)), dim3(256), 0, cv.wf, cv.bias, win, xm, y, M, cv.N, cv.K));
    else CK(launch_k(l, conv_naive_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, cv.wf, cv.bias, win, xm, y, M, cv.N, cv.K));
    return 0;
  }
  GemvP p = mk(cv.w, cv.bias, win, 0, y, cv.N, M, cv.N, cv.K);
  p.xmap = xm;
  return linear(l, p);
}

// ---- codec stages with B*T <= 8 rows (96 % of the codec's weights: 2048- and 1024-wide blocks, stem / up- / down-sampling convolutions
// next to them) as weight-stream programs (vv_stream.cuh: SP_WINDOW, SP_MIXER): two stages per Block1D instead of five kernels ------------
// Buffers: rows ping-pong between X[0] / X[1], FFN hidden sums between U[0] / U[1].  A block reads X[a], its owner CTA stores x1 into X[a^1]
// and the second linear accumulates there; a convolution accumulates into a ZEROED buffer -- zero-fill jobs ride on the stage after the
// buffer's last reader.
static bool codec_stream_stage(const vv_ctx* c, const Codec& k, int i) {
  const long long rows = (long long)c->d.max_batch * k.T[i];
  return k.T[i] <= 8 && rows <= 32;
}
static long long codec_x_floats(const vv_ctx* c) { return (long long)c->d.max_batch * 8192; }
static long long codec_u_floats(const vv_ctx* c) { return (long long)c->d.max_batch * 32768; }
static void window_op(SOp* o, const ConvL& cv, const float* src, int T_in, int T_out, int row_stride, float alpha, float beta) {
  o->pro = SP_WINDOW;
  SCodec& w = o->cod;
  memset(&w, 0, sizeof w);
  w.hist = cv.hist; w.next = cv.next; w.src = src; w.ctx = cv.ctx; w.T_in = T_in; w.T_out = T_out; w.stride = row_stride; w.cin = cv.Cin;
  w.alpha = alpha; w.beta = beta;
}
struct CodecBufs {
  float* X[2]; float* U[2];
  int cur = 0, ub = 0;
  explicit CodecBufs(vv_ctx* c) { X[0] = c->s_cx; X[1] = c->s_cx + codec_x_floats(c); U[0] = c->s_cu; U[1] = c->s_cu + codec_u_floats(c); }
};
// all blocks of one stage; rows enter in X[cur] and leave in X[cur]; if `zero_for_next` the buffer the FOLLOWING convolution accumulates
// into (= the input of the stage's last block) is zero-filled on that block's second linear
static int stage_ops(StreamBuilder& b, vv_ctx* c, CodecBufs& cb, const std::vector<Block>& blocks, int B, int T, bool zero_for_next, float* extra_zero,
                     long long extra_n) {
  for (size_t j = 0; j < blocks.size(); ++j) {
    const Block& blk = blocks[j];
    const int C = blk.C, M = B * T;
    SOp* o;
    {                                                          // mixer stage: x (X[cur]) -> x1 (X[cur^1]) + next history, channels over CTAs
      SOp& mx = b.push(SK_MIX, true);
      mx.M = M; mx.K = C; mx.x = cb.X[cb.cur]; mx.ldx = C;
      SCodec& w = mx.cod;
      memset(&w, 0, sizeof w);
      w.hist = blk.hist; w.next = blk.next; w.T_out = T; w.norm_w = blk.norm_w; w.dw_w = blk.dw_w; w.dw_b = blk.dw_b; w.gamma = blk.gamma;
      w.x1_out = cb.X[cb.cur ^ 1]; w.eps = c->d.codec_eps;
    }
    RET(b.gemv(blk.w1, blk.b1, cb.X[cb.cur ^ 1], C, cb.U[cb.ub], 4 * C, M, 4 * C, C, true, &o));
    o->pro = SP_RMSNORM; o->pro_w = blk.ffn_norm_w; o->pro_eps = c->d.codec_eps;
    o->init_dst = cb.U[cb.ub ^ 1]; o->init_n = codec_u_floats(c);          // hidden-sum buffer of the NEXT block (its reader finished two stages ago)
    RET(b.gemv(blk.w2, blk.b2, cb.U[cb.ub], 4 * C, cb.X[cb.cur ^ 1], C, M, C, 4 * C, true, &o));
    o->pro = SP_GELU; o->alpha_kind = SA_GAMMA; o->alpha = blk.ffn_gamma;
    if (j + 1 == blocks.size()) {
      if (zero_for_next) { o->init_dst = cb.X[cb.cur]; o->init_n = codec_x_floats(c); }
      if (extra_zero) { o->init2_dst = extra_zero; o->init2_n = extra_n; }
    }
    cb.cur ^= 1; cb.ub ^= 1;
  }
  return 0;
}

// decoder front: stem conv + the leading stages with <= 8 rows; *n_front = stages covered (at least stage 0: T = 1, B <= 8 rows), *out_x =
// where the last one leaves its rows
static int dec_front_stages(const vv_ctx* c) {
  int nf = 1;
  while (nf < c->d.n_stages - 1 && codec_stream_stage(c, c->dec, nf)) ++nf;
  return nf;
}
static int dec_front_prog(vv_ctx* c, const float* latent, const vv_ctx::StreamProg** out, int* n_front, float** out_x) {
  Codec& k = c->dec;
  const auto& d = c->d;
  const int B = d.max_batch;
  const int nf = dec_front_stages(c);
  *n_front = nf;
  char key[96];
  snprintf(key, sizeof key, "decf:%p", (const void*)latent);
  {
    auto hit = c->sprogs.find(key);
    if (hit != c->sprogs.end()) { *out = &hit->second; *out_x = c->dec_front_x; return 0; }
  }
  CodecBufs cb(c);
  StreamBuilder b(c);
  b.nop(false, cb.X[0], codec_x_floats(c));
  b.ops.back().init2_dst = cb.U[0]; b.ops.back().init2_n = codec_u_floats(c);
  SOp* o;
  RET(b.gemv(k.convs[0].w, k.convs[0].bias, nullptr, 0, cb.X[0], k.convs[0].N, B, k.convs[0].N, k.convs[0].K, true, &o));
  window_op(o, k.convs[0], latent, 1, 1, 1, 1.0f / c->speech_scale, -c->speech_bias);
  for (int i = 0; i < nf; ++i) {
    if (i > 0) {                                  // transposed conv into stage i: row (b, t) = [previous frame | frame t] -> s * Co outputs
      const ConvL& cv = k.convs[i];
      const int Tin = k.T[i - 1];
      RET(b.gemv(cv.w, cv.bias, nullptr, 0, cb.X[cb.cur ^ 1], cv.N, B * Tin, cv.N, cv.K, true, &o));
      window_op(o, cv, cb.X[cb.cur], Tin, Tin, 1, 1.f, 0.f);
      cb.cur ^= 1;
    }
    RET(stage_ops(b, c, cb, k.stages[i], B, k.T[i], i + 1 < nf, nullptr, 0));
  }
  *out_x = c->dec_front_x = cb.X[cb.cur];
  auto it = c->sprogs.find(key);
  if (it == c->sprogs.end()) {
    vv_ctx::StreamProg pr;
    RET(finish_stream(b, &pr));
    it = c->sprogs.emplace(key, pr).first;
  }
  *out = &it->second;
  return 0;
}

// encoder back: the trailing stages with <= 8 rows (at least the last one: T = 1, B <= 8 rows), each behind its strided conv, + the head
// conv.  `xin` = rows entering the conv of the first covered stage (produced by the kernel-per-stage path).
static int enc_back_first(const vv_ctx* c) {
  const Codec& k = c->enc;
  int f = c->d.n_stages - 1;
  while (f > 1 && codec_stream_stage(c, k, f - 1)) --f;
  return f;
}
static int enc_back_prog(vv_ctx* c, const float* xin, float* feat, const vv_ctx::StreamProg** out) {
  Codec& k = c->enc;
  const auto& d = c->d;
  const int B = d.max_batch, ns = d.n_stages, f = enc_back_first(c);
  char key[96];
  snprintf(key, sizeof key, "encb:%p:%p", (const void*)xin, (void*)feat);
  auto it = c->sprogs.find(key);
  if (it != c->sprogs.end()) { *out = &it->second; return 0; }
  CodecBufs cb(c);
  StreamBuilder b(c);
  b.nop(false, cb.X[0], codec_x_floats(c));
  b.ops.back().init2_dst = cb.U[0]; b.ops.back().init2_n = codec_u_floats(c);
  SOp* o;
  for (int i = f; i < ns; ++i) {
    const ConvL& cv = k.convs[i];
    const int Tin = k.T[i - 1], Tout = k.T[i];
    float* dst = (i == f) ? cb.X[0] : cb.X[cb.cur ^ 1];
    RET(b.gemv(cv.w, cv.bias, nullptr, 0, dst, cv.N, B * Tout, cv.N, cv.K, true, &o));      // strided conv: window rows [t*r, t*r + 2r)
    window_op(o, cv, i == f ? xin : cb.X[cb.cur], Tin, Tout, cv.stride, 1.f, 0.f);
    if (i > f) cb.cur ^= 1;
    const bool last = (i + 1 == ns);
    RET(stage_ops(b, c, cb, k.stages[i], B, Tout, !last, last ? feat : nullptr, (long long)B * d.semantic_vae_dim));
  }
  const ConvL& hd = k.convs[ns];
  RET(b.gemv(hd.w, hd.bias, nullptr, 0, feat, hd.N, B, hd.N, hd.K, true, &o));
  window_op(o, hd, cb.X[cb.cur], 1, 1, 1, 1.f, 0.f);
  vv_ctx::StreamProg pr;
  RET(finish_stream(b, &pr));
  it = c->sprogs.emplace(key, pr).first;
  *out = &it->second;
  return 0;
}

// ---- stage taps of one codec pass (vv_debug_codec_taps): every stage boundary of the kernel-per-stage path, the hand-off to / from the
// weight-stream program and the pass output, copied out [B][T][C] in pass order.  Production passes run with no sink.
enum { TAP_CONV = 0, TAP_BLOCK = 1, TAP_HANDOFF = 2, TAP_OUT = 3 };
struct TapMeta { int kind, stage, index, T, C; };
// kind, stage, index: TAP_CONV (i, 0) = output of stage i's convolution; TAP_BLOCK (i, j) = output of block j of stage i; TAP_HANDOFF
// (s, 0) = input of stage s where the stream program and the kernel-per-stage path meet; TAP_OUT (n_stages, 0) = the pass output
static void codec_tap_plan(const vv_ctx* c, int which, std::vector<TapMeta>* plan) {
  const int ns = c->d.n_stages;
  plan->clear();
  if (which == 0) {
    const Codec& k = c->dec;
    const int nf = dec_front_stages(c);
    plan->push_back({TAP_HANDOFF, nf, 0, k.T[nf - 1], k.C[nf - 1]});
    for (int i = nf; i < ns; ++i) {
      plan->push_back({TAP_CONV, i, 0, k.T[i], k.C[i]});
      for (int j = 0; j < (int)k.stages[i].size(); ++j) plan->push_back({TAP_BLOCK, i, j, k.T[i], k.C[i]});
    }
    plan->push_back({TAP_OUT, ns, 0, k.T[ns - 1], k.convs[ns].Cout});
  } else {
    const Codec& k = c->enc;
    const int stop = enc_back_first(c);
    for (int i = 0; i < stop; ++i) {
      plan->push_back({TAP_CONV, i, 0, k.T[i], k.C[i]});
      for (int j = 0; j < (int)k.stages[i].size(); ++j) plan->push_back({TAP_BLOCK, i, j, k.T[i], k.C[i]});
    }
    plan->push_back({TAP_HANDOFF, stop, 0, k.T[stop - 1], k.C[stop - 1]});
    plan->push_back({TAP_OUT, ns, 0, 1, k.convs[ns].Cout});
  }
}
struct TapSink {
  std::vector<TapMeta> plan;
  float* dst = nullptr;        // device, room for B * sum(T * C) floats
  const float* out = nullptr;  // the pass output buffer (the encoder's is written by its stream program)
  int B = 0;
  size_t next = 0;
  long long off = 0;
  int put(const L& l, int kind, int stage, int index, const float* src) {
    if (next >= plan.size() || plan[next].kind != kind || plan[next].stage != stage || plan[next].index != index)
      return fail(VV_ERR_STATE, "codec taps: tap %zu (kind %d, stage %d, index %d) is not the planned one", next, kind, stage, index);
    const long long n = (long long)B * plan[next].T * plan[next].C;
    CK(cudaMemcpyAsync(dst + off, src, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, l.s));
    off += n;
    ++next;
    return 0;
  }
};

static int enqueue_decode(const L& l, const int32_t* active, float* audio, const vv_ctx::StreamProg& front, int n_front, float* front_x,
                          TapSink* taps = nullptr) {
  vv_ctx* c = l.c;
  const auto& d = c->d;
  Codec& k = c->dec;
  const int B = d.max_batch, ns = d.n_stages;
  RET(launch_stream(l, front));                 // stem + stages [0, n_front) through the weight-stream kernel
  if (taps) RET(taps->put(l, TAP_HANDOFF, n_front, 0, front_x));
  float *xa = front_x, *xb = c->s_xb;
  for (int i = n_front; i < ns; ++i) {          // i >= 1: every remaining stage starts with its transposed conv
    const ConvL& cv = k.convs[i];
    const int Tin = k.T[i - 1];
    RET(assemble(l, xa, cv.hist, c->s_win, cv.next, B, Tin, 1, cv.Cin, nullptr, 0.f, 1.f, 0.f));
    RowMap xm; xm.T = Tin; xm.bs = (long long)(1 + Tin) * cv.Cin; xm.rs = cv.Cin;
    float* dst = (xa == c->s_xa) ? c->s_xb : c->s_xa;
    GemvP p = mk(cv.w, cv.bias, c->s_win, 0, dst, cv.N, B * Tin, cv.N, cv.K);
    p.xmap = xm;
    RET(linear(l, p));
    if (taps) RET(taps->put(l, TAP_CONV, i, 0, dst));
    xa = dst; xb = (xa == c->s_xa) ? c->s_xb : c->s_xa;
    for (int j = 0; j < (int)k.stages[i].size(); ++j) {
      RET(enqueue_block(l, k.stages[i][j], xa, xb, B, k.T[i], d.codec_eps));
      std::swap(xa, xb);
      if (taps) RET(taps->put(l, TAP_BLOCK, i, j, xa));
    }
  }
  const ConvL& hd = k.convs[ns];
  const int T = k.T[ns - 1];
  RET(assemble(l, xa, hd.hist, c->s_win, hd.next, B, T, 6, hd.Cin, nullptr, 0.f, 1.f, 0.f));
  RET(conv_apply(l, hd, c->s_win, audio, B, T, T));
  if (taps) RET(taps->put(l, TAP_OUT, ns, 0, audio));
  CK(launch_k(l, advance_kernel, dim3(k.n_segs, B, ADV_SLICES), dim3(256), 0, k.segs_dev, active));
  return 0;
}

// stages [0, n_stream_first) of the semantic encoder through the kernel-per-stage path; returns where their rows are (the stream program of
// the remaining stages was built against that pointer)
static float* encode_front_out(vv_ctx* c, int first) {
  // the ping-pong below is deterministic: stem -> s_xa, every conv and every block swaps
  const Codec& k = c->enc;
  bool in_a = true;
  for (int i = 0; i < first; ++i) {
    if (i > 0) in_a = !in_a;
    if (k.stages[i].size() & 1) in_a = !in_a;
  }
  return in_a ? c->s_xa : c->s_xb;
}
static int enqueue_encode(const L& l, const float* audio, const int32_t* active, const vv_ctx::StreamProg& back, TapSink* taps = nullptr) {
  vv_ctx* c = l.c;
  const auto& d = c->d;
  Codec& k = c->enc;
  const int B = d.max_batch;
  const int stop = enc_back_first(c);
  float *xa = c->s_xa, *xb = c->s_xb;
  int hop = k.T[0];
  RET(assemble(l, audio, k.convs[0].hist, c->s_win, k.convs[0].next, B, hop, 6, 1, nullptr, 0.f, 1.f, 0.f));
  RET(conv_apply(l, k.convs[0], c->s_win, xa, B, hop, hop));
  for (int i = 0; i < stop; ++i) {
    if (i > 0) {
      const ConvL& cv = k.convs[i];
      const int Tin = k.T[i - 1];
      RET(assemble(l, xa, cv.hist, c->s_win, cv.next, B, Tin, cv.ctx, cv.Cin, nullptr, 0.f, 1.f, 0.f));
      RET(conv_apply(l, cv, c->s_win, xb, B, k.T[i], Tin));
      std::swap(xa, xb);
    }
    if (taps) RET(taps->put(l, TAP_CONV, i, 0, xa));
    for (int j = 0; j < (int)k.stages[i].size(); ++j) {
      RET(enqueue_block(l, k.stages[i][j], xa, xb, B, k.T[i], d.codec_eps));
      std::swap(xa, xb);
      if (taps) RET(taps->put(l, TAP_BLOCK, i, j, xa));
    }
  }
  if (xa != encode_front_out(c, stop)) return fail(VV_ERR_STATE, "encoder hand-off buffer mismatch");
  if (taps) RET(taps->put(l, TAP_HANDOFF, stop, 0, xa));
  RET(launch_stream(l, back));                  // stages [stop, ns) + head conv through the weight-stream kernel
  if (taps) RET(taps->put(l, TAP_OUT, d.n_stages, 0, taps->out));
  CK(launch_k(l, advance_kernel, dim3(k.n_segs, B, ADV_SLICES), dim3(256), 0, k.segs_dev, active));
  return 0;
}

static int enqueue_connect(const L& l, const float* latent, const float* sem, const int32_t* active, float* embeds) {
  vv_ctx* c = l.c;
  const auto& d = c->d;
  const int H = d.hidden_size, B = d.max_batch;
  GemvP p = mk(c->ca_fc1, c->ca_b1, latent, 64, c->s_c1, H, B, H, 64);
  RET(linear(l, p));
  p = mk(c->ca_fc2, c->ca_b2, c->s_c1, H, c->s_e, H, B, H, H);
  p.pro = PRO_RMSNORM; p.pro_w = c->ca_n; p.pro_eps = 1e-6f;
  RET(linear(l, p));
  p = mk(c->cs_fc1, c->cs_b1, sem, d.semantic_vae_dim, c->s_c1, H, B, H, d.semantic_vae_dim);
  RET(linear(l, p));
  p = mk(c->cs_fc2, c->cs_b2, c->s_c1, H, c->s_e, H, B, H, H);
  p.pro = PRO_RMSNORM; p.pro_w = c->cs_n; p.pro_eps = 1e-6f; p.epi = EPI_RESID; p.res = c->s_e; p.ldres = H;
  RET(linear(l, p));
  CK(launch_k(l, select_embeds_kernel, dim3(B), dim3(256), 0, embeds, c->s_e, active, B, H));
  return 0;
}

extern "C" int vv_codec_decode_frame(vv_ctx* c, const float* latent, const int32_t* active, float* audio_out, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  CK(cudaSetDevice(c->device));
  char key[256];
  snprintf(key, sizeof key, "dec:%p:%p:%p", (const void*)latent, (const void*)active, (void*)audio_out);
  const vv_ctx::StreamProg* front; int nf; float* fx;
  RET(dec_front_prog(c, latent, &front, &nf, &fx));
  return run_cached(c, key, (cudaStream_t)stream, [&](const L& l) { return enqueue_decode(l, active, audio_out, *front, nf, fx); });
}
extern "C" int vv_semantic_encode_frame(vv_ctx* c, const float* audio, const int32_t* active, float* feat_out, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  CK(cudaSetDevice(c->device));
  char key[256];
  snprintf(key, sizeof key, "enc:%p:%p:%p", (const void*)audio, (const void*)active, (void*)feat_out);
  const vv_ctx::StreamProg* back;
  RET(enc_back_prog(c, encode_front_out(c, enc_back_first(c)), feat_out, &back));
  return run_cached(c, key, (cudaStream_t)stream, [&](const L& l) { return enqueue_encode(l, audio, active, *back); });
}
extern "C" int vv_debug_codec_taps(vv_ctx* c, int which, const float* in, const int32_t* active, float* out, float* taps, int64_t taps_floats,
                                   int32_t* meta, void* stream) {
  if (!c) return fail(VV_ERR_INVALID, "null ctx");
  if (!c->finalized) return fail(VV_ERR_STATE, "vv_debug_codec_taps: not finalized");
  if (which != 0 && which != 1) return fail(VV_ERR_INVALID, "vv_debug_codec_taps: which = %d (0 decoder, 1 semantic encoder)", which);
  TapSink sink;
  codec_tap_plan(c, which, &sink.plan);
  const int n = (int)sink.plan.size();
  long long need = 0;
  for (int i = 0; i < n; ++i) {
    const TapMeta& t = sink.plan[i];
    need += (long long)c->d.max_batch * t.T * t.C;
    if (meta) { int32_t* m = meta + 5 * i; m[0] = t.kind; m[1] = t.stage; m[2] = t.index; m[3] = t.T; m[4] = t.C; }
  }
  if (!taps) return n;
  if (taps_floats < need) return fail(VV_ERR_INVALID, "vv_debug_codec_taps: %lld floats of tap space, the pass needs %lld", (long long)taps_floats, need);
  if (!in || !active || !out) return fail(VV_ERR_INVALID, "vv_debug_codec_taps: null input, active set or output");
  CK(cudaSetDevice(c->device));
  sink.dst = taps; sink.out = out; sink.B = c->d.max_batch;
  L l{c, (cudaStream_t)stream};
  if (which == 0) {
    const vv_ctx::StreamProg* front; int nf; float* fx;
    RET(dec_front_prog(c, in, &front, &nf, &fx));
    RET(enqueue_decode(l, active, out, *front, nf, fx, &sink));
  } else {
    const vv_ctx::StreamProg* back;
    RET(enc_back_prog(c, encode_front_out(c, enc_back_first(c)), out, &back));
    RET(enqueue_encode(l, in, active, *back, &sink));
  }
  CK(cudaStreamSynchronize(l.s));
  if (sink.next != sink.plan.size()) return fail(VV_ERR_STATE, "vv_debug_codec_taps: the pass made %zu of %d taps", sink.next, n);
  return n;
}
extern "C" int vv_connect(vv_ctx* c, const float* latent, const float* sem, const int32_t* active, float* embeds, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  CK(cudaSetDevice(c->device));
  L l{c, (cudaStream_t)stream};
  return enqueue_connect(l, latent, sem, active, embeds);
}
extern "C" int vv_frame_tail(vv_ctx* c, const float* hidden, const float* noise, const int32_t* active, float cfg, float* latent_out,
                             float* audio_out, float* embeds, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  CK(cudaSetDevice(c->device));
  char key[320];
  RET(set_cfg(c, cfg, (cudaStream_t)stream));
  snprintf(key, sizeof key, "tail:%p:%p:%p:%p:%p:%p", (const void*)hidden, (const void*)noise, (const void*)active, (void*)latent_out,
           (void*)audio_out, (void*)embeds);
  const vv_ctx::StreamProg *sprog, *front, *back; int nf; float* fx;
  RET(sampler_stream_prog(c, noise, latent_out, &sprog));
  RET(dec_front_prog(c, latent_out, &front, &nf, &fx));
  RET(enc_back_prog(c, encode_front_out(c, enc_back_first(c)), c->s_feat, &back));
  return run_cached(c, key, (cudaStream_t)stream, [&](const L& l) {
    RET(enqueue_diffusion(l, hidden, *sprog));
    RET(enqueue_decode(l, active, audio_out, *front, nf, fx));
    RET(enqueue_encode(l, audio_out, active, *back));
    return enqueue_connect(l, latent_out, c->s_feat, active, embeds);
  });
}

// ------------------------------------------------------------------------------------------------
// a-9 voice prompts: non-streaming acoustic encoder + sampling + acoustic connector (vv_voice_encode)
// ------------------------------------------------------------------------------------------------
// Workspace = per-voice activations of one group of voices (two [T_i][C_i] buffers, per-row RMS factors, latent means) + a scratch region
// S for the GEMM operands of one row chunk.  The minimum holds one voice and 64-row chunks; more workspace means larger groups first,
// then longer chunks.  Every output row is computed the same way whatever the grouping, so results do not depend on the workspace size.
struct VoicePlan {
  std::vector<long long> T;        // rows per voice after conv i (T[0] = samples, T.back() = frames)
  long long maxTC = 0, F = 0;
  long long max_bpr = 0;           // largest scratch bytes per row of any GEMM
};
static long long align256(long long b) { return (b + 255) & ~255ll; }
static constexpr long long VOICE_CHUNK_MAX = 65535ll * 64;   // rows of one GEMM launch (grid.y = rows / 64)
static void voice_plan(const vv_ctx* c, long long T, VoicePlan* pl) {
  const VoiceEnc& v = c->venc;
  const int ns = (int)v.stages.size(), H = c->d.hidden_size;
  pl->T.assign(ns, 0);
  long long t = T;
  pl->max_bpr = 8ll * H;                                               // connector: fc1 output + operand planes
  for (int i = 0; i < ns; ++i) {
    if (i) t = (t + v.convs[i].stride - 1) / v.convs[i].stride;        // ceil: stride-alignment padding on the right
    pl->T[i] = t;
    pl->maxTC = std::max(pl->maxTC, t * v.C[i]);
    pl->max_bpr = std::max(pl->max_bpr, 32ll * v.C[i]);                // FFN: 4C hidden fp32 + 4C operand planes
    pl->max_bpr = std::max(pl->max_bpr, 4ll * v.convs[i].K);          // conv: window operand planes
  }
  pl->max_bpr = std::max(pl->max_bpr, 4ll * v.convs[ns].K);
  pl->F = t;
}
static long long voice_act_bytes(const vv_ctx* c, const VoicePlan& pl, long long g) {
  return 2 * align256(g * pl.maxTC * 4) + align256(g * pl.T[0] * 4) + align256(g * pl.F * c->d.acoustic_vae_dim * 4);
}
static long long voice_scratch_min(const VoicePlan& pl) { return 64 * pl.max_bpr + 512; }
static long long voice_chunk(long long S, long long bpr, long long M) {
  long long R = std::min(((S - 512) / bpr) & ~63ll, VOICE_CHUNK_MAX);
  return std::min(std::max(R, 64ll), M);
}
static int voice_check(vv_ctx* c, int n, int64_t T) {
  if (!c) return fail(VV_ERR_INVALID, "null ctx");
  if (!c->finalized) return fail(VV_ERR_STATE, "not finalized");
  if (!c->venc.present) return fail(VV_ERR_STATE, "voice encode: the checkpoint has no acoustic tokenizer encoder weights");
  if (n < 1 || T < 1 || T > (1ll << 30)) return fail(VV_ERR_INVALID, "voice encode: n = %d voices of T = %lld samples out of range", n, (long long)T);
  return 0;
}

extern "C" int64_t vv_voice_encode_workspace(vv_ctx* c, int n, int64_t T) {
  RET(voice_check(c, n, T));
  VoicePlan pl;
  voice_plan(c, T, &pl);
  return voice_act_bytes(c, pl, 1) + voice_scratch_min(pl);
}

static int voice_gemm(const L& l, const bf16* W, const float* bias, int N, int K, const bf16* hi, const bf16* lo, long long M, float* y, int ldy,
                      int epi = EPI_NONE, const float* gamma = nullptr) {
  GemvP p = mk(W, bias, nullptr, K, y, ldy, (int)M, N, K);
  p.epi = epi;
  if (epi == EPI_GAMMA_RESID) { p.epi_a = gamma; p.res = y; p.ldres = ldy; }     // in place: the operand is in the planes
  CK(launch_k(l, gemm_wgmma_kernel, dim3((N + WG_BM - 1) / WG_BM, (unsigned)((M + WG_BN - 1) / WG_BN)), dim3(128), (size_t)WG_SMEM, p, hi, lo));
  return 0;
}
static unsigned ew_grid(const vv_ctx* c, long long n) { return (unsigned)std::max(1ll, std::min((n + 255) / 256, (long long)c->sm_count * 16)); }

// y [nv][T_out][Cout] = causal conv of x [nv][T_in][Cin] (left pad k - s, right stride alignment, both as zeros)
static int voice_conv(const L& l, const ConvL& cv, const float* x, long long T_in, long long T_out, int nv, float* y, unsigned char* S, long long Sb) {
  const long long M = nv * T_out, R = voice_chunk(Sb, 4ll * cv.K, M);
  for (long long m0 = 0; m0 < M; m0 += R) {
    const long long r = std::min(R, M - m0);
    bf16* hi = (bf16*)S;
    bf16* lo = hi + r * cv.K;
    CK(launch_k(l, voice_window_split_kernel, dim3(ew_grid(l.c, r * cv.K / 4)), dim3(256), 0, x, (int)T_in, (int)T_out, cv.Cin, cv.stride,
                cv.ctx, cv.k * cv.Cin, cv.K, m0, (int)r, hi, lo));
    RET(voice_gemm(l, cv.w, cv.bias, cv.Cout, cv.K, hi, lo, r, y + m0 * cv.Cout, cv.Cout));
  }
  return 0;
}

// ---- stage taps of vv_voice_encode (vv_debug_voice_taps): every stage boundary, [n][T_k][C_k] per tap, back to back.  A group of voices
// writes its rows at voice offset v0 of every tap, so the layout does not depend on the grouping.  Production runs with no sink.
enum { VT_CONV = 0, VT_MIX = 1, VT_BLOCK = 2, VT_FC1 = 3, VT_EMBEDS = 4 };
// kind, stage, index: VT_CONV (i, 0) = output of stage i's convolution (i = n_stages: the head conv, the latent mean); VT_MIX (i, j) =
// x + gamma * dwconv7(RMSNorm(x)) of block j of stage i; VT_BLOCK (i, j) = output of that block; VT_FC1 / VT_EMBEDS (n_stages, 0) = the
// connector's fc1 output before its RMSNorm / the embeddings
static void voice_tap_plan(const vv_ctx* c, const VoicePlan& pl, std::vector<TapMeta>* plan) {
  const VoiceEnc& v = c->venc;
  const int ns = (int)v.stages.size();
  plan->clear();
  for (int i = 0; i < ns; ++i) {
    plan->push_back({VT_CONV, i, 0, (int)pl.T[i], v.C[i]});
    for (int j = 0; j < (int)v.stages[i].size(); ++j) {
      plan->push_back({VT_MIX, i, j, (int)pl.T[i], v.C[i]});
      plan->push_back({VT_BLOCK, i, j, (int)pl.T[i], v.C[i]});
    }
  }
  plan->push_back({VT_CONV, ns, 0, (int)pl.F, c->d.acoustic_vae_dim});
  plan->push_back({VT_FC1, ns, 0, (int)pl.F, c->d.hidden_size});
  plan->push_back({VT_EMBEDS, ns, 0, (int)pl.F, c->d.hidden_size});
}
struct VoiceTapSink {
  std::vector<TapMeta> plan;
  std::vector<long long> off;   // float offset of tap k: n * sum_{j<k} T_j * C_j
  float* dst = nullptr;         // device
  long long v0 = 0;             // first voice of the group being run
  size_t next = 0;              // the group's next tap
  // rows [r0, r0 + r) of the group's tap `next` (rows counted from the group's first voice); done: the tap is complete
  int put(const L& l, int kind, int stage, int index, const float* src, long long r0, long long r, bool done = true) {
    if (next >= plan.size() || plan[next].kind != kind || plan[next].stage != stage || plan[next].index != index)
      return fail(VV_ERR_STATE, "voice taps: tap %zu (kind %d, stage %d, index %d) is not the planned one", next, kind, stage, index);
    const TapMeta& t = plan[next];
    CK(cudaMemcpyAsync(dst + off[next] + (v0 * t.T + r0) * t.C, src, (size_t)(r * t.C) * sizeof(float), cudaMemcpyDeviceToDevice, l.s));
    if (done) ++next;
    return 0;
  }
};

// Block1D over x [nv][T][C] (result back in *x; *y is the other activation buffer); block j of stage i
static int voice_block(const L& l, const Block& b, float** x, float** y, float* inv, int nv, long long T, unsigned char* S, long long Sb,
                       VoiceTapSink* taps, int i, int j) {
  const int C = b.C;
  const float eps = l.c->d.codec_eps;
  const long long M = nv * T;
  CK(launch_k(l, voice_rms_kernel, dim3((unsigned)((M + 7) / 8)), dim3(256), 0, (const float*)*x, M, C, eps, inv));
  CK(launch_k(l, voice_dwconv_kernel, dim3(ew_grid(l.c, M * C)), dim3(256), 0, (const float*)*x, (const float*)inv, (const float*)b.norm_w,
              (const float*)b.dw_w, (const float*)b.dw_b, (const float*)b.gamma, *y, M, (int)T, C));
  std::swap(*x, *y);
  if (taps) RET(taps->put(l, VT_MIX, i, j, *x, 0, M));
  // FFN in row chunks (no halo): norm -> planes -> C x 4C GEMM + GELU -> planes -> 4C x C GEMM, gamma residual in place
  const long long R = voice_chunk(Sb, 32ll * C, M);
  float* hid = (float*)S;
  bf16* planes = (bf16*)(S + align256(R * 16 * C));
  for (long long m0 = 0; m0 < M; m0 += R) {
    const long long r = std::min(R, M - m0);
    float* xr = *x + m0 * C;
    CK(launch_k(l, voice_norm_split_kernel, dim3((unsigned)((r + 7) / 8)), dim3(256), 0, (const float*)xr, (const float*)b.ffn_norm_w, eps,
                (int)r, C, planes, planes + r * C));
    RET(voice_gemm(l, b.w1, b.b1, 4 * C, C, planes, planes + r * C, r, hid, 4 * C, EPI_GELU));
    CK(launch_k(l, split_bf16_kernel, dim3(ew_grid(l.c, r * C)), dim3(256), 0, (const float*)hid, dense_rows(4 * C), planes, planes + r * 4 * C,
                (int)r, 4 * C));
    RET(voice_gemm(l, b.w2, b.b2, C, 4 * C, planes, planes + r * 4 * C, r, xr, C, EPI_GAMMA_RESID, b.ffn_gamma));
  }
  if (taps) RET(taps->put(l, VT_BLOCK, i, j, *x, 0, M));
  return 0;
}

// what vv_voice_encode runs, with every stage boundary copied into `taps` when it is given
static int voice_run(vv_ctx* c, const char* who, const float* wavs, int n, int64_t T, const float* sigma, const float* eps, float* mean_out,
                     float* embeds_out, void* workspace, int64_t workspace_bytes, void* stream, VoiceTapSink* taps) {
  if (!wavs || !embeds_out || !workspace || (eps && !sigma)) return fail(VV_ERR_INVALID, "%s: null argument", who);
  if (((uintptr_t)workspace & 255) || ((uintptr_t)eps & 15)) return fail(VV_ERR_INVALID, "%s: workspace must be 256-byte and eps 16-byte aligned", who);
  VoicePlan pl;
  voice_plan(c, T, &pl);
  const long long smin = voice_scratch_min(pl), need = voice_act_bytes(c, pl, 1) + smin;
  if (workspace_bytes < need)
    return fail(VV_ERR_INVALID, "%s: workspace of %lld bytes is below the minimum %lld", who, (long long)workspace_bytes, need);
  long long g = n;
  while (g > 1 && voice_act_bytes(c, pl, g) + smin > workspace_bytes) --g;
  CK(cudaSetDevice(c->device));
  CK(cudaFuncSetAttribute(gemm_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM));
  const VoiceEnc& v = c->venc;
  const int ns = (int)v.stages.size(), D = c->d.acoustic_vae_dim, H = c->d.hidden_size;
  const long long F = pl.F;
  unsigned char* ws = (unsigned char*)workspace;
  float* bufA = (float*)ws;
  float* bufB = (float*)(ws + align256(g * pl.maxTC * 4));
  float* inv = (float*)(ws + 2 * align256(g * pl.maxTC * 4));
  float* mean = (float*)(ws + 2 * align256(g * pl.maxTC * 4) + align256(g * pl.T[0] * 4));
  unsigned char* S = ws + voice_act_bytes(c, pl, g);
  const long long Sb = workspace_bytes - voice_act_bytes(c, pl, g);
  L l{c, (cudaStream_t)stream};
  for (long long v0 = 0; v0 < n; v0 += g) {
    const int nv = (int)std::min<long long>(g, n - v0);
    if (taps) { taps->v0 = v0; taps->next = 0; }
    float *x = bufA, *y = bufB;
    for (int i = 0; i < ns; ++i) {
      if (i == 0) RET(voice_conv(l, v.convs[0], wavs + v0 * T, T, T, nv, x, S, Sb));
      else { RET(voice_conv(l, v.convs[i], x, pl.T[i - 1], pl.T[i], nv, y, S, Sb)); std::swap(x, y); }
      if (taps) RET(taps->put(l, VT_CONV, i, 0, x, 0, nv * pl.T[i]));
      for (int j = 0; j < (int)v.stages[i].size(); ++j) RET(voice_block(l, v.stages[i][j], &x, &y, inv, nv, pl.T[i], S, Sb, taps, i, j));
    }
    RET(voice_conv(l, v.convs[ns], x, F, F, nv, mean, S, Sb));
    if (taps) RET(taps->put(l, VT_CONV, ns, 0, mean, 0, nv * F));
    if (mean_out) CK(cudaMemcpyAsync(mean_out + v0 * F * D, mean, (size_t)nv * F * D * 4, cudaMemcpyDeviceToDevice, l.s));
    // x = mean + sigma * eps; feat = (x + bias) * scale; acoustic_connector = fc2(RMSNorm_1e-6(fc1(feat)))
    const long long M = nv * F, R = voice_chunk(Sb, 8ll * H, M);
    float* y1 = (float*)S;
    bf16* planes = (bf16*)(S + align256(R * 4 * H));
    for (long long m0 = 0; m0 < M; m0 += R) {
      const long long r = std::min(R, M - m0);
      CK(launch_k(l, voice_sample_split_kernel, dim3(ew_grid(c, r * D / 4)), dim3(256), 0, (const float*)mean, eps ? eps + v0 * F * D : nullptr,
                  sigma ? sigma + v0 : nullptr, (int)F, D, c->speech_bias, c->speech_scale, m0, (int)r, planes, planes + r * D));
      RET(voice_gemm(l, c->ca_fc1, c->ca_b1, H, D, planes, planes + r * D, r, y1, H));
      if (taps) RET(taps->put(l, VT_FC1, ns, 0, y1, m0, r, m0 + r == M));
      CK(launch_k(l, voice_norm_split_kernel, dim3((unsigned)((r + 7) / 8)), dim3(256), 0, (const float*)y1, (const float*)c->ca_n, 1e-6f, (int)r, H,
                  planes, planes + r * H));
      RET(voice_gemm(l, c->ca_fc2, c->ca_b2, H, H, planes, planes + r * H, r, embeds_out + (v0 * F + m0) * H, H));
    }
    if (taps) {
      RET(taps->put(l, VT_EMBEDS, ns, 0, embeds_out + v0 * F * H, 0, M));
      if (taps->next != taps->plan.size()) return fail(VV_ERR_STATE, "%s: a group made %zu of %zu taps", who, taps->next, taps->plan.size());
    }
  }
  return 0;
}

extern "C" int vv_voice_encode(vv_ctx* c, const float* wavs, int n, int64_t T, const float* sigma, const float* eps, float* mean_out,
                               float* embeds_out, void* workspace, int64_t workspace_bytes, void* stream) {
  RET(voice_check(c, n, T));
  return voice_run(c, "vv_voice_encode", wavs, n, T, sigma, eps, mean_out, embeds_out, workspace, workspace_bytes, stream, nullptr);
}

extern "C" int vv_debug_voice_taps(vv_ctx* c, const float* wavs, int n, int64_t T, const float* sigma, const float* eps, float* embeds_out,
                                   void* workspace, int64_t workspace_bytes, float* taps, int64_t taps_floats, int32_t* meta, void* stream) {
  RET(voice_check(c, n, T));
  VoicePlan pl;
  voice_plan(c, T, &pl);
  VoiceTapSink sink;
  voice_tap_plan(c, pl, &sink.plan);
  const int nt = (int)sink.plan.size();
  long long need = 0;
  for (int k = 0; k < nt; ++k) {
    const TapMeta& t = sink.plan[k];
    sink.off.push_back(need);
    need += (long long)n * t.T * t.C;
    if (meta) { int32_t* m = meta + 5 * k; m[0] = t.kind; m[1] = t.stage; m[2] = t.index; m[3] = t.T; m[4] = t.C; }
  }
  if (!taps) return nt;
  if (taps_floats < need)
    return fail(VV_ERR_INVALID, "vv_debug_voice_taps: %lld floats of tap space, the encoder needs %lld", (long long)taps_floats, need);
  sink.dst = taps;
  RET(voice_run(c, "vv_debug_voice_taps", wavs, n, T, sigma, eps, nullptr, embeds_out, workspace, workspace_bytes, stream, &sink));
  CK(cudaStreamSynchronize((cudaStream_t)stream));
  return nt;
}

// ------------------------------------------------------------------------------------------------
// f-2: native prompt prefill (vv_prefill.cuh).  Workspace = one chunk of R rows (R a multiple of 64): fp32 residual [R][H], operand
// buffer a1 [R][max(H, nq)] (norm output, attention output) and a2 [R][max(I, nq)] (Q, SwiGLU output), all bf16.  The minimum is one
// 64-row chunk; a larger workspace takes longer chunks, with the same result.
// ------------------------------------------------------------------------------------------------
static long long pf_bytes(const vv_ctx* c, long long R) {
  const auto& d = c->d;
  const long long nq = (long long)d.num_q_heads * d.head_dim;
  return align256(R * 4 * d.hidden_size) + align256(R * 2 * std::max<long long>(d.hidden_size, nq)) +
         align256(R * 2 * std::max<long long>(d.intermediate_size, nq));
}
static int pf_check(vv_ctx* c, int64_t n) {
  if (!c) return fail(VV_ERR_INVALID, "null ctx");
  if (!c->finalized) return fail(VV_ERR_STATE, "lm prefill: not finalized");
  if (n < 1) return fail(VV_ERR_INVALID, "lm prefill: n_tokens = %lld must be at least 1", (long long)n);
  const auto& d = c->d;
  if (d.head_dim != 64 && d.head_dim != 128) return fail(VV_ERR_INVALID, "lm prefill: head_dim %d (supported: 64, 128)", d.head_dim);
  if (d.hidden_size % 64 || d.intermediate_size % 64 || (d.num_q_heads * d.head_dim) % 64)
    return fail(VV_ERR_INVALID, "lm prefill: hidden / intermediate / q widths must be multiples of 64");
  return 0;
}
extern "C" int64_t vv_lm_prefill_workspace(vv_ctx* c, int64_t n_tokens) {
  RET(pf_check(c, n_tokens));
  return pf_bytes(c, 64);
}

// the checks and page reservation vv_lm_prefill and vv_debug_prefill_taps share; *R = rows per chunk
static int pf_begin(vv_ctx* c, const char* who, int seq, int64_t pos0, int64_t n, void* workspace, int64_t workspace_bytes, void* stream,
                    long long* R) {
  if ((uintptr_t)workspace & 255) return fail(VV_ERR_INVALID, "%s: workspace must be 256-byte aligned", who);
  const long long need = pf_bytes(c, 64);
  if (workspace_bytes < need)
    return fail(VV_ERR_INVALID, "%s: workspace of %lld bytes is below the minimum %lld", who, (long long)workspace_bytes, need);
  if (!c->kpool) return fail(VV_ERR_STATE, "%s: KV pool not initialised (vv_kv_init)", who);
  const auto& d = c->d;
  if (seq < 0 || seq >= 2 * d.max_batch) return fail(VV_ERR_INVALID, "%s: bad seq %d", who, seq);
  if (pos0 < 0 || pos0 + n > d.max_position_embeddings)
    return fail(VV_ERR_INVALID, "%s: positions [%lld, %lld) outside [0, %d)", who, (long long)pos0, (long long)(pos0 + n), d.max_position_embeddings);
  {
    const int64_t needp = (pos0 + n + KV_PAGE - 1) / KV_PAGE, have = (int64_t)c->seq_pages[seq].size();
    if (needp > c->max_pages || needp - have > (int64_t)c->free_pages.size())
      return fail(VV_ERR_NOMEM, "%s: KV page pool too small (seq %d needs %lld pages, holds %lld, %lld free)", who, seq, (long long)needp,
                  (long long)have, (long long)c->free_pages.size());
  }
  CK(cudaSetDevice(c->device));
  RET(vv_kv_reserve(c, seq, pos0 + n, stream));
  // rows per chunk: the largest multiple of 64 the workspace holds, at most the prompt (rounded up) and 65535 GEMM row tiles
  *R = std::min<long long>((n + 63) & ~63ll, 65535ll * PF_BM);
  while (*R > 64 && pf_bytes(c, *R) > workspace_bytes) *R -= 64;
  return 0;
}

// ---- per-kernel taps of one prefill layer (vv_debug_prefill_taps): what each kernel of the layer left, [n][cols] per tap, back to back.
// Production chunks run with no sink.
enum { PT_NORM1 = 0, PT_Q, PT_ATTN, PT_RESID1, PT_NORM2, PT_SWIGLU, PT_OUT, PT_COUNT };
struct PrefillTaps {
  unsigned char* dst = nullptr;  // device
  long long off[PT_COUNT];       // byte offset of tap k
  int cols[PT_COUNT], esz[PT_COUNT];
  long long c0 = 0;              // first row of the chunk being run
  PrefillTaps(const vv_ctx* c, long long n) {
    const auto& d = c->d;
    const int nq = d.num_q_heads * d.head_dim;
    const int cc[PT_COUNT] = {d.hidden_size, nq, nq, d.hidden_size, d.hidden_size, d.intermediate_size, d.hidden_size};
    const int ee[PT_COUNT] = {2, 2, 2, 4, 2, 2, 4};
    long long o = 0;
    for (int k = 0; k < PT_COUNT; ++k) { cols[k] = cc[k]; esz[k] = ee[k]; off[k] = o; o += n * cc[k] * ee[k]; }
  }
  long long bytes(long long n) const { return off[PT_COUNT - 1] + n * cols[PT_COUNT - 1] * esz[PT_COUNT - 1]; }
  int put(const L& l, int k, const void* src, int r) {
    CK(cudaMemcpyAsync(dst + off[k] + c0 * cols[k] * esz[k], src, (size_t)r * cols[k] * esz[k], cudaMemcpyDeviceToDevice, l.s));
    return 0;
  }
};

// decoder layer li over the r rows of one chunk at positions pos_base ..: residual x fp32 [r][H] updated in place, K/V into the pool;
// a1 / a2 the chunk's operand buffers (see pf_bytes)
static int prefill_layer(const L& l, int li, const int* page_row, long long pos_base, int r, float* x, bf16* a1, bf16* a2, PrefillTaps* taps) {
  vv_ctx* c = l.c;
  const auto& d = c->d;
  const int H = d.hidden_size, I = d.intermediate_size, nh = d.num_q_heads, nkv = d.num_kv_heads, hd = d.head_dim, nq = nh * hd;
  const int Nqkv = nq + 2 * nkv * hd;
  const size_t per_layer = (size_t)c->n_pages * nkv * KV_PAGE * hd;
  const float scale_log2 = 1.4426950408889634f / sqrtf((float)hd);
  auto gemm = [&](auto kern, const bf16* A, const bf16* W, int M, int N, int K, PfGemm p) -> int {
    p.A = A; p.W = W; p.M = M; p.N = N; p.K = K;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, PF_SMEM));
    CK(launch_k(l, kern, dim3((N + PF_BN - 1) / PF_BN, (M + PF_BM - 1) / PF_BM), dim3(256), (size_t)PF_SMEM, p));
    return 0;
  };
  const LmLayer& y = c->lm[li];
  PfGemm p;
  memset(&p, 0, sizeof p);
  CK(launch_k(l, pf_rmsnorm_kernel, dim3((r + 7) / 8), dim3(256), 0, (const float*)x, (const float*)y.ln1, d.rms_norm_eps, r, H, a1));
  if (taps) RET(taps->put(l, PT_NORM1, a1, r));
  p.bias = y.bqkv; p.out = a2; p.ldo = nq; p.kpool = c->kpool + per_layer * li; p.vpool = c->vpool + per_layer * li; p.page_row = page_row;
  p.nq = nq; p.kv_heads = nkv; p.pos_base = pos_base; p.inv_freq = c->inv_freq;
  if (hd == 128) RET(gemm(pf_gemm_kernel<PF_EPI_QKV, 128>, a1, y.wqkv, r, Nqkv, H, p));
  else RET(gemm(pf_gemm_kernel<PF_EPI_QKV, 64>, a1, y.wqkv, r, Nqkv, H, p));
  if (taps) RET(taps->put(l, PT_Q, a2, r));
  const dim3 ag((r + 63) / 64, nh);
  if (hd == 128) {
    CK(cudaFuncSetAttribute(pf_attn_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, PfAttnCfg<128>::SMEM));
    CK(launch_k(l, pf_attn_kernel<128>, ag, dim3(128), (size_t)PfAttnCfg<128>::SMEM, (const bf16*)a2, r, nh, nkv, (const bf16*)p.kpool,
                (const bf16*)p.vpool, page_row, pos_base, scale_log2, a1));
  } else {
    CK(cudaFuncSetAttribute(pf_attn_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, PfAttnCfg<64>::SMEM));
    CK(launch_k(l, pf_attn_kernel<64>, ag, dim3(128), (size_t)PfAttnCfg<64>::SMEM, (const bf16*)a2, r, nh, nkv, (const bf16*)p.kpool,
                (const bf16*)p.vpool, page_row, pos_base, scale_log2, a1));
  }
  if (taps) RET(taps->put(l, PT_ATTN, a1, r));
  memset(&p, 0, sizeof p);
  p.x = x; p.ldx = H;
  RET(gemm(pf_gemm_kernel<PF_EPI_RESID>, a1, y.wo, r, H, nq, p));
  if (taps) RET(taps->put(l, PT_RESID1, x, r));
  CK(launch_k(l, pf_rmsnorm_kernel, dim3((r + 7) / 8), dim3(256), 0, (const float*)x, (const float*)y.ln2, d.rms_norm_eps, r, H, a1));
  if (taps) RET(taps->put(l, PT_NORM2, a1, r));
  memset(&p, 0, sizeof p);
  p.out = a2; p.ldo = I;
  RET(gemm(pf_gemm_kernel<PF_EPI_SWIGLU>, a1, y.wgu, r, 2 * I, H, p));
  if (taps) RET(taps->put(l, PT_SWIGLU, a2, r));
  memset(&p, 0, sizeof p);
  p.x = x; p.ldx = H;
  RET(gemm(pf_gemm_kernel<PF_EPI_RESID>, a2, y.wdown, r, H, I, p));
  if (taps) RET(taps->put(l, PT_OUT, x, r));
  return 0;
}

extern "C" int vv_lm_prefill(vv_ctx* c, int seq, int64_t pos0, int64_t n, const float* embeds, float* hidden_last, void* workspace,
                             int64_t workspace_bytes, void* stream) {
  RET(pf_check(c, n));
  if (!embeds || !hidden_last || !workspace) return fail(VV_ERR_INVALID, "vv_lm_prefill: null argument");
  if (((uintptr_t)embeds & 15) || ((uintptr_t)hidden_last & 15)) return fail(VV_ERR_INVALID, "vv_lm_prefill: embeds / hidden_last must be 16-byte aligned");
  long long R;
  RET(pf_begin(c, "vv_lm_prefill", seq, pos0, n, workspace, workspace_bytes, stream, &R));
  const auto& d = c->d;
  const int H = d.hidden_size, nq = d.num_q_heads * d.head_dim;
  unsigned char* ws = (unsigned char*)workspace;
  float* x = (float*)ws;
  bf16* a1 = (bf16*)(ws + align256(R * 4 * H));
  bf16* a2 = (bf16*)(ws + align256(R * 4 * H) + align256(R * 2 * std::max(H, nq)));
  const int* page_row = c->page_table_dev + (size_t)seq * c->max_pages;
  L l{c, (cudaStream_t)stream};
  for (long long c0 = 0; c0 < n; c0 += R) {
    const int r = (int)std::min<long long>(R, n - c0);
    CK(cudaMemcpyAsync(x, embeds + c0 * H, (size_t)r * H * 4, cudaMemcpyDeviceToDevice, l.s));
    for (int li = 0; li < d.num_layers; ++li) RET(prefill_layer(l, li, page_row, pos0 + c0, r, x, a1, a2, nullptr));
    if (c0 + r == n) CK(launch_k(l, rows_norm_block_kernel, dim3(1), dim3(256), 0, (const float*)(x + (size_t)(r - 1) * H), (const float*)c->lm_norm, hidden_last, H, d.rms_norm_eps));
  }
  return 0;
}

extern "C" int vv_debug_prefill_taps(vv_ctx* c, int seq, int64_t pos0, int64_t n, int layer, const float* x_in, float* hidden_last,
                                     void* workspace, int64_t workspace_bytes, void* taps, int64_t taps_bytes, int32_t* meta, void* stream) {
  RET(pf_check(c, n));
  const auto& d = c->d;
  if (layer < 0 || layer >= d.num_layers) return fail(VV_ERR_INVALID, "vv_debug_prefill_taps: bad layer %d", layer);
  PrefillTaps sink(c, n);
  if (meta)
    for (int k = 0; k < PT_COUNT; ++k) { meta[3 * k] = k; meta[3 * k + 1] = sink.esz[k]; meta[3 * k + 2] = sink.cols[k]; }
  if (!taps) return PT_COUNT;
  if (taps_bytes < sink.bytes(n))
    return fail(VV_ERR_INVALID, "vv_debug_prefill_taps: %lld bytes of tap space, the layer needs %lld", (long long)taps_bytes, sink.bytes(n));
  if (!x_in || !workspace) return fail(VV_ERR_INVALID, "vv_debug_prefill_taps: null argument");
  if (((uintptr_t)x_in & 15) || ((uintptr_t)hidden_last & 15)) return fail(VV_ERR_INVALID, "vv_debug_prefill_taps: x_in / hidden_last must be 16-byte aligned");
  long long R;
  RET(pf_begin(c, "vv_debug_prefill_taps", seq, pos0, n, workspace, workspace_bytes, stream, &R));
  const int H = d.hidden_size, nq = d.num_q_heads * d.head_dim;
  unsigned char* ws = (unsigned char*)workspace;
  float* x = (float*)ws;
  bf16* a1 = (bf16*)(ws + align256(R * 4 * H));
  bf16* a2 = (bf16*)(ws + align256(R * 4 * H) + align256(R * 2 * std::max(H, nq)));
  const int* page_row = c->page_table_dev + (size_t)seq * c->max_pages;
  L l{c, (cudaStream_t)stream};
  sink.dst = (unsigned char*)taps;
  for (long long c0 = 0; c0 < n; c0 += R) {
    const int r = (int)std::min<long long>(R, n - c0);
    CK(cudaMemcpyAsync(x, x_in + c0 * H, (size_t)r * H * 4, cudaMemcpyDeviceToDevice, l.s));
    sink.c0 = c0;
    RET(prefill_layer(l, layer, page_row, pos0 + c0, r, x, a1, a2, &sink));
    if (hidden_last && c0 + r == n) CK(launch_k(l, rows_norm_block_kernel, dim3(1), dim3(256), 0, (const float*)(x + (size_t)(r - 1) * H), (const float*)c->lm_norm, hidden_last, H, d.rms_norm_eps));
  }
  CK(cudaStreamSynchronize(l.s));
  return PT_COUNT;
}

extern "C" int vv_embed_gather(vv_ctx* c, const int32_t* ids_dev, int64_t n, float* out, void* stream) {
  if (!c) return fail(VV_ERR_INVALID, "null ctx");
  if (!c->finalized) return fail(VV_ERR_STATE, "vv_embed_gather: not finalized");
  if (n < 1 || !ids_dev || !out) return fail(VV_ERR_INVALID, "vv_embed_gather: n = %lld ids / null argument", (long long)n);
  CK(cudaSetDevice(c->device));
  pf_embed_gather_kernel<<<(unsigned)std::min<int64_t>(n, 65535), 256, 0, (cudaStream_t)stream>>>(c->embed, ids_dev, n, c->d.vocab_size,
                                                                                                   c->d.hidden_size, out);
  CKL();
  c->launches++;
  return 0;
}

extern "C" int vv_debug_kv_read(vv_ctx* c, int seq, int layer, int64_t pos0, int64_t n, void* k_out, void* v_out, void* stream) {
  if (!c || !c->kpool) return fail(VV_ERR_STATE, "KV pool not initialised");
  const auto& d = c->d;
  if (seq < 0 || seq >= 2 * d.max_batch || layer < 0 || layer >= d.num_layers) return fail(VV_ERR_INVALID, "bad seq %d / layer %d", seq, layer);
  if (n < 1 || pos0 < 0 || pos0 + n > (int64_t)c->seq_pages[seq].size() * KV_PAGE)
    return fail(VV_ERR_INVALID, "vv_debug_kv_read: positions [%lld, %lld) outside the reserved range of seq %d", (long long)pos0, (long long)(pos0 + n), seq);
  const size_t per_layer = (size_t)c->n_pages * d.num_kv_heads * KV_PAGE * d.head_dim;
  pf_kv_read_kernel<<<(unsigned)std::min<int64_t>(n, 65535), 256, 0, (cudaStream_t)stream>>>(c->kpool + per_layer * layer, c->vpool + per_layer * layer,
                                                                                              c->page_table_dev + (size_t)seq * c->max_pages, d.num_kv_heads,
                                                                                              d.head_dim, pos0, n, (bf16*)k_out, (bf16*)v_out);
  CKL();
  c->launches++;
  return 0;
}

struct Rows { int v[16]; };
__global__ void state_zero_val_kernel(const StateSeg* __restrict__ segs, Rows r) {
  const int b = r.v[blockIdx.y];
  const StateSeg s = segs[blockIdx.x];
  float* dd = s.hist + (size_t)b * s.n;
  for (int i = threadIdx.x; i < s.n; i += blockDim.x) dd[i] = 0.f;
}
extern "C" int vv_codec_state_zero(vv_ctx* c, const int32_t* rows_host, int n, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  if (n < 1) return 0;
  if (n > c->d.max_batch) return fail(VV_ERR_INVALID, "too many rows");
  Rows r;
  for (int i = 0; i < 16; ++i) r.v[i] = i < n ? rows_host[i] : 0;
  for (int i = 0; i < n; ++i) if (r.v[i] < 0 || r.v[i] >= c->d.max_batch) return fail(VV_ERR_INVALID, "row %d out of range", r.v[i]);
  cudaStream_t s = (cudaStream_t)stream;
  state_zero_val_kernel<<<dim3(c->dec.n_segs, n), 256, 0, s>>>(c->dec.segs_dev, r);
  CKL();
  state_zero_val_kernel<<<dim3(c->enc.n_segs, n), 256, 0, s>>>(c->enc.segs_dev, r);
  CKL();
  c->launches += 2;
  return 0;
}
extern "C" int vv_codec_state_reset(vv_ctx* c, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  int rows[8];
  for (int i = 0; i < c->d.max_batch; ++i) rows[i] = i;
  return vv_codec_state_zero(c, rows, c->d.max_batch, stream);
}

extern "C" int vv_debug_gemv(vv_ctx* c, const void* w, const float* bias, const float* x, float* y, int M, int N, int K, int prologue,
                             const float* pro_w, float eps, int epilogue, void* stream) {
  if (!c) return fail(VV_ERR_INVALID, "null ctx");
  CK(cudaSetDevice(c->device));
  L l{c, (cudaStream_t)stream};
  const int ldy = epilogue == EPI_SWIGLU ? N / 2 : N;
  GemvP p = mk((const bf16*)w, bias, x, K, y, ldy, M, N, K);
  p.pro = prologue; p.pro_w = pro_w; p.pro_eps = eps; p.epi = epilogue;
  if (epilogue == EPI_RESID) { p.res = y; p.ldres = N; }
  return linear(l, p);
}

// linear() with the row map, strides, separate or in-place residual and epilogue operand of the codec's kernel-per-stage GEMMs (see the header)
extern "C" int vv_debug_gemv2(vv_ctx* c, const void* w, const float* bias, const float* x, int64_t ldx, int map_T, int64_t map_bs, float* y,
                              int64_t ldy, const float* res, int64_t ldres, int M, int N, int K, int prologue, const float* pro_w, float eps,
                              int epilogue, const float* epi_a, int64_t epi_lda, int32_t* info, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  if (!w || !x || !y || !info || M < 1 || N < 1 || K < 8) return fail(VV_ERR_INVALID, "vv_debug_gemv2: null operand or empty shape");
  if (prologue != PRO_NONE && prologue != PRO_RMSNORM && prologue != PRO_SILU) return fail(VV_ERR_INVALID, "vv_debug_gemv2: prologue %d", prologue);
  if (prologue == PRO_RMSNORM && !pro_w) return fail(VV_ERR_INVALID, "vv_debug_gemv2: RMSNorm needs its weight");
  const bool has_res = epilogue == EPI_RESID || epilogue == EPI_GATED_RESID || epilogue == EPI_GAMMA_RESID;
  if (epilogue != EPI_NONE && epilogue != EPI_GELU && epilogue != EPI_SILU && !has_res) return fail(VV_ERR_INVALID, "vv_debug_gemv2: epilogue %d", epilogue);
  if ((has_res && (!res || ldres < N || ldres > INT32_MAX)) || ((epilogue == EPI_GAMMA_RESID || epilogue == EPI_GATED_RESID) && !epi_a) ||
      (epilogue == EPI_GATED_RESID && epi_lda < N))
    return fail(VV_ERR_INVALID, "vv_debug_gemv2: missing residual / epilogue operand");
  if (ldx < 1 || map_T < 0 || map_bs < 0 || ldy < N || ldy > INT32_MAX) return fail(VV_ERR_INVALID, "vv_debug_gemv2: bad strides");
  CK(cudaSetDevice(c->device));
  L l{c, (cudaStream_t)stream};
  GemvP p = mk((const bf16*)w, bias, x, ldx, y, (int)ldy, M, N, K);
  if (map_T > 0) { p.xmap.T = map_T; p.xmap.bs = map_bs; }
  p.pro = prologue; p.pro_w = pro_w; p.pro_eps = eps; p.epi = epilogue;
  p.epi_a = epi_a; p.epi_lda = epi_lda; p.res = res; p.ldres = (int)ldres;
  RET(linear(l, p, info));
  CK(cudaStreamSynchronize(l.s));
  CKL();
  return 0;
}

// builds, runs and frees a one-off stream program (tests); returns the number of stages it ran (after the K split)
static int run_debug_stream(vv_ctx* c, StreamBuilder& b, void* stream) {
  vv_ctx::StreamProg pr;
  int rc = finish_stream(b, &pr);
  if (rc == 0) {
    L l{c, (cudaStream_t)stream};
    rc = launch_stream(l, pr);
    if (rc == 0 && cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess) rc = fail(VV_ERR_CUDA, "stream kernel: %s", cudaGetErrorString(cudaGetLastError()));
  }
  if (pr.ops) dfree(c, &pr.ops);
  if (pr.tmaps) dfree(c, &pr.tmaps);
  for (bf16* t : b.owned) dfree(c, &t);
  if (rc < 0) return rc;
  if (c->st_diag_host[0]) return fail(VV_ERR_CUDA, "stream kernel watchdog: code %u cta %u thread %u a %u b %u c %u", c->st_diag_host[0], c->st_diag_host[1],
                                      c->st_diag_host[2], c->st_diag_host[3], c->st_diag_host[4], c->st_diag_host[5]);
  return pr.n_ops;
}

// one linear through the weight-stream kernel (tests): y = [y +] alpha * (W pro(x) + bias); pro = SPro, alpha_kind = SAlpha
extern "C" int vv_debug_stream_gemv(vv_ctx* c, const void* w, const float* bias, const float* x, float* y, int M, int N, int K, int pro,
                                    const float* pro_w, float eps, int alpha_kind, const float* alpha, int accumulate, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  CK(cudaSetDevice(c->device));
  StreamBuilder b(c);
  b.fresh_weights = true;
  if (!accumulate) b.nop(false, y, (long long)M * N);
  SOp* o;
  RET(b.gemv((const bf16*)w, bias, x, pro == SP_SWIGLU ? 2LL * K : (long long)K, y, N, M, N, K, !accumulate, &o));
  o->pro = pro; o->pro_w = pro_w; o->pro_eps = eps; o->alpha_kind = alpha_kind; o->alpha = alpha; o->lda = N;
  const int rc = run_debug_stream(c, b, stream);
  return rc < 0 ? rc : 0;
}

// vv_debug_stream_gemv with the strides, AdaLN operands, store epilogue and K split exposed (see the header)
extern "C" int vv_debug_stream_gemv2(vv_ctx* c, const void* w, const float* bias, const float* x, int64_t ldx, float* y, int64_t ldy, int M, int N, int K,
                                     int pro, const float* pro_w, float eps, const float* pro_shift, const float* pro_scale, int64_t pro_ld,
                                     int alpha_kind, const float* alpha, int64_t lda, int store, int64_t operand_cap, void* stream) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  if (pro != SP_NONE && pro != SP_RMSNORM && pro != SP_ADALN && pro != SP_SWIGLU && pro != SP_GELU && pro != SP_SILU)
    return fail(VV_ERR_INVALID, "vv_debug_stream_gemv2: prologue %d not supported", pro);
  if (alpha_kind != SA_ONE && alpha_kind != SA_GATE && alpha_kind != SA_GAMMA) return fail(VV_ERR_INVALID, "vv_debug_stream_gemv2: alpha_kind %d", alpha_kind);
  if ((pro == SP_ADALN && (!pro_shift || !pro_scale)) || (alpha_kind != SA_ONE && !alpha))
    return fail(VV_ERR_INVALID, "vv_debug_stream_gemv2: missing AdaLN / alpha operand");
  if (ldx < (pro == SP_SWIGLU ? 2LL * K : (long long)K) || ldy < N || (alpha_kind == SA_GATE && lda < N) || (pro == SP_ADALN && pro_ld < K) ||
      ((uintptr_t)x & 15) || ldx % 4 || (pro == SP_ADALN && (pro_ld % 4 || ((uintptr_t)pro_shift & 15) || ((uintptr_t)pro_scale & 15))))
    return fail(VV_ERR_INVALID, "vv_debug_stream_gemv2: strides must cover the row and keep rows 16-byte aligned");
  CK(cudaSetDevice(c->device));
  StreamBuilder b(c);
  b.fresh_weights = true;
  b.operand_cap = operand_cap;
  SOp* o;
  RET(b.gemv((const bf16*)w, bias, x, ldx, y, ldy, M, N, K, false, &o));
  o->pro = pro; o->pro_w = pro_w; o->pro_eps = eps; o->pro_shift = pro_shift; o->pro_scale = pro_scale; o->pro_ld = pro_ld;
  o->alpha_kind = alpha_kind; o->alpha = alpha; o->lda = lda; o->store = store ? 1 : 0;
  return run_debug_stream(c, b, stream);
}
// clock stamps of the last traced stream launch (VV_STREAM_TRACE=<cta>): out [n_ops][12] int64; returns the number of stages, 0 if tracing is off.
// Stage kinds / shapes are appended per stage in out_meta [n_ops][4] = {kind, N, K, prologue}.
extern "C" int vv_stream_trace_read2(vv_ctx* c, long long* out, int max_ops) {     // [n_ops][sm_count][2] barrier arrival / release (ns)
  if (!c || !c->st_trace2) return 0;
  CK(cudaDeviceSynchronize());
  const int n = std::min(max_ops, c->st_trace_last_ops);
  CK(cudaMemcpy(out, c->st_trace2, (size_t)n * c->sm_count * 2 * sizeof(long long), cudaMemcpyDeviceToHost));
  return c->sm_count;
}
extern "C" int vv_stream_trace_read(vv_ctx* c, long long* out, int* out_meta, int max_ops, const char* prog_prefix) {
  if (!c || !c->st_trace) return 0;
  CK(cudaDeviceSynchronize());
  const int n = std::min(max_ops, c->st_trace_last_ops);
  CK(cudaMemcpy(out, c->st_trace, (size_t)n * ST_TRACE * sizeof(long long), cudaMemcpyDeviceToHost));
  for (auto& kv : c->sprogs) {
    if (kv.first.rfind(prog_prefix, 0) != 0 || kv.second.n_ops != c->st_trace_last_ops) continue;
    std::vector<SOp> ops(kv.second.n_ops);
    CK(cudaMemcpy(ops.data(), kv.second.ops, ops.size() * sizeof(SOp), cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) { out_meta[4 * i] = ops[i].kind; out_meta[4 * i + 1] = ops[i].N; out_meta[4 * i + 2] = ops[i].K; out_meta[4 * i + 3] = ops[i].pro; }
    break;
  }
  return n;
}
// watchdog record of the last stream kernel that trapped: out[0] = code (0 = none), out[1..5] = cta, thread, stage, iteration, extra
extern "C" int vv_stream_diag(vv_ctx* c, unsigned* out6) {
  if (!c || !c->st_diag_host) return fail(VV_ERR_STATE, "no context");
  for (int i = 0; i < 6; ++i) out6[i] = c->st_diag_host[i];
  return 0;
}

// time `iters` grid barriers of a cooperative launch with `per_sm` CTAs per SM (debug / profiling aid)
extern "C" int vv_debug_barrier_bench(vv_ctx* c, int iters, int per_sm, float* ms_out) {
  if (!c || !c->finalized) return fail(VV_ERR_STATE, "not finalized");
  CK(cudaSetDevice(c->device));
  cudaStream_t s;
  CK(cudaStreamCreate(&s));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = dim3(c->sm_count * per_sm); cfg.blockDim = dim3(256); cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative; attr[0].val.cooperative = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  float* sink = c->s_v;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  CK(cudaLaunchKernelEx(&cfg, barrier_bench_kernel, c->gridbar, 10, sink));
  CK(cudaEventRecord(e0, s));
  CK(cudaLaunchKernelEx(&cfg, barrier_bench_kernel, c->gridbar, iters, sink));
  CK(cudaEventRecord(e1, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaEventElapsedTime(ms_out, e0, e1));
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaStreamDestroy(s);
  return 0;
}
