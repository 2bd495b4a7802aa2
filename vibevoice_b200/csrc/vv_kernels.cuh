// vv_kernels.cuh -- hand-written sm_90a kernels of the VibeVoice generation hot path.
//
// Everything in the per-frame loop runs at M <= 2B rows against bf16 weight matrices, i.e. it is
// HBM-bandwidth bound (SURVEY 8d): the kernels below stream each weight byte exactly once with
// 16-byte coalesced loads, keep activations in fp32 (registers / shared memory), accumulate in
// fp32 and fuse the surrounding norm / modulation / activation / residual work into the GEMV
// prologue and epilogue so no activation round-trips through HBM more than once.
//
// Reference anchors (under vibevoice/modular of the reference project unless noted):
//   gemv prologues RMSNORM/ADALN      modular_vibevoice_diffusion_head.py:31-45, 158-161, 184-188;
//                                     transformers Qwen2RMSNorm (modeling_qwen2.py:249-266)
//   gemv epilogues SWIGLU/GATED_RESID modular_vibevoice_diffusion_head.py:116-123, 158-161
//   gemv epilogues GELU/GAMMA_RESID   modular_vibevoice_tokenizer.py:592-596, 670-682
//   assemble_window / dwconv_res      modular_vibevoice_tokenizer.py:327-382 (streaming SConv1d), 786-794
// (decode attention and the DPM-Solver++ update run only inside the weight-stream kernel: anchors at SAtt / SDpm in vv_stream.cuh)
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define VV_DEVINL __device__ __forceinline__

namespace vv {

typedef __nv_bfloat16 bf16;

enum Prologue { PRO_NONE = 0, PRO_RMSNORM = 1, PRO_ADALN = 2, PRO_SILU = 3 };
enum Epilogue { EPI_NONE = 0, EPI_RESID = 2, EPI_GATED_RESID = 3, EPI_GAMMA_RESID = 4, EPI_SWIGLU = 5, EPI_GELU = 6, EPI_SILU = 7 };

// row m of a logical [M, K] operand lives at base + (m / T) * bs + (m % T) * rs; rows may overlap
// (rs < K) -- that is how causal / strided / transposed convolutions read their input window.
struct RowMap {
  int T;
  long long bs;
  long long rs;
  VV_DEVINL long long off(int m) const { return (long long)(m / T) * bs + (long long)(m % T) * rs; }
};

static inline RowMap dense_rows(long long ld) { RowMap r; r.T = 1 << 30; r.bs = 0; r.rs = ld; return r; }

struct GemvP {
  const bf16* W;        // [N, K] row-major, K % 8 == 0
  const float* bias;    // [N] or null (added before the epilogue op)
  const float* x;       // fp32 activations
  RowMap xmap;
  float* y;             // [M, ldy]
  int ldy;
  int M, N, K;
  int pro;
  const float* pro_w;       // [K] norm weight (may be null for ADALN without affine)
  float pro_eps;
  const float* pro_shift;   // ADALN: [M, pro_ld]
  const float* pro_scale;
  long long pro_ld;
  int epi;
  const float* epi_a;       // GATED_RESID: gate [M, epi_lda]; GAMMA_RESID: gamma [N]
  long long epi_lda;
  const float* res;         // residual [M, ldres]
  int ldres;
  int WK;                   // warps splitting K inside a CTA (1,2,4,8); WR = 8 / WK row-quads per task
};

// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch: every hot-path kernel lets its successor start launching immediately
// (`pdl_trigger`) and blocks on its predecessor's completion (`pdl_wait`) only right before it touches
// activations -- weights never depend on a predecessor, so their first loads overlap the launch gap.
VV_DEVINL void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
VV_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

VV_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
VV_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
VV_DEVINL float silu_f(float x) { return x / (1.0f + __expf(-x)); }
VV_DEVINL float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

VV_DEVINL uint4 ldg_stream(const void* p) {  // weights are read once: bypass L1 allocation
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
VV_DEVINL void bf16x8_unpack(const uint4& u, float* f) {
  f[0] = __uint_as_float(u.x << 16); f[1] = __uint_as_float(u.x & 0xffff0000u);
  f[2] = __uint_as_float(u.y << 16); f[3] = __uint_as_float(u.y & 0xffff0000u);
  f[4] = __uint_as_float(u.z << 16); f[5] = __uint_as_float(u.z & 0xffff0000u);
  f[6] = __uint_as_float(u.w << 16); f[7] = __uint_as_float(u.w & 0xffff0000u);
}
VV_DEVINL float bf16_bits_to_f(unsigned short b) { return __uint_as_float(((unsigned)b) << 16); }

// position of element k inside the staged activation row: chunks of 256, inside a chunk the 8
// values a lane consumes are split into two float4 planes so both LDS.128 are bank-conflict free.
VV_DEVINL int xs_pos(int k) {
  int c = k >> 8, kk = k & 255;
  int lane = kk >> 3, j = kk & 7;
  return (c << 8) + ((j >> 2) << 7) + (lane << 2) + (j & 3);
}

VV_DEVINL void epi_store_e(const GemvP& p, int epi, int m, int n, float v) {
  // n indexes the weight row; bias already added; `epi` may be a compile-time constant at the call site
  switch (epi) {
    case EPI_RESID: v += p.res[(long long)m * p.ldres + n]; break;
    case EPI_GATED_RESID: v = p.res[(long long)m * p.ldres + n] + p.epi_a[(long long)m * p.epi_lda + n] * v; break;
    case EPI_GAMMA_RESID: v = p.res[(long long)m * p.ldres + n] + p.epi_a[n] * v; break;
    case EPI_GELU: v = gelu_erf_f(v); break;
    case EPI_SILU: v = silu_f(v); break;
    default: break;
  }
  p.y[(long long)m * p.ldy + n] = v;
}
VV_DEVINL void epi_store(const GemvP& p, int m, int n, float v) { epi_store_e(p, p.epi, m, n, v); }

// ---------------------------------------------------------------------------------------------
// GEMV: y[m, n] = epi( sum_k W[n,k] * pro(x)[m,k] + bias[n] ),  M <= 16 (blocks of MB rows).
// CTA = 8 warps arranged as WR row-quads x WK k-splits; persistent over row-quad tasks.
//  * weights stream from HBM straight into registers, 16 B / lane / load, software-pipelined one
//    256-element chunk ahead; the first chunk of a CTA's first task is requested BEFORE the
//    activation block is staged, so the HBM latency of the weights overlaps the prologue;
//  * the staged activation block pro(x) lives in shared memory (fp32, bank-conflict-free planes).
// ---------------------------------------------------------------------------------------------
template <int MB>
__global__ void __launch_bounds__(256) gemv_kernel(GemvP p) {
  extern __shared__ __align__(16) float smem_f[];
  const int K = p.K, N = p.N;
  const int Kp = (K + 255) & ~255;
  float* xs = smem_f;                   // [MB][Kp]
  float* red = smem_f + MB * Kp;        // [2][8 warps][4*MB]
  __shared__ float s_part[MB][8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int WK = p.WK, WR = 8 / WK;
  const int wr = warp / WK, wk = warp % WK;
  const int ntasks = (N + 4 * WR - 1) / (4 * WR);
  const int nchunks = (K + 255) >> 8;
  const int klane = lane * 8;

  auto load_chunk = [&](uint4 (&wv)[4], const bf16* const (&wrow)[4], int c) {
    if (c < nchunks && (c << 8) + klane < K) {
#pragma unroll
      for (int r = 0; r < 4; ++r) wv[r] = ldg_stream(wrow[r] + (c << 8));
    } else {
#pragma unroll
      for (int r = 0; r < 4; ++r) wv[r] = make_uint4(0u, 0u, 0u, 0u);
    }
  };
  auto set_rows = [&](const bf16* (&wrow)[4], int task) {
    const int r0 = (task * WR + wr) * 4;
#pragma unroll
    for (int r = 0; r < 4; ++r) wrow[r] = p.W + (size_t)min(r0 + r, N - 1) * K + klane;
  };

  pdl_trigger();
  for (int m0 = 0; m0 < p.M; m0 += MB) {
    __syncthreads();
    int task = blockIdx.x;
    const bf16* wrow[4];
    uint4 cur[4], nxt[4];
    int c = wk;
    if (task < ntasks) {
      set_rows(wrow, task);
      load_chunk(cur, wrow, c);            // two chunks per warp are in flight while the activations are staged
      load_chunk(nxt, wrow, c + WK);
    }
    pdl_wait();                            // predecessor's activations are complete and visible from here on
    // ---- stage pro(x) for rows m0..m0+MB-1: one pass over x (values parked in registers across the norm reduction) ----
    const bool need_inv = (p.pro == PRO_RMSNORM || p.pro == PRO_ADALN);
    const int K4 = K >> 2;
    constexpr int XR = 4;                  // float4 per thread per row kept in registers (covers K <= 4096)
    const bool one_pass = (K4 <= XR * 256);
    for (int m = 0; m < MB; ++m) {
      const bool valid = (m0 + m < p.M);
      const float* xr = p.x + (valid ? p.xmap.off(m0 + m) : 0);
      float4 xv[XR];
      float inv = 1.f;
      if (need_inv) {
        float ss = 0.f;
        if (one_pass) {
#pragma unroll
          for (int i = 0; i < XR; ++i) {
            const int q = tid + i * 256;
            xv[i] = (valid && q < K4) ? *reinterpret_cast<const float4*>(xr + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
            ss += xv[i].x * xv[i].x + xv[i].y * xv[i].y + xv[i].z * xv[i].z + xv[i].w * xv[i].w;
          }
        } else if (valid) {
          for (int q = tid; q < K4; q += 256) { const float4 v = *reinterpret_cast<const float4*>(xr + 4 * q); ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w; }
        }
        ss = warp_sum(ss);
        if (lane == 0) s_part[m][warp] = ss;
        __syncthreads();
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += s_part[m][i];
        inv = rsqrtf(t / (float)K + p.pro_eps);
      }
      auto xform_store = [&](int k, float4 v, bool have) {
        if (valid && k < K) {
          if (!have) v = *reinterpret_cast<const float4*>(xr + k);
          if (p.pro == PRO_RMSNORM) {
            const float4 w = *reinterpret_cast<const float4*>(p.pro_w + k);
            v.x *= inv * w.x; v.y *= inv * w.y; v.z *= inv * w.z; v.w *= inv * w.w;
          } else if (p.pro == PRO_ADALN) {
            float4 w = make_float4(1.f, 1.f, 1.f, 1.f);
            if (p.pro_w) w = *reinterpret_cast<const float4*>(p.pro_w + k);
            const long long o = (long long)(m0 + m) * p.pro_ld + k;
            const float4 sc = *reinterpret_cast<const float4*>(p.pro_scale + o);
            const float4 sh = *reinterpret_cast<const float4*>(p.pro_shift + o);
            v.x = v.x * inv * w.x * (1.f + sc.x) + sh.x; v.y = v.y * inv * w.y * (1.f + sc.y) + sh.y;
            v.z = v.z * inv * w.z * (1.f + sc.z) + sh.z; v.w = v.w * inv * w.w * (1.f + sc.w) + sh.w;
          } else if (p.pro == PRO_SILU) {
            v.x = silu_f(v.x); v.y = silu_f(v.y); v.z = silu_f(v.z); v.w = silu_f(v.w);
          }
        } else {
          v = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        *reinterpret_cast<float4*>(xs + m * Kp + xs_pos(k)) = v;
      };
#pragma unroll
      for (int i = 0; i < XR; ++i) {
        const int q = tid + i * 256;
        if (q < (Kp >> 2)) xform_store(q << 2, xv[i], need_inv && one_pass);
      }
      for (int q = tid + XR * 256; q < (Kp >> 2); q += 256) xform_store(q << 2, make_float4(0.f, 0.f, 0.f, 0.f), false);
    }
    __syncthreads();

    int parity = 0;
    while (task < ntasks) {
      float acc[4][MB];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int m = 0; m < MB; ++m) acc[r][m] = 0.f;
      // residual / gate operands of this task's outputs are requested now, consumed after the reduction
      float pre_res = 0.f, pre_gate = 1.f;
      const bool has_res = (p.epi == EPI_RESID || p.epi == EPI_GATED_RESID || p.epi == EPI_GAMMA_RESID);
      if (has_res && tid < WR * 4 * MB) {
        const int q = tid / (4 * MB), r = (tid / MB) % 4, m = tid % MB;
        const int n = (task * WR + q) * 4 + r;
        if (n < N && m0 + m < p.M) {
          pre_res = p.res[(long long)(m0 + m) * p.ldres + n];
          if (p.epi == EPI_GATED_RESID) pre_gate = p.epi_a[(long long)(m0 + m) * p.epi_lda + n];
          else if (p.epi == EPI_GAMMA_RESID) pre_gate = p.epi_a[n];
        }
      }
      while (c < nchunks) {
        uint4 nn[4];
        load_chunk(nn, wrow, c + 2 * WK);
        float xv[MB][8];
#pragma unroll
        for (int m = 0; m < MB; ++m) {
          const float4 a = *reinterpret_cast<const float4*>(xs + m * Kp + (c << 8) + (lane << 2));
          const float4 b = *reinterpret_cast<const float4*>(xs + m * Kp + (c << 8) + 128 + (lane << 2));
          xv[m][0] = a.x; xv[m][1] = a.y; xv[m][2] = a.z; xv[m][3] = a.w;
          xv[m][4] = b.x; xv[m][5] = b.y; xv[m][6] = b.z; xv[m][7] = b.w;
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          float wf[8];
          bf16x8_unpack(cur[r], wf);
#pragma unroll
          for (int m = 0; m < MB; ++m)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[r][m] = fmaf(wf[j], xv[m][j], acc[r][m]);
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) { cur[r] = nxt[r]; nxt[r] = nn[r]; }
        c += WK;
      }
      // next task's first chunks go out before this task's reduction
      const int this_task = task;
      task += gridDim.x;
      c = wk;
      if (task < ntasks) {
        set_rows(wrow, task);
        load_chunk(cur, wrow, c);
        load_chunk(nxt, wrow, c + WK);
      }
      // ---- reduce: lanes -> lane 0; k-split warps -> shared ----
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int m = 0; m < MB; ++m) acc[r][m] = warp_sum(acc[r][m]);
      float* rbuf = red + parity * (8 * 4 * MB);
      if (lane == 0) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int m = 0; m < MB; ++m) rbuf[warp * (4 * MB) + r * MB + m] = acc[r][m];
      }
      __syncthreads();
      // ---- epilogue: one thread per (row-quad, r, m) ----
      if (p.epi == EPI_SWIGLU) {
        if (tid < WR * 2 * MB) {
          const int q = tid / (2 * MB), pr = (tid / MB) % 2, m = tid % MB;
          const int n0 = (this_task * WR + q) * 4 + pr * 2;
          if (n0 + 1 < N && m0 + m < p.M) {
            float g = 0.f, u = 0.f;
            for (int s = 0; s < WK; ++s) {
              g += rbuf[(q * WK + s) * (4 * MB) + (pr * 2) * MB + m];
              u += rbuf[(q * WK + s) * (4 * MB) + (pr * 2 + 1) * MB + m];
            }
            if (p.bias) { g += p.bias[n0]; u += p.bias[n0 + 1]; }
            p.y[(long long)(m0 + m) * p.ldy + (n0 >> 1)] = silu_f(g) * u;
          }
        }
      } else {
        if (tid < WR * 4 * MB) {
          const int q = tid / (4 * MB), r = (tid / MB) % 4, m = tid % MB;
          const int n = (this_task * WR + q) * 4 + r;
          if (n < N && m0 + m < p.M) {
            float v = 0.f;
            for (int s = 0; s < WK; ++s) v += rbuf[(q * WK + s) * (4 * MB) + r * MB + m];
            if (p.bias) v += p.bias[n];
            if (has_res) v = pre_res + pre_gate * v;
            else if (p.epi == EPI_GELU) v = gelu_erf_f(v);
            else if (p.epi == EPI_SILU) v = silu_f(v);
            p.y[(long long)(m0 + m) * p.ldy + n] = v;
          }
        }
      }
      parity ^= 1;
      // double-buffered `red`: the next task writes the other half, the one after is fenced by
      // the next __syncthreads, so no trailing barrier is needed here.
    }
  }
}

// ---------------------------------------------------------------------------------------------
// mbarrier / bulk-copy primitives (shared by the weight-stream kernel in vv_stream.cuh)
// ---------------------------------------------------------------------------------------------
VV_DEVINL unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
VV_DEVINL void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
VV_DEVINL void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
VV_DEVINL void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
VV_DEVINL void mbar_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok = 0;
  const unsigned a = smem_u32(bar);
  while (!ok) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(a), "r"(parity) : "memory");
  }
}
VV_DEVINL void bulk_g2s(void* smem_dst, const void* gsrc, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
VV_DEVINL void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// Tensor-core GEMM for the codec stages with many rows (M > 8): C[M,N] = A[M,K] * W[N,K]^T.
// A is fp32 in global memory and is split on the fly into bf16 hi + bf16 lo (A = hi + lo up to
// 2^-16 relative), W is bf16, so two bf16 MMAs per tile reproduce the fp32-activation result of
// the GEMV path to ~1e-5 while running on the tensor pipe.  CTA tile 32 x 64 x 64, 4 warps, W
// streamed with a 3-stage cp.async ring, A register-prefetched one k-step ahead.
// (mma.sync m16n8k16.)
// ---------------------------------------------------------------------------------------------
VV_DEVINL void cp_async16(void* smem, const void* gmem, int src_bytes) {
  unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(sa), "l"(gmem), "r"(src_bytes));
}
VV_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::); }
template <int N_> VV_DEVINL void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N_)); }
VV_DEVINL void ldmatrix_x4(unsigned (&r)[4], const void* smem) {
  unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(sa));
}
VV_DEVINL void mma_bf16_16816(float (&d)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
VV_DEVINL unsigned pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<unsigned*>(&v);
}

constexpr int MM_BM = 32, MM_BN = 64, MM_BK = 64, MM_ST = 3, MM_LD = MM_BK + 8;   // +8 bf16 = 16 B row pad (ldmatrix conflict-free)
__global__ void __launch_bounds__(128) gemm_mma_kernel(GemvP p) {
  __shared__ __align__(16) bf16 Ah[MM_BM][MM_LD];
  __shared__ __align__(16) bf16 Al[MM_BM][MM_LD];
  __shared__ __align__(16) bf16 Ws[MM_ST][MM_BN][MM_LD];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bm = blockIdx.y * MM_BM, bn = blockIdx.x * MM_BN;
  const int K = p.K, nk_all = (K + MM_BK - 1) / MM_BK;
  // split-K (gridDim.z > 1): only launched for in-place residual epilogues (y == res); each split atomically adds its
  // scaled partial into y, split 0 also adds the bias.  Few-CTA, long-K shapes (codec FFN2) get z-times the parallelism.
  const int kz = blockIdx.z, nz = gridDim.z;
  const int kt0 = (int)(((long long)nk_all * kz) / nz), kt1 = (int)(((long long)nk_all * (kz + 1)) / nz);
  const int nk = kt1 - kt0;
  // A loader: thread -> row tid/4, 16 consecutive k at (tid%4)*16
  const int ar = tid >> 2, ac = (tid & 3) * 16;
  const float* arow = (bm + ar < p.M) ? p.x + p.xmap.off(bm + ar) : nullptr;
  // W loader: 64 rows x 64 k bf16 = 512 x 16 B; thread handles 4 of them
  auto load_w = [&](int stage, int kt) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + i * 128, r = idx >> 3, c = (idx & 7) * 8;
      const int n = bn + r, k = (kt0 + kt) * MM_BK + c;
      const bool ok = (n < p.N) && (k < K);
      cp_async16(&Ws[stage][r][c], p.W + (size_t)(ok ? n : 0) * K + (ok ? k : 0), ok ? 16 : 0);
    }
  };
  float4 areg[4];
  float a_inv = 1.f;            // PRO_RMSNORM: row scale, applied together with the norm weight while converting A
  auto load_a = [&](int kt) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = (kt0 + kt) * MM_BK + ac + i * 4;
      areg[i] = (arow && k < K) ? *reinterpret_cast<const float4*>(arow + k) : make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.pro == PRO_RMSNORM && arow && k < K) {
        const float4 wv = *reinterpret_cast<const float4*>(p.pro_w + k);
        areg[i].x *= a_inv * wv.x; areg[i].y *= a_inv * wv.y; areg[i].z *= a_inv * wv.z; areg[i].w *= a_inv * wv.w;
      } else if (p.pro == PRO_ADALN && arow && k < K) {
        float4 wv = make_float4(1.f, 1.f, 1.f, 1.f);
        if (p.pro_w) wv = *reinterpret_cast<const float4*>(p.pro_w + k);
        const long long o = (long long)(bm + ar) * p.pro_ld + k;
        const float4 sc = *reinterpret_cast<const float4*>(p.pro_scale + o);
        const float4 sh = *reinterpret_cast<const float4*>(p.pro_shift + o);
        areg[i].x = areg[i].x * a_inv * wv.x * (1.f + sc.x) + sh.x; areg[i].y = areg[i].y * a_inv * wv.y * (1.f + sc.y) + sh.y;
        areg[i].z = areg[i].z * a_inv * wv.z * (1.f + sc.z) + sh.z; areg[i].w = areg[i].w * a_inv * wv.w * (1.f + sc.w) + sh.w;
      } else if (p.pro == PRO_SILU && arow && k < K) {
        areg[i].x = silu_f(areg[i].x); areg[i].y = silu_f(areg[i].y); areg[i].z = silu_f(areg[i].z); areg[i].w = silu_f(areg[i].w);
      }
    }
  };
  auto store_a = [&]() {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float v[4] = {areg[i].x, areg[i].y, areg[i].z, areg[i].w};
      float h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { h[j] = __bfloat162float(__float2bfloat16_rn(v[j])); l[j] = v[j] - h[j]; }
      *reinterpret_cast<uint2*>(&Ah[ar][ac + i * 4]) = make_uint2(pack_bf16(h[0], h[1]), pack_bf16(h[2], h[3]));
      *reinterpret_cast<uint2*>(&Al[ar][ac + i * 4]) = make_uint2(pack_bf16(l[0], l[1]), pack_bf16(l[2], l[3]));
    }
  };
  float acc[2][2][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

  pdl_trigger();
#pragma unroll
  for (int s_ = 0; s_ < MM_ST - 1; ++s_) { if (s_ < nk) load_w(s_, s_); cp_async_commit(); }
  pdl_wait();
  if (p.pro == PRO_RMSNORM || p.pro == PRO_ADALN) {   // 4 threads share a row: each sums a quarter of it, combined with two shuffles
    float ss = 0.f;
    if (arow) for (int k = (tid & 3) * 4; k < K; k += 16) { const float4 v = *reinterpret_cast<const float4*>(arow + k); ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w; }
    ss += __shfl_xor_sync(0xffffffffu, ss, 1);
    ss += __shfl_xor_sync(0xffffffffu, ss, 2);
    a_inv = rsqrtf(ss / (float)K + p.pro_eps);
  }
  load_a(0);
  for (int kt = 0; kt < nk; ++kt) {
    __syncthreads();                       // previous step's readers of Ah/Al and of the stage about to be refilled are done
    store_a();
    if (kt + MM_ST - 1 < nk) load_w((kt + MM_ST - 1) % MM_ST, kt + MM_ST - 1);
    cp_async_commit();
    if (kt + 1 < nk) load_a(kt + 1);
    cp_async_wait<MM_ST - 1>();            // stage kt has landed
    __syncthreads();
    const int st = kt % MM_ST;
#pragma unroll
    for (int kk = 0; kk < MM_BK; kk += 16) {
      unsigned ah[2][4], al[2][4], bw[4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        ldmatrix_x4(ah[mt], &Ah[mt * 16 + (lane & 15)][kk + (lane >> 4) * 8]);
        ldmatrix_x4(al[mt], &Al[mt * 16 + (lane & 15)][kk + (lane >> 4) * 8]);
      }
      // B fragments for this warp's two n-tiles (16 rows of W): lanes 0-7 n0..7 @k, 8-15 n0..7 @k+8, 16-23 n8..15 @k, 24-31 n8..15 @k+8
      ldmatrix_x4(bw, &Ws[st][warp * 16 + (lane & 7) + ((lane >> 4) << 3)][kk + ((lane >> 3) & 1) * 8]);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        mma_bf16_16816(acc[mt][0], ah[mt], bw[0], bw[1]);
        mma_bf16_16816(acc[mt][0], al[mt], bw[0], bw[1]);
        mma_bf16_16816(acc[mt][1], ah[mt], bw[2], bw[3]);
        mma_bf16_16816(acc[mt][1], al[mt], bw[2], bw[3]);
      }
    }
  }
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int m = bm + mt * 16 + (lane >> 2) + (q >> 1) * 8;
        const int n = bn + warp * 16 + nt * 8 + (lane & 3) * 2 + (q & 1);
        if (p.epi == EPI_SWIGLU) {                 // (gate, up) = (even, odd) weight rows = (c0,c1) / (c2,c3) of one thread
          if ((q & 1) == 0 && m < p.M && n + 1 < p.N) {
            const float g_ = acc[mt][nt][q] + (p.bias ? p.bias[n] : 0.f), u_ = acc[mt][nt][q + 1] + (p.bias ? p.bias[n + 1] : 0.f);
            p.y[(long long)m * p.ldy + (n >> 1)] = silu_f(g_) * u_;
          }
        } else if (m < p.M && n < p.N) {
          if (nz == 1) {
            epi_store(p, m, n, acc[mt][nt][q] + (p.bias ? p.bias[n] : 0.f));
          } else {
            float v = acc[mt][nt][q] + ((kz == 0 && p.bias) ? p.bias[n] : 0.f);
            if (p.epi == EPI_GAMMA_RESID) v *= p.epi_a[n];
            else if (p.epi == EPI_GATED_RESID) v *= p.epi_a[(long long)m * p.epi_lda + n];
            atomicAdd(p.y + (long long)m * p.ldy + n, v);
          }
        }
      }
}

// ---------------------------------------------------------------------------------------------
// Deep-ring variant of gemm_mma_kernel for the codec GEMMs with M > 8 (FFNs, transposed convs); prologue none or RMSNorm.
// Why: these GEMMs are tiny (K = 32..2048, <= 112 CTAs) and each CTA used to pay one L2/DRAM round trip PER k-step
// (A register-prefetched one step ahead, W two steps ahead).  Here BOTH operands arrive by cp.async into a 6-stage ring -- fp32 A tile [32 x 64] and bf16 W tile [64 x 64] per stage --
// so up to five k-steps (usually the whole K of a split) are in flight from the first instruction and a CTA pays ~one round trip in
// total.  The fp32 A tile is converted to the bf16 hi/lo mma fragments straight from shared memory (LDS.64 per fragment register,
// row stride 72 floats = conflict-free), which also removes the second __syncthreads and the Ah/Al staging of the old kernel.
// Same tile (32 x 64 x 64, 4 warps, warp = 16 output columns), same split-K / epilogue semantics, same hi+lo accuracy.
// ---------------------------------------------------------------------------------------------
constexpr int MR_ST = 6, MR_ALD = MM_BK + 8;   // 72-float rows: a half-warp LDS.64 (4 rows x 8 words) hits 32 distinct banks
constexpr int MR_A_BYTES = MM_BM * MR_ALD * 4, MR_W_BYTES = MM_BN * MM_LD * 2, MR_STAGE = MR_A_BYTES + MR_W_BYTES;
constexpr int MR_SMEM = MR_ST * MR_STAGE;
constexpr int MR_MAXK_NORM = 512;                  // PRO_RMSNORM: the norm weight row is staged in shared memory behind the ring (2 CTAs/SM must still fit)
constexpr int MR_SMEM_NORM = MR_SMEM + MR_MAXK_NORM * 4;
// RMS / EPI >= 0: prologue and epilogue kind as compile-time facts (the codec tail launches this kernel 68 times per frame and every
// launch runs its path once from a cold instruction cache); -1 = decided at run time.
template <int RMS, int EPI>
__global__ void __launch_bounds__(128) gemm_mma_ring_kernel(GemvP p) {
  extern __shared__ __align__(16) unsigned char mr_smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bm = blockIdx.y * MM_BM, bn = blockIdx.x * MM_BN;
  const int K = p.K, nk_all = (K + MM_BK - 1) / MM_BK;
  const int kz = blockIdx.z, nz = gridDim.z;
  const int kt0 = (int)(((long long)nk_all * kz) / nz), kt1 = (int)(((long long)nk_all * (kz + 1)) / nz);
  const int nk = kt1 - kt0;
  auto a_tile = [&](int stage) { return reinterpret_cast<float*>(mr_smem + stage * MR_STAGE); };
  auto w_tile = [&](int stage) { return reinterpret_cast<bf16*>(mr_smem + stage * MR_STAGE + MR_A_BYTES); };
  auto load_w = [&](int stage, int kt) {          // 64 rows x 8 chunks of 16 B
    bf16* wt = w_tile(stage);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + i * 128, r = idx >> 3, c = (idx & 7) * 8;
      const int n = bn + r, k = (kt0 + kt) * MM_BK + c;
      const bool ok = (n < p.N) && (k < K);
      cp_async16(wt + r * MM_LD + c, p.W + (size_t)(ok ? n : 0) * K + (ok ? k : 0), ok ? 16 : 0);
    }
  };
  // A loader: 32 rows x 16 chunks of 16 B (4 floats); thread -> row tid/4, chunks (tid%4) + 4 i  (a row's 4 threads cover 64 B runs)
  const int ar = tid >> 2;
  const float* arow = (bm + ar < p.M) ? p.x + p.xmap.off(bm + ar) : nullptr;
  auto load_a = [&](int stage, int kt) {
    float* at = a_tile(stage) + ar * MR_ALD;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = ((tid & 3) + 4 * i) * 4, k = (kt0 + kt) * MM_BK + c;
      const bool ok = arow && (k < K);
      cp_async16(at + c, ok ? arow + k : p.x, ok ? 16 : 0);
    }
  };
  float acc[2][2][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;
  // PRO_RMSNORM (never combined with split-K): y = W (x * inv_rms(x) * g) = inv_rms(x) * (W (x * g)) -- the per-row scalar commutes
  // with the GEMM, so the tile multiplies x * g (g = norm weight, applied while building fragments), every thread accumulates the
  // squares of the raw x values it converts anyway, and the row scale is applied to the accumulator in the epilogue.  No separate
  // normalisation pass, no extra read of x.
  const bool rms = RMS >= 0 ? (RMS != 0) : (p.pro == PRO_RMSNORM);
  const int epi = EPI >= 0 ? EPI : p.epi;
  float* gk = reinterpret_cast<float*>(mr_smem + MR_SMEM);
  float ss[2][2] = {{0.f, 0.f}, {0.f, 0.f}};

  pdl_trigger();
  if (rms) for (int i = tid * 4; i < K; i += 128 * 4) cp_async16(gk + i, p.pro_w + i, 16);
#pragma unroll
  for (int s_ = 0; s_ < MR_ST - 1; ++s_) if (s_ < nk) load_w(s_, s_);      // weights do not depend on the predecessor grid
  pdl_wait();
#pragma unroll
  for (int s_ = 0; s_ < MR_ST - 1; ++s_) { if (s_ < nk) load_a(s_, s_); cp_async_commit(); }   // group s_ completes => W(all issued) and A(s_) landed
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<MR_ST - 2>();            // stage kt has landed (this thread's copies) ...
    __syncthreads();                       // ... and everyone's; all warps are also done reading stage kt-1
    if (kt + MR_ST - 1 < nk) { load_w((kt + MR_ST - 1) % MR_ST, kt + MR_ST - 1); load_a((kt + MR_ST - 1) % MR_ST, kt + MR_ST - 1); }
    cp_async_commit();
    const int st = kt % MR_ST;
    const float* at = a_tile(st);
    const bf16* wt = w_tile(st);
#pragma unroll
    for (int kk = 0; kk < MM_BK; kk += 16) {
      unsigned ah[2][4], al[2][4], bw[4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        // m16n8k16 A fragment: reg0 = (row g, k 2t..2t+1), reg1 = (row g+8, same k), reg2 = (row g, k+8..), reg3 = (row g+8, k+8..)
        const float* a0 = at + (mt * 16 + (lane >> 2)) * MR_ALD + kk + (lane & 3) * 2;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float2 v = *reinterpret_cast<const float2*>(a0 + (q & 1) * 8 * MR_ALD + (q >> 1) * 8);
          if (rms) {
            ss[mt][q & 1] = fmaf(v.x, v.x, fmaf(v.y, v.y, ss[mt][q & 1]));
            const int kg = min((kt0 + kt) * MM_BK + kk + (lane & 3) * 2 + (q >> 1) * 8, K - 2);   // columns >= K hold zeros
            const float2 g = *reinterpret_cast<const float2*>(gk + kg);
            v.x *= g.x; v.y *= g.y;
          }
          const float hx = __bfloat162float(__float2bfloat16_rn(v.x)), hy = __bfloat162float(__float2bfloat16_rn(v.y));
          ah[mt][q] = pack_bf16(hx, hy);
          al[mt][q] = pack_bf16(v.x - hx, v.y - hy);
        }
      }
      ldmatrix_x4(bw, wt + (warp * 16 + (lane & 7) + ((lane >> 4) << 3)) * MM_LD + kk + ((lane >> 3) & 1) * 8);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        mma_bf16_16816(acc[mt][0], ah[mt], bw[0], bw[1]);
        mma_bf16_16816(acc[mt][0], al[mt], bw[0], bw[1]);
        mma_bf16_16816(acc[mt][1], ah[mt], bw[2], bw[3]);
        mma_bf16_16816(acc[mt][1], al[mt], bw[2], bw[3]);
      }
    }
  }
  if (rms) {
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {                 // a row's 64 columns per k-step live in the 4 lanes of a quad
        float t = ss[mt][h];
        t += __shfl_xor_sync(0xffffffffu, t, 1);
        t += __shfl_xor_sync(0xffffffffu, t, 2);
        ss[mt][h] = rsqrtf(t / (float)K + p.pro_eps);
      }
  }
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int m = bm + mt * 16 + (lane >> 2) + (q >> 1) * 8;
        const int n = bn + warp * 16 + nt * 8 + (lane & 3) * 2 + (q & 1);
        if (m < p.M && n < p.N) {
          if (nz == 1) {
            epi_store_e(p, epi, m, n, acc[mt][nt][q] * (rms ? ss[mt][q >> 1] : 1.f) + (p.bias ? p.bias[n] : 0.f));
          } else {
            float v = acc[mt][nt][q] + ((kz == 0 && p.bias) ? p.bias[n] : 0.f);
            if (epi == EPI_GAMMA_RESID) v *= p.epi_a[n];
            else if (epi == EPI_GATED_RESID) v *= p.epi_a[(long long)m * p.epi_lda + n];
            atomicAdd(p.y + (long long)m * p.ldy + n, v);
          }
        }
      }
}

// ---------------------------------------------------------------------------------------------
// Warpgroup GEMM (Hopper wgmma) for the wide M > 8 GEMMs: D^T[128 x 64] += W[128 x K] * A[64 x K]^T ("swap-AB": the weight rows fill
// the MMA M dimension as two m64 halves, the MMA N dimension holds up to 64 activation rows).
//   * operands in shared memory, K-major, 128-byte swizzle (8-row atoms of 8 x 128 B, stride byte offset 1024 B); W tiles and the
//     activation planes arrive by cp.async into swizzled positions (three stages, requested two k-blocks ahead); activations are
//     pre-split fp32 -> bf16 hi + bf16 lo (split_bf16_kernel) and both halves are multiplied into the SAME accumulator (two MMAs),
//     so the result keeps ~fp32-activation accuracy;
//   * the CTA is one warpgroup: wgmma.mma_async m64n64k16 from shared memory, fp32 accumulators in registers (64 per thread);
//   * epilogue straight from the accumulator fragments, fused bias / activation / residual.
// ---------------------------------------------------------------------------------------------
constexpr int WG_BM = 128, WG_BN = 64, WG_BK = 64;
constexpr int WG_STAGE = WG_BM * 128 + 2 * WG_BN * 128;          // W 16 KB + A_hi 8 KB + A_lo 8 KB
constexpr int WG_NST = 3;                                       // shared-memory stages (operands are requested two k-blocks ahead)
constexpr int WG_SMEM = WG_NST * WG_STAGE + 1024;               // + slack for 1024 B alignment

// shared-memory matrix descriptor of a K-major bf16 operand with 128-byte swizzle: start address, leading byte offset (unused for this
// layout, 16 B), stride byte offset 1024 B (one 8-row atom), layout type 1 = SWIZZLE_128B.  A k-step of 16 elements (32 B) inside the
// atom is +2 on the start-address field; 64 rows further is +512.
VV_DEVINL unsigned long long wgmma_desc_sw128(unsigned smem_addr) {
  return (unsigned long long)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
VV_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
VV_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N_> VV_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N_) : "memory"); }
// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands K-major in shared memory.  Accumulator fragment: register i of thread
// (warp w of the warpgroup, lane l) holds row 16 w + l / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (l & 3) + (i & 1).
VV_DEVINL void wgmma_m64n16(float (&d)[8], unsigned long long a, unsigned long long b, int accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "l"(a), "l"(b), "r"(accumulate) : "memory");
}
VV_DEVINL void wgmma_m64n32(float (&d)[16], unsigned long long a, unsigned long long b, int accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(a), "l"(b), "r"(accumulate) : "memory");
}
VV_DEVINL void wgmma_m64n64(float (&d)[32], unsigned long long a, unsigned long long b, int accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(a), "l"(b), "r"(accumulate) : "memory");
}

// fp32 activations [M, K] (RowMap) -> dense bf16 planes hi, lo [M, K] with x = hi + lo (|err| <= 2^-17 |x|)
__global__ void split_bf16_kernel(const float* __restrict__ x, RowMap xmap, bf16* __restrict__ hi, bf16* __restrict__ lo, int M, int K) {
  pdl_trigger();
  pdl_wait();
  const long long n4 = (long long)M * (K >> 2);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / (K >> 2)), k = (int)(i % (K >> 2)) << 2;
    const float4 v = *reinterpret_cast<const float4*>(x + xmap.off(m) + k);
    const float h0 = __bfloat162float(__float2bfloat16_rn(v.x)), h1 = __bfloat162float(__float2bfloat16_rn(v.y));
    const float h2 = __bfloat162float(__float2bfloat16_rn(v.z)), h3 = __bfloat162float(__float2bfloat16_rn(v.w));
    *reinterpret_cast<uint2*>(hi + (size_t)m * K + k) = make_uint2(pack_bf16(h0, h1), pack_bf16(h2, h3));
    *reinterpret_cast<uint2*>(lo + (size_t)m * K + k) = make_uint2(pack_bf16(v.x - h0, v.y - h1), pack_bf16(v.z - h2, v.w - h3));
  }
}

__global__ void __launch_bounds__(128) gemm_wgmma_kernel(GemvP p, const bf16* __restrict__ a_hi, const bf16* __restrict__ a_lo) {
  extern __shared__ unsigned char wg_raw[];
  const unsigned raw_addr = smem_u32(wg_raw);
  unsigned char* sm = wg_raw + ((1024u - (raw_addr & 1023u)) & 1023u);      // 1024 B aligned (swizzle atom)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bn = blockIdx.x * WG_BM;       // weight rows (output features) of this CTA
  const int bm = blockIdx.y * WG_BN;       // activation rows
  const int K = p.K, nk = (K + WG_BK - 1) / WG_BK;

  // one stage = W tile [128 x 64] + A_hi [64 x 64] + A_lo [64 x 64], all bf16, rows of 128 B, 16-byte chunks XOR-swizzled by (row & 7)
  auto load_w = [&](int stage, int kb) {   // 128 rows x 8 chunks: 8 cp.async per thread
    unsigned char* wt = sm + stage * WG_STAGE;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + i * 128, r = idx >> 3, c = idx & 7;
      const int n = bn + r, k = kb * WG_BK + c * 8;
      const bool ok = (n < p.N) && (k < K);
      cp_async16(wt + r * 128 + ((c ^ (r & 7)) << 4), p.W + (size_t)(ok ? n : 0) * K + (ok ? k : 0), ok ? 16 : 0);
    }
  };
  auto load_a = [&](int stage, int kb) {   // 2 planes x 64 rows x 8 chunks: 8 cp.async per thread
    unsigned char* ah = sm + stage * WG_STAGE + WG_BM * 128;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + i * 128, pl = idx >> 9, r = (idx >> 3) & 63, c = idx & 7;
      const int m = bm + r, k = kb * WG_BK + c * 8;
      const bool ok = (m < p.M) && (k < K);
      const bf16* src = (pl ? a_lo : a_hi) + (size_t)(ok ? m : 0) * K + (ok ? k : 0);
      cp_async16(ah + pl * (WG_BN * 128) + r * 128 + ((c ^ (r & 7)) << 4), src, ok ? 16 : 0);
    }
  };
  float acc[2][32];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[h][i] = 0.f;

  pdl_trigger();
  load_w(0, 0);                                       // weights never depend on the predecessor grid
  if (nk > 1) load_w(1, 1);
  pdl_wait();
  load_a(0, 0);
  cp_async_commit();                                   // group 0 = W(0), W(1), A(0)
  if (nk > 1) load_a(1, 1);
  cp_async_commit();                                   // group 1 = A(1)
  for (int kb = 0; kb < nk; ++kb) {
    const int st = kb % WG_NST;
    cp_async_wait<1>();                                                 // this thread's copies of k-block kb have landed
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy smem writes -> visible to the tensor core (async proxy)
    __syncthreads();                                                    // ... and everyone's
    const unsigned wbase = smem_u32(sm + st * WG_STAGE);
    const unsigned long long dw = wgmma_desc_sw128(wbase), dh = wgmma_desc_sw128(wbase + WG_BM * 128),
                             dl = wgmma_desc_sw128(wbase + WG_BM * 128 + WG_BN * 128);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < WG_BK / 16; ++k) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        wgmma_m64n64(acc[h], dw + 512 * h + 2 * k, dh + 2 * k, 1);
        wgmma_m64n64(acc[h], dw + 512 * h + 2 * k, dl + 2 * k, 1);
      }
    }
    wgmma_commit();
    if (kb + 2 < nk) {
      wgmma_wait<1>();                     // this thread's MMAs of k-block kb-1 are done ...
      __syncthreads();                     // ... and every warp's: stage (kb+2)%3 == (kb-1)%3 may be refilled
      load_w((kb + 2) % WG_NST, kb + 2);
      load_a((kb + 2) % WG_NST, kb + 2);
    }
    cp_async_commit();
  }
  wgmma_wait<0>();
  // epilogue: rows of the fragment = weight rows n, columns = activation rows m
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n = bn + h * 64 + warp * 16 + (lane >> 2) + 8 * e;
      if (n >= p.N) continue;
      const float bias = p.bias ? p.bias[n] : 0.f;
#pragma unroll
      for (int j = 0; j < WG_BN / 8; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int m = bm + 8 * j + 2 * (lane & 3) + c;
          if (m < p.M) epi_store(p, m, n, acc[h][4 * j + 2 * e + c] + bias);
        }
    }
}

// thread-per-output small-K product with fp32 weights (encoder stem conv 1->32 k7, decoder head conv 32->1 k7)
__global__ void conv_naive_kernel(const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ x,
                                  RowMap xmap, float* __restrict__ y, int M, int N, int K) {
  pdl_trigger();
  pdl_wait();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)M * N) return;
  const int m = (int)(idx / N), n = (int)(idx % N);
  const float* xr = x + xmap.off(m);
  const float* wr = W + (size_t)n * K;
  float acc = bias ? bias[n] : 0.f;
  for (int k = 0; k < K; ++k) acc = fmaf(wr[k], xr[k], acc);
  y[idx] = acc;
}

// same product, one WARP per output: for long windows (decoder head conv: K = 7 x 32 = 224, N = 1) the thread-per-output loop is a
// 224-deep dependent FMA chain on 13 CTAs; here the lanes split K (coalesced 128 B reads of the window) and shuffle-reduce.
__global__ void __launch_bounds__(256) conv_warp_kernel(const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ x,
                                                        RowMap xmap, float* __restrict__ y, int M, int N, int K) {
  pdl_trigger();
  pdl_wait();
  const long long idx = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (idx >= (long long)M * N) return;
  const int m = (int)(idx / N), n = (int)(idx % N);
  const float* xr = x + xmap.off(m);
  const float* wr = W + (size_t)n * K;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) acc = fmaf(wr[k], xr[k], acc);
  acc = warp_sum(acc);
  if (lane == 0) y[idx] = acc + (bias ? bias[n] : 0.f);
}

// y[m,:] = rmsnorm(x[m,:]) * w   (one warp per row)
__global__ void rows_norm_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y,
                                 int M, int C, float eps) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (size_t)row * C;
  float ss = 0.f;
  for (int c = lane; c < C; c += 32) { float v = xr[c]; ss += v * v; }
  ss = warp_sum(ss);
  const float inv = rsqrtf(ss / (float)C + eps);
  for (int c = lane; c < C; c += 32) y[(size_t)row * C + c] = xr[c] * inv * (w ? w[c] : 1.f);
}

// ---------------------------------------------------------------------------------------------
// Streaming conv state.  win[b] = [hist[b] (ctx rows) ; f(src[b]) (T rows)], and the last ctx rows
// of the window are staged into hist_next[b]; `advance_kernel` commits hist_next -> hist for the
// rows that actually took this frame (a-8: VibeVoiceTokenizerStreamingCache, tokenizer.py:193-256).
// f = affine (alpha*x+beta) or RMSNorm*w.
// ---------------------------------------------------------------------------------------------
__global__ void assemble_window_kernel(const float* __restrict__ src, const float* __restrict__ hist,
                                       float* __restrict__ win, float* __restrict__ hist_next, int B, int T, int ctx, int C,
                                       const float* __restrict__ norm_w, float eps, float alpha, float beta) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int R = ctx + T;
  if (row >= B * R) return;
  const int b = row / R, j = row % R;
  float* wr = win + ((size_t)b * R + j) * C;
  float* hn = (j >= T) ? hist_next + ((size_t)b * ctx + (j - T)) * C : nullptr;
  if (j < ctx) {
    const float* hr = hist + ((size_t)b * ctx + j) * C;
    for (int c = lane; c < C; c += 32) { float v = hr[c]; wr[c] = v; if (hn) hn[c] = v; }
  } else {
    const float* sr = src + ((size_t)b * T + (j - ctx)) * C;
    float inv = 1.f;
    if (norm_w) {
      float ss = 0.f;
      for (int c = lane; c < C; c += 32) { float v = sr[c]; ss += v * v; }
      ss = warp_sum(ss);
      inv = rsqrtf(ss / (float)C + eps);
    }
    for (int c = lane; c < C; c += 32) {
      float v = norm_w ? sr[c] * inv * norm_w[c] : sr[c] * alpha + beta;
      wr[c] = v;
      if (hn) hn[c] = v;
    }
  }
}

// block-per-row variants for wide channels (C >= 512, few rows): the single-warp versions are a latency chain
__global__ void __launch_bounds__(256) assemble_window_block_kernel(const float* __restrict__ src, const float* __restrict__ hist,
                                                                    float* __restrict__ win, float* __restrict__ hist_next, int B, int T,
                                                                    int ctx, int C, const float* __restrict__ norm_w, float eps, float alpha,
                                                                    float beta) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x, tid = threadIdx.x;
  const int R = ctx + T;
  const int b = row / R, j = row % R;
  float* wr = win + ((size_t)b * R + j) * C;
  float* hn = (j >= T) ? hist_next + ((size_t)b * ctx + (j - T)) * C : nullptr;
  __shared__ float sp[8];
  if (j < ctx) {
    const float* hr = hist + ((size_t)b * ctx + j) * C;
    for (int c = tid; c < C; c += 256) { float v = hr[c]; wr[c] = v; if (hn) hn[c] = v; }
  } else {
    const float* sr = src + ((size_t)b * T + (j - ctx)) * C;
    float inv = 1.f;
    if (norm_w) {
      float ss = 0.f;
      for (int c = tid; c < C; c += 256) { float v = sr[c]; ss += v * v; }
      ss = warp_sum(ss);
      if ((tid & 31) == 0) sp[tid >> 5] = ss;
      __syncthreads();
      float t = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) t += sp[i];
      inv = rsqrtf(t / (float)C + eps);
    }
    for (int c = tid; c < C; c += 256) {
      float v = norm_w ? sr[c] * inv * norm_w[c] : sr[c] * alpha + beta;
      wr[c] = v;
      if (hn) hn[c] = v;
    }
  }
}
__global__ void __launch_bounds__(256) rows_norm_block_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y,
                                                              int C, float eps) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x, tid = threadIdx.x;
  const float* xr = x + (size_t)row * C;
  __shared__ float sp[8];
  float ss = 0.f;
  for (int c = tid; c < C; c += 256) { float v = xr[c]; ss += v * v; }
  ss = warp_sum(ss);
  if ((tid & 31) == 0) sp[tid >> 5] = ss;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) t += sp[i];
  const float inv = rsqrtf(t / (float)C + eps);
  for (int c = tid; c < C; c += 256) y[(size_t)row * C + c] = xr[c] * inv * (w ? w[c] : 1.f);
}

// out = x + gamma * (bias + sum_j w[j][c] * win[t+j][c])   (depthwise causal conv k=7 + layer scale + residual)
__global__ void dwconv_res_kernel(const float* __restrict__ x, const float* __restrict__ win, const float* __restrict__ w /*[7][C]*/,
                                  const float* __restrict__ bias, const float* __restrict__ gamma, float* __restrict__ out,
                                  int B, int T, int C) {
  pdl_trigger();
  pdl_wait();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * T * C) return;
  const int c = (int)(idx % C);
  const long long bt = idx / C;
  const int t = (int)(bt % T), b = (int)(bt / T);
  const float* wp = win + ((size_t)b * (T + 6) + t) * C + c;
  float acc = bias[c];
#pragma unroll
  for (int j = 0; j < 7; ++j) acc = fmaf(w[j * C + c], wp[(size_t)j * C], acc);
  out[idx] = x[idx] + gamma[c] * acc;
}

struct StateSeg { float* hist; float* next; int n; };   // n floats per batch row

constexpr int ADV_SLICES = 8;     // CTAs per (segment, batch row): the widest histories (6 x 2048 floats) are a latency chain for one CTA
__global__ void advance_kernel(const StateSeg* __restrict__ segs, const int* __restrict__ active) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.y;
  if (active && !active[b]) return;
  const StateSeg s = segs[blockIdx.x];
  float* d = s.hist + (size_t)b * s.n;
  const float* a = s.next + (size_t)b * s.n;
  for (int i = blockIdx.z * blockDim.x + threadIdx.x; i < s.n; i += gridDim.z * blockDim.x) d[i] = a[i];
}

// ---------------------------------------------------------------------------------------------
// LLM decode step pieces
// ---------------------------------------------------------------------------------------------
constexpr int KV_PAGE = 64;     // tokens per page
constexpr int HD = 128;         // head_dim of both shipped models (configs/*.json)

struct KvView {
  bf16* kpool; bf16* vpool;     // this layer: [n_pages][kv_heads][KV_PAGE][HD]
  const int* page_table;        // [n_seq][max_pages]
  int max_pages;
  const int* kv_len;            // [n_seq] committed length
  const int* row_mode;          // [n_seq] 0 skip / 1 run
  int kv_heads, q_heads;
};

constexpr int ATT_MAXG = 8;     // q heads per kv head (6 for 1.5B, 7 for 7B)
constexpr int AT2_LD = HD + 8;  // row stride (bf16) of the stream kernel's attention Q tile: +8 = 16 B pad, ldmatrix conflict-free
VV_DEVINL void ldmatrix_x4_trans(unsigned (&r)[4], const void* smem) {
  unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(sa));
}

// logits over the valid ids + constrained argmax (VibeVoiceTokenConstraintProcessor + argmax, :53-66, :498)
__global__ void __launch_bounds__(256) lm_head_argmax_kernel(const float* __restrict__ hidden, const bf16* __restrict__ w_valid,
                                                             const int* __restrict__ valid_ids, int n_valid, int H,
                                                             float* __restrict__ logits, int* __restrict__ tokens) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ float red[8][8];
  float acc[8];
#pragma unroll
  for (int v = 0; v < 8; ++v) acc[v] = 0.f;
  const float* hr = hidden + (size_t)b * H;
  for (int k = tid; k < H; k += 256) {
    const float x = hr[k];
#pragma unroll
    for (int v = 0; v < 8; ++v) if (v < n_valid) acc[v] = fmaf(__bfloat162float(w_valid[(size_t)v * H + k]), x, acc[v]);
  }
#pragma unroll
  for (int v = 0; v < 8; ++v) { acc[v] = warp_sum(acc[v]); if (lane == 0) red[warp][v] = acc[v]; }
  __syncthreads();
  if (tid == 0) {
    int best = 0; float bv = -INFINITY;
    for (int v = 0; v < n_valid; ++v) {
      float t = 0.f;
      for (int w = 0; w < 8; ++w) t += red[w][v];
      logits[(size_t)b * n_valid + v] = t;
      if (t > bv) { bv = t; best = v; }     // strict > : lowest id wins ties (valid_ids ascending)
    }
    tokens[b] = valid_ids[best];
  }
}

// ---------------------------------------------------------------------------------------------
// diffusion sampler glue
// ---------------------------------------------------------------------------------------------
// c_all[i][r][:] = silu(condp[r][:] + temb[i][:])   for all steps i (sample-independent t-embedding)
__global__ void head_cond_prep_kernel(const float* __restrict__ condp, const float* __restrict__ temb, float* __restrict__ c_all,
                                      int n_steps, int R, int H) {
  pdl_trigger();
  pdl_wait();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)n_steps * R * H) return;
  const int k = (int)(idx % H);
  const int r = (int)((idx / H) % R);
  const int i = (int)(idx / ((long long)H * R));
  c_all[idx] = silu_f(condp[(size_t)r * H + k] + temb[(size_t)i * H + k]);
}

// one DPM-Solver++ step (update formula at SDpm, vv_stream.cuh); kn: per-step noise gain (sde-dpmsolver++), 0 for the ODE solver
struct DpmCoef { float a0, s0, ks, kx, rinv; int order; float kn; };

// embeds[b] = active[b] ? e_new[b] : embeds[b];  embeds[B+b] = embeds[b]  (negative stream is fed the same input, :579-581)
__global__ void select_embeds_kernel(float* __restrict__ embeds, const float* __restrict__ e_new, const int* __restrict__ active,
                                     int B, int H) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.x;
  const bool a = active[b] != 0;
  for (int k = threadIdx.x; k < H; k += blockDim.x) {
    const float v = a ? e_new[(size_t)b * H + k] : embeds[(size_t)b * H + k];
    embeds[(size_t)b * H + k] = v;
    embeds[(size_t)(B + b) * H + k] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// load-time repack kernels (run once in vv_finalize_weights)
// ---------------------------------------------------------------------------------------------
__global__ void cvt_f32_to_bf16_kernel(const float* __restrict__ s, bf16* __restrict__ d, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) d[i] = __float2bfloat16_rn(s[i]);
}
__global__ void cvt_f16_to_bf16_kernel(const __half* __restrict__ s, bf16* __restrict__ d, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) d[i] = __float2bfloat16_rn(__half2float(s[i]));
}
__global__ void cvt_bf16_to_f32_kernel(const bf16* __restrict__ s, float* __restrict__ d, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) d[i] = __bfloat162float(s[i]);
}
__global__ void cvt_f16_to_f32_kernel(const __half* __restrict__ s, float* __restrict__ d, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) d[i] = __half2float(s[i]);
}
// out[2j] = a[j], out[2j+1] = b[j]   (rows of length K)
__global__ void interleave_rows_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, bf16* __restrict__ out, size_t rows, size_t K) {
  const size_t n = rows * K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / K, k = i % K;
    out[(2 * r) * K + k] = a[i];
    out[(2 * r + 1) * K + k] = b[i];
  }
}
// Conv1d weight [Co][Ci][k] -> window-GEMV form [Co][j*Ci + ci]
__global__ void repack_conv_kernel(const bf16* __restrict__ w, bf16* __restrict__ out, int Co, int Ci, int k) {
  const size_t n = (size_t)Co * Ci * k;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int j = (int)(i % k); const int ci = (int)((i / k) % Ci); const size_t co = i / ((size_t)k * Ci);
    out[co * ((size_t)k * Ci) + (size_t)j * Ci + ci] = w[i];
  }
}
// ConvTranspose1d weight [Ci][Co][k=2s] -> [(j*Co + co)][half*Ci + ci], half 0 = previous frame (tap j+s), half 1 = current frame (tap j)
__global__ void repack_convtr_kernel(const bf16* __restrict__ w, bf16* __restrict__ out, int Ci, int Co, int s) {
  const int k = 2 * s;
  const size_t n = (size_t)Ci * Co * k;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int tap = (int)(i % k); const int co = (int)((i / k) % Co); const int ci = (int)(i / ((size_t)k * Co));
    const int j = tap % s, half = (tap >= s) ? 0 : 1;
    out[((size_t)j * Co + co) * (2 * (size_t)Ci) + (size_t)half * Ci + ci] = w[i];
  }
}
// depthwise [C][1][7] fp32 -> [7][C];  generic small conv [Co][Ci][k] fp32 -> [Co][j*Ci+ci]
__global__ void repack_dw_kernel(const float* __restrict__ w, float* __restrict__ out, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < C * 7) { const int c = i / 7, j = i % 7; out[j * C + c] = w[i]; }
}
__global__ void repack_conv_f32_kernel(const float* __restrict__ w, float* __restrict__ out, int Co, int Ci, int k) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Co * Ci * k) { const int j = i % k, ci = (i / k) % Ci, co = i / (k * Ci); out[co * (k * Ci) + j * Ci + ci] = w[i]; }
}
__global__ void tile_bias_kernel(const float* __restrict__ b, float* __restrict__ out, int Co, int s) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Co * s) out[i] = b[i % Co];
}
__global__ void gather_rows_kernel(const bf16* __restrict__ table, const int* __restrict__ ids, bf16* __restrict__ out, int H) {
  const bf16* r = table + (size_t)ids[blockIdx.x] * H;
  for (int k = threadIdx.x; k < H; k += blockDim.x) out[(size_t)blockIdx.x * H + k] = r[k];
}
// sinusoidal timestep features (diffusion_head.py:66-88): [n_steps][256] = [cos(t f_j) | sin(t f_j)]
__global__ void timestep_feat_kernel(const float* __restrict__ t, const float* __restrict__ freqs /*[128]*/, float* __restrict__ out, int n_steps) {
  const int i = blockIdx.x, j = threadIdx.x;   // 256 threads
  if (i >= n_steps) return;
  const float a = t[i] * freqs[j & 127];
  out[i * 256 + j] = (j < 128) ? cosf(a) : sinf(a);
}
// KV hand-off from a prefill: src [n_tokens][kv_heads][HD] bf16 -> pages
__global__ void kv_write_kernel(const bf16* __restrict__ k, const bf16* __restrict__ v, bf16* __restrict__ kpool, bf16* __restrict__ vpool,
                                const int* __restrict__ page_row, int kv_heads, int hd, long long pos0, long long n_tokens) {
  const long long t = blockIdx.x;
  if (t >= n_tokens) return;
  const long long pos = pos0 + t;
  const int page = page_row[pos / KV_PAGE];
  const int slot = (int)(pos % KV_PAGE);
  for (int i = threadIdx.x; i < kv_heads * hd; i += blockDim.x) {
    const int h = i / hd, d = i % hd;
    const size_t o = (((size_t)page * kv_heads + h) * KV_PAGE + slot) * hd + d;
    kpool[o] = k[(size_t)t * kv_heads * hd + i];
    vpool[o] = v[(size_t)t * kv_heads * hd + i];
  }
}

}  // namespace vv
