// vv_prefill.cuh -- native LM prompt prefill (SURVEY f-2): the decoder stack over thousands of prompt tokens of ONE sequence.
//
// The per-frame kernels stream weights at M <= 16 rows; the prompt is the opposite case (M = thousands of rows, tensor-core bound), so it
// gets its own kernels, driven by vv_lm_prefill in vv_runtime.cu:
//   pf_rmsnorm_kernel   RMSNorm of the fp32 residual rows -> bf16 GEMM operand (Qwen2RMSNorm, modeling_qwen2.py:249-266)
//   pf_gemm_kernel      wgmma GEMM, bf16 activations x the engine's packed bf16 weights, fp32 accumulators, fused epilogues:
//                         QKV   bias -> RoPE -> K/V rounded to bf16 straight into the paged pool, bf16 Q
//                         RESID fp32 residual add (O and down projections)
//                         SWIGLU silu(gate) * up of the row-interleaved gate/up weight -> bf16 operand of the down projection
//   pf_attn_kernel      causal flash attention over the paged pool (online softmax, fp32 statistics, bf16 P), GQA, head_dim 64 / 128
// Numerics: transformers Qwen2DecoderLayer (modeling_qwen2.py:116-174, 203-245) with bf16 GEMM operands, a bf16 KV cache and bf16 Q / P --
// oracle.vv_oracle.qwen2_forward(act_bf16=True) with kv_bf16 up to summation order.  No split-K, and every query walks its keys in page
// order whatever rows share its CTA, so results do not depend on how the tokens are chunked.
#pragma once
#include "vv_kernels.cuh"

namespace vv {

// ---------------------------------------------------------------------------------------------
// RMSNorm rows: x fp32 [M][H] -> out bf16 [M][H] = bf16(x * rsqrt(mean(x^2) + eps) * w); one warp per row
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pf_rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w, float eps, int M, int H,
                                                         bf16* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (size_t)row * H;
  float ss = 0.f;
  for (int k = lane * 4; k < H; k += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + k);
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  ss = warp_sum(ss);
  const float inv = rsqrtf(ss / (float)H + eps);
  bf16* o = out + (size_t)row * H;
  for (int k = lane * 4; k < H; k += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + k);
    const float4 g = *reinterpret_cast<const float4*>(w + k);
    *reinterpret_cast<uint2*>(o + k) = make_uint2(pack_bf16(v.x * inv * g.x, v.y * inv * g.y), pack_bf16(v.z * inv * g.z, v.w * inv * g.w));
  }
}

// ---------------------------------------------------------------------------------------------
// GEMM: C[M x N] = A[M x K] * W[N x K]^T, A bf16 activations (dense rows of K), W the packed bf16 weight (row-major [N][K]).
//   * CTA tile 128 activation rows x 128 weight rows; two warpgroups, each wgmma.mma_async m64n128k16 over its 64 rows (activations are
//     the MMA M side, so output features run along the fragment columns and a gate/up pair of the interleaved weight sits in one thread);
//   * both operands K-major in shared memory with the 128-byte swizzle, filled by cp.async through a 4-stage ring (three k-blocks ahead);
//   * epilogue straight from the accumulator fragments.  Every output element is one chain of k-block MMAs: no split-K.
// ---------------------------------------------------------------------------------------------
constexpr int PF_BM = 128, PF_BN = 128, PF_BK = 64, PF_NST = 4;
constexpr int PF_STAGE = PF_BM * 128 + PF_BN * 128;                    // A 16 KB + W 16 KB
constexpr int PF_SMEM = PF_NST * PF_STAGE + 1024;
enum { PF_EPI_QKV = 0, PF_EPI_RESID = 1, PF_EPI_SWIGLU = 2 };

struct PfGemm {
  const bf16* A;                // [M][K]
  const bf16* W;                // [N][K]
  int M, N, K;
  const float* bias;            // QKV: [N]
  float* x; int ldx;            // RESID: x[m][n] += C
  bf16* out; int ldo;           // QKV: Q [M][nq]; SWIGLU: [M][N/2]
  // QKV: K/V rows of positions pos_base + m go to the paged pool of this layer ([n_pages][kv_heads][KV_PAGE][hd])
  bf16* kpool; bf16* vpool; const int* page_row;
  int nq, kv_heads;             // q features; kv heads (head_dim is the kernel's template argument)
  long long pos_base;
  const float* inv_freq;        // [hd/2]
};

// D[64 x 128] += A[64 x 16] * B[128 x 16]^T, both K-major in shared memory (fragment layout as wgmma_m64n16, columns 0..127)
VV_DEVINL void wgmma_m64n128(float (&d)[64], unsigned long long a, unsigned long long b) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(a), "l"(b), "r"(1) : "memory");
}

template <int EPI, int HD_ = 128>      // HD_: head_dim, used by the QKV epilogue only
__global__ void __launch_bounds__(256) pf_gemm_kernel(PfGemm p) {
  extern __shared__ unsigned char pf_raw[];
  const unsigned raw_addr = smem_u32(pf_raw);
  unsigned char* sm = pf_raw + ((1024u - (raw_addr & 1023u)) & 1023u);      // 1024 B aligned (swizzle atom)
  const int tid = threadIdx.x, lane = tid & 31, warp = (tid >> 5) & 3, wg = tid >> 7;
  const int bn = blockIdx.x * PF_BN;       // weight rows (output features)
  const int bm = blockIdx.y * PF_BM;       // activation rows
  const int K = p.K, nk = K / PF_BK;        // K % 64 == 0 (checked by the host)

  auto load_w = [&](int stage, int kb) {   // 128 rows x 8 16-byte chunks: 4 per thread
    unsigned char* wt = sm + stage * PF_STAGE + PF_BM * 128;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + i * 256, r = idx >> 3, c = idx & 7;
      const int n = bn + r;
      const bool ok = n < p.N;
      cp_async16(wt + r * 128 + ((c ^ (r & 7)) << 4), p.W + (size_t)(ok ? n : 0) * K + kb * PF_BK + c * 8, ok ? 16 : 0);
    }
  };
  auto load_a = [&](int stage, int kb) {
    unsigned char* at = sm + stage * PF_STAGE;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + i * 256, r = idx >> 3, c = idx & 7;
      const int m = bm + r;
      const bool ok = m < p.M;
      cp_async16(at + r * 128 + ((c ^ (r & 7)) << 4), p.A + (size_t)(ok ? m : 0) * K + kb * PF_BK + c * 8, ok ? 16 : 0);
    }
  };
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;

  pdl_trigger();
#pragma unroll
  for (int s = 0; s < PF_NST - 1; ++s)
    if (s < nk) load_w(s, s);                                          // weights never depend on the predecessor grid
  pdl_wait();
#pragma unroll
  for (int s = 0; s < PF_NST - 1; ++s) {
    if (s < nk) load_a(s, s);
    cp_async_commit();                                                 // group s (group 0 also holds the early weight tiles)
  }
  for (int kb = 0; kb < nk; ++kb) {
    const int st = kb % PF_NST;
    cp_async_wait<PF_NST - 2>();                                       // this thread's copies of k-block kb have landed
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy smem writes -> visible to the tensor core
    __syncthreads();                                                   // ... and everyone's
    const unsigned base = smem_u32(sm + st * PF_STAGE);
    const unsigned long long da = wgmma_desc_sw128(base + wg * 64 * 128), dw = wgmma_desc_sw128(base + PF_BM * 128);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < PF_BK / 16; ++k) wgmma_m64n128(acc, da + 2 * k, dw + 2 * k);
    wgmma_commit();
    wgmma_wait<1>();                                                   // k-block kb-1 is done in this warpgroup ...
    __syncthreads();                                                   // ... and in the other: its stage may be refilled
    if (kb + PF_NST - 1 < nk) {
      load_w((kb + PF_NST - 1) % PF_NST, kb + PF_NST - 1);
      load_a((kb + PF_NST - 1) % PF_NST, kb + PF_NST - 1);
    }
    cp_async_commit();
  }
  wgmma_wait<0>();

  // fragment register i: activation row 16 warp + lane/4 + 8 ((i >> 1) & 1), feature column 8 (i >> 2) + 2 (lane & 3) + (i & 1)
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int m = bm + wg * 64 + warp * 16 + (lane >> 2) + 8 * e;
    if (m >= p.M) continue;
    if (EPI == PF_EPI_RESID) {
      float* xr = p.x + (size_t)m * p.ldx;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int n = bn + 8 * j + 2 * (lane & 3);
        if (n >= p.N) continue;
        float2 v = *reinterpret_cast<float2*>(xr + n);
        v.x += acc[4 * j + 2 * e];
        v.y += acc[4 * j + 2 * e + 1];
        *reinterpret_cast<float2*>(xr + n) = v;
      }
    } else if (EPI == PF_EPI_SWIGLU) {
      bf16* o = p.out + (size_t)m * p.ldo;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int n = bn + 8 * j + 2 * (lane & 3);                    // even: gate row n/2, odd: up row n/2
        if (n >= p.N) continue;
        const float g = acc[4 * j + 2 * e], u = acc[4 * j + 2 * e + 1];
        o[n >> 1] = __float2bfloat16_rn(g / (1.0f + expf(-g)) * u);
      }
    } else {
      // QKV: heads are hd-aligned and tiles 128-aligned, so dims d and d + hd/2 of a head are registers j and j + hd/16 of this thread
      const long long pos = p.pos_base + m;
      constexpr int hd = HD_, half = HD_ / 2;
      const int nkvd = p.kv_heads * hd;
      const int page = p.page_row[pos / KV_PAGE], slot = (int)(pos % KV_PAGE);
      float v[16][2];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int n = bn + 8 * j + 2 * (lane & 3);
        const bool ok = n < p.N;
        v[j][0] = acc[4 * j + 2 * e] + (ok ? p.bias[n] : 0.f);
        v[j][1] = acc[4 * j + 2 * e + 1] + (ok ? p.bias[n + 1] : 0.f);
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int n = bn + 8 * j + 2 * (lane & 3);
        if (n >= p.N) continue;
        const int d = (8 * j) % hd + 2 * (lane & 3);                   // bn is a multiple of 128, hence of hd
        if (n < p.nq + nkvd) {                                         // q or k: rotate the (d, d + hd/2) pairs from the first half
          if ((8 * j) % hd >= half) continue;
          constexpr int JP = HD_ / 16;                                 // partner register offset: dims d + hd/2 (same head, same tile)
          const int jp = j + JP;
          float o1[2], o2[2];
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            float sn, cs;
            sincosf((float)pos * p.inv_freq[d + c], &sn, &cs);
            const float x1 = v[j][c], x2 = v[jp][c];
            o1[c] = x1 * cs - x2 * sn;
            o2[c] = x2 * cs + x1 * sn;
          }
          const unsigned lo = pack_bf16(o1[0], o1[1]), hi = pack_bf16(o2[0], o2[1]);
          if (n < p.nq) {
            bf16* q = p.out + (size_t)m * p.ldo + (n - d);
            *reinterpret_cast<unsigned*>(q + d) = lo;
            *reinterpret_cast<unsigned*>(q + d + half) = hi;
          } else {
            const int h = (n - p.nq) / hd;
            bf16* kr = p.kpool + (((size_t)page * p.kv_heads + h) * KV_PAGE + slot) * hd;
            *reinterpret_cast<unsigned*>(kr + d) = lo;
            *reinterpret_cast<unsigned*>(kr + d + half) = hi;
          }
        } else {
          const int h = (n - p.nq - nkvd) / hd;
          bf16* vr = p.vpool + (((size_t)page * p.kv_heads + h) * KV_PAGE + slot) * hd;
          *reinterpret_cast<unsigned*>(vr + d) = pack_bf16(v[j][0], v[j][1]);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Causal flash attention of one 64-row query tile and one query head over the paged pool of the sequence (CTA = 4 warps x 16 rows).
// Key tiles are pages: tile t holds positions [64 t, 64 t + 64), read K/V [64][hd] contiguous per kv head, double-buffered with cp.async.
// S = Q K^T with mma.sync m16n8k16 (bf16 Q, bf16 K), online softmax in fp32 (exp2 of log2e-scaled scores), O += bf16(P) V.  A query walks
// tiles 0, 1, ... in order; a tile that is entirely in a query's future is an exact no-op for it (scale 1, weight 0), so the result of a
// row does not depend on which rows share its CTA.
// ---------------------------------------------------------------------------------------------
template <int HD_>
struct PfAttnCfg {
  static constexpr int LD = HD_ + 8;                                   // +16 B row pad: ldmatrix conflict-free
  static constexpr int SMEM = 5 * 64 * LD * 2;                         // Q + 2 x K + 2 x V
};

template <int HD_>
__global__ void __launch_bounds__(128) pf_attn_kernel(const bf16* __restrict__ q, int M, int q_heads, int kv_heads, const bf16* __restrict__ kpool,
                                                      const bf16* __restrict__ vpool, const int* __restrict__ page_row, long long pos_base,
                                                      float scale_log2, bf16* __restrict__ out) {
  constexpr int LD = PfAttnCfg<HD_>::LD, NT = HD_ / 8, KS = HD_ / 16, CH = HD_ / 8;   // CH: 16-byte chunks per row
  extern __shared__ __align__(16) unsigned char pa_smem[];
  bf16 (*Qs)[LD] = reinterpret_cast<bf16 (*)[LD]>(pa_smem);
  bf16 (*Ks)[64][LD] = reinterpret_cast<bf16 (*)[64][LD]>(pa_smem + 64 * LD * 2);
  bf16 (*Vs)[64][LD] = reinterpret_cast<bf16 (*)[64][LD]>(pa_smem + 3 * 64 * LD * 2);
  pdl_trigger();
  const int qt = gridDim.x - 1 - blockIdx.x;                          // longest (latest) query tiles first
  const int h = blockIdx.y, g = h / (q_heads / kv_heads);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int m0 = qt * 64;
  const int ldq = q_heads * HD_;
  const long long kv_end = pos_base + M;                               // keys at or beyond it are not written yet
  const long long last_pos = pos_base + min(m0 + 63, M - 1);
  const int n_tiles = (int)(last_pos / 64) + 1;
  const long long warp_lo = pos_base + m0 + warp * 16, warp_hi = warp_lo + 15;
  pdl_wait();

  for (int i = tid; i < 64 * CH; i += 128) {
    const int r = i / CH, c = (i % CH) * 8;
    const bool ok = m0 + r < M;
    cp_async16(&Qs[r][c], q + (size_t)(ok ? m0 + r : 0) * ldq + h * HD_ + c, ok ? 16 : 0);
  }
  auto prefetch = [&](int t, int buf) {
    const size_t base = ((size_t)page_row[t] * kv_heads + g) * KV_PAGE * HD_;
    for (int i = tid; i < 64 * CH; i += 128) {
      const int r = i / CH, c = (i % CH) * 8;
      const int nb = ((long long)t * 64 + r < kv_end) ? 16 : 0;
      cp_async16(&Ks[buf][r][c], kpool + base + (size_t)r * HD_ + c, nb);
      cp_async16(&Vs[buf][r][c], vpool + base + (size_t)r * HD_ + c, nb);
    }
  };
  prefetch(0, 0);
  cp_async_commit();

  unsigned qa[KS][4];
  float o[NT][4];
#pragma unroll
  for (int i = 0; i < NT; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const long long p0 = warp_lo + (lane >> 2), p1 = p0 + 8;           // this thread's two query positions

  for (int t = 0; t < n_tiles; ++t) {
    const int buf = t & 1;
    if (t + 1 < n_tiles) prefetch(t + 1, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    if (t == 0) {
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) ldmatrix_x4(qa[ks], &Qs[warp * 16 + (lane & 15)][ks * 16 + (lane >> 4) * 8]);
    }
    const long long k0 = (long long)t * 64;
    if (k0 <= warp_hi) {                                               // else every key of the tile is in this warp's future
      float s[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < KS; ++ks)
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {
          unsigned kb[4];
          ldmatrix_x4(kb, &Ks[buf][jp * 16 + (lane & 7) + ((lane >> 4) << 3)][ks * 16 + ((lane >> 3) & 1) * 8]);
          mma_bf16_16816(s[2 * jp], qa[ks], kb[0], kb[1]);
          mma_bf16_16816(s[2 * jp + 1], qa[ks], kb[2], kb[3]);
        }
      const bool diag = k0 + 63 > warp_lo;
      float mt[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float v = s[j][c] * scale_log2;
          if (diag) {
            const long long kp = k0 + j * 8 + 2 * (lane & 3) + (c & 1);
            if (kp > ((c & 2) ? p1 : p0)) v = -INFINITY;
          }
          s[j][c] = v;
          mt[c >> 1] = fmaxf(mt[c >> 1], v);
        }
      float corr[2], msafe[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mt[r] = fmaxf(mt[r], __shfl_xor_sync(0xffffffffu, mt[r], 1));
        mt[r] = fmaxf(mt[r], __shfl_xor_sync(0xffffffffu, mt[r], 2));
        const float mn = fmaxf(m_run[r], mt[r]);
        msafe[r] = (mn == -INFINITY) ? 0.f : mn;
        corr[r] = exp2f(m_run[r] - msafe[r]);
        m_run[r] = mn;
        l_run[r] *= corr[r];
      }
#pragma unroll
      for (int i = 0; i < NT; ++i) { o[i][0] *= corr[0]; o[i][1] *= corr[0]; o[i][2] *= corr[1]; o[i][3] *= corr[1]; }
      unsigned pa[4][4];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float e0 = exp2f(s[j][0] - msafe[0]), e1 = exp2f(s[j][1] - msafe[0]);
        const float e2 = exp2f(s[j][2] - msafe[1]), e3 = exp2f(s[j][3] - msafe[1]);
        l_run[0] += e0 + e1;
        l_run[1] += e2 + e3;
        pa[j >> 1][(j & 1) * 2] = pack_bf16(e0, e1);
        pa[j >> 1][(j & 1) * 2 + 1] = pack_bf16(e2, e3);
      }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int np = 0; np < HD_ / 16; ++np) {
          unsigned vb[4];
          ldmatrix_x4_trans(vb, &Vs[buf][kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8][np * 16 + (lane >> 4) * 8]);
          mma_bf16_16816(o[2 * np], pa[kk], vb[0], vb[1]);
          mma_bf16_16816(o[2 * np + 1], pa[kk], vb[2], vb[3]);
        }
    }
    __syncthreads();
  }
  cp_async_wait<0>();
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const int r0 = m0 + warp * 16 + (lane >> 2);
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int m = r0 + 8 * e;
    if (m >= M) continue;
    const float inv = 1.f / l_run[e];
    bf16* orow = out + (size_t)m * ldq + h * HD_;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
      *reinterpret_cast<unsigned*>(orow + nt * 8 + 2 * (lane & 3)) = pack_bf16(o[nt][2 * e] * inv, o[nt][2 * e + 1] * inv);
  }
}

// embedding rows of device token ids: out[r] = fp32(table[ids[r]]); ids outside [0, vocab) give zero rows instead of reading out of bounds
__global__ void pf_embed_gather_kernel(const bf16* __restrict__ table, const int* __restrict__ ids, long long n, int vocab, int H,
                                       float* __restrict__ out) {
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    const int id = ids[r];
    const bool ok = id >= 0 && id < vocab;
    for (int k = threadIdx.x; k < H; k += blockDim.x) out[r * H + k] = ok ? __bfloat162float(table[(size_t)id * H + k]) : 0.f;
  }
}

// the inverse of kv_write_kernel: pages of one sequence / layer -> [n][kv_heads][hd] bf16
__global__ void pf_kv_read_kernel(const bf16* __restrict__ kpool, const bf16* __restrict__ vpool, const int* __restrict__ page_row, int kv_heads,
                                  int hd, long long pos0, long long n, bf16* __restrict__ k, bf16* __restrict__ v) {
  for (long long t = blockIdx.x; t < n; t += gridDim.x) {
    const long long pos = pos0 + t;
    const int page = page_row[pos / KV_PAGE], slot = (int)(pos % KV_PAGE);
    for (int i = threadIdx.x; i < kv_heads * hd; i += blockDim.x) {
      const int hh = i / hd, d = i % hd;
      const size_t src = (((size_t)page * kv_heads + hh) * KV_PAGE + slot) * hd + d;
      if (k) k[t * kv_heads * hd + i] = kpool[src];
      if (v) v[t * kv_heads * hd + i] = vpool[src];
    }
  }
}

}  // namespace vv
