// vv_voice.cuh -- non-streaming acoustic tokenizer encoder for voice prompts (a-9): the elementwise / row kernels around the wgmma
// GEMM (gemm_wgmma_kernel), which runs every convolution, FFN linear and connector linear of the encoder.
//
// Reference anchors (under vibevoice/modular of the reference project):
//   padding of every conv       modular_vibevoice_tokenizer.py:327-382 (SConv1d, non-streaming: pad_total = k - s on the left, stride
//                               alignment zeros on the right)
//   Block1D                     modular_vibevoice_tokenizer.py:620-684
//   encoder                     modular_vibevoice_tokenizer.py:384-418, 776-813
//   sampling                    modular_vibevoice_tokenizer.py:966-991, modeling_vibevoice_inference.py:149-163
//
// Activations are time-major [voice][t][C] fp32.  Every GEMM operand is a pair of dense bf16 planes hi + lo (x = hi + lo), as
// split_bf16_kernel makes them; the kernels below write those planes straight from the windowed / normalised / sampled rows, so no
// padded or normalised fp32 copy of an activation is ever stored.  Element offsets are 64-bit throughout.
#pragma once
#include "vv_kernels.cuh"

namespace vv {

VV_DEVINL void store_split4(bf16* __restrict__ hi, bf16* __restrict__ lo, long long off, float a, float b, float c, float d) {
  const float h0 = __bfloat162float(__float2bfloat16_rn(a)), h1 = __bfloat162float(__float2bfloat16_rn(b));
  const float h2 = __bfloat162float(__float2bfloat16_rn(c)), h3 = __bfloat162float(__float2bfloat16_rn(d));
  *reinterpret_cast<uint2*>(hi + off) = make_uint2(pack_bf16(h0, h1), pack_bf16(h2, h3));
  *reinterpret_cast<uint2*>(lo + off) = make_uint2(pack_bf16(a - h0, b - h1), pack_bf16(c - h2, d - h3));
}

// Window operand of a causal strided conv as planes [M][Kp]: output row m0 + r (voice v = row / T_out, frame t = row % T_out) reads input
// rows t*stride - pad + j, j < k, of voice v; element kk = j*Cin + ci (the tap-major weight layout).  Rows outside [0, T_in) and the
// padding columns kk >= k*Cin read as zero.  Kp % 4 == 0.
__global__ void __launch_bounds__(256) voice_window_split_kernel(const float* __restrict__ x, int T_in, int T_out, int Cin, int stride,
                                                                 int pad, int Kreal, int Kp, long long m0, int M, bf16* __restrict__ hi,
                                                                 bf16* __restrict__ lo) {
  pdl_trigger();
  pdl_wait();
  const int K4 = Kp >> 2;
  const long long n4 = (long long)M * K4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / K4;
    const int kk = (int)(i - r * K4) << 2;
    const long long row = m0 + r;
    const long long v = row / T_out;
    const int t = (int)(row - v * T_out);
    const float* xv = x + v * T_in * (long long)Cin;
    float e[4];
    if ((Cin & 3) == 0) {               // the 4 elements share one input row
      const int j = kk / Cin, ci = kk - j * Cin, ti = t * stride - pad + j;
      if (kk < Kreal && ti >= 0 && ti < T_in) {
        const float4 q = *reinterpret_cast<const float4*>(xv + (long long)ti * Cin + ci);
        e[0] = q.x; e[1] = q.y; e[2] = q.z; e[3] = q.w;
      } else {
        e[0] = e[1] = e[2] = e[3] = 0.f;
      }
    } else {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int k = kk + u, j = k / Cin, ci = k - j * Cin, ti = t * stride - pad + j;
        e[u] = (k < Kreal && ti >= 0 && ti < T_in) ? xv[(long long)ti * Cin + ci] : 0.f;
      }
    }
    store_split4(hi, lo, r * Kp + kk, e[0], e[1], e[2], e[3]);
  }
}

// planes [M][C] of RMSNorm(x[m]) * w (one warp per row, C % 4 == 0); x rows are C floats apart
__global__ void __launch_bounds__(256) voice_norm_split_kernel(const float* __restrict__ x, const float* __restrict__ w, float eps, int M, int C,
                                                               bf16* __restrict__ hi, bf16* __restrict__ lo) {
  pdl_trigger();
  pdl_wait();
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const float4* xr = reinterpret_cast<const float4*>(x + row * C);
  const int C4 = C >> 2;
  float ss = 0.f;
  for (int c = lane; c < C4; c += 32) { const float4 q = xr[c]; ss += q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w; }
  ss = warp_sum(ss);
  const float inv = rsqrtf(ss / (float)C + eps);
  for (int c = lane; c < C4; c += 32) {
    const float4 q = xr[c];
    const float4 g = reinterpret_cast<const float4*>(w)[c];
    store_split4(hi, lo, row * C + 4 * c, q.x * inv * g.x, q.y * inv * g.y, q.z * inv * g.z, q.w * inv * g.w);
  }
}

// inv[m] = 1 / sqrt(mean(x[m]^2) + eps) (one warp per row)
__global__ void __launch_bounds__(256) voice_rms_kernel(const float* __restrict__ x, long long M, int C, float eps, float* __restrict__ inv) {
  pdl_trigger();
  pdl_wait();
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const float4* xr = reinterpret_cast<const float4*>(x + row * C);
  float ss = 0.f;
  for (int c = lane; c < (C >> 2); c += 32) { const float4 q = xr[c]; ss += q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w; }
  ss = warp_sum(ss);
  if (lane == 0) inv[row] = rsqrtf(ss / (float)C + eps);
}

// Block1D mixer half: out = x + gamma * (bias + sum_j w[j] * n[t - 6 + j]) with n = RMSNorm(x) * norm_w and n[t < 0] = 0 (causal
// depthwise k = 7, per voice of T rows).  `out` must not alias `x`.
__global__ void __launch_bounds__(256) voice_dwconv_kernel(const float* __restrict__ x, const float* __restrict__ inv, const float* __restrict__ norm_w,
                                                           const float* __restrict__ w /*[7][C]*/, const float* __restrict__ bias,
                                                           const float* __restrict__ gamma, float* __restrict__ out, long long rows, int T, int C) {
  pdl_trigger();
  pdl_wait();
  const long long n = rows * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / C;
    const int c = (int)(i - row * C);
    const int t = (int)(row % T);
    float acc = bias[c];
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      const int d = 6 - j;
      if (t >= d) acc = fmaf(w[j * C + c], x[i - (long long)d * C] * inv[row - d] * norm_w[c], acc);
    }
    out[i] = x[i] + gamma[c] * acc;
  }
}

// connector operand: planes [M][D] of (mean + sigma[v] * eps + bias) * scale for rows m0 .. m0 + M (voice v = row / F); eps == null: no noise
__global__ void __launch_bounds__(256) voice_sample_split_kernel(const float* __restrict__ mean, const float* __restrict__ eps,
                                                                 const float* __restrict__ sigma, int F, int D, float bias, float scale,
                                                                 long long m0, int M, bf16* __restrict__ hi, bf16* __restrict__ lo) {
  pdl_trigger();
  pdl_wait();
  const int D4 = D >> 2;
  const long long n4 = (long long)M * D4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / D4;
    const int k = (int)(i - r * D4) << 2;
    const long long off = (m0 + r) * D + k;
    const float4 q = *reinterpret_cast<const float4*>(mean + off);
    float a = q.x, b = q.y, c = q.z, d = q.w;
    if (eps) {
      const float s = sigma[(m0 + r) / F];
      const float4 e = *reinterpret_cast<const float4*>(eps + off);
      a += s * e.x; b += s * e.y; c += s * e.z; d += s * e.w;
    }
    store_split4(hi, lo, r * D + k, (a + bias) * scale, (b + bias) * scale, (c + bias) * scale, (d + bias) * scale);
  }
}

VV_DEVINL float to_f32(float v) { return v; }
VV_DEVINL float to_f32(bf16 v) { return __bfloat162float(v); }

// Conv1d weight [Co][Ci][k] (fp32 or bf16) -> bf16 [Co][Kp] tap-major (column j*Ci + ci), zero columns from k*Ci to Kp
template <class T>
__global__ void repack_conv_pad_kernel(const T* __restrict__ w, bf16* __restrict__ out, int Co, int Ci, int k, int Kp) {
  const long long n = (long long)Co * Kp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i / Kp), kk = (int)(i % Kp);
    float v = 0.f;
    if (kk < k * Ci) {
      const int j = kk / Ci, ci = kk % Ci;
      v = to_f32(w[((long long)co * Ci + ci) * k + j]);
    }
    out[i] = __float2bfloat16_rn(v);
  }
}

}  // namespace vv
