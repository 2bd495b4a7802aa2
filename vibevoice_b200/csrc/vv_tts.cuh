// vv_tts.cuh -- the two per-token modules of the streaming-0.5B variant that sit outside the decoder stack
// (reference vibevoice/modular/modeling_vibevoice_streaming.py:42-53, 124-131; used at
// modeling_vibevoice_streaming_inference.py:290-291 and :691-696):
//   tts_type_embed_kernel  dst[row] = src[row'] + tts_input_types[type]   (type 1 = text, 0 = speech) for every TTS-LM input row
//   eos_prob_kernel        sigmoid(fc2 . relu(fc1 . h + b1) + b2)   the end-of-speech classifier on the last TTS-LM hidden state of n rows
// Both read fp32 weights: the checkpoint's values are kept exactly (an EOS decision near 0.5 must not move with a bf16 rounding).
#pragma once
#include "vv_kernels.cuh"

namespace vv {

constexpr int TTS_MAX_ROWS = 16;                    // 2 * max_batch rows at most
struct TtsRows { int dst[TTS_MAX_ROWS]; int src[TTS_MAX_ROWS]; int type[TTS_MAX_ROWS]; int n; };

// One fp32 add per element, as `src[s] + tts_input_types.weight[type]` is in PyTorch: dst[rows.dst[i]] = src[rows.src[i]] + types[rows.type[i]].
// Every element is read and written by the same thread, and a thread reads all its sources before it writes, so a source row may also
// be a destination row.
__global__ void tts_type_embed_kernel(const float* src, const float* __restrict__ types, TtsRows rows, float* dst, int H) {
  pdl_trigger();
  pdl_wait();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= H) return;
  float v[TTS_MAX_ROWS];
#pragma unroll
  for (int i = 0; i < TTS_MAX_ROWS; ++i)            // static indices: the row lists stay in the parameter bank
    if (i < rows.n) v[i] = src[(size_t)rows.src[i] * H + k] + types[(size_t)rows.type[i] * H + k];
#pragma unroll
  for (int i = 0; i < TTS_MAX_ROWS; ++i)
    if (i < rows.n) dst[(size_t)rows.dst[i] * H + k] = v[i];
}

constexpr int EOS_THREADS = 256;
constexpr int EOS_ROWS_PER_CTA = EOS_THREADS / 32;  // one fc1 row per warp
constexpr int EOS_MAX_ROWS = 8;                     // hidden rows per launch (max_batch <= 8 TTS-LM positive rows)
struct EosRows { int row[EOS_MAX_ROWS]; int n; };

// BinaryClassifier of n hidden rows in one launch.  Warp w of CTA b computes fc1 row j = b * 8 + w for all n rows (it reads the fc1 row
// once; each row keeps its own lane-strided fmaf chain in k order, then the fixed xor tree), and thread r of the CTA adds row r's fc2 terms
// in fc1-row order into partial[r][b].  The last CTA to finish (integer ticket) adds each row's partials in CTA order, so a row's result
// depends neither on scheduling nor on the other rows: it is bit-identical to the same row alone.  The ticket is reset for the next call by
// that CTA.  partial / ticket: device workspace of EOS_MAX_ROWS * gridDim.x floats and one unsigned (zero before the first call).
__global__ void __launch_bounds__(EOS_THREADS) eos_prob_kernel(const float* __restrict__ h, EosRows rows, const float* __restrict__ w1,
                                                               const float* __restrict__ b1, const float* __restrict__ w2,
                                                               const float* __restrict__ b2, int H, float* __restrict__ partial,
                                                               unsigned* __restrict__ ticket, float* __restrict__ prob_out,
                                                               float* __restrict__ logit_out) {
  extern __shared__ float sh[];                     // h rows [n][H]
  __shared__ float terms[EOS_MAX_ROWS][EOS_ROWS_PER_CTA];
  __shared__ bool last;
  pdl_trigger();
  pdl_wait();
  const int n = rows.n;
  for (int r = 0; r < n; ++r)
    for (int k = threadIdx.x; k < H; k += EOS_THREADS) sh[r * H + k] = h[(size_t)rows.row[r] * H + k];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x * EOS_ROWS_PER_CTA + warp;
  float t[EOS_MAX_ROWS];
#pragma unroll
  for (int r = 0; r < EOS_MAX_ROWS; ++r) t[r] = 0.f;
  if (j < H) {
    const float* wr = w1 + (size_t)j * H;
    float acc[EOS_MAX_ROWS];
#pragma unroll
    for (int r = 0; r < EOS_MAX_ROWS; ++r) acc[r] = 0.f;
    for (int k = lane; k < H; k += 32) {
      const float w = wr[k];
#pragma unroll
      for (int r = 0; r < EOS_MAX_ROWS; ++r)
        if (r < n) acc[r] = fmaf(w, sh[r * H + k], acc[r]);
    }
#pragma unroll
    for (int r = 0; r < EOS_MAX_ROWS; ++r)
      if (r < n) t[r] = w2[j] * fmaxf(warp_sum(acc[r]) + b1[j], 0.f);
  }
  if (lane == 0) {
#pragma unroll
    for (int r = 0; r < EOS_MAX_ROWS; ++r)
      if (r < n) terms[r][warp] = t[r];
  }
  __syncthreads();
  if (threadIdx.x < n) {
    float s = 0.f;
    for (int w = 0; w < EOS_ROWS_PER_CTA; ++w) s += terms[threadIdx.x][w];
    partial[threadIdx.x * gridDim.x + blockIdx.x] = s;
    __threadfence();
  }
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last || threadIdx.x >= n) return;
  __threadfence();
  const volatile float* p = partial + threadIdx.x * gridDim.x;
  float s = 0.f;
  for (int b = 0; b < (int)gridDim.x; ++b) s += p[b];
  const float logit = s + b2[0];
  prob_out[threadIdx.x] = 1.f / (1.f + expf(-logit));
  if (logit_out) logit_out[threadIdx.x] = logit;
  if (threadIdx.x == 0) *ticket = 0u;
}

}  // namespace vv
