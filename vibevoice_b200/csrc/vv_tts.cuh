// vv_tts.cuh -- the two per-token modules of the streaming-0.5B variant that sit outside the decoder stack
// (reference vibevoice/modular/modeling_vibevoice_streaming.py:42-53, 124-131; used at
// modeling_vibevoice_streaming_inference.py:290-291 and :691-696):
//   tts_type_embed_kernel  dst[row] = src + tts_input_types[type]   (type 1 = text, 0 = speech) for every TTS-LM input row
//   eos_prob_kernel        sigmoid(fc2 . relu(fc1 . h + b1) + b2)   the end-of-speech classifier on the last TTS-LM hidden state
// Both read fp32 weights: the checkpoint's values are kept exactly (an EOS decision near 0.5 must not move with a bf16 rounding).
#pragma once
#include "vv_kernels.cuh"

namespace vv {

constexpr int TTS_MAX_ROWS = 16;                    // 2 * max_batch rows at most
struct TtsRows { int row[TTS_MAX_ROWS]; int n; };

// One fp32 add per element, as `src + tts_input_types.weight[type]` is in PyTorch.  Every element is read and written by the same
// thread, so src may be one of the destination rows.
__global__ void tts_type_embed_kernel(const float* src, const float* __restrict__ types, int type_id, TtsRows rows, float* dst, int H) {
  pdl_trigger();
  pdl_wait();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= H) return;
  const float v = src[k] + types[(size_t)type_id * H + k];
#pragma unroll
  for (int i = 0; i < TTS_MAX_ROWS; ++i)            // static indices: the row list stays in the parameter bank
    if (i < rows.n) dst[(size_t)rows.row[i] * H + k] = v;
}

constexpr int EOS_THREADS = 256;
constexpr int EOS_ROWS_PER_CTA = EOS_THREADS / 32;  // one fc1 row per warp

// BinaryClassifier in one launch.  Warp w of CTA b computes fc1 row j = b * 8 + w (lane-strided dot product, then a fixed xor tree),
// and thread 0 of the CTA adds its rows' fc2 terms in row order into partial[b].  The last CTA to finish (integer ticket) adds the
// partials in CTA order, so the result does not depend on scheduling: two calls give the same bits.  The ticket is reset for the next
// call by that CTA.  partial / ticket: device workspace of gridDim.x floats and one unsigned (zero before the first call).
__global__ void __launch_bounds__(EOS_THREADS) eos_prob_kernel(const float* __restrict__ h, const float* __restrict__ w1,
                                                               const float* __restrict__ b1, const float* __restrict__ w2,
                                                               const float* __restrict__ b2, int H, float* __restrict__ partial,
                                                               unsigned* __restrict__ ticket, float* __restrict__ prob_out,
                                                               float* __restrict__ logit_out) {
  extern __shared__ float sh[];                     // h [H]
  __shared__ float terms[EOS_ROWS_PER_CTA];
  __shared__ bool last;
  pdl_trigger();
  pdl_wait();
  for (int k = threadIdx.x; k < H; k += EOS_THREADS) sh[k] = h[k];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x * EOS_ROWS_PER_CTA + warp;
  float t = 0.f;
  if (j < H) {
    const float* wr = w1 + (size_t)j * H;
    float acc = 0.f;
    for (int k = lane; k < H; k += 32) acc = fmaf(wr[k], sh[k], acc);
    acc = warp_sum(acc);
    t = w2[j] * fmaxf(acc + b1[j], 0.f);
  }
  if (lane == 0) terms[warp] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < EOS_ROWS_PER_CTA; ++w) s += terms[w];
    partial[blockIdx.x] = s;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  const volatile float* p = partial;
  float s = 0.f;
  for (int b = 0; b < (int)gridDim.x; ++b) s += p[b];
  const float logit = s + b2[0];
  prob_out[0] = 1.f / (1.f + expf(-logit));
  if (logit_out) logit_out[0] = logit;
  *ticket = 0u;
}

}  // namespace vv
