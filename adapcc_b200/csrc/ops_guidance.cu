// Classifier-free guidance for GPT-2 generation: the guided scores of HuggingFace's
// UnbatchedClassifierFreeGuidanceLogitsProcessor, computed on the device between the LM head and the sampler inside the
// same CUDA graph replay. The logits hold 2B rows: row b is prompt b's (c), row B + b its negative prompt's (u).
//
//   guidance_mix_kernel : one 1024-thread CTA per row pair b. Three passes over the first `vocab` columns of both rows:
//                         1. the maxima mc, mu;
//                         2. Sc = sum_i exp(c_i - mc), Su = sum_i exp(u_i - mu) (two passes rather than an online
//                            rescale, so every term is rounded the same way and the error bound stays simple);
//                         3. lc = (c_i - mc) - log Sc, lu = (u_i - mu) - log Su, and row b's column i becomes
//                            scale * (lc - lu) + lu, HuggingFace's order of operations.
//                         Row b's padding columns and rows [B, 2B) are not written.
//
// Every sum runs in fp32 in an order fixed by the thread layout: thread t adds columns t, t + 1024, ... in index order,
// a 5-level shuffle butterfly adds the lanes and every warp adds the 32 warp partials with a second butterfly. Each
// operation is correctly rounded (__fsub_rn / __fadd_rn / __fmul_rn: no contraction into FMAs). A row's bits therefore
// depend on its two input rows, vocab and the scale only, not on B, and there is no host sync, so the launch can be
// captured in a graph. ops/guidance.py has the fp64 definition the tests compare against (DESIGN.md §4a).
#include <cmath>

#include "block_reduce.cuh"
#include "common.h"

namespace adapcc {

constexpr int kGuideThreads = kRowThreads;
constexpr int kGuideUnroll = 4;              // columns per thread and row in flight at once

__global__ void __launch_bounds__(kGuideThreads) guidance_mix_kernel(float* logits, int ld, int vocab, int B,
                                                                     float scale) {
  __shared__ float2 s_part[kRowWarps];
  float* c = logits + (long long)blockIdx.x * ld;
  const float* u = logits + (long long)(blockIdx.x + B) * ld;
  constexpr int kStride = kGuideThreads * kGuideUnroll;

  float2 m = make_float2(-INFINITY, -INFINITY);
  for (int i0 = threadIdx.x; i0 < vocab; i0 += kStride) {
#pragma unroll
    for (int k = 0; k < kGuideUnroll; ++k) {
      const int i = i0 + k * kGuideThreads;
      if (i < vocab) m = make_float2(fmaxf(m.x, c[i]), fmaxf(m.y, u[i]));
    }
  }
  m = block_reduce_f2<true>(m, s_part);

  float2 s = make_float2(0.f, 0.f);
  for (int i0 = threadIdx.x; i0 < vocab; i0 += kStride) {
    float ec[kGuideUnroll], eu[kGuideUnroll];
#pragma unroll
    for (int k = 0; k < kGuideUnroll; ++k) {          // loads and exponentials first, then the adds in index order
      const int i = i0 + k * kGuideThreads;
      ec[k] = i < vocab ? expf(__fsub_rn(c[i], m.x)) : 0.f;
      eu[k] = i < vocab ? expf(__fsub_rn(u[i], m.y)) : 0.f;
    }
#pragma unroll
    for (int k = 0; k < kGuideUnroll; ++k) {
      if (i0 + k * kGuideThreads < vocab) s = make_float2(__fadd_rn(s.x, ec[k]), __fadd_rn(s.y, eu[k]));
    }
  }
  s = block_reduce_f2<false>(s, s_part);

  const float log_sc = logf(s.x), log_su = logf(s.y);
  for (int i0 = threadIdx.x; i0 < vocab; i0 += kStride) {
#pragma unroll
    for (int k = 0; k < kGuideUnroll; ++k) {
      const int i = i0 + k * kGuideThreads;
      if (i < vocab) {
        const float lc = __fsub_rn(__fsub_rn(c[i], m.x), log_sc);
        const float lu = __fsub_rn(__fsub_rn(u[i], m.y), log_su);
        c[i] = __fadd_rn(__fmul_rn(scale, __fsub_rn(lc, lu)), lu);
      }
    }
  }
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// logits fp32 [2B, ld]: rows [0, B) the prompts', rows [B, 2B) the negative prompts'; row b's first `vocab` columns
// are overwritten with the guided scores of rows b and B + b
int adapcc_guidance_mix(float* logits, int ld, int vocab, int B, float scale, void* stream) {
  if (B < 1 || B > 65535 || vocab < 1 || ld < vocab) {
    set_error("guidance_mix: need 1 <= B <= 65535 and 1 <= vocab <= ld (B=%d vocab=%d ld=%d)", B, vocab, ld);
    return -1;
  }
  if (!std::isfinite(scale)) {
    set_error("guidance_mix: need a finite scale (got %g)", (double)scale);
    return -1;
  }
  if (!logits) {
    set_error("guidance_mix: null pointer");
    return -1;
  }
  guidance_mix_kernel<<<B, kGuideThreads, 0, (cudaStream_t)stream>>>(logits, ld, vocab, B, scale);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
