// DoLa layer-contrast decoding for GPT-2 generation (Chuang et al. 2023; HuggingFace's `dola_layers`): the layer choice
// and the contrast of ops/dola.py, computed on the device between the LM head and the repetition controls inside the
// same CUDA graph replay. The logits hold (1 + n_cand)·B rows: row b is row b's final logits f, row B + j·B + b the
// logits q_j of its j-th candidate layer's residual stream through the same tied head.
//
//   dola_divergence_kernel : one 1024-thread CTA per (candidate j, row b). Two passes over the first `vocab` columns of
//                            f and q_j give the maxima mf, mq and the log-sums lsf = log sum_i exp(f_i - mf),
//                            lsq = log sum_i exp(q_i - mq). With more than one candidate a third pass forms
//                            lf_i = (f_i - mf) - lsf, lq_i = (q_i - mq) - lsq, M_i = 0.5 (exp lf_i + exp lq_i) and sums
//                            M_i (log M_i - lf_i) and M_i (log M_i - lq_i) over the ids with M_i > 0; their means over
//                            vocab give KL1 and KL2, and JS_j = 0.5 (KL1 + KL2). The (j, b) CTA writes JS_j, mq and lsq
//                            to `work`; every CTA of row b computes mf and lsf the same way, so they get the same bits,
//                            and the j = 0 CTA writes them.
//   dola_contrast_kernel   : one 1024-thread CTA per row b. It picks c, the first j with the largest JS_j (0 for one
//                            candidate), sets thr = fl32(max_i lf_i + fl32(ln 0.1)) and overwrites row b's first `vocab`
//                            columns with lf_i - lq_c,i where lf_i >= thr and -inf elsewhere. Rows [B, (1 + n_cand)·B)
//                            and the padding columns are not written.
//
// Every sum runs in fp32 in an order fixed by the thread layout: thread t adds columns t, t + 1024, ... in index order
// and block_reduce.cuh adds the threads. Each add, subtract and multiply is correctly rounded (no contraction into
// FMAs), and expf / logf are the full-precision functions. A row's bits therefore depend on its own 1 + n_cand logit rows
// and vocab only, not on B, and there is no host sync, so both launches can be captured in a graph. ops/dola.py has
// the fp64 definition the tests compare against (DESIGN.md §4a).
#include <cmath>

#include "block_reduce.cuh"
#include "common.h"

namespace adapcc {

constexpr int kDolaUnroll = 4;               // columns per thread and row in flight at once
constexpr int kDolaMaxLayers = 16;           // candidate layers per call (ops.DOLA_MAX_LAYERS)
constexpr int kDolaWork = 4;                 // fp32 words per (candidate, row) slot of the work buffer
constexpr float kLnTenth = -2.302585092994045684f;   // fl32(ln 0.1): HuggingFace's relative_top = 0.1

// The maxima (pass 1) and log-sums (pass 2) of rows f and q over their first `vocab` columns, as (f, q) pairs.
__device__ __forceinline__ void dola_row_stats(const float* f, const float* q, int vocab, float2* s_part, float2& m,
                                               float2& ls) {
  constexpr int kStride = kRowThreads * kDolaUnroll;
  m = make_float2(-INFINITY, -INFINITY);
  for (int i0 = threadIdx.x; i0 < vocab; i0 += kStride) {
#pragma unroll
    for (int k = 0; k < kDolaUnroll; ++k) {
      const int i = i0 + k * kRowThreads;
      if (i < vocab) m = make_float2(fmaxf(m.x, f[i]), fmaxf(m.y, q[i]));
    }
  }
  m = block_reduce_f2<true>(m, s_part);

  float2 s = make_float2(0.f, 0.f);
  for (int i0 = threadIdx.x; i0 < vocab; i0 += kStride) {
    float ef[kDolaUnroll], eq[kDolaUnroll];
#pragma unroll
    for (int k = 0; k < kDolaUnroll; ++k) {            // loads and exponentials first, then the adds in index order
      const int i = i0 + k * kRowThreads;
      ef[k] = i < vocab ? expf(__fsub_rn(f[i], m.x)) : 0.f;
      eq[k] = i < vocab ? expf(__fsub_rn(q[i], m.y)) : 0.f;
    }
#pragma unroll
    for (int k = 0; k < kDolaUnroll; ++k) {
      if (i0 + k * kRowThreads < vocab) s = make_float2(__fadd_rn(s.x, ef[k]), __fadd_rn(s.y, eq[k]));
    }
  }
  s = block_reduce_f2<false>(s, s_part);
  ls = make_float2(logf(s.x), logf(s.y));
}

template <bool kJS>
__global__ void __launch_bounds__(kRowThreads) dola_divergence_kernel(const float* logits, int ld, int vocab, int B,
                                                                      float* work) {
  __shared__ float2 s_part[kRowWarps];
  const int j = blockIdx.x, b = blockIdx.y, n_cand = gridDim.x;
  const float* f = logits + (long long)b * ld;
  const float* q = logits + ((long long)(j + 1) * B + b) * ld;
  float2 m, ls;
  dola_row_stats(f, q, vocab, s_part, m, ls);

  float js = 0.f;
  if (kJS) {
    constexpr int kStride = kRowThreads * kDolaUnroll;
    float2 s = make_float2(0.f, 0.f);
    for (int i0 = threadIdx.x; i0 < vocab; i0 += kStride) {
      float t1[kDolaUnroll], t2[kDolaUnroll];
#pragma unroll
      for (int k = 0; k < kDolaUnroll; ++k) {
        const int i = i0 + k * kRowThreads;
        t1[k] = t2[k] = 0.f;
        if (i < vocab) {
          const float lf = __fsub_rn(__fsub_rn(f[i], m.x), ls.x);
          const float lq = __fsub_rn(__fsub_rn(q[i], m.y), ls.y);
          const float mid = __fmul_rn(0.5f, __fadd_rn(expf(lf), expf(lq)));
          if (mid > 0.f) {                             // a term with M_i = 0 is 0, as in torch's kl_div
            const float lm = logf(mid);
            t1[k] = __fmul_rn(mid, __fsub_rn(lm, lf));
            t2[k] = __fmul_rn(mid, __fsub_rn(lm, lq));
          }
        }
      }
#pragma unroll
      for (int k = 0; k < kDolaUnroll; ++k) s = make_float2(__fadd_rn(s.x, t1[k]), __fadd_rn(s.y, t2[k]));
    }
    s = block_reduce_f2<false>(s, s_part);
    const float v = (float)vocab;
    js = __fmul_rn(0.5f, __fadd_rn(__fdiv_rn(s.x, v), __fdiv_rn(s.y, v)));
  }
  if (threadIdx.x == 0) {
    float* w = work + ((long long)j * B + b) * kDolaWork;
    w[0] = js;
    w[1] = m.y;
    w[2] = ls.y;
    if (j == 0) {
      float* wf = work + ((long long)n_cand * B + b) * kDolaWork;
      wf[0] = m.x;
      wf[1] = ls.x;
    }
  }
}

__global__ void __launch_bounds__(kRowThreads) dola_contrast_kernel(float* logits, int ld, int vocab, int B,
                                                                    int n_cand, const float* work) {
  const int b = blockIdx.x;
  int c = 0;
  float best = work[(long long)b * kDolaWork];
  for (int j = 1; j < n_cand; ++j) {                   // the first maximum in the candidates' order
    const float js = work[((long long)j * B + b) * kDolaWork];
    if (js > best) best = js, c = j;
  }
  const float* wc = work + ((long long)c * B + b) * kDolaWork;
  const float* wf = work + ((long long)n_cand * B + b) * kDolaWork;
  const float mq = wc[1], lsq = wc[2], mf = wf[0], lsf = wf[1];
  const float thr = __fadd_rn(__fsub_rn(__fsub_rn(mf, mf), lsf), kLnTenth);   // max_i lf_i = (mf - mf) - lsf
  float* f = logits + (long long)b * ld;
  const float* q = logits + ((long long)(c + 1) * B + b) * ld;
  constexpr int kStride = kRowThreads * kDolaUnroll;
  for (int i0 = threadIdx.x; i0 < vocab; i0 += kStride) {
#pragma unroll
    for (int k = 0; k < kDolaUnroll; ++k) {
      const int i = i0 + k * kRowThreads;
      if (i < vocab) {
        const float lf = __fsub_rn(__fsub_rn(f[i], mf), lsf);
        f[i] = lf >= thr ? __fsub_rn(lf, __fsub_rn(__fsub_rn(q[i], mq), lsq)) : -INFINITY;
      }
    }
  }
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// fp32 words of dola_contrast's work buffer for B rows and n_cand candidates
long long adapcc_dola_work_numel(int B, int n_cand) { return (long long)(n_cand + 1) * B * kDolaWork; }

// logits fp32 [(1 + n_cand)·B, ld]: rows [0, B) the final logits, row B + j·B + b candidate j's of row b; row b's first
// `vocab` columns are overwritten with its DoLa scores. work: adapcc_dola_work_numel(B, n_cand) fp32 words.
int adapcc_dola_contrast(float* logits, int ld, int vocab, int B, int n_cand, float* work, void* stream) {
  if (B < 1 || B > 65535 || n_cand < 1 || n_cand > kDolaMaxLayers || vocab < 1 || ld < vocab) {
    set_error("dola_contrast: need 1 <= B <= 65535, 1 <= n_cand <= %d and 1 <= vocab <= ld (B=%d n_cand=%d vocab=%d "
              "ld=%d)", kDolaMaxLayers, B, n_cand, vocab, ld);
    return -1;
  }
  if (!logits || !work) {
    set_error("dola_contrast: null pointer");
    return -1;
  }
  const dim3 grid(n_cand, B);
  if (n_cand > 1)
    dola_divergence_kernel<true><<<grid, kRowThreads, 0, (cudaStream_t)stream>>>(logits, ld, vocab, B, work);
  else
    dola_divergence_kernel<false><<<grid, kRowThreads, 0, (cudaStream_t)stream>>>(logits, ld, vocab, B, work);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  dola_contrast_kernel<<<B, kRowThreads, 0, (cudaStream_t)stream>>>(logits, ld, vocab, B, n_cand, work);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
