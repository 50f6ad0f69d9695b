// The sampled row of the on-device sampler: the inverse-CDF pick, the survivors a draw decided from, SynthID's
// tournament and draw_row, the definition's steps 1-7 by one CTA of 1024 threads. ops_sample.cu draws every token of
// generate and of speculative decoding through it; ops_synthid.cu holds its SynthID instantiation, in a translation
// unit of its own, so the register allocation ptxas gives the shared __noinline__ filters, and with it the SASS of the
// other sampling kernels, does not depend on that kernel.
#pragma once

#include <climits>
#include <cmath>
#include <cstdint>

#include "device_prims.cuh"
#include "sample_filter.cuh"
#include "synthid.cuh"

namespace adapcc {

__device__ __forceinline__ float philox_uniform(uint32_t w) { return (float)(w >> 8) * 0x1p-24f; }

// The inverse-CDF pick over s_x[0, V) by the whole CTA: the ids with `counts(x)` count, with weight `weight(x)`. Returns the smallest counting i whose inclusive prefix of weights exceeds u Z' (Z', the total, goes to `zp`), or
// the largest counting id when rounding leaves none, or -1 when no id counts. Thread t owns the contiguous ids
// [t C, t C + C) (C odd, so a warp's reads hit 32 different banks); prefix = (sum of the lower threads' chunks, by a
// shuffle scan and warp totals in order) + the running sum inside the chunk.
template <class Counts, class Weight>
__device__ __forceinline__ int scan_pick(const float* s_x, SampleSmem& sm, int V, Counts counts, Weight weight, float u,
                                         float& zp) {
  const int tid = threadIdx.x;
  const int C = ((V + kSampleThreads - 1) / kSampleThreads) | 1;
  const int i0 = min(tid * C, V), i1 = min(i0 + C, V);
  float run = 0.f;
  int last = -1;
  for (int i = i0; i < i1; ++i) {
    const float x = s_x[i];
    if (counts(x)) {
      run += weight(x);
      last = i;
    }
  }
  const int lane = tid & 31, warp = tid >> 5;
  float inc = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  float excl = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane == 0) excl = 0.f;
  __syncthreads();
  if (lane == 31) sm.f[warp] = inc;
  __syncthreads();
  // offset of this warp: an inclusive shuffle scan over the warp totals (lane w holds warp w's), the same in
  // every warp; Z' is its last element
  float tot = sm.f[lane];
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float y = __shfl_up_sync(0xffffffffu, tot, o);
    if (lane >= o) tot += y;
  }
  zp = __shfl_sync(0xffffffffu, tot, 31);
  float off = __shfl_sync(0xffffffffu, tot, (warp + 31) & 31);
  if (warp == 0) off = 0.f;
  excl = off + excl;
  const float target = u * zp;
  int found = INT_MAX;
  if (i0 < i1) {
    float acc = 0.f;
    for (int i = i0; i < i1; ++i) {
      const float x = s_x[i];
      if (counts(x)) {
        acc += weight(x);
        if (excl + acc > target) {
          found = i;
          break;
        }
      }
    }
  }
  // the first crossing over the block; when rounding leaves none, the largest counting id
  const unsigned long long first = 0xFFFFFFFFull - block_max(sm, 0xFFFFFFFFull - (unsigned long long)found);
  return first != (unsigned long long)INT_MAX ? (int)first
                                              : (int)block_max(sm, (unsigned long long)(last + 1)) - 1;
}

// What a draw decided from: the survivors are the ids with f2key(s_x[i]) >= tau, with weights expf(s_x[i] - m) and
// total zp. No survivor (greedy, or no finite logit): tau above every key, zp = 0.
struct RowCut {
  uint32_t tau;
  float m, zp;
};

__device__ __forceinline__ float cut_prob(float x, const RowCut& c) {
  return f2key(x) >= c.tau ? expf(x - c.m) / c.zp : 0.f;
}

// SynthID's tournament (DESIGN.md §4a, step 6b) over the survivors {f2key(s_x[i]) >= tau} of a row with maximum m and
// context hash hc, by the whole CTA: s_x becomes p' (0 off the survivors). p_i = e_i / Z' with e_i = exp(x_i - m);
// then for each layer l, mass = the sum of p_i over the ids with g_l = 1 (per-thread loops in index order, then
// block_sum2's fixed tree) and p_i <- p_i ((1 + g_l) - mass). Thread t owns the ids t + 1024 k (k < 56), so one
// layer's g-values of its ids fit in a 64-bit mask, and each pass applies the previous layer's update while it
// computes the next layer's g-values and partial mass. Ids whose p is not positive take no further part.
static __device__ __noinline__ void synthid_tournament(float* s_x, SampleSmem& sm, int V, uint32_t tau, float m,
                                                       const SynthIDArgs& w, unsigned long long hc) {
  const int tid = threadIdx.x;
  float z = 0.f, unused = 0.f;
  for (int i = tid; i < V; i += kSampleThreads) {
    const float x = s_x[i];
    if (f2key(x) >= tau) z += expf(x - m);
  }
  block_sum2(sm, z, unused);
  for (int i = tid; i < V; i += kSampleThreads) {
    const float x = s_x[i];
    s_x[i] = f2key(x) >= tau ? __fdiv_rn(expf(x - m), z) : 0.f;
  }
  float mass = 0.f;                                 // the previous layer's, and its g-values in gm
  unsigned long long gm = 0ull;
  for (int l = 0;; ++l) {
    const bool last = l == w.depth;
    const unsigned long long key = last ? 0ull : w.keys[l];
    unsigned long long gn = 0ull;
    float part = 0.f;
    for (int i = tid, k = 0; i < V; i += kSampleThreads, ++k) {
      float p = s_x[i];
      if (!(p > 0.f)) continue;
      if (l > 0) {
        p *= (((gm >> k) & 1ull) ? 2.f : 1.f) - mass;
        s_x[i] = p;
      }
      if (!last && p > 0.f && synthid_g(w, synthid_acc(synthid_acc(hc, (unsigned long long)i), key))) {
        gn |= 1ull << k;
        part += p;
      }
    }
    if (last) break;
    unused = 0.f;
    block_sum2(sm, part, unused);
    mass = part;
    gm = gn;
  }
  __syncthreads();                                  // the draw reads other threads' ids
}

// One row of the definition (DESIGN.md §4a, steps 1-7) by the whole CTA: the logits row `l`, the tokens generated so
// far `step` (the min-length rule), the Philox counter `pos` and the row's seed. Returns the token, the same in every
// thread. sample_tokens_kernel, sample_slots_kernel and spec_slots_kernel all draw through it, so their tokens are the
// same bits. With `cut`, it also returns the survivors; s_x then still holds the row they are read from. The SynthID
// instantiation (kSynthID) runs the tournament of step 6b with context hash hc when `sid` is set (a step that is
// neither skipped nor repeated) and draws from p' (the arg-max of p' at temperature 0); without `sid` it is the row
// of the other instantiation.
template <bool kSynthID = false>
__device__ __forceinline__ int draw_row(float* s_x, SampleSmem& sm, const SampleArgs& a, const float* l, int step,
                                        int pos, long long seed, RowCut* cut = nullptr,
                                        const SynthIDArgs* sid = nullptr, unsigned long long hc = 0ull) {
  if (cut) *cut = RowCut{0xFFFFFFFFu, 0.f, 0.f};
  const int V = a.vocab;
  unsigned long long best;
  const int present = row_prologue(s_x, sm, l, V, a.temperature, step, a.min_new, a.suppress, a.n_suppress, best);
  int token = 0;                                    // a row without a finite logit draws id 0
  if (present > 0 && a.temperature == 0.f) {
    token = (int)(0xFFFFFFFFu - (uint32_t)best);
    if constexpr (kSynthID) {
      if (sid) {                                    // p: the softmax over every finite id; the arg-max of p'
        synthid_tournament(s_x, sm, V, kNegInfKey + 1, key2f((uint32_t)(best >> 32)), *sid, hc);
        unsigned long long pb = 0ull;
        for (int i = threadIdx.x; i < V; i += kSampleThreads) {
          const float p = s_x[i];
          if (p > 0.f) pb = max(pb, ((unsigned long long)f2key(p) << 32) | (0xFFFFFFFFu - (uint32_t)i));
        }
        pb = block_max(sm, pb);
        if (pb) token = (int)(0xFFFFFFFFu - (uint32_t)pb);
      }
    }
  } else if (present > 0) {
    const uint32_t mkey = (uint32_t)(best >> 32);
    const float m = key2f(mkey);
    int kept = present;
    if (a.top_h > 0.f) {
      __shared__ unsigned long long s_sel[kTopHN];
      __shared__ int s_n;
      kept = top_h_row(s_x, sm, V, present, m, a.top_h, 1, s_sel, &s_n);
    }
    uint32_t tau = row_tau(s_x, sm, V, a.top_k, a.top_p, 1, kept, mkey, m);
    if (a.f.on()) {
      filter_row(s_x, sm, V, a.f, tau, m, mkey);
      tau = kNegInfKey + 1;                         // the survivors are the finite ids
    }
    // the draw: the smallest i whose inclusive prefix of surviving weights exceeds u Z'
    const uint32_t w0 = philox4((uint32_t)pos, (uint32_t)(unsigned long long)seed,
                                (uint32_t)((unsigned long long)seed >> 32)).x;
    float zp;
    if constexpr (kSynthID) {
      if (sid) {                                    // the same rule and word over p'
        synthid_tournament(s_x, sm, V, tau, m, *sid, hc);
        token = scan_pick(s_x, sm, V, [](float x) { return x > 0.f; }, [](float x) { return x; },
                          philox_uniform(w0), zp);
        return token;
      }
    }
    token = scan_pick(s_x, sm, V, [tau](float x) { return f2key(x) >= tau; }, [m](float x) { return expf(x - m); },
                      philox_uniform(w0), zp);
    if (cut) *cut = RowCut{tau, m, zp};
  }
  return token;
}

// Launches sample_tokens_synthid_kernel (ops_synthid.cu) on B rows: the body of adapcc_sample_tokens_synthid without
// the step increment. Returns 0 or -1 with the error set.
int sample_tokens_synthid_launch(const SampleArgs& a, const SynthIDArgs& w, int B, cudaStream_t stream);

}  // namespace adapcc
