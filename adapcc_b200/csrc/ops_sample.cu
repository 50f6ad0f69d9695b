// Token sampling for GPT-2 generation: the tied LM head in bf16 and one seeded top-k / top-p draw per row, both on the
// device, so a whole generation step (decode, head, sample) can be replayed from one CUDA graph without a host sync.
//
//   lm_head : out[b, i] = sum_d h[b, d] * W[i, d] (bf16 in, fp32 out). Memory bound at GPT-2's batch sizes, so W is
//             streamed once per call for all rows: the h rows sit in shared memory, a warp holds kHeadRows rows of W in
//             registers and forms their dot products with every h row. Lane l owns the 8-element chunks l, l + 32, ...
//             of d; each lane adds its chunks in order and a shuffle tree adds the lanes. The order depends on D only,
//             so a row's bits do not depend on B, on the other rows or on which warp handles which rows of W.
//   sample  : one CTA of 1024 threads per row; the row's x_i = l_i / temperature stay in shared memory for all passes.
//             The top-k threshold and the top-p cut-off are found by bisection over the order-preserving integer
//             encoding of x (counts for top-k, masses for top-p), with no sort. The draw is an inclusive scan over the
//             surviving weights in index order.
//   slots   : the draws of assisted generation, one CTA per verify slot or draft (grid (slots, B)), through the same
//             row body as `sample`, with a per-slot Philox counter and step (DESIGN.md §4a). A draft draw can also
//             write the draft's filtered weights, which rejection-sampling verification reads.
//   spec    : rejection-sampling verification of a round, one CTA per verify slot (grid (k + 1, B)): the slot's draw,
//             the acceptance of its draft and the residual draw, each from its own Philox word (DESIGN.md §4a).
//
// Every floating-point sum runs in fp32 in an order fixed by the thread layout (per-thread loops in index order,
// shuffle trees, warp partials added in warp order), never by arrival. A row's token depends on its logits, its seed,
// its position and the scalars only: not on B, nor on graph replay versus eager launch. DESIGN.md §4a has the
// definition the kernel implements; ops/sampling.py evaluates the same definition in fp64.
#include <cuda_bf16.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <mutex>

#include "common.h"
#include "device_prims.cuh"

namespace adapcc {

constexpr int kHeadThreads = 256;
constexpr int kHeadRows = 4;                 // rows of W per warp and iteration
constexpr int kHeadMaxChunks = 4;            // 8-element chunks of d per lane: D <= 32 * 8 * 4 = 1024
constexpr int kHeadMaxD = 32 * 8 * kHeadMaxChunks;
constexpr int kHeadMaxB = 64;                // h in shared memory: 64 x 1024 x 2 B = 128 KB at most
constexpr int kSampleThreads = 1024;
constexpr int kSampleWarps = kSampleThreads / 32;
constexpr int kSampleMaxVocab = 56 * 1024;   // x of a row in shared memory: 224 KB
constexpr int kSampleMaxList = 1024;
constexpr int kOpsMaxDevices = 64;
constexpr int kSlotMaxSlots = 16;            // verify slots per row (LOOKUP_MAX_TOKENS + 1)
constexpr uint32_t kNegInfKey = 0x007FFFFFu; // key(-inf): ids at -inf (removed ones included) are never candidates

__global__ void __launch_bounds__(kHeadThreads)
lm_head_logits_kernel(const __nv_bfloat16* __restrict__ h, int ld_h, const __nv_bfloat16* __restrict__ W, int V, int D,
                      float* __restrict__ out, int B) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  __nv_bfloat16* s_h = reinterpret_cast<__nv_bfloat16*>(s_raw);   // [B, D]
  const int nvec = D >> 3;
  for (int i = threadIdx.x; i < B * nvec; i += kHeadThreads) {
    const int b = i / nvec, c = i - b * nvec;
    *reinterpret_cast<uint4*>(s_h + (long long)b * D + c * 8) =
        *reinterpret_cast<const uint4*>(h + (long long)b * ld_h + c * 8);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = blockIdx.x * (kHeadThreads / 32) + (threadIdx.x >> 5);
  const int stride = gridDim.x * (kHeadThreads / 32) * kHeadRows;
  for (int r0 = warp * kHeadRows; r0 < V; r0 += stride) {
    uint4 w[kHeadRows][kHeadMaxChunks];
#pragma unroll
    for (int r = 0; r < kHeadRows; ++r)
#pragma unroll
      for (int j = 0; j < kHeadMaxChunks; ++j) {
        const int c = lane + 32 * j;
        w[r][j] = (r0 + r < V && c < nvec) ? __ldg(reinterpret_cast<const uint4*>(W + (long long)(r0 + r) * D + c * 8))
                                           : make_uint4(0u, 0u, 0u, 0u);
      }
    for (int b = 0; b < B; ++b) {
      float acc[kHeadRows];
#pragma unroll
      for (int r = 0; r < kHeadRows; ++r) acc[r] = 0.f;
#pragma unroll
      for (int j = 0; j < kHeadMaxChunks; ++j) {
        const int c = lane + 32 * j;
        if (c < nvec) {
          float hv[8];
          unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(s_h + (long long)b * D + c * 8), hv);
#pragma unroll
          for (int r = 0; r < kHeadRows; ++r) {
            float wv[8];
            unpack<__nv_bfloat16>(w[r][j], wv);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[r] = fmaf(hv[e], wv[e], acc[r]);
          }
        }
      }
#pragma unroll
      for (int r = 0; r < kHeadRows; ++r)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
      float v = acc[0];
#pragma unroll
      for (int r = 1; r < kHeadRows; ++r) v = lane == r ? acc[r] : v;
      if (lane < kHeadRows && r0 + lane < V) out[(long long)b * V + r0 + lane] = v;
    }
  }
}

// ---- sampling --------------------------------------------------------------------------------------------------------
struct SampleArgs {
  const float* logits;       // [B, ld], the first `vocab` columns used
  int ld, vocab;
  float temperature, top_p;
  int top_k;
  const long long* seeds;    // [B]
  const int* pos;            // [B]: position of the token being drawn (the Philox counter)
  int* step;                 // tokens generated so far (read here, incremented by step_incr_kernel)
  int min_new;
  const int* suppress;       // ids removed while *step < min_new
  int n_suppress;
  const int* stop;           // ids that end a row
  int n_stop;
  int* done;                 // [B]
  long long* next_ids;       // [B]
  long long* tokens;         // [B, max_new]
  int max_new;
  // truncation filters after top-p (DESIGN.md §4a); `filters` is set iff one of them is on
  float min_p, typical_p, epsilon, eta;
  bool filters;
};

// order-preserving: a < b (floats, no NaN) <=> key(a) < key(b)
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// the four output words of Philox4x32-10 (Salmon et al., SC'11) for counter (c0, 0, 0, 0) and key (k0, k1): the draw
// uses word 0; rejection-sampling verification uses word 1 for the acceptance test and word 2 for the residual draw,
// so neither depends on the draw that produced the draft
__device__ __forceinline__ uint4 philox4(uint32_t c0, uint32_t k0, uint32_t k1) {
  uint32_t c1 = 0u, c2 = 0u, c3 = 0u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

struct SampleSmem {
  float f[kSampleWarps];
  float g[kSampleWarps];
  int i[3][kSampleWarps];
  unsigned long long u[kSampleWarps];
};

// every thread gets the block sums: a shuffle tree per warp, then each warp adds the 32 warp partials with the same
// shuffle tree (lane w holds warp w's partial), so the order is fixed and every warp gets the same bits
__device__ __forceinline__ void block_sum(SampleSmem& sm, float& f, int& a, int& b, int& c) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    f += __shfl_xor_sync(0xffffffffu, f, o);
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  __syncthreads();                                  // the previous reduction's readers are done with the buffers
  if (lane == 0) {
    sm.f[warp] = f;
    sm.i[0][warp] = a;
    sm.i[1][warp] = b;
    sm.i[2][warp] = c;
  }
  __syncthreads();
  f = sm.f[lane];
  a = sm.i[0][lane];
  b = sm.i[1][lane];
  c = sm.i[2][lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    f += __shfl_xor_sync(0xffffffffu, f, o);
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
}

// two fp32 block sums with the same fixed order as block_sum
__device__ __forceinline__ void block_sum2(SampleSmem& sm, float& f, float& g) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    f += __shfl_xor_sync(0xffffffffu, f, o);
    g += __shfl_xor_sync(0xffffffffu, g, o);
  }
  __syncthreads();
  if (lane == 0) {
    sm.f[warp] = f;
    sm.g[warp] = g;
  }
  __syncthreads();
  f = sm.f[lane];
  g = sm.g[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    f += __shfl_xor_sync(0xffffffffu, f, o);
    g += __shfl_xor_sync(0xffffffffu, g, o);
  }
}

__device__ __forceinline__ unsigned long long block_max(SampleSmem& sm, unsigned long long v) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) sm.u[warp] = v;
  __syncthreads();
  v = sm.u[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// z = sum of e_i = exp(x_i - m) and s1 = sum of e_i (x_i - m) over the finite ids, in block_sum's fixed order
__device__ __forceinline__ void row_moments(const float* s_x, SampleSmem& sm, int V, float m, float& z, float& s1) {
  z = 0.f;
  s1 = 0.f;
  for (int i = threadIdx.x; i < V; i += kSampleThreads) {
    const float x = s_x[i];
    if (x != -INFINITY) {
      const float y = x - m, e = expf(y);
      z += e;
      s1 += e * y;
    }
  }
  block_sum2(sm, z, s1);
}

// The truncation filters after top-p, in HuggingFace's order: min-p, typical, epsilon, eta. The kept set {key >= tau}
// is first written into the row (-inf for every other id), and each filter removes ids the same way, so afterwards
// the survivors are exactly the finite ids. A filter that is off costs nothing; p_i = e_i / Z over the current
// survivors, with e_i = exp(x_i - m) and m the row maximum, which top-k, top-p and min-p always keep.
__device__ __noinline__ void filter_row(float* s_x, SampleSmem& sm, const SampleArgs& a, uint32_t tau, float m,
                                        uint32_t mkey) {
  const int tid = threadIdx.x, V = a.vocab;
  // materialise top-k / top-p; min-p keeps e_i >= min_p, i.e. p_i >= min_p p_max
  for (int i = tid; i < V; i += kSampleThreads) {
    const float x = s_x[i];
    if (f2key(x) < tau || (a.min_p > 0.f && expf(x - m) < a.min_p)) s_x[i] = -INFINITY;
  }
  uint32_t kmax = mkey;                             // key of the largest survivor: typical may remove the maximum
  if (a.typical_p < 1.f) {
    // H = log Z - mu with mu = sum p_i (x_i - m), so the deviation |-log p_i - H| is d_i = |(x_i - m) - mu|. The
    // cut-off d* is the smallest d with G(d) = (mass of d_i <= d) >= p Z, found by bisection over the order-preserving
    // keys of d. Invariant: G(lo) < p Z <= G(hi); G(lo) is carried and each pass adds the mass in (lo, mid]. Once no
    // key lies strictly inside the half that holds d*, that half's upper end is d*. hi starts at key(+inf), so rounding
    // that keeps every G below p Z keeps every id.
    float z, s1;
    row_moments(s_x, sm, V, m, z, s1);
    const float mu = s1 / z, pz = a.typical_p * z;
    uint32_t lo = f2key(0.f) - 1, hi = f2key(INFINITY);
    float g_lo = 0.f;
    while (hi - lo > 1) {
      const uint32_t mid = lo + (hi - lo) / 2;
      float s = 0.f;
      int nl = 0, nh = 0, unused = 0;
      for (int i = tid; i < V; i += kSampleThreads) {
        const float x = s_x[i];
        if (x != -INFINITY) {
          const uint32_t k = f2key(fabsf((x - m) - mu));
          if (k > lo && k <= hi) {
            if (k <= mid) s += expf(x - m);
            nl += k < mid;
            nh += k > mid && k < hi;
          }
        }
      }
      block_sum(sm, s, nl, nh, unused);
      const float g = g_lo + s;
      if (g >= pz) {
        hi = mid;
        if (nl == 0) break;
      } else {
        lo = mid;
        g_lo = g;
        if (nh == 0) break;
      }
    }
    unsigned long long best = 0;
    for (int i = tid; i < V; i += kSampleThreads) {
      const float x = s_x[i];
      if (x != -INFINITY) {
        if (f2key(fabsf((x - m) - mu)) > hi) s_x[i] = -INFINITY;
        else best = max(best, (unsigned long long)f2key(x));
      }
    }
    kmax = (uint32_t)block_max(sm, best);
  }
  // epsilon keeps p_i >= epsilon, eta keeps p_i >= min(eta, sqrt(eta) exp(-H)) with exp(-H) Z = exp(mu); both keep
  // the largest survivors (ties together) as well, which only matters when no p_i reaches the threshold
  for (int f = 0; f < 2; ++f) {
    const float c = f == 0 ? a.epsilon : a.eta;
    if (!(c > 0.f)) continue;
    float z, s1;
    row_moments(s_x, sm, V, m, z, s1);
    const float t = f == 0 ? c * z : fminf(c * z, sqrtf(c) * expf(s1 / z));
    for (int i = tid; i < V; i += kSampleThreads) {
      const float x = s_x[i];
      if (x != -INFINITY && expf(x - m) < t && f2key(x) != kmax) s_x[i] = -INFINITY;
    }
  }
  __syncthreads();                                  // the draw reads other threads' ids
}

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

// One row of the definition (DESIGN.md §4a, steps 1-7) by the whole CTA: the logits row `l`, the tokens generated so
// far `step` (the min-length rule), the Philox counter `pos` and the row's seed. Returns the token, the same in every
// thread. sample_tokens_kernel, sample_slots_kernel and spec_slots_kernel all draw through it, so their tokens are the
// same bits. With `cut`, it also returns the survivors; s_x then still holds the row they are read from.
__device__ __forceinline__ int draw_row(float* s_x, SampleSmem& sm, const SampleArgs& a, const float* l, int step,
                                        int pos, long long seed, RowCut* cut = nullptr) {
  if (cut) *cut = RowCut{0xFFFFFFFFu, 0.f, 0.f};
  const int tid = threadIdx.x, V = a.vocab;
  const bool greedy = a.temperature == 0.f;
  for (int i = tid; i < V; i += kSampleThreads) s_x[i] = greedy ? l[i] : __fdiv_rn(l[i], a.temperature);
  __syncthreads();
  if (step < a.min_new) {                           // the min-length rule comes before any filtering
    for (int j = tid; j < a.n_suppress; j += kSampleThreads) {
      const int id = a.suppress[j];
      if (id >= 0 && id < V) s_x[id] = -INFINITY;
    }
    __syncthreads();
  }
  // the maximum (lowest index on a tie) and the number of candidates
  unsigned long long best = 0;
  int present = 0, z1 = 0, z2 = 0;
  for (int i = tid; i < V; i += kSampleThreads) {
    const uint32_t k = f2key(s_x[i]);
    if (k > kNegInfKey) {
      ++present;
      best = max(best, ((unsigned long long)k << 32) | (0xFFFFFFFFu - (uint32_t)i));
    }
  }
  best = block_max(sm, best);
  float fz = 0.f;
  block_sum(sm, fz, present, z1, z2);
  int token = 0;                                    // a row without a finite logit draws id 0
  if (present > 0 && greedy) {
    token = (int)(0xFFFFFFFFu - (uint32_t)best);
  } else if (present > 0) {
    const uint32_t mkey = (uint32_t)(best >> 32);
    const float m = key2f(mkey);
    uint32_t tau = kNegInfKey + 1;                  // candidates are the ids with key >= tau
    if (a.top_k > 0 && a.top_k < present) {
      // tau = the k-th largest key counted with multiplicity. Invariant: count(key >= lo) >= k > count(key >= hi).
      // Stops early once no key lies strictly between lo and hi: lo is then the k-th largest key.
      uint32_t lo = kNegInfKey + 1, hi = mkey + 1;
      int cnt_hi = 0;
      while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        int c = 0, nl = 0, nh = 0;
        for (int i = tid; i < V; i += kSampleThreads) {
          const uint32_t k = f2key(s_x[i]);
          if (k > lo && k < hi) {
            c += k >= mid;
            nl += k < mid;
            nh += k > mid;
          }
        }
        float f = 0.f;
        block_sum(sm, f, c, nl, nh);
        if (cnt_hi + c >= a.top_k) {
          lo = mid;
          if (nh == 0) break;
        } else {
          hi = mid;
          cnt_hi += c;
          if (nl == 0) break;
        }
      }
      tau = lo;
    }
    float z = 0.f;
    int u0 = 0, u1 = 0, u2 = 0;
    for (int i = tid; i < V; i += kSampleThreads) {
      const float x = s_x[i];
      if (f2key(x) >= tau) z += expf(x - m);
    }
    block_sum(sm, z, u0, u1, u2);
    const float pz = a.top_p * z;
    if (a.top_p < 1.f && pz < z) {
      // top-p: keep i iff F(key_i) <= p Z, F(t) = the mass of candidates with key > t (non-increasing in t).
      // Invariant: F(lo) > p Z >= F(hi); F(hi) is carried, each pass adds the mass in (mid, hi]. Once no candidate key
      // lies strictly between lo and hi, the kept set is key >= hi.
      uint32_t lo = tau - 1, hi = mkey;
      float f_hi = 0.f;
      while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        float s = 0.f;
        int nl = 0, nh = 0, unused = 0;
        for (int i = tid; i < V; i += kSampleThreads) {
          const float x = s_x[i];
          const uint32_t k = f2key(x);
          if (k > lo && k <= hi) {
            if (k > mid) s += expf(x - m);
            nl += k < mid;
            nh += k > mid && k < hi;
          }
        }
        block_sum(sm, s, nl, nh, unused);
        const float f = f_hi + s;
        if (f <= pz) {
          hi = mid;
          f_hi = f;
          if (nl == 0) break;
        } else {
          lo = mid;
          if (nh == 0) break;
        }
      }
      tau = hi;
    }
    if (a.filters) {
      filter_row(s_x, sm, a, tau, m, mkey);
      tau = kNegInfKey + 1;                         // the survivors are the finite ids
    }
    // the draw: the smallest i whose inclusive prefix of surviving weights exceeds u Z'
    const uint32_t w0 = philox4((uint32_t)pos, (uint32_t)(unsigned long long)seed,
                                (uint32_t)((unsigned long long)seed >> 32)).x;
    float zp;
    token = scan_pick(s_x, sm, V, [tau](float x) { return f2key(x) >= tau; }, [m](float x) { return expf(x - m); },
                      philox_uniform(w0), zp);
    if (cut) *cut = RowCut{tau, m, zp};
  }
  return token;
}

__global__ void __launch_bounds__(kSampleThreads, 1)
sample_tokens_kernel(const __grid_constant__ SampleArgs a) {
  extern __shared__ float s_x[];                    // [vocab]
  __shared__ SampleSmem sm;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int step = *a.step;                         // incremented by the next kernel on the stream, after every CTA
  long long* tok_out = a.tokens + (long long)b * a.max_new + step;
  if (a.done[b]) {                                  // a finished row keeps done set and pads its reply with -1
    if (tid == 0) {
      if (step < a.max_new) *tok_out = -1;
      a.next_ids[b] = 0;
    }
    return;
  }
  const int token = draw_row(s_x, sm, a, a.logits + (long long)b * a.ld, step, a.pos[b], a.seeds[b]);
  if (tid == 0) {
    bool stopped = false;
    for (int j = 0; j < a.n_stop; ++j) stopped |= a.stop[j] == token;
    a.next_ids[b] = token;
    if (step < a.max_new) *tok_out = stopped ? -1 : token;
    if (stopped) a.done[b] = 1;
  }
}

__global__ void step_incr_kernel(int* step) { *step += 1; }

// ---- per-slot draws of speculative decoding (DESIGN.md §4a, assisted generation) -------------------------------------
struct SlotArgs {
  SampleArgs s;              // logits [B * kq, ld], the scalars, suppress list and seeds [B]; the rest unused
  int B, kq, S, slot0;       // kq logits rows per row b; CTA x draws slot j = slot0 + x of S slots per row
  const int* lens;           // [B]: the row's cached tokens; slot j draws the token at sequence index lens + j + 1
  const int* emitted;        // [B]: tokens emitted so far; slot j is generated step emitted + j
  const int* done;           // [B]
  const int* nq;             // [B]: the row's real verify slots
  int* g;                    // verify: g[b * S + j] (slot j real iff j < nq)
  long long* ids;            // draft: ids[b * S + j + 1] and next[b] (draft j + 1 real iff j + 1 < nq; else 0)
  long long* next;
  float* q;                  // draft, optional: the filtered weights of draft step j, q[(b * (S - 1) + j) * vocab + i]
  float* zq;                 // ... (0 off the survivors) and their total zq[b * (S - 1) + j]
};

__global__ void __launch_bounds__(kSampleThreads, 1)
sample_slots_kernel(const __grid_constant__ SlotArgs a) {
  extern __shared__ float s_x[];                    // [vocab]
  __shared__ SampleSmem sm;
  const int x = blockIdx.x, b = blockIdx.y, j = a.slot0 + x;
  const bool draft = a.ids != nullptr;
  if (a.done[b] || j + (draft ? 1 : 0) >= a.nq[b]) {   // a done row or a pad slot: nothing is drawn
    if (draft && threadIdx.x == 0) {
      a.ids[(long long)b * a.S + j + 1] = 0;
      a.next[b] = 0;
    }
    return;
  }
  RowCut cut;
  const int token = draw_row(s_x, sm, a.s, a.s.logits + ((long long)b * a.kq + x) * a.s.ld, a.emitted[b] + j,
                             a.lens[b] + j + 1, a.s.seeds[b], &cut);
  if (threadIdx.x == 0) {
    if (draft) {
      a.ids[(long long)b * a.S + j + 1] = token;
      a.next[b] = token;
    } else {
      a.g[(long long)b * a.S + j] = token;
    }
  }
  if (a.q) {                                        // the draft's distribution at this step, for rejection sampling
    const long long r = (long long)b * (a.S - 1) + j;
    float* q = a.q + r * a.s.vocab;
    for (int i = threadIdx.x; i < a.s.vocab; i += kSampleThreads) {
      const float v = s_x[i];
      q[i] = f2key(v) >= cut.tau ? expf(v - cut.m) : 0.f;
    }
    if (threadIdx.x == 0) a.zq[r] = cut.zp;
  }
}

// ---- rejection-sampling verification (DESIGN.md §4a) ------------------------------------------------------------------
struct SpecArgs {
  SlotArgs t;                // the model's slots: logits [B * S, ld] (kq = S, slot0 = 0), g [B * S]; ids, q unused
  const long long* ids;      // [B * S]: draft j + 1 in slot j + 1
  const float* q;            // [B, S - 1, vocab] and [B, S - 1]: the draft's weights and totals (sample_slots_kernel)
  const float* zq;
  int* acc;                  // [B * S]: draft j + 1 accepted, for j < nq - 1
  int* last;                 // [B * S]: the round's last token if it ends at slot j: t_j for j < nq - 1, else g_j
};

// CTA (j, b): draws g_j as sample_slots_kernel does; for a slot with a real draft d = d_{j+1} it also decides d
// (accepted iff v Q_j(d) < P_j(d), v from Philox word 1 at lens + j + 1) and draws the residual t_j from
// max(0, P_j - Q_j) with rho_d = 0 (word 2 at lens + j + 1; g_j when no weight is left). No slot depends on another.
__global__ void __launch_bounds__(kSampleThreads, 1)
spec_slots_kernel(const __grid_constant__ SpecArgs a) {
  extern __shared__ float s_x[];                    // [vocab]
  __shared__ SampleSmem sm;
  const SlotArgs& t = a.t;
  const int j = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, V = t.s.vocab;
  const int nq = t.nq[b];
  if (t.done[b] || j >= nq) return;
  const int L = t.lens[b];
  const long long seed = t.s.seeds[b];
  const long long o = (long long)b * t.S + j;
  RowCut cut;
  const int token = draw_row(s_x, sm, t.s, t.s.logits + o * t.s.ld, t.emitted[b] + j, L + j + 1, seed, &cut);
  if (j + 1 >= nq) {                                // the last real slot: a round that gets here emits g_j
    if (tid == 0) {
      t.g[o] = token;
      a.last[o] = token;
    }
    return;
  }
  const long long r = (long long)b * (t.S - 1) + j;
  const float* wq = a.q + r * V;
  const float zq = a.zq[r];
  const long long dl = a.ids[o + 1];
  const int d = dl >= 0 && dl < V ? (int)dl : -1;
  const uint4 w = philox4((uint32_t)(L + j + 1), (uint32_t)(unsigned long long)seed,
                          (uint32_t)((unsigned long long)seed >> 32));
  if (tid == 0) {
    const float pd = d >= 0 ? cut_prob(s_x[d], cut) : 0.f;
    const float qd = d >= 0 && zq > 0.f ? wq[d] / zq : 0.f;
    t.g[o] = token;
    a.acc[o] = philox_uniform(w.y) * qd < pd;       // strict: an id with P = 0 is never accepted
  }
  __syncthreads();                                  // s_x[d] is read before the row becomes the residual
  for (int i = tid; i < V; i += kSampleThreads) {
    const float p = cut_prob(s_x[i], cut), q = zq > 0.f ? wq[i] / zq : 0.f;
    s_x[i] = i == d ? 0.f : fmaxf(0.f, p - q);
  }
  __syncthreads();
  float zr;
  const int res = scan_pick(s_x, sm, V, [](float x) { return x > 0.f; }, [](float x) { return x; },
                            philox_uniform(w.z), zr);
  if (tid == 0) a.last[o] = res >= 0 ? res : token;
}

// The checks and set-up shared by adapcc_sample_slots and adapcc_spec_slots; fills `s` or sets the error.
static int slot_args(const char* who, const float* logits, int ld, int vocab, int B, int kq, int S, int slot0,
                     bool draft, float temperature, int top_k, float top_p, float min_p, float typical_p,
                     float epsilon, float eta, const long long* seeds, const int* lens, const int* emitted,
                     const int* done, const int* nq, int min_new, const int* suppress, int n_suppress, SampleArgs& s) {
  if (B < 1 || B > 65535 || S < 1 || S > kSlotMaxSlots || kq < 1 || (draft && kq != 1) || slot0 < 0 ||
      slot0 + kq + (draft ? 1 : 0) > S || vocab < 1 || vocab > kSampleMaxVocab || ld < vocab) {
    set_error("%s: need 1 <= B <= 65535, 1 <= S <= %d, kq >= 1 (1 for drafts), 0 <= slot0, slot0 + kq (+ 1 for "
              "drafts) <= S, 1 <= vocab <= %d, ld >= vocab (B=%d S=%d kq=%d slot0=%d vocab=%d ld=%d)", who,
              kSlotMaxSlots, kSampleMaxVocab, B, S, kq, slot0, vocab, ld);
    return -1;
  }
  if (!(temperature >= 0.f) || top_k < 0 || !(top_p > 0.f && top_p <= 1.f) || !(min_p >= 0.f && min_p <= 1.f) ||
      !(typical_p > 0.f && typical_p <= 1.f) || !(epsilon >= 0.f && epsilon < 1.f) || !(eta >= 0.f && eta < 1.f)) {
    set_error("%s: need temperature >= 0, top_k >= 0, 0 < top_p <= 1, 0 <= min_p <= 1, 0 < typical_p <= 1, 0 <= "
              "epsilon < 1, 0 <= eta < 1 (got %g, %d, %g, %g, %g, %g, %g)", who, temperature, top_k, top_p, min_p,
              typical_p, epsilon, eta);
    return -1;
  }
  if (n_suppress < 0 || n_suppress > kSampleMaxList || (n_suppress && !suppress)) {
    set_error("%s: a suppress list of at most %d ids (got %d)", who, kSampleMaxList, n_suppress);
    return -1;
  }
  if (!logits || !seeds || !lens || !emitted || !done || !nq) {
    set_error("%s: null pointer", who);
    return -1;
  }
  s = SampleArgs{logits, ld, vocab, temperature, top_p, top_k, seeds, nullptr, nullptr, min_new, suppress, n_suppress,
                 nullptr, 0, nullptr, nullptr, nullptr, 1, min_p, typical_p, epsilon, eta,
                 min_p > 0.f || typical_p < 1.f || epsilon > 0.f || eta > 0.f};
  return 0;
}

// the row of a sampling kernel in shared memory, once per device
template <class Kernel>
static int allow_row_smem(const char* who, Kernel kernel, std::once_flag* once, cudaError_t* setup) {
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kOpsMaxDevices) { set_error("%s: device %d out of range", who, dev); return -1; }
  std::call_once(once[dev], [&] {
    setup[dev] = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kSampleMaxVocab * (int)sizeof(float));
  });
  CUDA_TRY(setup[dev]);
  return 0;
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// h: bf16 [B, ld_h] (the first D columns used); w: bf16 [V, D] contiguous; out: fp32 [B, V] contiguous
int adapcc_lm_head_logits(const void* h, int ld_h, const void* w, int V, int D, void* out, int B, void* stream) {
  if (B < 1 || B > kHeadMaxB || V < 1 || D < 8 || D > kHeadMaxD || D % 8 != 0 || ld_h < D || ld_h % 8 != 0) {
    set_error("lm_head_logits: need 1 <= B <= %d, V >= 1, D a multiple of 8 in [8, %d], ld_h >= D and a multiple of "
              "8 (B=%d V=%d D=%d ld_h=%d)", kHeadMaxB, kHeadMaxD, B, V, D, ld_h);
    return -1;
  }
  if (((uintptr_t)h | (uintptr_t)w) & 15 || (uintptr_t)out & 3) {
    set_error("lm_head_logits: h and w must be 16-byte aligned, out 4-byte aligned");
    return -1;
  }
  static std::once_flag once[kOpsMaxDevices];
  static cudaError_t setup[kOpsMaxDevices];
  static int sms[kOpsMaxDevices];
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kOpsMaxDevices) { set_error("lm_head_logits: device %d out of range", dev); return -1; }
  std::call_once(once[dev], [&] {
    setup[dev] = cudaFuncSetAttribute(lm_head_logits_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kHeadMaxB * kHeadMaxD * 2);
    if (setup[dev] == cudaSuccess) setup[dev] = cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
  });
  CUDA_TRY(setup[dev]);
  const size_t smem = (size_t)B * D * 2;
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lm_head_logits_kernel, kHeadThreads, smem));
  const int rows_per_cta = (kHeadThreads / 32) * kHeadRows;
  const int grid = std::max(1, std::min((V + rows_per_cta - 1) / rows_per_cta, std::max(1, per_sm) * sms[dev]));
  lm_head_logits_kernel<<<grid, kHeadThreads, smem, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)h, ld_h, (const __nv_bfloat16*)w, V, D, (float*)out, B);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// logits: fp32 [B, ld]; seeds int64 [B]; pos int32 [B]; step: int32 [1] on the device; suppress / stop: int32 lists
// on the device (may be null when empty); done int32 [B]; next_ids int64 [B]; tokens int64 [B, max_new]; the
// filters are off at min_p = 0, typical_p = 1, epsilon = 0 and eta = 0
int adapcc_sample_tokens_filtered(const float* logits, int ld, int vocab, int B, float temperature, int top_k,
                                  float top_p, float min_p, float typical_p, float epsilon, float eta,
                                  const long long* seeds, const int* pos, int* step, int min_new, const int* suppress,
                                  int n_suppress, const int* stop, int n_stop, int* done, long long* next_ids,
                                  long long* tokens, int max_new, void* stream) {
  if (B < 1 || vocab < 1 || vocab > kSampleMaxVocab || ld < vocab || max_new < 1) {
    set_error("sample_tokens: need B >= 1, 1 <= vocab <= %d, ld >= vocab, max_new >= 1 (B=%d vocab=%d ld=%d "
              "max_new=%d)", kSampleMaxVocab, B, vocab, ld, max_new);
    return -1;
  }
  if (!(temperature >= 0.f) || top_k < 0 || !(top_p > 0.f && top_p <= 1.f)) {
    set_error("sample_tokens: need temperature >= 0, top_k >= 0, 0 < top_p <= 1 (got %g, %d, %g)", temperature, top_k,
              top_p);
    return -1;
  }
  if (!(min_p >= 0.f && min_p <= 1.f) || !(typical_p > 0.f && typical_p <= 1.f) || !(epsilon >= 0.f && epsilon < 1.f) ||
      !(eta >= 0.f && eta < 1.f)) {
    set_error("sample_tokens: need 0 <= min_p <= 1, 0 < typical_p <= 1, 0 <= epsilon < 1, 0 <= eta < 1 (got %g, %g, "
              "%g, %g)", min_p, typical_p, epsilon, eta);
    return -1;
  }
  if (n_suppress < 0 || n_stop < 0 || n_suppress > kSampleMaxList || n_stop > kSampleMaxList ||
      (n_suppress && !suppress) || (n_stop && !stop)) {
    set_error("sample_tokens: suppress / stop lists of at most %d ids (got %d, %d)", kSampleMaxList, n_suppress, n_stop);
    return -1;
  }
  if (!logits || !seeds || !pos || !step || !done || !next_ids || !tokens) {
    set_error("sample_tokens: null pointer");
    return -1;
  }
  static std::once_flag once[kOpsMaxDevices];
  static cudaError_t setup[kOpsMaxDevices];
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kOpsMaxDevices) { set_error("sample_tokens: device %d out of range", dev); return -1; }
  std::call_once(once[dev], [&] {
    setup[dev] = cudaFuncSetAttribute(sample_tokens_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kSampleMaxVocab * (int)sizeof(float));
  });
  CUDA_TRY(setup[dev]);
  SampleArgs a{logits, ld, vocab, temperature, top_p, top_k, seeds, pos, step, min_new, suppress, n_suppress,
               stop, n_stop, done, next_ids, tokens, max_new, min_p, typical_p, epsilon, eta,
               min_p > 0.f || typical_p < 1.f || epsilon > 0.f || eta > 0.f};
  cudaStream_t s = (cudaStream_t)stream;
  sample_tokens_kernel<<<B, kSampleThreads, (size_t)vocab * sizeof(float), s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  step_incr_kernel<<<1, 1, 0, s>>>(step);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// logits fp32 [B * kq, ld]; seeds int64 [B]; lens, emitted, done, nq int32 [B]; suppress: int32 list (null when
// empty). Verify draws: g int32 [B * S], ids = next = q = zq = null. Draft draws (kq = 1: draft j + 1 needs draft j):
// ids int64 [B * S] and next int64 [B], g null; optionally (temperature > 0) the draft's weights q fp32
// [B, S - 1, vocab] and totals zq fp32 [B, S - 1] of step slot0, both or neither.
int adapcc_sample_slots(const float* logits, int ld, int vocab, int B, int kq, int S, int slot0, float temperature,
                        int top_k, float top_p, float min_p, float typical_p, float epsilon, float eta,
                        const long long* seeds, const int* lens, const int* emitted, const int* done, const int* nq,
                        int min_new, const int* suppress, int n_suppress, int* g, long long* ids, long long* next,
                        float* q, float* zq, void* stream) {
  const bool draft = ids != nullptr;
  SampleArgs s;
  if (slot_args("sample_slots", logits, ld, vocab, B, kq, S, slot0, draft, temperature, top_k, top_p, min_p,
                typical_p, epsilon, eta, seeds, lens, emitted, done, nq, min_new, suppress, n_suppress, s))
    return -1;
  if ((draft ? (!next || g) : (!g || next)) || !q != !zq || (q && (!draft || !(temperature > 0.f)))) {
    set_error("sample_slots: not exactly one of g and (ids, next), or q / zq without the other, or not with a draft "
              "draw at temperature > 0");
    return -1;
  }
  static std::once_flag once[kOpsMaxDevices];
  static cudaError_t setup[kOpsMaxDevices];
  if (allow_row_smem("sample_slots", sample_slots_kernel, once, setup)) return -1;
  SlotArgs a{s, B, kq, S, slot0, lens, emitted, done, nq, g, ids, next, q, zq};
  sample_slots_kernel<<<dim3(kq, B), kSampleThreads, (size_t)vocab * sizeof(float), (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// Rejection-sampling verification of a round, one CTA per slot: logits fp32 [B * S, ld]; seeds int64 [B]; lens,
// emitted, done, nq int32 [B]; suppress int32 list (null when empty); ids int64 [B * S] (the drafts); q fp32
// [B, S - 1, vocab] and zq fp32 [B, S - 1] (sample_slots' draft weights); g, acc, last int32 [B * S]. temperature > 0.
int adapcc_spec_slots(const float* logits, int ld, int vocab, int B, int S, float temperature, int top_k, float top_p,
                      float min_p, float typical_p, float epsilon, float eta, const long long* seeds, const int* lens,
                      const int* emitted, const int* done, const int* nq, int min_new, const int* suppress,
                      int n_suppress, const long long* ids, const float* q, const float* zq, int* g, int* acc,
                      int* last, void* stream) {
  SampleArgs s;
  if (slot_args("spec_slots", logits, ld, vocab, B, S, S, 0, false, temperature, top_k, top_p, min_p, typical_p,
                epsilon, eta, seeds, lens, emitted, done, nq, min_new, suppress, n_suppress, s))
    return -1;
  if (S < 2 || !(temperature > 0.f)) {
    set_error("spec_slots: need S >= 2 and temperature > 0 (got %d, %g)", S, temperature);
    return -1;
  }
  if (!ids || !q || !zq || !g || !acc || !last) {
    set_error("spec_slots: null pointer");
    return -1;
  }
  static std::once_flag once[kOpsMaxDevices];
  static cudaError_t setup[kOpsMaxDevices];
  if (allow_row_smem("spec_slots", spec_slots_kernel, once, setup)) return -1;
  SlotArgs t{s, B, S, S, 0, lens, emitted, done, nq, g, nullptr, nullptr, nullptr, nullptr};
  SpecArgs a{t, ids, q, zq, acc, last};
  spec_slots_kernel<<<dim3(S, B), kSampleThreads, (size_t)vocab * sizeof(float), (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// adapcc_sample_tokens_filtered with every filter off
int adapcc_sample_tokens(const float* logits, int ld, int vocab, int B, float temperature, int top_k, float top_p,
                         const long long* seeds, const int* pos, int* step, int min_new, const int* suppress,
                         int n_suppress, const int* stop, int n_stop, int* done, long long* next_ids, long long* tokens,
                         int max_new, void* stream) {
  return adapcc_sample_tokens_filtered(logits, ld, vocab, B, temperature, top_k, top_p, 0.f, 1.f, 0.f, 0.f, seeds, pos,
                                       step, min_new, suppress, n_suppress, stop, n_stop, done, next_ids, tokens,
                                       max_new, stream);
}

}  // extern "C"
