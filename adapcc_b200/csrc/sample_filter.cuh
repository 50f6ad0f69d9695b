// The row prologue and filter of the on-device sampler (ops_sample.cu) and of sampled beam search (ops_beam.cu): one
// CTA of 1024 threads holds a row's values x_i in shared memory. Top-h (entropy-bounded truncation over the row's 100
// largest values) removes ids in place first; the top-k threshold and the top-p cut-off are found by bisection
// over the order-preserving integer encoding of x (counts for top-k, masses for top-p), with no sort; the truncation
// filters after top-p (min-p, typical, epsilon, eta) remove ids from the row in place. Also the counter convention
// of the Philox4x32-10 draws both samplers make (the generator is philox.cuh), and the block reductions in their
// fixed order (per-thread loops in index order, shuffle trees, the 32 warp partials added by the same shuffle tree in
// warp order).
#pragma once

#include <cmath>
#include <cstdint>

#include "philox.cuh"

namespace adapcc {

constexpr int kSampleThreads = 1024;
constexpr int kSampleWarps = kSampleThreads / 32;
constexpr int kSampleMaxVocab = 56 * 1024;   // x of a row in shared memory: 224 KB
constexpr uint32_t kNegInfKey = 0x007FFFFFu; // key(-inf): ids at -inf (removed ones included) are never candidates

constexpr int kTopHN = 100;                   // top-h looks at the row's 100 largest values (HuggingFace's top_n)

// The truncation filters after top-p (DESIGN.md §4a), each off at its neutral value. min_keep is HuggingFace's
// min_tokens_to_keep: 1 in the sampler and stochastic beam search, max(2, 1 + n_stop) in beam sampling.
struct FilterArgs {
  float min_p, typical_p, epsilon, eta;
  int min_keep;
  __host__ __device__ bool on() const { return min_p > 0.f || typical_p < 1.f || epsilon > 0.f || eta > 0.f; }
};

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
  float top_h;               // top-h before top-k (0: off)
  FilterArgs f;              // the truncation filters after top-p (min_keep 1)
};

// order-preserving: a < b (floats, no NaN) <=> key(a) < key(b)
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// counter (c0, 0, 0, 0): a token draw uses word 0; rejection-sampling verification uses word 1 for the acceptance
// test and word 2 for the residual draw, so neither depends on the draw that produced the draft
__device__ __forceinline__ uint4 philox4(uint32_t c0, uint32_t k0, uint32_t k1) {
  return philox4(c0, 0u, 0u, 0u, k0, k1);
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

// The start of every sampled row, by the whole CTA: s_x[i] = x_i = l_i / T for the logits row l (l_i itself at T = 0),
// then, while step < min_new, the suppressed ids at -inf (the min-length rule comes before any filtering). Returns the
// number of finite ids; `best` gets their block maximum (key << 32) | ~i, a tie to the lower id. The sampler's draw_row
// and sampled beam search's row kernels all begin here, so their rows are the same bits.
__device__ __forceinline__ int row_prologue(float* s_x, SampleSmem& sm, const float* l, int V, float T, int step,
                                            int min_new, const int* suppress, int n_suppress,
                                            unsigned long long& best) {
  const int tid = threadIdx.x;
  for (int i = tid; i < V; i += kSampleThreads) s_x[i] = T == 0.f ? l[i] : __fdiv_rn(l[i], T);
  __syncthreads();
  if (step < min_new) {
    for (int j = tid; j < n_suppress; j += kSampleThreads) {
      const int id = suppress[j];
      if (id >= 0 && id < V) s_x[id] = -INFINITY;
    }
    __syncthreads();
  }
  best = 0;
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
  return present;
}

// The k-th largest key f2key(s_x[i]) counted with multiplicity, for 0 < k < (number of finite ids); mkey is the
// largest. Invariant: count(key >= lo) >= k > count(key >= hi). Stops early once no key lies strictly between lo and
// hi: lo is then the k-th largest key.
__device__ __forceinline__ uint32_t kth_key(const float* s_x, SampleSmem& sm, int V, int k, uint32_t mkey) {
  const int tid = threadIdx.x;
  uint32_t lo = kNegInfKey + 1, hi = mkey + 1;
  int cnt_hi = 0;
  while (hi - lo > 1) {
    const uint32_t mid = lo + (hi - lo) / 2;
    int c = 0, nl = 0, nh = 0;
    for (int i = tid; i < V; i += kSampleThreads) {
      const uint32_t key = f2key(s_x[i]);
      if (key > lo && key < hi) {
        c += key >= mid;
        nl += key < mid;
        nh += key > mid;
      }
    }
    float f = 0.f;
    block_sum(sm, f, c, nl, nh);
    if (cnt_hi + c >= k) {
      lo = mid;
      if (nh == 0) break;
    } else {
      hi = mid;
      cnt_hi += c;
      if (nl == 0) break;
    }
  }
  return lo;
}

// Top-k, then top-p, over the row's `present` finite values (mkey: the largest key, m: its value). Returns tau: the
// kept ids are those with f2key(s_x[i]) >= tau. top-k keeps the k' = max(top_k, min_keep) largest values (top_k = 0:
// off); top-p keeps i iff the weight of the kept values strictly larger than x_i is <= top_p Z, and always the
// min_keep largest values. Tied values are kept or dropped together. The sampler passes min_keep = 1, beam sampling
// max(2, 1 + n_stop) (HuggingFace's min_tokens_to_keep with beams).
__device__ __forceinline__ uint32_t row_tau(const float* s_x, SampleSmem& sm, int V, int top_k, float top_p,
                                            int min_keep, int present, uint32_t mkey, float m) {
  const int tid = threadIdx.x;
  uint32_t tau = kNegInfKey + 1;                    // candidates are the ids with key >= tau
  const int k = top_k > 0 && top_k < min_keep ? min_keep : top_k;
  if (k > 0 && k < present) tau = kth_key(s_x, sm, V, k, mkey);
  float z = 0.f;
  int u0 = 0, u1 = 0, u2 = 0;
  for (int i = tid; i < V; i += kSampleThreads) {
    const float x = s_x[i];
    if (f2key(x) >= tau) z += expf(x - m);
  }
  block_sum(sm, z, u0, u1, u2);
  const float pz = top_p * z;
  if (top_p < 1.f && pz < z) {
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
        const uint32_t key = f2key(x);
        if (key > lo && key <= hi) {
          if (key > mid) s += expf(x - m);
          nl += key < mid;
          nh += key > mid && key < hi;
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
    // the min_keep largest values stay (the largest one always does)
    if (min_keep > 1) tau = min(tau, min_keep < present ? kth_key(s_x, sm, V, min_keep, mkey) : kNegInfKey + 1);
  }
  return tau;
}

// The truncation filters after top-p, in HuggingFace's order: min-p, typical, epsilon, eta. The kept set {key >= tau}
// is first written into the row (-inf for every other id), and each filter removes ids the same way, so afterwards
// the survivors are exactly the finite ids. A filter that is off costs nothing; p_i = e_i / Z over the current
// survivors, with e_i = exp(x_i - m) and m the row maximum, which top-k, top-p and min-p always keep. Every filter
// also keeps f.min_keep ids (HuggingFace's min_tokens_to_keep): min-p, epsilon and eta the min_keep largest values,
// typical the min_keep smallest deviations, ties together. At min_keep = 1 that adds no pass and changes no bits.
static __device__ __noinline__ void filter_row(float* s_x, SampleSmem& sm, int V, FilterArgs f, uint32_t tau, float m,
                                               uint32_t mkey) {
  const int tid = threadIdx.x;
  // materialise top-k / top-p; min-p keeps e_i >= min_p, i.e. p_i >= min_p p_max
  const bool mp = f.min_p > 0.f, mp_floor = mp && f.min_keep > 1;
  for (int i = tid; i < V; i += kSampleThreads) {
    const float x = s_x[i];
    if (f2key(x) < tau || (mp && !mp_floor && expf(x - m) < f.min_p)) s_x[i] = -INFINITY;
  }
  if (mp_floor) {                                   // min-p over the materialised survivors, above their floor
    const uint32_t kk = kth_key(s_x, sm, V, f.min_keep, mkey);
    for (int i = tid; i < V; i += kSampleThreads) {
      const float x = s_x[i];
      if (x != -INFINITY && expf(x - m) < f.min_p && f2key(x) < kk) s_x[i] = -INFINITY;
    }
  }
  uint32_t kmax = mkey;                             // key of the largest survivor: typical may remove the maximum
  if (f.typical_p < 1.f) {
    // H = log Z - mu with mu = sum p_i (x_i - m), so the deviation |-log p_i - H| is d_i = |(x_i - m) - mu|. The
    // cut-off d* is the smallest d with G(d) = (mass of d_i <= d) >= p Z and N(d) = (count of d_i <= d) >= min_keep,
    // found by bisection over the order-preserving keys of d. Invariant: not both at lo, both at hi; G(lo) and N(lo)
    // are carried and each pass adds the mass and count in (lo, mid]. Once no key lies strictly inside the half that
    // holds d*, that half's upper end is d*. hi starts at key(+inf), so rounding that keeps every G below p Z keeps
    // every id. With min_keep = 1, G >= p Z > 0 already implies N >= 1.
    float z, s1;
    row_moments(s_x, sm, V, m, z, s1);
    const float mu = s1 / z, pz = f.typical_p * z;
    uint32_t lo = f2key(0.f) - 1, hi = f2key(INFINITY);
    float g_lo = 0.f;
    int n_lo = 0;
    while (hi - lo > 1) {
      const uint32_t mid = lo + (hi - lo) / 2;
      float s = 0.f;
      int nl = 0, nh = 0, cnt = 0;
      for (int i = tid; i < V; i += kSampleThreads) {
        const float x = s_x[i];
        if (x != -INFINITY) {
          const uint32_t k = f2key(fabsf((x - m) - mu));
          if (k > lo && k <= hi) {
            if (k <= mid) {
              s += expf(x - m);
              ++cnt;
            }
            nl += k < mid;
            nh += k > mid && k < hi;
          }
        }
      }
      block_sum(sm, s, nl, nh, cnt);
      const float g = g_lo + s;
      if (g >= pz && n_lo + cnt >= f.min_keep) {
        hi = mid;
        if (nl == 0) break;
      } else {
        lo = mid;
        g_lo = g;
        n_lo += cnt;
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
  // the min_keep largest survivors (ties together) as well, which only matters when fewer reach the threshold
  for (int e = 0; e < 2; ++e) {
    const float c = e == 0 ? f.epsilon : f.eta;
    if (!(c > 0.f)) continue;
    float z, s1;
    row_moments(s_x, sm, V, m, z, s1);
    const float t = e == 0 ? c * z : fminf(c * z, sqrtf(c) * expf(s1 / z));
    const uint32_t kk = f.min_keep > 1 ? kth_key(s_x, sm, V, f.min_keep, kmax) : kmax;
    for (int i = tid; i < V; i += kSampleThreads) {
      const float x = s_x[i];
      if (x != -INFINITY && expf(x - m) < t && f2key(x) < kk) s_x[i] = -INFINITY;
    }
  }
  __syncthreads();                                  // the draw reads other threads' ids
}

// The M best keys f2key(s_x[i]) of a row of 1024 threads (all finite ones when there are at most M; else those above
// the M-th largest key, and of the ones equal to it the lowest ids) as (key << 32) | ~i, best first: emit(r, v) for
// r < M, v = 0 past the count. s_sel holds M entries. Returns the largest key.
template <class Emit>
__device__ __forceinline__ uint32_t row_best_keys(const float* s_x, SampleSmem& sm, int V, int M,
                                                  unsigned long long* s_sel, int* s_n, Emit emit) {
  const int tid = threadIdx.x;
  unsigned long long best = 0;
  int cnt = 0, z1 = 0, z2 = 0;
  float fz = 0.f;
  for (int i = tid; i < V; i += kSampleThreads) {
    const uint32_t k = f2key(s_x[i]);
    if (k > kNegInfKey) {
      ++cnt;
      best = max(best, (unsigned long long)k);
    }
  }
  best = block_max(sm, best);
  block_sum(sm, fz, cnt, z1, z2);
  uint32_t thr = kNegInfKey;                          // taken: key > thr, or key == thr and id < cut
  int cut = 0;
  if (cnt > M) {
    thr = kth_key(s_x, sm, V, M, (uint32_t)best);
    int gt = 0, eq = 0, unused = 0;
    for (int i = tid; i < V; i += kSampleThreads) {
      const uint32_t k = f2key(s_x[i]);
      gt += k > thr;
      eq += k == thr;
    }
    block_sum(sm, fz, gt, eq, unused);
    const int need = M - gt;
    cut = V;
    if (eq > need) {                                  // tied at the M-th key: the smallest cut with need ids below it
      int lo = 0, hi = V;
      while (hi - lo > 1) {
        const int mid = lo + (hi - lo) / 2;
        int c = 0, u0 = 0, u1 = 0;
        for (int i = tid; i < mid; i += kSampleThreads) c += f2key(s_x[i]) == thr;
        block_sum(sm, fz, c, u0, u1);
        if (c >= need) hi = mid;
        else lo = mid;
      }
      cut = hi;
    }
  }
  if (tid == 0) *s_n = 0;
  __syncthreads();
  for (int i = tid; i < V; i += kSampleThreads) {
    const uint32_t k = f2key(s_x[i]);
    if (k > thr || (k == thr && i < cut)) s_sel[atomicAdd(s_n, 1)] = ((unsigned long long)k << 32) |
                                                                     (0xFFFFFFFFu - (uint32_t)i);
  }
  __syncthreads();
  const int n = *s_n;
  // best first: a key's place is the number of larger keys (the keys are distinct)
  for (int e = tid; e < M; e += kSampleThreads) {
    if (e >= n) {
      emit(e, 0ull);
      continue;
    }
    const unsigned long long v = s_sel[e];
    int r = 0;
    for (int f = 0; f < n; ++f) r += s_sel[f] > v;
    emit(r, v);
  }
  return (uint32_t)best;
}

// Top-h (HuggingFace's TopHLogitsWarper, entropy-bounded truncation), after row_prologue and before row_tau, on the
// row's `present` > 0 finite values with maximum m. The n = min(100, present) largest, ordered by value descending with
// ties to the lower id (row_best_keys), have p_r = e_r / Z over those n and h_r = -p_r log p_r = p_r (log Z - (x_r -
// m)); the longest prefix whose running sum of h_r is <= top_h H (H = sum of all n h_r) survives, and at least the
// first min(min_keep, n) entries (the row maximum always). Every other id goes to -inf; returns the survivors' count.
// The sums run on warp 0: lane l owns entries 4l .. 4l + 3 and adds them in order, a shuffle tree adds the lanes for
// Z and H and a shuffle scan for the running sums, so the order is fixed. s_sel holds kTopHN entries.
static __device__ __noinline__ int top_h_row(float* s_x, SampleSmem& sm, int V, int present, float m, float top_h,
                                             int min_keep, unsigned long long* s_sel, int* s_n) {
  const int tid = threadIdx.x, n = min(present, kTopHN);
  int my_r = -1;
  unsigned long long my_v = 0;
  row_best_keys(s_x, sm, V, kTopHN, s_sel, s_n, [&](int r, unsigned long long v) {
    my_r = r;
    my_v = v;
  });
  __syncthreads();                                  // every rank is counted before the entries move to their places
  if (my_r >= 0) s_sel[my_r] = my_v;
  __syncthreads();
  if (tid < 32) {
    const int lane = tid;
    float y[4], e[4], z = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int r = 4 * lane + q;
      y[q] = r < n ? key2f((uint32_t)(s_sel[r] >> 32)) - m : 0.f;
      e[q] = r < n ? expf(y[q]) : 0.f;
      z += e[q];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    const float lz = logf(z);
    float h[4], hl = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      h[q] = __fdiv_rn(e[q], z) * (lz - y[q]);
      hl += h[q];
    }
    float H = hl, inc = hl;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) H += __shfl_xor_sync(0xffffffffu, H, o);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    float run = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) run = 0.f;
    const float tau = top_h * H;
    int c = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      run += h[q];
      c += 4 * lane + q < n && run <= tau;          // a prefix: the running sum never falls
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) *s_n = max(c, min(max(min_keep, 1), n));
  }
  __syncthreads();
  const int c = *s_n;
  const unsigned long long last = s_sel[c - 1];
  for (int i = tid; i < V; i += kSampleThreads) {
    const uint32_t k = f2key(s_x[i]);
    if (k > kNegInfKey && (((unsigned long long)k << 32) | (0xFFFFFFFFu - (uint32_t)i)) < last) s_x[i] = -INFINITY;
  }
  __syncthreads();                                  // the draw and row_best_keys read other threads' ids
  return c;
}

}  // namespace adapcc
