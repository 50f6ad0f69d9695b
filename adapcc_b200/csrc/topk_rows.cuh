// The per-row top-N pass of beam selection (ops_beam.cu) and contrastive search (ops_contrastive.cu): one 512-thread
// CTA reads a logits row from global memory and finds its N best candidates as 64-bit keys (order-preserving float
// bits of the ranked value, then the inverted id, so a tie goes to the lower id). Each thread keeps its four best keys
// in registers; each warp takes its N best by N rounds of a warp maximum (a lane that runs out of kept keys rescans its
// ids below the last winner), and warp 0 merges the 16 warp lists into the row's N best.
//
// The ranked value is c_i = s + ((l_i - m) - lz) (beam search: a beam's candidate score) or, with kRaw, the logit l_i
// itself (contrastive search ranks by logit). Every fp32 sum runs in an order fixed by the thread layout.
#pragma once

#include <cmath>
#include <cstdint>

namespace adapcc {

constexpr int kBeamThreads = 512;
constexpr int kBeamWarps = kBeamThreads / 32;
constexpr uint32_t kBeamNegInfKey = 0x007FFFFFu;      // key(-inf): candidates at -inf are never taken

__device__ __forceinline__ uint32_t beam_f2key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float beam_key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// every thread gets the same bits: a shuffle tree per warp, then the warp partials by the same tree in warp order
__device__ __forceinline__ float beam_block_sum(float* red, float v) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = lane < kBeamWarps ? red[lane] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float beam_block_max(float* red, float v) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = lane < kBeamWarps ? red[lane] : -INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

struct RowView {
  const float* l;
  const uint32_t* bits;        // removed ids (null: none)
  int V;
  float s, m, lz;
  __device__ __forceinline__ bool removed(int i) const { return bits && ((bits[i >> 5] >> (i & 31)) & 1u); }
};

// this thread's four best candidate keys strictly below `bound`, best first (0: none)
template <bool kRaw>
__device__ __forceinline__ void scan_top4(const RowView& rv, unsigned long long bound, unsigned long long (&t)[4]) {
  t[0] = t[1] = t[2] = t[3] = 0ull;
  for (int i = threadIdx.x; i < rv.V; i += kBeamThreads) {
    if (rv.removed(i)) continue;
    const float c = kRaw ? __ldg(rv.l + i) : rv.s + ((__ldg(rv.l + i) - rv.m) - rv.lz);
    const uint32_t k32 = beam_f2key(c);
    if (k32 <= kBeamNegInfKey) continue;
    const unsigned long long key = ((unsigned long long)k32 << 32) | (0xFFFFFFFFu - (uint32_t)i);
    if (key >= bound || key <= t[3]) continue;
    t[3] = key;
#pragma unroll
    for (int q = 3; q > 0; --q)
      if (t[q] > t[q - 1]) {
        const unsigned long long x = t[q];
        t[q] = t[q - 1];
        t[q - 1] = x;
      }
  }
}

// The row's N best keys, best first, into out[0..N) (0: fewer than N candidates), written by lane 0 of warp 0.
// s_top: kBeamWarps * N zeroed shared entries (a barrier after zeroing them precedes the call); every thread calls it.
template <bool kRaw>
__device__ __forceinline__ void row_top_keys(const RowView& rv, int N, unsigned long long* s_top,
                                             unsigned long long* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long t[4];
  scan_top4<kRaw>(rv, ~0ull, t);
  bool more = t[3] != 0ull;                           // four kept: the thread may hold further candidates
  for (int r = 0; r < N; ++r) {
    const unsigned long long w = warp_max_u64(t[0]);
    if (w == 0ull) break;
    if (lane == 0) s_top[warp * N + r] = w;
    if (t[0] == w) {
      t[0] = t[1];
      t[1] = t[2];
      t[2] = t[3];
      t[3] = 0ull;
      if (t[0] == 0ull && more) {
        scan_top4<kRaw>(rv, w, t);
        more = t[3] != 0ull;
      }
    }
  }
  __syncthreads();
  if (warp == 0) {
    unsigned long long bound = ~0ull;
    for (int r = 0; r < N; ++r) {
      unsigned long long best = 0ull;
      for (int e = lane; e < kBeamWarps * N; e += 32) {
        const unsigned long long v = s_top[e];
        if (v < bound && v > best) best = v;
      }
      best = warp_max_u64(best);
      if (lane == 0) out[r] = best;
      bound = best;
    }
  }
}

}  // namespace adapcc
