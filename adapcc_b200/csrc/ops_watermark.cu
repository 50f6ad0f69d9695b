// Green-list watermarking for GPT-2 generation (Kirchenbauer et al. 2023): the bias applied to each row's fp32 logits
// after the repetition controls, inside the same CUDA graph replay, and the detector's counts. The definition, with
// the keyed Philox hash that picks the green ids, is in ops/watermark.py.
//
//   watermark_kernel       : a 2-D grid, kWmChunk vocabulary ids per CTA x one row per grid row, so one row alone
//                            still spreads over the SMs. Each CTA reads its row's length and the last w ids of the
//                            sequence the repetition-control kernel keeps (seq, lens), computes the lefthash seed once
//                            (thread 0, then shared memory) or loads the selfhash window, and each thread tests its
//                            ids, adding delta (one __fadd_rn) to the green ones. Only green logits are read and
//                            written. The grid depends on R and vocab only and nothing is read on the host, so one
//                            graph capture serves every token.
//   watermark_count_kernel : one CTA per row of a right-padded [B, T] id matrix, the row in shared memory. Every
//                            scored position computes its seed from the ids before it and tests its id; with
//                            ignore_repeated the position is dropped when an earlier scored position holds the same
//                            n-gram (the compare-against-earlier scheme of rule 3 in ops_repeats.cu). Per-thread
//                            integer counts are reduced in a fixed shuffle / shared-memory tree, no atomics, so the
//                            counts are exact.
#include <cmath>
#include <cstdint>

#include "common.h"
#include "philox.cuh"

namespace adapcc {

constexpr int kWmThreads = 128;
constexpr int kWmPerThread = 4;
constexpr int kWmChunk = kWmThreads * kWmPerThread;   // vocabulary ids per CTA
constexpr int kWmMaxWidth = 8;
constexpr int kWmMaxLen = 1024;                        // sequence positions per row of the bias (GPT-2's n_positions)
constexpr int kWmCountThreads = 256;
constexpr int kWmCountMaxLen = 8192;                   // ids per row of the detector
constexpr uint32_t kTagCtx = 0x57435458u, kTagSelf = 0x57534C46u, kTagGreen = 0x5747524Eu;

struct WatermarkKey {
  uint32_t k0, k1;             // K mod 2^32, K >> 32
  uint32_t theta;              // round(gamma 2^32)
  int selfhash, width;
};

__device__ __forceinline__ bool wm_green(uint32_t v, uint32_t s0, uint32_t s1, uint32_t theta) {
  return philox4(v, 0u, 0u, kTagGreen, s0, s1).x < theta;
}

// the lefthash seed after the w ids ending at ctx_end (ctx_end[-1] the last)
__device__ __forceinline__ uint2 wm_lefthash_seed(const int* ctx_end, const WatermarkKey& k) {
  uint32_t s0 = k.k0, s1 = k.k1;
  for (int i = 1; i <= k.width; ++i) {
    const uint4 o = philox4((uint32_t)ctx_end[-i], (uint32_t)i, 0u, kTagCtx, s0, s1);
    s0 = o.x;
    s1 = o.y;
  }
  return make_uint2(s0, s1);
}

__device__ __forceinline__ unsigned long long wm_self_h(uint32_t x, uint32_t v, const WatermarkKey& k) {
  const uint4 o = philox4(x, v, 0u, kTagSelf, k.k0, k.k1);
  return ((unsigned long long)o.y << 32) | o.x;
}

// the selfhash test of v with the w - 1 ids before it ending at win_end
__device__ __forceinline__ bool wm_self_green(uint32_t v, const int* win_end, const WatermarkKey& k) {
  unsigned long long m = wm_self_h(v, v, k);
  for (int i = 1; i < k.width; ++i) m = min(m, wm_self_h((uint32_t)win_end[-i], v, k));
  return wm_green(v, (uint32_t)m, (uint32_t)(m >> 32), k.theta);
}

struct WatermarkArgs {
  float* logits;               // [R, ld], the first `vocab` columns used
  int ld, vocab;
  const int* seq;              // [R, t_max]: row r's sequence is seq[r, :lens[r]]
  int t_max;
  const int* lens;             // [R]
  float delta;
  WatermarkKey key;
};

__global__ void __launch_bounds__(kWmThreads) watermark_kernel(const __grid_constant__ WatermarkArgs a) {
  __shared__ uint2 s_seed;
  __shared__ int s_win[kWmMaxWidth];
  const int r = blockIdx.y, tid = threadIdx.x;
  const WatermarkKey& k = a.key;
  const int L = min(max(a.lens[r], 0), a.t_max);
  if (L < k.width - k.selfhash) return;                // too short a sequence: the row is unchanged (uniform exit)
  const int* s = a.seq + (long long)r * a.t_max;
  if (k.selfhash) {
    if (tid < k.width - 1) s_win[tid] = s[L - k.width + 1 + tid];
  } else if (tid == 0) {
    s_seed = wm_lefthash_seed(s + L, k);
  }
  __syncthreads();
  float* l = a.logits + (long long)r * a.ld;
  const int v0 = blockIdx.x * kWmChunk + tid;
#pragma unroll
  for (int q = 0; q < kWmPerThread; ++q) {
    const int v = v0 + q * kWmThreads;
    if (v >= a.vocab) break;
    const bool g = k.selfhash ? wm_self_green((uint32_t)v, s_win + k.width - 1, k)
                              : wm_green((uint32_t)v, s_seed.x, s_seed.y, k.theta);
    if (g) l[v] = __fadd_rn(l[v], a.delta);
  }
}

struct WatermarkCountArgs {
  const int* ids;              // [B, T]
  int T;
  const int* lens;             // [B]
  const int* scored_from;      // [B]
  int ignore_repeated;
  int* counts;                 // [B, 2]: scored, green
  WatermarkKey key;
};

__global__ void __launch_bounds__(kWmCountThreads) watermark_count_kernel(const __grid_constant__ WatermarkCountArgs a) {
  extern __shared__ int s_ids[];                       // [T]
  __shared__ int s_part[2][kWmCountThreads / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const WatermarkKey& k = a.key;
  const int L = min(max(a.lens[b], 0), a.T);
  const int* row = a.ids + (long long)b * a.T;
  for (int j = tid; j < L; j += kWmCountThreads) s_ids[j] = row[j];
  __syncthreads();
  const int n = k.width + 1 - k.selfhash;              // the n-gram: the seed's window and the id
  const int lo = max(a.scored_from[b], k.width - k.selfhash);
  int scored = 0, green = 0;
  for (int j = lo + tid; j < L; j += kWmCountThreads) {
    if (a.ignore_repeated) {
      bool seen = false;
      for (int e = lo; e < j && !seen; ++e) {
        bool same = true;
        for (int q = 0; q < n && same; ++q) same = s_ids[e - q] == s_ids[j - q];
        seen = same;
      }
      if (seen) continue;
    }
    const uint32_t v = (uint32_t)s_ids[j];
    bool g;
    if (k.selfhash) {
      g = wm_self_green(v, s_ids + j, k);
    } else {
      const uint2 sd = wm_lefthash_seed(s_ids + j, k);
      g = wm_green(v, sd.x, sd.y, k.theta);
    }
    ++scored;
    green += g;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    scored += __shfl_xor_sync(0xffffffffu, scored, o);
    green += __shfl_xor_sync(0xffffffffu, green, o);
  }
  if ((tid & 31) == 0) {
    s_part[0][tid >> 5] = scored;
    s_part[1][tid >> 5] = green;
  }
  __syncthreads();
  if (tid == 0) {
    int ns = 0, ng = 0;
    for (int w = 0; w < kWmCountThreads / 32; ++w) {
      ns += s_part[0][w];
      ng += s_part[1][w];
    }
    a.counts[2 * b] = ns;
    a.counts[2 * b + 1] = ng;
  }
}

bool wm_key(WatermarkKey& k, int selfhash, int width, unsigned k0, unsigned k1, unsigned theta, const char* who) {
  if ((selfhash != 0 && selfhash != 1) || width < 1 || width > kWmMaxWidth || theta < 1u) {
    set_error("%s: need scheme 0 or 1, 1 <= width <= %d and theta >= 1 (got %d, %d, %u)", who, kWmMaxWidth, selfhash,
              width, theta);
    return false;
  }
  k = WatermarkKey{k0, k1, theta, selfhash, width};
  return true;
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// logits fp32 [R, ld]; seq int32 [R, t_max]; lens int32 [R]; selfhash 0 (lefthash) or 1; width w in [1, 8]; k0, k1 the
// hashing key's words; theta the green threshold; delta finite. In place, no host sync.
int adapcc_watermark(float* logits, int ld, int vocab, int R, const int* seq, int t_max, const int* lens, int selfhash,
                     int width, unsigned k0, unsigned k1, unsigned theta, float delta, void* stream) {
  if (R < 1 || R > 65535 || vocab < 1 || ld < vocab || t_max < 1 || t_max > kWmMaxLen) {
    set_error("watermark: need 1 <= R <= 65535, 1 <= vocab <= ld and 1 <= t_max <= %d (R=%d vocab=%d ld=%d t_max=%d)",
              kWmMaxLen, R, vocab, ld, t_max);
    return -1;
  }
  if (!logits || !seq || !lens) {
    set_error("watermark: null pointer");
    return -1;
  }
  if (!std::isfinite(delta)) {
    set_error("watermark: need a finite delta (got %g)", (double)delta);
    return -1;
  }
  WatermarkArgs a{logits, ld, vocab, seq, t_max, lens, delta, {}};
  if (!wm_key(a.key, selfhash, width, k0, k1, theta, "watermark")) return -1;
  const dim3 grid((vocab + kWmChunk - 1) / kWmChunk, R);
  watermark_kernel<<<grid, kWmThreads, 0, (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// ids int32 [B, T]; lens, scored_from int32 [B]; counts int32 [B, 2] out (scored, green); the key as above.
int adapcc_watermark_count(const int* ids, int T, int B, const int* lens, const int* scored_from, int selfhash,
                           int width, unsigned k0, unsigned k1, unsigned theta, int ignore_repeated, int* counts,
                           void* stream) {
  if (B < 1 || T < 1 || T > kWmCountMaxLen) {
    set_error("watermark_count: need B >= 1 and 1 <= T <= %d (B=%d T=%d)", kWmCountMaxLen, B, T);
    return -1;
  }
  if (!ids || !lens || !scored_from || !counts) {
    set_error("watermark_count: null pointer");
    return -1;
  }
  WatermarkCountArgs a{ids, T, lens, scored_from, ignore_repeated != 0, counts, {}};
  if (!wm_key(a.key, selfhash, width, k0, k1, theta, "watermark_count")) return -1;
  watermark_count_kernel<<<B, kWmCountThreads, (size_t)T * sizeof(int), (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
