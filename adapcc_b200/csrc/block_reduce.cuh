// The fixed-order block reduction of the 1024-thread row kernels that must give the same bits for a row whatever else
// is in the batch (ops_guidance.cu, ops_dola.cu): a 5-level shuffle butterfly adds (or takes the maximum of) the lanes
// of each warp, and every warp then combines the 32 warp partials with a second butterfly, so each thread gets the same
// result, computed in an order fixed by the thread layout alone. Every add is correctly rounded (__fadd_rn).
#pragma once

namespace adapcc {

constexpr int kRowThreads = 1024;
constexpr int kRowWarps = kRowThreads / 32;

// The block-wide max (kMax) or sum of both components of v; s_part holds kRowWarps entries.
template <bool kMax>
__device__ __forceinline__ float2 block_reduce_f2(float2 v, float2* s_part) {
  static_assert(kRowWarps == 32, "the second butterfly reads one warp partial per lane");
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float x = __shfl_xor_sync(0xffffffffu, v.x, o), y = __shfl_xor_sync(0xffffffffu, v.y, o);
    v = kMax ? make_float2(fmaxf(v.x, x), fmaxf(v.y, y)) : make_float2(__fadd_rn(v.x, x), __fadd_rn(v.y, y));
  }
  const int lane = threadIdx.x & 31;
  if (lane == 0) s_part[threadIdx.x >> 5] = v;
  __syncthreads();
  v = s_part[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float x = __shfl_xor_sync(0xffffffffu, v.x, o), y = __shfl_xor_sync(0xffffffffu, v.y, o);
    v = kMax ? make_float2(fmaxf(v.x, x), fmaxf(v.y, y)) : make_float2(__fadd_rn(v.x, x), __fadd_rn(v.y, y));
  }
  __syncthreads();                                    // s_part is free for the next reduction
  return v;
}

}  // namespace adapcc
