// Training dropout masks as a pure function of (seed, step, site, row, column): the definition of ops/dropout.py
// (DESIGN.md §4a), shared by the fused add-LayerNorm (ops_norm.cu), the fused embedding sum (ops_embed.cu) and the
// stand-alone kernel (ops_dropout.cu). Nothing is stored for the backward: it evaluates the same function again.
//
// One Philox4x32-10 call covers the 8 consecutive columns 8 vec .. 8 vec + 7 of one row (one 16-byte bf16 vector):
// counter (row, vec, site, step), key = the 64-bit seed as (low, high) words. Column 8 vec + i uses 16-bit half i of
// the four output words: half 2 j is the LOW half of word j, half 2 j + 1 its HIGH half. An element is kept iff its
// half >= thr = round(p * 65536), and a kept element is multiplied by scale = 65536 / (65536 - thr) in fp32.
#pragma once

#include <cstdint>

#include "common.h"
#include "philox.cuh"

namespace adapcc {

struct DropArgs {
  const long long* seed;     // [1] on the device
  const int* step;           // [1] on the device: the training forwards run so far
  uint32_t site, thr;
  float scale;
};

// host side: the launch arguments of an entry point `who`, checked (seed int64 [1] and step int32 [1] on the device)
inline bool drop_args(const char* who, const void* seed, const void* step, int site, unsigned int thr, float scale,
                      DropArgs* out) {
  if (!seed || !step || site < 0 || thr > 65535u) {
    set_error("%s: seed and step are required, site >= 0, thr <= 65535", who);
    return false;
  }
  *out = DropArgs{(const long long*)seed, (const int*)step, (uint32_t)site, thr, scale};
  return true;
}

struct DropKey {
  uint32_t k0, k1, step;
};

__device__ __forceinline__ DropKey drop_key(const DropArgs& a) {
  const unsigned long long s = (unsigned long long)*a.seed;
  return DropKey{(uint32_t)s, (uint32_t)(s >> 32), (uint32_t)*a.step};
}

// bit i of the result: column 8 vec + i of `row` is kept
__device__ __forceinline__ uint32_t drop_keep8(uint32_t row, uint32_t vec, const DropArgs& a, const DropKey& k) {
  const uint4 w = philox4(row, vec, a.site, k.step, k.k0, k.k1);
  const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
  uint32_t keep = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    keep |= (uint32_t)((ws[j] & 0xffffu) >= a.thr) << (2 * j);
    keep |= (uint32_t)((ws[j] >> 16) >= a.thr) << (2 * j + 1);
  }
  return keep;
}

// f[i] = keep_i ? f[i] * scale : 0. The product is rounded on its own (never contracted into a following add), so the
// result is the fp32 value a reference gets from mask * scale * x.
__device__ __forceinline__ void drop_apply(float (&f)[8], uint32_t keep, float scale) {
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = (keep >> i) & 1u ? __fmul_rn(f[i], scale) : 0.f;
}

}  // namespace adapcc
