// Decode attention: one new token per row against a per-layer KV cache, split over the keys ("flash-decoding").
//
// GPT-2 generation with a cache runs, per layer and step, softmax(q . K[0..L]^T / sqrt(Dh)) . V[0..L] for every
// (row b, head h), L = lens[b] keys already cached plus the new one. That is a matrix-vector product over the cache:
// memory bound, and one (b, h) pair is far too little work for one CTA at B * H = 12. So the keys are cut into splits
// of kDecodeSplit keys, one CTA each:
//
//   split   : grid (splits of t_max, H, B). A CTA whose first key lies beyond L exits at once, so the launch depends
//             on t_max only and a captured decode step stays valid whatever the lengths are at replay. The CTA that
//             holds key L reads the new k / v from qkv, uses them for key L and then stores them into the cache at
//             position L: no CTA ever reads the new key back from the cache. Each CTA writes (max, sum, acc[Dh]) of its
//             keys in fp32 to `work`.
//   combine : one CTA per (b, h) rescales and adds the partials of splits 0, 1, ... in that order and writes bf16.
//
// Every sum runs in an order fixed by the thread layout (shuffle trees, shared-memory partials added in index order),
// never by arrival: a row's output bits depend on its q, its cached K / V and lens[b] only — not on B, the other rows
// or graph replay versus eager launch. lens is only read here; the caller advances it after the last layer.
// A row with lens[b] outside [0, t_max) is left alone: no cache write, output row zero.
#include <cuda_bf16.h>

#include <cmath>

#include "common.h"
#include "device_prims.cuh"

namespace adapcc {

// Keys per split. Split + combine timed back to back on an H100 80GB HBM3 (400 W), H = 12, Dh = 64, t_max = 1024,
// S = 64 / 128 / 256 at lens 128 / 512 / 1023: 9.3-9.9 / 10.6-11.3 / 10.7-15.7 us at B * H = 12 and 10.2-12.9 /
// 11.7-12.3 / 11.6-16.7 us at B * H = 96. 64 is fastest in five of the six cases (128 by 5 % at B * H = 96,
// lens 1023): at GPT-2's batch sizes more, shorter splits keep more SMs busy (DESIGN.md §4b).
constexpr int kDecodeSplit = 64;
constexpr int kDecodeThreads = 128;
constexpr int kDecodeMaxDh = 128;

struct DecodeArgs {
  const __nv_bfloat16* qkv;   // [B, qkv_stride]: q | k | v, each H * Dh
  __nv_bfloat16* k_cache;     // [B, H, t_max, Dh]
  __nv_bfloat16* v_cache;
  const int* lens;            // [B]
  float* work;                // [B, H, n_splits, Dh + 2]
  __nv_bfloat16* out;         // [B, H * Dh]
  int H, Dh, t_max, qkv_stride, n_splits;
};

template <int S>
__global__ void __launch_bounds__(kDecodeThreads)
decode_attn_split_kernel(const __grid_constant__ DecodeArgs a) {
  __shared__ float s_p[S];                          // scores, then exp(score - max)
  __shared__ float s_acc[kDecodeThreads * 8];       // per key group: its partial P.V
  __shared__ float s_red[kDecodeThreads / 32];
  const int s = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int L = a.lens[b];
  if (L < 0 || L >= a.t_max) return;
  const int j0 = s * S;
  if (j0 > L) return;
  const int n = min(S, L + 1 - j0);                 // keys of this split: j0 .. j0 + n - 1
  const int Dh = a.Dh, nvec = Dh >> 3, D = a.H * Dh;
  int G = 1;                                        // lanes per key: 8 elements (16 bytes) each, a power of two <= 16
  while (G < nvec) G <<= 1;
  const int tid = threadIdx.x, c = tid & (G - 1), grp = tid / G, ngrp = kDecodeThreads / G;
  const bool act = c < nvec;
  const __nv_bfloat16* qrow = a.qkv + (long long)b * a.qkv_stride + h * Dh;
  const long long head = ((long long)b * a.H + h) * a.t_max * Dh;
  __nv_bfloat16* kc = a.k_cache + head;
  __nv_bfloat16* vc = a.v_cache + head;
  const float scale = 1.0f / sqrtf((float)Dh);

  float q[8];
  if (act) unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(qrow + c * 8), q);
  // 1. scores: G lanes per key, a shuffle tree over the G partial dot products. The loop bound is the same for every
  //    lane of a warp, so the shuffles always see full warps.
#pragma unroll 4
  for (int base = 0; base < n; base += ngrp) {
    const int jj = base + grp, j = j0 + jj;
    float d = 0.f;
    if (act && jj < n) {
      float k[8];
      unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(j == L ? qrow + D + c * 8 : kc + (long long)j * Dh + c * 8), k);
#pragma unroll
      for (int e = 0; e < 8; ++e) d = fmaf(q[e], k[e], d);
    }
    for (int o = G >> 1; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (c == 0 && jj < n) s_p[jj] = d * scale;
  }
  __syncthreads();
  // 2. max and sum of exp over the split (max is exact in any order; the sum's order is fixed by the layout)
  const int lane = tid & 31, warp = tid >> 5;
  float m = -INFINITY;
  for (int jj = tid; jj < n; jj += kDecodeThreads) m = fmaxf(m, s_p[jj]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) s_red[warp] = m;
  __syncthreads();
  m = s_red[0];
#pragma unroll
  for (int w = 1; w < kDecodeThreads / 32; ++w) m = fmaxf(m, s_red[w]);
  __syncthreads();                                  // every thread has read s_red before it is reused
  float l = 0.f;
  for (int jj = tid; jj < n; jj += kDecodeThreads) {
    const float p = expf(s_p[jj] - m);
    s_p[jj] = p;
    l += p;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
  if (lane == 0) s_red[warp] = l;
  __syncthreads();
  // 3. P.V: key group grp takes keys grp, grp + ngrp, ...; lane c of the group owns elements 8c .. 8c + 7
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  if (act) {
#pragma unroll 4
    for (int jj = grp; jj < n; jj += ngrp) {
      const int j = j0 + jj;
      float v[8];
      unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(j == L ? qrow + 2 * D + c * 8 : vc + (long long)j * Dh + c * 8), v);
      const float p = s_p[jj];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = fmaf(p, v[e], acc[e]);
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) s_acc[grp * (G * 8) + c * 8 + e] = acc[e];
  __syncthreads();
  float* w = a.work + (((long long)b * a.H + h) * a.n_splits + s) * (Dh + 2);
  if (tid < Dh) {
    float r = 0.f;
    for (int g = 0; g < ngrp; ++g) r += s_acc[g * (G * 8) + tid];
    w[2 + tid] = r;
  }
  // the new token's k / v go into the cache last: this CTA read them from qkv above, no other CTA reads position L
  if (L < j0 + S && tid < nvec) {
    *reinterpret_cast<uint4*>(kc + (long long)L * Dh + tid * 8) = *reinterpret_cast<const uint4*>(qrow + D + tid * 8);
    *reinterpret_cast<uint4*>(vc + (long long)L * Dh + tid * 8) = *reinterpret_cast<const uint4*>(qrow + 2 * D + tid * 8);
  }
  if (tid == 0) {
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kDecodeThreads / 32; ++i) sum += s_red[i];
    w[0] = m;
    w[1] = sum;
  }
}

// one CTA per (h, b): out[b, h * Dh + t] = sum_s acc_s[t] e^(m_s - M) / sum_s l_s e^(m_s - M), splits in index order
template <int S>
__global__ void __launch_bounds__(kDecodeMaxDh)
decode_attn_combine_kernel(const __grid_constant__ DecodeArgs a) {
  const int h = blockIdx.x, b = blockIdx.y, t = threadIdx.x, Dh = a.Dh;
  if (t >= Dh) return;
  __nv_bfloat16* o = a.out + (long long)b * a.H * Dh + h * Dh;
  const int L = a.lens[b];
  if (L < 0 || L >= a.t_max) {
    o[t] = __float2bfloat16_rn(0.f);
    return;
  }
  const int ns = L / S + 1;
  const float* w = a.work + ((long long)b * a.H + h) * a.n_splits * (Dh + 2);
  float M = -INFINITY;
  for (int s = 0; s < ns; ++s) M = fmaxf(M, w[s * (Dh + 2)]);
  float l = 0.f, acc = 0.f;
  for (int s = 0; s < ns; ++s) {
    const float* ws = w + s * (Dh + 2);
    const float f = expf(ws[0] - M);
    l = fmaf(ws[1], f, l);
    acc = fmaf(ws[2 + t], f, acc);
  }
  o[t] = __float2bfloat16_rn(acc / l);
}

inline int decode_splits(int t_max) { return (t_max + kDecodeSplit - 1) / kDecodeSplit; }

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// fp32 elements of the `work` buffer adapcc_decode_attn needs for this shape
long long adapcc_decode_attn_work(int B, int H, int Dh, int t_max) {
  if (B < 1 || H < 1 || Dh < 1 || t_max < 1) return 0;
  return (long long)B * H * decode_splits(t_max) * (Dh + 2);
}

// qkv: bf16 [B, qkv_stride] (q | k | v of the new token, H * Dh each); k_cache / v_cache: bf16 [B, H, t_max, Dh];
// lens: int32 [B] (keys already cached; read only); out: bf16 [B, H * Dh]; work: fp32, adapcc_decode_attn_work elements
int adapcc_decode_attn(const void* qkv, void* k_cache, void* v_cache, const int* lens, void* out, int B, int H, int Dh,
                       int t_max, int qkv_stride, void* work, void* stream) {
  if (B < 1 || H < 1 || B > 65535 || H > 65535 || t_max < 1) {
    set_error("decode_attn: need 1 <= B, H <= 65535 and t_max >= 1 (B=%d H=%d t_max=%d)", B, H, t_max);
    return -1;
  }
  if (Dh < 8 || Dh > kDecodeMaxDh || Dh % 8 != 0) {
    set_error("decode_attn: head dim must be a multiple of 8 in [8, %d], got %d", kDecodeMaxDh, Dh);
    return -1;
  }
  if (qkv_stride < 3 * H * Dh || qkv_stride % 8 != 0) {
    set_error("decode_attn: qkv row stride %d must be a multiple of 8 and >= 3 * H * Dh = %d", qkv_stride, 3 * H * Dh);
    return -1;
  }
  if (((uintptr_t)qkv | (uintptr_t)k_cache | (uintptr_t)v_cache | (uintptr_t)out) & 15) {
    set_error("decode_attn: qkv, caches and output must be 16-byte aligned");
    return -1;
  }
  if (!lens || !work || ((uintptr_t)lens | (uintptr_t)work) & 3) {
    set_error("decode_attn: lens and work must be non-null and 4-byte aligned");
    return -1;
  }
  DecodeArgs a{};
  a.qkv = (const __nv_bfloat16*)qkv;
  a.k_cache = (__nv_bfloat16*)k_cache;
  a.v_cache = (__nv_bfloat16*)v_cache;
  a.lens = lens;
  a.work = (float*)work;
  a.out = (__nv_bfloat16*)out;
  a.H = H;
  a.Dh = Dh;
  a.t_max = t_max;
  a.qkv_stride = qkv_stride;
  a.n_splits = decode_splits(t_max);
  cudaStream_t s = (cudaStream_t)stream;
  decode_attn_split_kernel<kDecodeSplit><<<dim3(a.n_splits, H, B), kDecodeThreads, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  decode_attn_combine_kernel<kDecodeSplit><<<dim3(H, B), kDecodeMaxDh, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
