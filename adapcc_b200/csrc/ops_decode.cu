// Decode attention: new tokens against a per-layer KV cache, split over the keys ("flash-decoding"). One split kernel
// and one combine kernel serve decode_attn (one new token per row), cand_attn (contrastive search: k candidates of one
// position per row, the cache read only) and verify_attn (prompt lookup: a row's last token and its drafts at
// consecutive positions).
//
// GPT-2 generation with a cache runs, per layer and step, softmax(q . K[0..P]^T / sqrt(Dh)) . V[0..P] for every
// (query, head h): a matrix-vector product over the cache, memory bound, and one (query, h) pair is far too little
// work for one CTA at B * H = 12. So the keys are cut into splits of kDecodeSplit keys, one CTA each.
//
// Cache row b has kq queries; query j of row b is row b * kq + j of qkv, out and work, and L = lens[b].
//   real queries : none if L is outside [0, t_max) (nothing written, every output of the row zero); otherwise all kq,
//                  or, with nq, min(nq[b], kq, t_max - L) (at least 0). A pad query's output is zero.
//   position     : query j sits at P = L + chain * j (chain 0: decode and candidates; 1: verify) and attends keys 0..P.
//   keys, values : position p < L from the cache; p >= L from the c_attn output of query j - (P - p) (with chain 0 the
//                  query itself, with chain 1 slot p - L). No CTA ever reads a position >= L from the cache.
//   new k / v    : the CTA whose split holds P stores query j's, after its reads: into side_k / side_v row b * kq + j
//                  when side buffers are given (the cache stays read only), otherwise into the cache at P.
//
//   split   : grid (splits of t_max, H, B). A CTA whose first key lies beyond every real query's P exits at once, so
//             the launch depends on t_max, B and kq only and a captured step stays valid whatever the lengths are at
//             replay. The CTA runs its row's real queries one after the other and writes (max, sum, acc[Dh]) of each
//             query's keys in fp32 to `work`. With kq > 1 or side buffers it first stages its split's cached K / V
//             tile in shared memory, so every cached element is read once per CTA for all kq queries; otherwise (one
//             query, decode_attn and verify_attn at k = 0) it reads the cache directly.
//   combine : grid (H, kq, B), one CTA per (head, query): rescales and adds the partials of splits
//             0 .. P / kDecodeSplit in that order and writes bf16.
//
// Every sum runs in an order fixed by the thread layout (shuffle trees, shared-memory partials added in index order),
// never by arrival: a query's output bits depend on its q, the keys and values it attends and P only, not on B, kq,
// the other queries, the staging or graph replay versus eager launch. So a candidate or a verify slot is
// bit-identical to decode_attn at the same keys. lens and nq are only read here.
//
// fp8 cache (decode_attn with k_scale / v_scale): every cached key and value vector is Dh e4m3 bytes q and an fp32
// power-of-two scale 2^e, read as fl32(q) * 2^e (ops/kvcache.py, DESIGN.md §4a). Scaling by a power of two commutes
// with every fp32 product and sum, so the kernel multiplies a key's dot product by its scale once and folds the value's
// scale into its weight p, and gives the bits of the bf16 kernel on a bf16 cache holding the dequantized values. The
// new token attends to its own k / v unquantized (from qkv); the CTA that stores them quantizes them.
#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include <cmath>
#include <cstdint>
#include <type_traits>

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
constexpr int kDecodeMaxQueries = 16;               // kq: contrastive candidates, prompt-lookup slots

struct DecodeArgs {
  const __nv_bfloat16* qkv;   // [B * kq, qkv_stride]: q | k | v of each query, H * Dh each
  __nv_bfloat16* k_cache;     // [B, H, t_max, Dh]; never written when side_k is given
  __nv_bfloat16* v_cache;
  const int* lens;            // [B]
  const int* nq;              // [B]: real queries of each row (null: all kq)
  float* work;                // [B * kq, H, n_splits, Dh + 2]
  __nv_bfloat16* out;         // [B * kq, H * Dh]
  __nv_bfloat16* side_k;      // [B * kq, H * Dh]: each query's new key (null: it goes into the cache)
  __nv_bfloat16* side_v;
  int kq, chain, H, Dh, t_max, qkv_stride, n_splits;
  float* k_scale;             // [B, H, t_max]: with an fp8 cache (k_cache / v_cache then hold e4m3 bytes); else null
  float* v_scale;
};

// fl32 of 8 e4m3 bytes (exact: e4m3 -> f16 -> f32)
__device__ __forceinline__ void unpack_fp8(uint2 v, float* f) {
  const uint32_t w[2] = {v.x, v.y};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w[i >> 1] >> (16 * (i & 1))), __NV_E4M3);
    const float2 t = __half22float2(__half2(h));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

// Quantizes one bf16 vector of 8 * nvec elements (ops/kvcache.py): lane c < nvec of the 16-lane group holds elements
// 8c .. 8c + 7 in x (own) and writes their bytes to q + 8c; lane 0 writes the scale. Every lane of the warp calls it
// (the group's max is a shuffle). amax is the largest |x| as bits: NaN > inf > any finite value, so the max is exact
// in any order and a non-finite vector is seen whatever its other elements are.
__device__ __forceinline__ void quantize_fp8(const uint4 x4, bool own, int c, uint8_t* q, float* scale) {
  float x[8];
  unpack<__nv_bfloat16>(x4, x);
  unsigned m = 0;
  if (own) {
#pragma unroll
    for (int e = 0; e < 8; ++e) m = max(m, __float_as_uint(fabsf(x[e])));
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  const float amax = __uint_as_float(m);
  const bool finite = amax <= 3.402823466e38f;
  const int ex = finite && amax > 0.f ? ilogbf(amax) - 7 : 0;       // amax * 2^-ex in [128, 256)
  if (!own) return;
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = make_float2(ldexpf(x[2 * i], -ex), ldexpf(x[2 * i + 1], -ex));
    w[i] = finite ? (uint32_t)__nv_cvt_float2_to_fp8x2(t, __NV_SATFINITE, __NV_E4M3) : 0u;
  }
  *reinterpret_cast<uint2*>(q + c * 8) = make_uint2(w[0] | (w[1] << 16), w[2] | (w[3] << 16));
  if (c == 0) *scale = finite ? ldexpf(1.f, ex) : __int_as_float(0x7fc00000);
}

// real queries of cache row b, whose length is L
__device__ __forceinline__ int decode_queries(const DecodeArgs& a, int b, int L) {
  if (L < 0 || L >= a.t_max) return 0;
  return a.nq ? max(0, min(a.nq[b], min(a.kq, a.t_max - L))) : a.kq;
}

// kStaged is chosen at launch: staging the tile costs 37 KB of shared memory and more than twice the registers, which
// only pays when several queries read it. The unstaged kernel runs one query and stores into the cache; keeping side
// buffers out of it keeps it at 32 registers (36 with them, which cost decode up to 3 % at 96 (row, head) pairs).
// T is the cache element: __nv_bfloat16, or uint8_t for an fp8 cache (unstaged only).
template <bool kStaged, typename T>
__global__ void __launch_bounds__(kDecodeThreads) decode_attn_split_kernel(const __grid_constant__ DecodeArgs a) {
  constexpr bool kFp8 = std::is_same<T, uint8_t>::value;
  static_assert(!(kStaged && kFp8), "the staged variant reads a bf16 cache only");
  constexpr int S = kDecodeSplit;
  __shared__ float s_p[S];                          // scores, then exp(score - max)
  __shared__ float s_acc[kDecodeThreads * 8];       // per key group: its partial P.V
  __shared__ float s_red[kDecodeThreads / 32];
  const int s = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int L = a.lens[b];
  const int nq = decode_queries(a, b, L);
  const int j0 = s * S;
  if (nq == 0 || j0 > L + a.chain * (nq - 1)) return;
  const int Dh = a.Dh, nvec = Dh >> 3, D = a.H * Dh;
  int G = 1;                                        // lanes per key: 8 elements (16 bytes) each, a power of two <= 16
  while (G < nvec) G <<= 1;
  const int tid = threadIdx.x, c = tid & (G - 1), grp = tid / G, ngrp = kDecodeThreads / G;
  const bool act = c < nvec;
  const long long head = ((long long)b * a.H + h) * a.t_max * Dh;
  T* kc = reinterpret_cast<T*>(a.k_cache) + head;
  T* vc = reinterpret_cast<T*>(a.v_cache) + head;
  const T* tk = kc + (long long)j0 * Dh;             // the split's cached keys and values: key jj at jj * Dh
  const T* tv = vc + (long long)j0 * Dh;
  const long long sh = ((long long)b * a.H + h) * a.t_max + j0;     // fp8: the scale of key jj at sh + jj
  if constexpr (kStaged) {
    __shared__ __align__(16) __nv_bfloat16 s_k[S * kDecodeMaxDh];
    __shared__ __align__(16) __nv_bfloat16 s_v[S * kDecodeMaxDh];
    const int np = min(S, L - j0);                  // cached keys of this split (none if it starts at L or later)
    for (int e = tid; e < np * nvec; e += kDecodeThreads) {
      const int jj = e / nvec, cc = e - jj * nvec;
      *reinterpret_cast<uint4*>(s_k + jj * Dh + cc * 8) = *reinterpret_cast<const uint4*>(tk + jj * Dh + cc * 8);
      *reinterpret_cast<uint4*>(s_v + jj * Dh + cc * 8) = *reinterpret_cast<const uint4*>(tv + jj * Dh + cc * 8);
    }
    __syncthreads();
    tk = s_k;
    tv = s_v;
  }
  const float scale = 1.0f / sqrtf((float)Dh);
  const int lane = tid & 31, warp = tid >> 5;
  // unstaged: kq == 1, and the one query is real after the exit above, sits at P = L and owns the only new key
  const int nrun = kStaged ? nq : 1;
  for (int qi = 0; qi < nrun; ++qi) {
    const int P = L + a.chain * qi;                 // this query's position: keys 0 .. P
    if (j0 > P) continue;                           // uniform across the CTA
    const int n = min(S, P + 1 - j0);               // keys of this split: j0 .. j0 + n - 1
    const long long bq = (long long)b * a.kq + qi;
    const __nv_bfloat16* qrow = a.qkv + bq * a.qkv_stride + h * Dh;
    const __nv_bfloat16* qnew = qrow - (long long)(P - L) * a.qkv_stride;   // the query whose new key sits at L
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
        if constexpr (kFp8) {
          if (j < L)
            unpack_fp8(*reinterpret_cast<const uint2*>(tk + jj * Dh + c * 8), k);
          else
            unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(qrow + D + c * 8), k);
        } else {
          unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(
              j >= L ? (kStaged ? qnew + (long long)(j - L) * a.qkv_stride : qrow) + D + c * 8
                     : tk + jj * Dh + c * 8), k);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) d = fmaf(q[e], k[e], d);
      }
      for (int o = G >> 1; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      if constexpr (kFp8) {
        if (c == 0 && jj < n) s_p[jj] = (j < L ? d * a.k_scale[sh + jj] : d) * scale;
      } else {
        if (c == 0 && jj < n) s_p[jj] = d * scale;
      }
    }
    __syncthreads();
    // 2. max and sum of exp over the split (max is exact in any order; the sum's order is fixed by the layout)
    float m = -INFINITY;
    for (int jj = tid; jj < n; jj += kDecodeThreads) m = fmaxf(m, s_p[jj]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) s_red[warp] = m;
    __syncthreads();
    m = s_red[0];
#pragma unroll
    for (int w = 1; w < kDecodeThreads / 32; ++w) m = fmaxf(m, s_red[w]);
    __syncthreads();                                // every thread has read s_red before it is reused
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
        float p = s_p[jj];
        if constexpr (kFp8) {
          if (j < L) {
            unpack_fp8(*reinterpret_cast<const uint2*>(tv + jj * Dh + c * 8), v);
            p *= a.v_scale[sh + jj];
          } else {
            unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(qrow + 2 * D + c * 8), v);
          }
        } else {
          unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(
              j >= L ? (kStaged ? qnew + (long long)(j - L) * a.qkv_stride : qrow) + 2 * D + c * 8
                     : tv + jj * Dh + c * 8), v);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = fmaf(p, v[e], acc[e]);
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) s_acc[grp * (G * 8) + c * 8 + e] = acc[e];
    __syncthreads();
    float* w = a.work + ((bq * a.H + h) * a.n_splits + s) * (Dh + 2);
    if (tid < Dh) {
      float r = 0.f;
      for (int g = 0; g < ngrp; ++g) r += s_acc[g * (G * 8) + tid];
      w[2 + tid] = r;
    }
    // the query's new k / v are stored last: this CTA read them from qkv above, and no CTA reads position P from the
    // cache
    if constexpr (kFp8) {
      if (P < j0 + S && tid < 32) {                 // warp 0: lanes 0 .. nvec - 1 hold the vector
        const long long ps = ((long long)b * a.H + h) * a.t_max + P;
        const bool own = tid < nvec;
        const int c8 = own ? tid * 8 : 0;
        quantize_fp8(*reinterpret_cast<const uint4*>(qrow + D + c8), own, tid, kc + (long long)P * Dh,
                     a.k_scale + ps);
        quantize_fp8(*reinterpret_cast<const uint4*>(qrow + 2 * D + c8), own, tid, vc + (long long)P * Dh,
                     a.v_scale + ps);
      }
    } else if (P < j0 + S && tid < nvec) {
      const bool side = kStaged && a.side_k;
      __nv_bfloat16* nk = side ? a.side_k + bq * D + h * Dh : kc + (long long)P * Dh;
      __nv_bfloat16* nv = side ? a.side_v + bq * D + h * Dh : vc + (long long)P * Dh;
      const uint4 k4 = *reinterpret_cast<const uint4*>(qrow + D + tid * 8);
      const uint4 v4 = *reinterpret_cast<const uint4*>(qrow + 2 * D + tid * 8);
      *reinterpret_cast<uint4*>(nk + tid * 8) = k4;
      *reinterpret_cast<uint4*>(nv + tid * 8) = v4;
    }
    if (tid == 0) {
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < kDecodeThreads / 32; ++i) sum += s_red[i];
      w[0] = m;
      w[1] = sum;
    }
    if (qi + 1 < nrun) __syncthreads();             // s_p, s_red and s_acc are reused by the next query
  }
}

// one CTA per (h, query j, row b): out[b * kq + j, h * Dh + t] = sum_s acc_s[t] e^(m_s - M) / sum_s l_s e^(m_s - M)
// over splits 0 .. P / kDecodeSplit in index order; zero for a query that is not real. b and j come from the grid:
// deriving them from a (H, B * kq) grid by a division made decode up to 8 % slower at lens 1023.
__global__ void __launch_bounds__(kDecodeMaxDh) decode_attn_combine_kernel(const __grid_constant__ DecodeArgs a) {
  const int h = blockIdx.x, j = blockIdx.y, b = blockIdx.z, t = threadIdx.x, Dh = a.Dh;
  if (t >= Dh) return;
  const long long bq = (long long)b * a.kq + j;
  __nv_bfloat16* o = a.out + bq * a.H * Dh + h * Dh;
  const float* w = a.work + (bq * a.H + h) * a.n_splits * (Dh + 2);
  const int L = a.lens[b];
  // j < decode_queries(a, b, L) given j < kq, spelled out as one uniform test; with the call and a signed division
  // below, a combine took about 0.1 us longer
  if (L < 0 || L >= a.t_max || (a.nq && (j >= a.nq[b] || j >= a.t_max - L))) {
    o[t] = __float2bfloat16_rn(0.f);
    return;
  }
  const int ns = (unsigned)(L + a.chain * j) / kDecodeSplit + 1;   // P >= 0 for a real query
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

// Prefill of an fp8 cache: positions [0, T) of one layer from the c_attn output kv [B, T, 3 * H * Dh] (k at H * Dh,
// v at 2 * H * Dh), read in place. One CTA per (position t, row b); each 16-lane group quantizes one vector (the k
// and v of every head in turn), so the grid depends on the shapes only. 2H vectors and an even number of groups per
// CTA keep the loop bound uniform across each warp, as the shuffles need.
constexpr int kQuantThreads = 256;

__global__ void __launch_bounds__(kQuantThreads) kv_quantize_kernel(const __nv_bfloat16* kv, uint8_t* k, uint8_t* v,
                                                                    float* k_scale, float* v_scale, int H, int Dh,
                                                                    int T, int t_max) {
  const int t = blockIdx.x, b = blockIdx.y, D = H * Dh;
  const int c = threadIdx.x & 15;
  const bool own = c < (Dh >> 3);
  const __nv_bfloat16* row = kv + ((long long)b * T + t) * 3 * D;
  for (int g = threadIdx.x >> 4; g < 2 * H; g += kQuantThreads / 16) {
    const int h = g >> 1, isv = g & 1;
    const uint4 x = own ? *reinterpret_cast<const uint4*>(row + (1 + isv) * D + h * Dh + c * 8) : make_uint4(0, 0, 0, 0);
    const long long cell = ((long long)b * H + h) * t_max + t;
    quantize_fp8(x, own, c, (isv ? v : k) + cell * Dh, (isv ? v_scale : k_scale) + cell);
  }
}

inline int decode_splits(int t_max) { return (t_max + kDecodeSplit - 1) / kDecodeSplit; }

// Checks the arguments of the C entry point `who` (the prefix of its errors), whose rows hold 1..max_kq queries, and
// launches split and combine. a.n_splits is filled in here.
static int decode_attn_launch(const char* who, int max_kq, DecodeArgs a, int B, void* stream) {
  const int kq = a.kq, H = a.H, Dh = a.Dh, t_max = a.t_max;
  if (B < 1 || H < 1 || kq < 1 || kq > max_kq || B > 65535 || H > 65535 || (long long)B * kq > 65535 || t_max < 1) {
    set_error("%s: need 1 <= B, H, B * kq <= 65535, 1 <= kq <= %d and t_max >= 1 (B=%d kq=%d H=%d t_max=%d)", who,
              max_kq, B, kq, H, t_max);
    return -1;
  }
  if (Dh < 8 || Dh > kDecodeMaxDh || Dh % 8 != 0) {
    set_error("%s: head dim must be a multiple of 8 in [8, %d], got %d", who, kDecodeMaxDh, Dh);
    return -1;
  }
  if (a.qkv_stride < 3 * H * Dh || a.qkv_stride % 8 != 0) {
    set_error("%s: qkv row stride %d must be a multiple of 8 and >= 3 * H * Dh = %d", who, a.qkv_stride, 3 * H * Dh);
    return -1;
  }
  if (((uintptr_t)a.qkv | (uintptr_t)a.k_cache | (uintptr_t)a.v_cache | (uintptr_t)a.out | (uintptr_t)a.side_k |
       (uintptr_t)a.side_v) & 15) {
    set_error("%s: qkv, caches, output and side buffers must be 16-byte aligned", who);
    return -1;
  }
  if (!a.lens || !a.work || ((uintptr_t)a.lens | (uintptr_t)a.nq | (uintptr_t)a.work) & 3) {
    set_error("%s: lens and work must be non-null, and lens, nq and work 4-byte aligned", who);
    return -1;
  }
  if (!a.k_scale != !a.v_scale || ((uintptr_t)a.k_scale | (uintptr_t)a.v_scale) & 3 ||
      (a.k_scale && (kq != 1 || a.side_k))) {
    set_error("%s: k_scale and v_scale must both be null or both 4-byte aligned, and an fp8 cache takes one query per "
              "row and no side buffers", who);
    return -1;
  }
  a.n_splits = decode_splits(t_max);
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid(a.n_splits, H, B);
  if (a.k_scale)
    decode_attn_split_kernel<false, uint8_t><<<grid, kDecodeThreads, 0, s>>>(a);
  else if (kq == 1 && !a.side_k)
    decode_attn_split_kernel<false, __nv_bfloat16><<<grid, kDecodeThreads, 0, s>>>(a);
  else
    decode_attn_split_kernel<true, __nv_bfloat16><<<grid, kDecodeThreads, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  decode_attn_combine_kernel<<<dim3(H, kq, B), kDecodeMaxDh, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// fp32 elements of the `work` buffer adapcc_decode_attn needs for this shape
long long adapcc_decode_attn_work(int B, int H, int Dh, int t_max) {
  if (B < 1 || H < 1 || Dh < 1 || t_max < 1) return 0;
  return (long long)B * H * decode_splits(t_max) * (Dh + 2);
}

// qkv: bf16 [B, qkv_stride] (q | k | v of the new token, H * Dh each); k_cache / v_cache: bf16 [B, H, t_max, Dh];
// lens: int32 [B] (keys already cached; read only); out: bf16 [B, H * Dh]; work: fp32, adapcc_decode_attn_work elements.
// k_scale / v_scale: null for a bf16 cache; with an fp8 cache (k_cache / v_cache e4m3 bytes [B, H, t_max, Dh]) fp32
// [B, H, t_max], the scale of each cached vector
int adapcc_decode_attn(const void* qkv, void* k_cache, void* v_cache, const int* lens, void* out, int B, int H, int Dh,
                       int t_max, int qkv_stride, void* work, void* k_scale, void* v_scale, void* stream) {
  DecodeArgs a{(const __nv_bfloat16*)qkv, (__nv_bfloat16*)k_cache, (__nv_bfloat16*)v_cache, lens, nullptr,
               (float*)work, (__nv_bfloat16*)out, nullptr, nullptr, /*kq=*/1, /*chain=*/0, H, Dh, t_max, qkv_stride};
  a.k_scale = (float*)k_scale;
  a.v_scale = (float*)v_scale;
  return decode_attn_launch("decode_attn", 1, a, B, stream);
}

// Prefill of one layer's fp8 cache: positions [0, T) of every row. kv: bf16 [B, T, 3 * H * Dh] contiguous (the c_attn
// output); k_cache / v_cache: e4m3 bytes [B, H, t_max, Dh]; k_scale / v_scale: fp32 [B, H, t_max]
int adapcc_kv_quantize(const void* kv, void* k_cache, void* v_cache, void* k_scale, void* v_scale, int B, int T, int H,
                       int Dh, int t_max, void* stream) {
  if (B < 1 || B > 65535 || H < 1 || T < 1 || T > t_max || Dh < 8 || Dh > kDecodeMaxDh || Dh % 8 != 0) {
    set_error("kv_quantize: need 1 <= B <= 65535, H >= 1, 1 <= T <= t_max and Dh a multiple of 8 in [8, %d] (B=%d "
              "T=%d H=%d Dh=%d t_max=%d)", kDecodeMaxDh, B, T, H, Dh, t_max);
    return -1;
  }
  if (!kv || !k_cache || !v_cache || !k_scale || !v_scale) {
    set_error("kv_quantize: null pointer");
    return -1;
  }
  if (((uintptr_t)kv & 15) || (((uintptr_t)k_cache | (uintptr_t)v_cache) & 7) ||
      (((uintptr_t)k_scale | (uintptr_t)v_scale) & 3)) {
    set_error("kv_quantize: kv must be 16-byte, the caches 8-byte and the scales 4-byte aligned");
    return -1;
  }
  kv_quantize_kernel<<<dim3(T, B), kQuantThreads, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)kv, (uint8_t*)k_cache, (uint8_t*)v_cache, (float*)k_scale, (float*)v_scale, H, Dh, T,
      t_max);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// Contrastive-search candidates: kq queries per row, all at position lens[b]. qkv: bf16 [B * kq, qkv_stride];
// k_cache / v_cache: bf16 [B, H, t_max, Dh] (read only); lens: int32 [B]; out: bf16 [B * kq, H * Dh]; side_k / side_v:
// bf16 [B * kq, H * Dh], each candidate's new k / v; work: fp32, adapcc_decode_attn_work(B * kq, ...) elements
int adapcc_cand_attn(const void* qkv, const void* k_cache, const void* v_cache, const int* lens, void* out,
                     void* side_k, void* side_v, int B, int kq, int H, int Dh, int t_max, int qkv_stride, void* work,
                     void* stream) {
  if (!side_k || !side_v) {                         // without them the kernel would store into the cache
    set_error("cand_attn: side_k and side_v must be non-null");
    return -1;
  }
  const DecodeArgs a{(const __nv_bfloat16*)qkv, (__nv_bfloat16*)const_cast<void*>(k_cache),
                     (__nv_bfloat16*)const_cast<void*>(v_cache), lens, nullptr, (float*)work, (__nv_bfloat16*)out,
                     (__nv_bfloat16*)side_k, (__nv_bfloat16*)side_v, kq, /*chain=*/0, H, Dh, t_max, qkv_stride};
  return decode_attn_launch("cand_attn", kDecodeMaxQueries, a, B, stream);
}

// Prompt-lookup verify slots: slot j of row b at position lens[b] + j, the first nq[b] real. qkv: bf16
// [B * kq, qkv_stride]; k_cache / v_cache: bf16 [B, H, t_max, Dh]; lens, nq: int32 [B] (read only); out: bf16
// [B * kq, H * Dh]; work: fp32, adapcc_decode_attn_work(B * kq, ...) elements
int adapcc_verify_attn(const void* qkv, void* k_cache, void* v_cache, const int* lens, const int* nq, void* out, int B,
                       int kq, int H, int Dh, int t_max, int qkv_stride, void* work, void* stream) {
  if (!nq) {                                        // without it every slot would count as real
    set_error("verify_attn: nq must be non-null");
    return -1;
  }
  const DecodeArgs a{(const __nv_bfloat16*)qkv, (__nv_bfloat16*)k_cache, (__nv_bfloat16*)v_cache, lens, nq,
                     (float*)work, (__nv_bfloat16*)out, nullptr, nullptr, kq, /*chain=*/1, H, Dh, t_max, qkv_stride};
  return decode_attn_launch("verify_attn", kDecodeMaxQueries, a, B, stream);
}

}  // extern "C"
