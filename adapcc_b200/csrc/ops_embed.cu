// Fused embedding sum (forward + backward) for the transformer workloads.
//
// GPT-2's input layer is x[t] = wte[ids[t]] + wpe[pos[t]] + wte[token_type[t]]
// (/root/reference/models/gpt2/train_gpt2_ddp.py:157-159 -> transformers' GPT2Model): three gathers and two adds
// forward, and — the expensive part — three sort-based `embedding_dense_backward` passes (16 radix-sort launches,
// segment scans) plus two 77 MB accumulate kernels backward. Here:
//
//   forward : one kernel, one warp per token row, the K looked-up rows summed in fp32 registers, bf16 out.
//   backward: three small launches, no sort, no host-visible sizes (CUDA-graph capturable), bit-for-bit repeatable:
//     1. claim   : every lookup (k, t) does atomicMin(owner[table_k, idx], lookup id) — the smallest lookup id that
//                  hits a table row becomes the row's OWNER for this step — and atomicMax(maxbits[table_k, idx],
//                  max |dY[t, :]|) (the float bits of a non-negative value order like the integers);
//     2. scatter : every lookup adds its dY row into the owner's scratch row as 64-bit FIXED POINT (red.add.u64),
//                  scaled by 2^shift with shift = 62 - lookup_bits - (exponent(row max) + 1), lookup_bits =
//                  ceil(log2(#lookups)): every entry becomes the integer round(float(entry * 2^shift)), no sum can
//                  overflow, the resolution is 2^-46 or finer of the row's largest entry, and integer addition gives
//                  the same bits in every order (an fp32 red.add would not: duplicates — repeated tokens, the two
//                  token-type rows hit by thousands of tokens — arrive in a different order every run); rows hit
//                  many times within a 64-lookup tile are pre-summed as the same integers in int64 registers first;
//     3. commit  : each owner converts its scratch row S back, grad = bf16_rn(float(old) + float(double(S) * 2^-shift))
//                  (NaN if the row's dY held a non-finite value), into the table's bf16 gradient row (which may already
//                  hold another contribution, e.g. the tied LM head's dW), zeroes the scratch row and releases the owner
//                  and maxbits slots, so all work buffers are back to their initial state for the next step.
//   Neither the order duplicates arrive in nor how the scatter groups them changes a bit of the result
//   (tests/test_gpu_kernels_reference.py checks it against an exact emulation of this arithmetic).
//   Lookups that share a table (ids and token types both index wte) share owner slots, so a row hit through both is
//   still committed exactly once.
//
// With dropout (DROP; dropout.cuh) the output row is drop(sum): the forward masks and scales the fp32 sum before the
// one bf16 rounding, and the backward's dY entry is everywhere replaced by the fp32 value mask * scale * dY[t, c], the
// mask recomputed from (seed, step, site, t, c >> 3). claim takes the row maximum of THOSE values and scatter converts
// THOSE values, so the shift still bounds every integer that is added, and each lookup of token t still contributes one
// integer per column that depends on (t, c) alone. The sum of integers is therefore still independent of arrival order
// and of the hot / direct grouping: the repeatability argument above holds unchanged.
#include <cuda_bf16.h>

#include <climits>

#include "common.h"
#include "device_prims.cuh"
#include "dropout.cuh"

namespace adapcc {

constexpr int kEmbedMaxLookups = 4;

struct EmbedFwdArgs {
  const __nv_bfloat16* table[kEmbedMaxLookups];
  const long long* idx[kEmbedMaxLookups];
  int K;
};

struct EmbedBwdArgs {
  const long long* idx[kEmbedMaxLookups];
  __nv_bfloat16* grad[kEmbedMaxLookups];
  int owner_base[kEmbedMaxLookups];      // first owner slot of lookup k's table
  int K;
};

// y[t, :] = [drop](sum_k table_k[idx_k[t], :]); D % 8 == 0; one warp per row.
template <bool DROP>
__global__ void __launch_bounds__(256)
embed_sum_fwd_kernel(const __grid_constant__ EmbedFwdArgs a, int n, int D, __nv_bfloat16* __restrict__ out,
                     const DropArgs drop) {
  const int warp = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (warp >= n) return;
  DropKey dkey{};
  if constexpr (DROP) dkey = drop_key(drop);
  const int nvec = D >> 3;
  const __nv_bfloat16* rows[kEmbedMaxLookups];
#pragma unroll
  for (int k = 0; k < kEmbedMaxLookups; ++k)
    rows[k] = k < a.K ? a.table[k] + a.idx[k][warp] * (long long)D : nullptr;
  for (int c = lane; c < nvec; c += 32) {
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
    for (int k = 0; k < kEmbedMaxLookups; ++k) {
      if (k < a.K) {
        float f[8];
        unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(rows[k] + c * 8), f);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += f[i];
      }
    }
    if constexpr (DROP) drop_apply(acc, drop_keep8(warp, c, drop, dkey), drop.scale);
    st16(out + (long long)warp * D + c * 8, pack<__nv_bfloat16>(acc));
  }
}

// one warp per lookup
template <bool DROP>
__global__ void __launch_bounds__(256)
embed_bwd_claim_kernel(const __grid_constant__ EmbedBwdArgs a, int n, int D, const __nv_bfloat16* __restrict__ dy,
                       int* __restrict__ owner, unsigned int* __restrict__ maxbits, const DropArgs drop) {
  const int i = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (i >= a.K * n) return;
  DropKey dkey{};
  if constexpr (DROP) dkey = drop_key(drop);
  const int k = i / n, t = i - k * n;
  const int slot = a.owner_base[k] + (int)a.idx[k][t];
  unsigned int m = 0;
  for (int c = lane; c < (D >> 3); c += 32) {
    float f[8];
    unpack<__nv_bfloat16>(ld16(dy + (long long)t * D + c * 8), f);
    if constexpr (DROP) drop_apply(f, drop_keep8(t, c, drop, dkey), drop.scale);
#pragma unroll
    for (int e = 0; e < 8; ++e) m = max(m, __float_as_uint(fabsf(f[e])));      // NaN / inf order above every finite
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) {
    atomicMin(owner + slot, i);
    atomicMax(maxbits + slot, m);
  }
}

// 2^shift scales a row whose largest |entry| has float bits `mb` so that up to 2^lookup_bits such entries sum below 2^62
__device__ __forceinline__ int embed_shift(unsigned int mb, int lookup_bits) {
  const int ex = (int)((mb >> 23) & 0xffu);
  const int e = ex == 0 ? -126 : ex - 127;                   // |entry| < 2^(e + 1)
  return 62 - lookup_bits - (e + 1);
}

// one dY entry as fixed point: round(v * 2^shift); every path through the scatter adds exactly these integers
__device__ __forceinline__ long long to_fixed(float v, int shift) { return __float2ll_rn(ldexpf(v, shift)); }

__device__ __forceinline__ void red_add_fixed(long long* p, long long q) {
  atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)q);
}

// scratch[owner, :] += dY[t, :] (fixed point) for a TILE of 64 consecutive lookups per CTA. Rows hit by many lookups of the tile (the
// two token-type rows are hit by every token) are first summed in int64 registers and leave as ONE reduction per tile
// and thread group instead of one per lookup: up to 4 "hot" owners per tile (>= 4 hits), found with 64 x 64 compares
// in shared memory. Everything else (token ids, positions: mostly unique inside a tile) goes straight to the scratch
// row. Both paths add the same integers, so when a tile has more than 4 candidates, which of them become hot (warp
// order decides) does not change any bit of the result.
constexpr int kEmbTile = 64, kEmbHot = 4, kEmbGroup = 128;       // 2 thread groups x 128 threads; group g: lookups j = g mod 2

template <bool DROP>
__global__ void __launch_bounds__(2 * kEmbGroup)
embed_bwd_scatter_kernel(const __grid_constant__ EmbedBwdArgs a, int n, int D, const __nv_bfloat16* __restrict__ dy,
                         const int* __restrict__ owner, const unsigned int* __restrict__ maxbits,
                         long long* __restrict__ scratch, int lookup_bits, const DropArgs drop) {
  __shared__ int s_own[kEmbTile];
  __shared__ int s_row[kEmbTile];
  __shared__ int s_shift[kEmbTile];
  __shared__ int s_hot_key[kEmbHot];
  __shared__ int s_hot_of[kEmbTile];
  __shared__ int s_nhot;
  const int total = a.K * n;
  const int i0 = blockIdx.x * kEmbTile;
  const int j = threadIdx.x;
  if (j == 0) s_nhot = 0;
  if (j < kEmbTile) {
    const int i = i0 + j;
    int own = -1, row = 0, shift = 0;
    if (i < total) {
      const int k = i / n;
      row = i - k * n;
      const int slot = a.owner_base[k] + (int)a.idx[k][row];
      own = owner[slot];
      shift = embed_shift(maxbits[slot], lookup_bits);
    }
    s_own[j] = own;
    s_row[j] = row;
    s_shift[j] = shift;
  }
  __syncthreads();
  if (j < kEmbTile && s_own[j] >= 0) {
    const int own = s_own[j];
    int cnt = 0;
    bool first = true;
    for (int i2 = 0; i2 < kEmbTile; ++i2) {
      if (s_own[i2] == own) {
        ++cnt;
        if (i2 < j) first = false;
      }
    }
    if (first && cnt >= 4) {
      const int slot = atomicAdd(&s_nhot, 1);
      if (slot < kEmbHot) s_hot_key[slot] = own;
    }
  }
  __syncthreads();
  const int nhot = min(s_nhot, kEmbHot);
  if (j < kEmbTile) {
    int h = -1;
    for (int q = 0; q < nhot; ++q)
      if (s_hot_key[q] == s_own[j]) h = q;
    s_hot_of[j] = h;
  }
  __syncthreads();
  const int g = threadIdx.x / kEmbGroup, tg = threadIdx.x - g * kEmbGroup;
  const int nvec = D >> 3;
  DropKey dkey{};
  if constexpr (DROP) dkey = drop_key(drop);
  for (int c = tg; c < nvec; c += kEmbGroup) {
    long long acc[kEmbHot][8];
#pragma unroll
    for (int q = 0; q < kEmbHot; ++q)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[q][e] = 0;
    for (int jj = g; jj < kEmbTile; jj += 2) {
      const int own = s_own[jj];
      if (own < 0) continue;
      float f[8];
      unpack<__nv_bfloat16>(ld16(dy + (long long)s_row[jj] * D + c * 8), f);
      if constexpr (DROP) drop_apply(f, drop_keep8(s_row[jj], c, drop, dkey), drop.scale);
      const int h = s_hot_of[jj];
      if (h < 0) {
        long long* dst = scratch + (long long)own * D + c * 8;
#pragma unroll
        for (int e = 0; e < 8; ++e) red_add_fixed(dst + e, to_fixed(f[e], s_shift[jj]));
      } else {
#pragma unroll
        for (int q = 0; q < kEmbHot; ++q)
          if (q == h) {
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[q][e] += to_fixed(f[e], s_shift[jj]);
          }
      }
    }
#pragma unroll
    for (int q = 0; q < kEmbHot; ++q)
      if (q < nhot) {
        long long* dst = scratch + (long long)s_hot_key[q] * D + c * 8;
#pragma unroll
        for (int e = 0; e < 8; ++e) red_add_fixed(dst + e, acc[q][e]);
      }
  }
}

// one warp per lookup; only owners act: grad[idx, :] += scratch[i, :]; scratch[i, :] = 0; owner / maxbits slots released
__global__ void __launch_bounds__(256)
embed_bwd_commit_kernel(const __grid_constant__ EmbedBwdArgs a, int n, int D, int* __restrict__ owner,
                        unsigned int* __restrict__ maxbits, long long* __restrict__ scratch, int lookup_bits) {
  const int i = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (i >= a.K * n) return;
  const int k = i / n, t = i - k * n;
  const long long row = a.idx[k][t];
  int* slot = owner + a.owner_base[k] + (int)row;
  if (*slot != i) return;                       // warp-uniform: every lane reads the same word
  unsigned int* mb_slot = maxbits + (slot - owner);
  const unsigned int mb = *mb_slot;
  const bool finite = mb < 0x7f800000u;
  const int shift = embed_shift(mb, lookup_bits);
  long long* s = scratch + (long long)i * D;
  __nv_bfloat16* g = a.grad[k] + row * (long long)D;
  const int nvec = D >> 3;
  for (int c = lane; c < nvec; c += 32) {
    float f[8];
    unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(g + c * 8), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      f[e] += finite ? (float)ldexp((double)s[c * 8 + e], -shift) : __int_as_float(0x7fc00000);
      s[c * 8 + e] = 0;
    }
    *reinterpret_cast<uint4*>(g + c * 8) = pack<__nv_bfloat16>(f);
  }
  __syncwarp();
  if (lane == 0) {
    *slot = INT_MAX;
    *mb_slot = 0u;
  }
}

__global__ void embed_fill_int_kernel(int* p, long long n, int v) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// tables[k]: bf16 [rows_k, D]; idx[k]: int64 [n]; out: bf16 [n, D]; drop: optional dropout of the sum
static int embed_fwd_launch(void* const* tables, void* const* idx, int K, int n, int D, void* out, void* stream,
                            const DropArgs* drop) {
  if (n <= 0) return 0;
  if (K < 1 || K > kEmbedMaxLookups || D % 8 != 0) { set_error("embed_sum_fwd: 1 <= K <= %d lookups, D %% 8 == 0", kEmbedMaxLookups); return -1; }
  EmbedFwdArgs a{};
  a.K = K;
  for (int k = 0; k < K; ++k) {
    if (((uintptr_t)tables[k] | (uintptr_t)out) & 15) { set_error("embed_sum_fwd: tables / output must be 16-byte aligned"); return -1; }
    a.table[k] = (const __nv_bfloat16*)tables[k];
    a.idx[k] = (const long long*)idx[k];
  }
  const int wpb = 8;
  const int grid = (n + wpb - 1) / wpb;
  if (drop)
    embed_sum_fwd_kernel<true><<<grid, wpb * 32, 0, (cudaStream_t)stream>>>(a, n, D, (__nv_bfloat16*)out, *drop);
  else
    embed_sum_fwd_kernel<false><<<grid, wpb * 32, 0, (cudaStream_t)stream>>>(a, n, D, (__nv_bfloat16*)out, DropArgs{});
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

int adapcc_embed_sum_fwd(void* const* tables, void* const* idx, int K, int n, int D, void* out, void* stream) {
  return embed_fwd_launch(tables, idx, K, n, D, out, stream, nullptr);
}

// The sum under dropout (dropout.cuh): seed int64 [1] and step int32 [1] on the device, site / thr / scale of the
// definition; row t of the output is row t of the mask.
int adapcc_embed_sum_drop_fwd(void* const* tables, void* const* idx, int K, int n, int D, void* out, const void* seed,
                              const void* step, int site, unsigned int thr, float scale, void* stream) {
  DropArgs d;
  if (!drop_args("embed_sum_drop_fwd", seed, step, site, thr, scale, &d)) return -1;
  return embed_fwd_launch(tables, idx, K, n, D, out, stream, &d);
}

// owner: int32 [sum of distinct table rows], all INT_MAX between calls; maxbits: uint32, same size, all zero between
// calls; scratch: int64 [K * n, D], all zero between calls (adapcc_embed_bwd_reset establishes all three).
// grads[k]: bf16 [rows_k, D], accumulated into. drop: the forward's dropout, applied to dy as it is read.
static int embed_bwd_launch(const void* dy, void* const* idx, void* const* grads, const int* owner_base, int K, int n,
                            int D, int* owner, unsigned int* maxbits, long long* scratch, void* stream,
                            const DropArgs* drop) {
  if (n <= 0) return 0;
  if (K < 1 || K > kEmbedMaxLookups || D % 8 != 0) { set_error("embed_sum_bwd: 1 <= K <= %d lookups, D %% 8 == 0", kEmbedMaxLookups); return -1; }
  if ((long long)K * n >= INT_MAX) { set_error("embed_sum_bwd: too many lookups"); return -1; }
  EmbedBwdArgs a{};
  a.K = K;
  for (int k = 0; k < K; ++k) {
    if (((uintptr_t)grads[k] | (uintptr_t)dy | (uintptr_t)scratch) & 15) { set_error("embed_sum_bwd: buffers must be 16-byte aligned"); return -1; }
    a.idx[k] = (const long long*)idx[k];
    a.grad[k] = (__nv_bfloat16*)grads[k];
    a.owner_base[k] = owner_base[k];
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int total = K * n;
  int lookup_bits = 0;                               // total <= 2^lookup_bits
  while ((1LL << lookup_bits) < (long long)total) ++lookup_bits;
  const int wpb = 8;
  const __nv_bfloat16* dyb = (const __nv_bfloat16*)dy;
  const int cgrid = (total + wpb - 1) / wpb, sgrid = (total + kEmbTile - 1) / kEmbTile;
  if (drop) {
    embed_bwd_claim_kernel<true><<<cgrid, wpb * 32, 0, s>>>(a, n, D, dyb, owner, maxbits, *drop);
    embed_bwd_scatter_kernel<true><<<sgrid, 2 * kEmbGroup, 0, s>>>(a, n, D, dyb, owner, maxbits, scratch, lookup_bits,
                                                                   *drop);
  } else {
    embed_bwd_claim_kernel<false><<<cgrid, wpb * 32, 0, s>>>(a, n, D, dyb, owner, maxbits, DropArgs{});
    embed_bwd_scatter_kernel<false><<<sgrid, 2 * kEmbGroup, 0, s>>>(a, n, D, dyb, owner, maxbits, scratch, lookup_bits,
                                                                    DropArgs{});
  }
  embed_bwd_commit_kernel<<<(total + wpb - 1) / wpb, wpb * 32, 0, s>>>(a, n, D, owner, maxbits, scratch, lookup_bits);
  CUDA_TRY(cudaGetLastError());
  count_launch(3);
  return 0;
}

int adapcc_embed_sum_bwd(const void* dy, void* const* idx, void* const* grads, const int* owner_base, int K, int n,
                         int D, int* owner, unsigned int* maxbits, long long* scratch, void* stream) {
  return embed_bwd_launch(dy, idx, grads, owner_base, K, n, D, owner, maxbits, scratch, stream, nullptr);
}

int adapcc_embed_sum_drop_bwd(const void* dy, void* const* idx, void* const* grads, const int* owner_base, int K, int n,
                              int D, int* owner, unsigned int* maxbits, long long* scratch, const void* seed,
                              const void* step, int site, unsigned int thr, float scale, void* stream) {
  DropArgs d;
  if (!drop_args("embed_sum_drop_bwd", seed, step, site, thr, scale, &d)) return -1;
  return embed_bwd_launch(dy, idx, grads, owner_base, K, n, D, owner, maxbits, scratch, stream, &d);
}

int adapcc_embed_bwd_reset(int* owner, unsigned int* maxbits, long long n_owner, long long* scratch,
                           long long scratch_elems, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (n_owner > 0) embed_fill_int_kernel<<<(int)std::min<long long>(1024, (n_owner + 255) / 256), 256, 0, s>>>(owner, n_owner, INT_MAX);
  if (n_owner > 0) CUDA_TRY(cudaMemsetAsync(maxbits, 0, (size_t)n_owner * sizeof(unsigned int), s));
  if (scratch_elems > 0) CUDA_TRY(cudaMemsetAsync(scratch, 0, (size_t)scratch_elems * sizeof(long long), s));
  CUDA_TRY(cudaGetLastError());
  if (n_owner > 0) count_launch();
  return 0;
}

}  // extern "C"
