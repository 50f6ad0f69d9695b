// Prompt-lookup speculative decoding for greedy GPT-2 generation on the device, so a verify step is one CUDA graph
// replay: the model on k + 1 slots per row, the LM head, then acceptance and the next drafts. The definition is in
// ops/lookup.py and DESIGN.md §4a.
//
//   verify_attn    : decode attention of a row's nq[b] real slots (its last token, then its drafts). Slot j sits at
//                    position lens[b] + j and attends over the cached keys 0..lens[b]-1 plus the new keys of its row's
//                    slots 0..j, read from their c_attn output. Grid (splits of t_max, H, B) as in
//                    decode_attn_split_kernel (ops_decode.cu): each CTA stages its split's cached K / V tile in shared
//                    memory once and runs the slots over it one after the other, each with the decode kernel's thread
//                    layout, split size and summation order, so slot j's output is bit-identical to decode_attention_
//                    with lens = lens[b] + j on a cache that already holds slots 0..j-1. The CTA whose split holds
//                    position lens[b] + j stores slot j's k / v there; no CTA reads a position >= lens[b] from the cache.
//   verify_combine : the decode kernel's combine, with slot j's length lens[b] + j; a pad slot's output is zero.
//   lk_argmax      : grid (slots, B), 512 threads: each real slot's arg-max (topk_rows.cuh with N = 1, ties to the lower
//                    id); suppress_ids are removed while emitted[b] + j < min_new.
//   lk_accept      : one thread per row: emits g_0, g_1, ... while the draft of the next slot equals the token just
//                    emitted, stopping at a stop id (sets done, not written), at max_new tokens (sets done) or at the
//                    first rejected draft; appends the emitted ids to the row's sequence, advances lens and emitted.
//   lk_draft       : one CTA per row: the earliest earlier occurrence of the sequence's last m tokens (m from the
//                    n-gram size down to 1); the tokens after it are the drafts. Writes the next step's ids, positions
//                    and real-slot count.
//
// Every grid depends on B, k and t_max only, so one capture serves every step. A row's results depend only on its own
// logits, cache and sequence.
#include <cuda_bf16.h>

#include <climits>
#include <cmath>
#include <cstdint>

#include "common.h"
#include "device_prims.cuh"
#include "topk_rows.cuh"

namespace adapcc {

constexpr int kLkSplit = 64;                        // = kDecodeSplit (ops_decode.cu): the same splits, the same bits
constexpr int kLkAttnThreads = 128;                 // = kDecodeThreads
constexpr int kLkMaxDh = 128;                       // = kDecodeMaxDh
constexpr int kLkMaxSlots = 16;                     // k + 1: the row's last token and up to 15 drafts
constexpr int kLkMaxNgram = 16;
constexpr int kLkMaxIds = 1024;                     // ids per suppress / stop list
constexpr int kLkDraftThreads = 256;

struct VerifyArgs {
  const __nv_bfloat16* qkv;   // [B * kq, qkv_stride]: q | k | v of each slot, H * Dh each
  __nv_bfloat16* k_cache;     // [B, H, t_max, Dh]
  __nv_bfloat16* v_cache;
  const int* lens;            // [B]
  const int* nq;              // [B]: real slots of each row
  float* work;                // [B * kq, H, n_splits, Dh + 2]
  __nv_bfloat16* out;         // [B * kq, H * Dh]
  int kq, H, Dh, t_max, qkv_stride, n_splits;
};

// real slots of row b: nq[b] clamped to [0, kq] and to the positions left in the cache (0 for a row outside it)
__device__ __forceinline__ int verify_slots(const VerifyArgs& a, int b, int L) {
  if (L < 0 || L >= a.t_max) return 0;
  return max(0, min(a.nq[b], min(a.kq, a.t_max - L)));
}

template <int S>
__global__ void __launch_bounds__(kLkAttnThreads) verify_attn_split_kernel(const __grid_constant__ VerifyArgs a) {
  __shared__ __align__(16) __nv_bfloat16 s_k[S * kLkMaxDh];   // the split's cached keys and values, shared by the
  __shared__ __align__(16) __nv_bfloat16 s_v[S * kLkMaxDh];   // row's slots
  __shared__ float s_p[S];
  __shared__ float s_acc[kLkAttnThreads * 8];
  __shared__ float s_red[kLkAttnThreads / 32];
  const int s = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int L = a.lens[b];
  const int nq = verify_slots(a, b, L);
  const int j0 = s * S;
  if (nq == 0 || j0 > L + nq - 1) return;
  const int np = min(S, L - j0);                    // cached keys of this split (none if it starts at L or later)
  const int Dh = a.Dh, nvec = Dh >> 3, D = a.H * Dh;
  int G = 1;
  while (G < nvec) G <<= 1;
  const int tid = threadIdx.x, c = tid & (G - 1), grp = tid / G, ngrp = kLkAttnThreads / G;
  const bool act = c < nvec;
  const long long head = ((long long)b * a.H + h) * a.t_max * Dh;
  __nv_bfloat16* kc = a.k_cache + head;
  __nv_bfloat16* vc = a.v_cache + head;
  for (int e = tid; e < np * nvec; e += kLkAttnThreads) {
    const int jj = e / nvec, cc = e - jj * nvec;
    const long long g = (long long)(j0 + jj) * Dh + cc * 8;
    *reinterpret_cast<uint4*>(s_k + jj * Dh + cc * 8) = *reinterpret_cast<const uint4*>(kc + g);
    *reinterpret_cast<uint4*>(s_v + jj * Dh + cc * 8) = *reinterpret_cast<const uint4*>(vc + g);
  }
  __syncthreads();
  const float scale = 1.0f / sqrtf((float)Dh);
  const int lane = tid & 31, warp = tid >> 5;
  const __nv_bfloat16* rowq = a.qkv + (long long)b * a.kq * a.qkv_stride + h * Dh;   // slot 0 of the row, head h
  for (int qi = 0; qi < nq; ++qi) {
    const int Lq = L + qi;                          // this slot's position: keys 0 .. Lq
    if (j0 > Lq) continue;                          // uniform across the CTA
    const int n = min(S, Lq + 1 - j0);
    const long long bq = (long long)b * a.kq + qi;
    const __nv_bfloat16* qrow = rowq + (long long)qi * a.qkv_stride;
    float q[8];
    if (act) unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(qrow + c * 8), q);
    // 1. scores (decode_attn_split_kernel's layout and order); key j >= L is slot j - L's new key
#pragma unroll 4
    for (int base = 0; base < n; base += ngrp) {
      const int jj = base + grp, j = j0 + jj;
      float d = 0.f;
      if (act && jj < n) {
        float k[8];
        unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(
            j >= L ? rowq + (long long)(j - L) * a.qkv_stride + D + c * 8 : s_k + jj * Dh + c * 8), k);
#pragma unroll
        for (int e = 0; e < 8; ++e) d = fmaf(q[e], k[e], d);
      }
      for (int o = G >> 1; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      if (c == 0 && jj < n) s_p[jj] = d * scale;
    }
    __syncthreads();
    // 2. max and sum of exp over the split
    float m = -INFINITY;
    for (int jj = tid; jj < n; jj += kLkAttnThreads) m = fmaxf(m, s_p[jj]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) s_red[warp] = m;
    __syncthreads();
    m = s_red[0];
#pragma unroll
    for (int w = 1; w < kLkAttnThreads / 32; ++w) m = fmaxf(m, s_red[w]);
    __syncthreads();
    float l = 0.f;
    for (int jj = tid; jj < n; jj += kLkAttnThreads) {
      const float p = expf(s_p[jj] - m);
      s_p[jj] = p;
      l += p;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
    if (lane == 0) s_red[warp] = l;
    __syncthreads();
    // 3. P.V
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    if (act) {
#pragma unroll 4
      for (int jj = grp; jj < n; jj += ngrp) {
        const int j = j0 + jj;
        float v[8];
        unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(
            j >= L ? rowq + (long long)(j - L) * a.qkv_stride + 2 * D + c * 8 : s_v + jj * Dh + c * 8), v);
        const float p = s_p[jj];
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
    // the slot's k / v go into the cache at Lq: position Lq >= L is read from qkv by every CTA, never from the cache
    if (Lq < j0 + S && tid < nvec) {
      *reinterpret_cast<uint4*>(kc + (long long)Lq * Dh + tid * 8) = *reinterpret_cast<const uint4*>(qrow + D + tid * 8);
      *reinterpret_cast<uint4*>(vc + (long long)Lq * Dh + tid * 8) =
          *reinterpret_cast<const uint4*>(qrow + 2 * D + tid * 8);
    }
    if (tid == 0) {
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < kLkAttnThreads / 32; ++i) sum += s_red[i];
      w[0] = m;
      w[1] = sum;
    }
    __syncthreads();                                // s_p, s_red and s_acc are reused by the next slot
  }
}

// one CTA per (h, slot row): decode_attn_combine_kernel with the slot's length lens[b] + j
template <int S>
__global__ void __launch_bounds__(kLkMaxDh) verify_attn_combine_kernel(const __grid_constant__ VerifyArgs a) {
  const int h = blockIdx.x, bq = blockIdx.y, t = threadIdx.x, Dh = a.Dh;
  if (t >= Dh) return;
  __nv_bfloat16* o = a.out + (long long)bq * a.H * Dh + h * Dh;
  const int b = bq / a.kq, qi = bq - b * a.kq;
  const int L = a.lens[b];
  if (qi >= verify_slots(a, b, L)) {
    o[t] = __float2bfloat16_rn(0.f);
    return;
  }
  const int ns = (L + qi) / S + 1;
  const float* w = a.work + ((long long)bq * a.H + h) * a.n_splits * (Dh + 2);
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

// ---- acceptance ----------------------------------------------------------------------------------------------------
struct AcceptArgs {
  const float* logits;         // [B * ls, ld]: slot j of row b in row b * ls + j, the first `vocab` columns used
  int ld, vocab, B, kq, ls;    // kq: slots per row of ids / g; ls: slots per row of logits (1 or kq)
  const int* emitted;          // [B]: tokens emitted so far (advanced by lk_accept)
  int min_new;
  const int* suppress;         // ids removed while emitted + j < min_new
  int n_suppress;
  int* g;                      // [B * kq]: each real slot's arg-max
  const long long* ids;        // [B * kq]: the step's input ids (slot j > 0: draft j)
  const int* nq;               // [B]
  int* seq;                    // [B, t_max]: each row's sequence (prompt, then its emitted tokens)
  int t_max;
  int* lens;                   // [B]: cached tokens = |sequence| - 1; advanced here
  int* emitted_w;              // = emitted, written by lk_accept
  int* done;                   // [B]
  const int* stop;
  int n_stop;
  long long* tokens;           // [B, max_new]
  int max_new;
  int* steps;                  // [B]: verify steps per live row (null: not counted)
};

__device__ __forceinline__ int accept_slots(const AcceptArgs& a, int b) { return max(0, min(a.nq[b], a.ls)); }

__global__ void __launch_bounds__(kBeamThreads, 1) lk_argmax_kernel(const __grid_constant__ AcceptArgs a) {
  extern __shared__ uint32_t s_bits[];
  __shared__ unsigned long long s_top[kBeamWarps];
  __shared__ unsigned long long s_best[1];
  const int j = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, V = a.vocab;
  if (a.done[b] || j >= accept_slots(a, b)) return;
  const bool sup = a.emitted[b] + j < a.min_new && a.n_suppress > 0;
  if (sup) {
    for (int w = tid; w < (V + 31) / 32; w += kBeamThreads) s_bits[w] = 0u;
    __syncthreads();
    for (int i = tid; i < a.n_suppress; i += kBeamThreads) {
      const int id = a.suppress[i];
      if (id >= 0 && id < V) atomicOr(&s_bits[id >> 5], 1u << (id & 31));
    }
  }
  if (tid < kBeamWarps) s_top[tid] = 0ull;
  if (tid == 0) s_best[0] = 0ull;
  __syncthreads();
  RowView rv{a.logits + ((long long)b * a.ls + j) * a.ld, sup ? s_bits : nullptr, V, 0.f, 0.f, 0.f};
  row_top_keys<true>(rv, 1, s_top, s_best);
  __syncthreads();
  if (tid == 0) {
    const unsigned long long key = s_best[0];
    a.g[(long long)b * a.kq + j] = key ? (int)(0xFFFFFFFFu - (uint32_t)key) : 0;   // no live id: id 0
  }
}

__global__ void lk_accept_kernel(const __grid_constant__ AcceptArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B || a.done[b]) return;
  const int nq = accept_slots(a, b), L = a.lens[b];
  int e = a.emitted[b], c = 0, done = 0;
  int* s = a.seq + (long long)b * a.t_max;
  for (int j = 0; j < nq; ++j) {
    const int t = a.g[(long long)b * a.kq + j];
    if (L + 1 + c < a.t_max) s[L + 1 + c] = t;
    ++c;
    ++e;
    bool is_stop = false;
    for (int q = 0; q < a.n_stop; ++q) is_stop |= a.stop[q] == t;
    if (is_stop) {
      done = 1;
      break;
    }
    if (e <= a.max_new) a.tokens[(long long)b * a.max_new + e - 1] = t;
    if (e >= a.max_new) {
      done = 1;
      break;
    }
    if (j + 1 < nq && a.ids[(long long)b * a.kq + j + 1] != t) break;   // draft j + 1 rejected
  }
  a.lens[b] = L + c;
  a.emitted_w[b] = e;
  if (done) a.done[b] = 1;
  if (a.steps) a.steps[b] += 1;
}

// ---- drafts --------------------------------------------------------------------------------------------------------
struct DraftArgs {
  const int* seq;              // [B, t_max]
  int t_max, B, kq, ngram, max_new;
  const int* lens;             // [B]: the sequence is seq[b, 0 .. lens[b]]
  const int* emitted;          // [B]
  const int* done;             // [B]
  long long* ids;              // [B * kq]: slot 0 the last token, then the drafts, 0 in a pad slot
  long long* pos;              // [B * kq]: lens[b] + j, clamped to t_max - 1
  int* nq;                     // [B]: 1 + drafts, 0 for a done row
};

__global__ void __launch_bounds__(kLkDraftThreads) lk_draft_kernel(const __grid_constant__ DraftArgs a) {
  __shared__ int s_first;
  const int b = blockIdx.x, tid = threadIdx.x, K = a.kq - 1;
  const int L = min(max(a.lens[b], 0), a.t_max - 1), slen = L + 1;
  const int* s = a.seq + (long long)b * a.t_max;
  const bool live = !a.done[b];
  const int r = live ? min(K, a.max_new - a.emitted[b] - 1) : 0;   // drafts this row may take
  int start = -1, nd = 0;
  if (r > 0) {
    for (int m = min(a.ngram, slen - 1); m >= 1; --m) {
      if (tid == 0) s_first = INT_MAX;
      __syncthreads();
      for (int i = tid; i + m < slen; i += kLkDraftThreads) {       // windows whose continuation is non-empty
        bool eq = true;
        for (int t = 0; t < m && eq; ++t) eq = s[i + t] == s[slen - m + t];
        if (eq) {
          atomicMin(&s_first, i);
          break;                                      // this thread's later windows start later
        }
      }
      __syncthreads();
      const int first = s_first;
      __syncthreads();                                // s_first is reset for the next m
      if (first != INT_MAX) {
        start = first + m;
        nd = min(r, slen - start);
        break;
      }
    }
  }
  if (tid < a.kq) {
    const long long o = (long long)b * a.kq + tid;
    a.ids[o] = !live ? 0 : tid == 0 ? s[L] : tid <= nd ? s[start + tid - 1] : 0;
    a.pos[o] = min(L + tid, a.t_max - 1);
  }
  if (tid == 0) a.nq[b] = live ? 1 + nd : 0;
}

inline int lk_splits(int t_max) { return (t_max + kLkSplit - 1) / kLkSplit; }

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// qkv: bf16 [B * kq, qkv_stride]; k_cache / v_cache: bf16 [B, H, t_max, Dh]; lens, nq: int32 [B] (read only); out: bf16
// [B * kq, H * Dh]; work: fp32, adapcc_decode_attn_work(B * kq, ...) elements
int adapcc_verify_attn(const void* qkv, void* k_cache, void* v_cache, const int* lens, const int* nq, void* out, int B,
                       int kq, int H, int Dh, int t_max, int qkv_stride, void* work, void* stream) {
  if (B < 1 || H < 1 || kq < 1 || kq > kLkMaxSlots || B > 65535 || H > 65535 || (long long)B * kq > 65535 ||
      t_max < 1) {
    set_error("verify_attn: need 1 <= B, H, B * kq <= 65535, 1 <= kq <= %d and t_max >= 1 (B=%d kq=%d H=%d t_max=%d)",
              kLkMaxSlots, B, kq, H, t_max);
    return -1;
  }
  if (Dh < 8 || Dh > kLkMaxDh || Dh % 8 != 0) {
    set_error("verify_attn: head dim must be a multiple of 8 in [8, %d], got %d", kLkMaxDh, Dh);
    return -1;
  }
  if (qkv_stride < 3 * H * Dh || qkv_stride % 8 != 0) {
    set_error("verify_attn: qkv row stride %d must be a multiple of 8 and >= 3 * H * Dh = %d", qkv_stride, 3 * H * Dh);
    return -1;
  }
  if (((uintptr_t)qkv | (uintptr_t)k_cache | (uintptr_t)v_cache | (uintptr_t)out) & 15) {
    set_error("verify_attn: qkv, caches and output must be 16-byte aligned");
    return -1;
  }
  if (!lens || !nq || !work || ((uintptr_t)lens | (uintptr_t)nq | (uintptr_t)work) & 3) {
    set_error("verify_attn: lens, nq and work must be non-null and 4-byte aligned");
    return -1;
  }
  VerifyArgs a{};
  a.qkv = (const __nv_bfloat16*)qkv;
  a.k_cache = (__nv_bfloat16*)k_cache;
  a.v_cache = (__nv_bfloat16*)v_cache;
  a.lens = lens;
  a.nq = nq;
  a.work = (float*)work;
  a.out = (__nv_bfloat16*)out;
  a.kq = kq;
  a.H = H;
  a.Dh = Dh;
  a.t_max = t_max;
  a.qkv_stride = qkv_stride;
  a.n_splits = lk_splits(t_max);
  cudaStream_t s = (cudaStream_t)stream;
  verify_attn_split_kernel<kLkSplit><<<dim3(a.n_splits, H, B), kLkAttnThreads, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  verify_attn_combine_kernel<kLkSplit><<<dim3(H, B * kq), kLkMaxDh, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// logits fp32 [B * ls, ld]; suppress / stop int32 lists (null when empty); g int32, ids int64 [B * kq]; nq, seq
// [B, t_max], lens, emitted, done int32; tokens int64 [B, max_new]; steps int32 [B] or null
int adapcc_lookup_accept(const float* logits, int ld, int vocab, int B, int kq, int ls, int min_new,
                         const int* suppress, int n_suppress, const int* stop, int n_stop, int* g, const long long* ids,
                         const int* nq, int* seq, int t_max, int* lens, int* emitted, int* done, long long* tokens,
                         int max_new, int* steps, void* stream) {
  if (B < 1 || B > 65535 || kq < 1 || kq > kLkMaxSlots || (ls != 1 && ls != kq) || vocab < 1 || ld < vocab ||
      t_max < 1 || max_new < 1) {
    set_error("lookup_accept: need 1 <= B <= 65535, 1 <= kq <= %d, ls in {1, kq}, 1 <= vocab <= ld, t_max, max_new "
              ">= 1 (B=%d kq=%d ls=%d vocab=%d ld=%d)", kLkMaxSlots, B, kq, ls, vocab, ld);
    return -1;
  }
  if (n_suppress < 0 || n_suppress > kLkMaxIds || (n_suppress && !suppress) || n_stop < 0 || n_stop > kLkMaxIds ||
      (n_stop && !stop)) {
    set_error("lookup_accept: at most %d suppressed and %d stop ids (got %d, %d)", kLkMaxIds, kLkMaxIds, n_suppress,
              n_stop);
    return -1;
  }
  if (!logits || !g || !ids || !nq || !seq || !lens || !emitted || !done || !tokens) {
    set_error("lookup_accept: null pointer");
    return -1;
  }
  const size_t bits = n_suppress > 0 && min_new > 0 ? (size_t)(vocab + 31) / 32 * sizeof(uint32_t) : 0;
  if (bits > 200 * 1024) {
    set_error("lookup_accept: suppression needs vocab <= %d (got %d)", 200 * 1024 * 8, vocab);
    return -1;
  }
  if (bits > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(lk_argmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bits));
  AcceptArgs a{logits, ld, vocab, B, kq, ls, emitted, min_new, suppress, n_suppress, g, ids, nq, seq, t_max, lens,
               emitted, done, stop, n_stop, tokens, max_new, steps};
  cudaStream_t s = (cudaStream_t)stream;
  lk_argmax_kernel<<<dim3(ls, B), kBeamThreads, bits, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  lk_accept_kernel<<<(B + 63) / 64, 64, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// seq int32 [B, t_max]; lens, emitted, done int32 [B]; ids, pos int64 [B * kq]; nq int32 [B]
int adapcc_lookup_draft(const int* seq, int t_max, int B, int kq, int ngram, int max_new, const int* lens,
                        const int* emitted, const int* done, long long* ids, long long* pos, int* nq, void* stream) {
  if (B < 1 || B > 65535 || kq < 1 || kq > kLkMaxSlots || ngram < 1 || ngram > kLkMaxNgram || t_max < 1 ||
      max_new < 1) {
    set_error("lookup_draft: need 1 <= B <= 65535, 1 <= kq <= %d, 1 <= ngram <= %d, t_max, max_new >= 1 (B=%d kq=%d "
              "ngram=%d)", kLkMaxSlots, kLkMaxNgram, B, kq, ngram);
    return -1;
  }
  if (!seq || !lens || !emitted || !done || !ids || !pos || !nq) {
    set_error("lookup_draft: null pointer");
    return -1;
  }
  DraftArgs a{seq, t_max, B, kq, ngram, max_new, lens, emitted, done, ids, pos, nq};
  lk_draft_kernel<<<B, kLkDraftThreads, 0, (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
