// Contrastive search for GPT-2 generation (Su et al., "A Contrastive Framework for Neural Text Generation") on the
// device, so a token is one CUDA graph replay: candidate decode step, re-rank and commit, LM head, repetition controls,
// candidate selection. The definition is in ops/contrastive.py and DESIGN.md §4a. The candidates' attention is
// adapcc_cand_attn in ops_decode.cu; this file selects the candidates, re-ranks them and commits the winner.
//
//   cs_select     : one 512-thread CTA per row: the k largest logits (topk_rows.cuh, ranked by the logit itself, ties
//                   to the lower id), each with p = expf(l - m) / Z over the remaining ids; suppress_ids are removed
//                   while step < min_new. Writes the ids into the candidate step's input buffer.
//   cs_sim        : grid (chunks of kCsSimPos context positions, B): max over the chunk of cos(h_j, c) for the row's k
//                   candidate hidden states h_j (staged in shared memory, norms computed per CTA in a fixed order) and
//                   its context vectors c (read once per CTA for all k candidates, with their stored norms).
//   cs_commit     : one CTA per row: max over chunks (exact in any order), score (1 - a) p - a s, argmax (ties to the
//                   lower rank); writes the token, done and the winner's id, appends its hidden state and norm to the
//                   context, copies its side-buffer k / v into the cache at lens[b] for every layer and advances lens.
//
// Every grid depends on t_max, B and k only, so one capture serves every token. Every fp32 sum runs in an order fixed
// by the thread layout; a row's results depend only on its own logits, cache, context and candidates.
#include <cuda_bf16.h>

#include <cmath>
#include <cstdint>

#include "common.h"
#include "device_prims.cuh"
#include "topk_rows.cuh"

namespace adapcc {

constexpr int kCsMaxK = 16;                         // candidates per row
constexpr int kCsMaxD = 1024;                       // hidden size (four 16-byte vectors per lane)
constexpr int kCsSimPos = 64;                       // context positions per cs_sim CTA
constexpr int kCsSimThreads = 256;
constexpr int kCsMaxSuppress = 1024;
constexpr int kCsMaxStop = 1024;

// ---- candidate selection -----------------------------------------------------------------------------------------
struct SelectArgs {
  const float* logits;         // [B, ld], the first `vocab` columns used
  int ld, vocab, kq;
  const int* step;             // tokens emitted so far
  int min_new;
  const int* suppress;         // ids removed while *step < min_new
  int n_suppress;
  const int* done;             // [B]
  long long* next_ids;         // [B * k]: the candidate step's input (0 in an invalid slot)
  int* cand_tok;               // [B * k]: candidate ids, -1 in an invalid slot
  float* cand_p;               // [B * k]: their probabilities
};

__global__ void __launch_bounds__(kBeamThreads, 1) cs_select_kernel(const __grid_constant__ SelectArgs a) {
  extern __shared__ uint32_t s_bits[];
  __shared__ float s_red[kBeamWarps];
  __shared__ unsigned long long s_top[kBeamWarps * kCsMaxK];
  __shared__ unsigned long long s_best[kCsMaxK];
  __shared__ float s_mz[2];
  const int row = blockIdx.x, tid = threadIdx.x, K = a.kq, V = a.vocab;
  long long* nxt = a.next_ids + (long long)row * K;
  int* tok = a.cand_tok + (long long)row * K;
  float* cp = a.cand_p + (long long)row * K;
  if (a.done[row]) {
    if (tid < K) {
      nxt[tid] = 0;
      tok[tid] = -1;
      cp[tid] = 0.f;
    }
    return;
  }
  const bool sup = *a.step < a.min_new && a.n_suppress > 0;
  if (sup) {
    for (int w = tid; w < (V + 31) / 32; w += kBeamThreads) s_bits[w] = 0u;
    __syncthreads();
    for (int j = tid; j < a.n_suppress; j += kBeamThreads) {
      const int id = a.suppress[j];
      if (id >= 0 && id < V) atomicOr(&s_bits[id >> 5], 1u << (id & 31));
    }
  }
  for (int e = tid; e < kBeamWarps * K; e += kBeamThreads) s_top[e] = 0ull;
  if (tid < K) s_best[tid] = 0ull;
  __syncthreads();
  RowView rv{a.logits + (long long)row * a.ld, sup ? s_bits : nullptr, V, 0.f, 0.f, 0.f};
  float m = -INFINITY;
  for (int i = tid; i < V; i += kBeamThreads)
    if (!rv.removed(i)) m = fmaxf(m, __ldg(rv.l + i));
  m = beam_block_max(s_red, m);
  if (m > -INFINITY) {                                // uniform across the CTA
    float z = 0.f;
    for (int i = tid; i < V; i += kBeamThreads)
      if (!rv.removed(i)) z += expf(__ldg(rv.l + i) - m);
    z = beam_block_sum(s_red, z);
    if (tid == 0) {
      s_mz[0] = m;
      s_mz[1] = z;
    }
    row_top_keys<true>(rv, K, s_top, s_best);
  }
  __syncthreads();
  if (tid < K) {
    const unsigned long long key = s_best[tid];
    if (key) {
      const int id = (int)(0xFFFFFFFFu - (uint32_t)key);
      nxt[tid] = id;
      tok[tid] = id;
      cp[tid] = expf(beam_key2f((uint32_t)(key >> 32)) - s_mz[0]) / s_mz[1];
    } else {
      nxt[tid] = 0;
      tok[tid] = -1;
      cp[tid] = 0.f;
    }
  }
}

// ---- re-rank and commit ------------------------------------------------------------------------------------------
// Euclidean norm of a D-vector by one warp: lane c takes 16-byte vectors c, c + 32, ... (squares by fmaf in element
// order), then a shuffle tree. Every lane gets the same bits.
__device__ __forceinline__ float warp_norm(const __nv_bfloat16* x, int D) {
  const int lane = threadIdx.x & 31, nvec = D >> 3;
  float ss = 0.f;
  for (int c = lane; c < nvec; c += 32) {
    float v[8];
    unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(x + c * 8), v);
#pragma unroll
    for (int e = 0; e < 8; ++e) ss = fmaf(v[e], v[e], ss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  return sqrtf(ss);
}

struct RerankArgs {
  const __nv_bfloat16* hc;     // [B * k, ldh]: the candidates' final hidden states
  int ldh, kq, D, B;
  const int* cand_tok;         // [B * k], -1: invalid
  const float* cand_p;         // [B * k]
  float alpha;
  __nv_bfloat16* ctx;          // [B, t_max, D]: the rows' context of hidden states
  float* ctx_norm;             // [B, t_max]
  int t_max, n_chunks;
  float* sim;                  // [B, n_chunks, k]: per chunk, max cos of each candidate
  int* lens;                   // [B]: context length = cached tokens; advanced here
  int* done;                   // [B]
  const int* stop;
  int n_stop;
  const int* step;             // tokens emitted so far (read; incremented by cs_incr_kernel)
  long long* tokens;           // [B, max_new]
  int max_new;
  long long* win_ids;          // [B]: the emitted candidate's id (0 for a row without a candidate)
  __nv_bfloat16* win_h;        // [B, D]: its hidden state (the LM head's input)
  const __nv_bfloat16* side;   // [n_layer, 2, B * k, H * Dh]: the candidates' new keys and values
  __nv_bfloat16* k_cache;      // [n_layer, B, H, t_max, Dh]
  __nv_bfloat16* v_cache;
  int n_layer, H, Dh;
};

__global__ void __launch_bounds__(kCsSimThreads) cs_sim_kernel(const __grid_constant__ RerankArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  __nv_bfloat16* s_h = reinterpret_cast<__nv_bfloat16*>(s_raw);   // [k, D]
  __shared__ float s_hn[kCsMaxK];
  __shared__ float s_best[kCsSimThreads / 32][kCsMaxK];
  const int chunk = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int K = a.kq, D = a.D, nvec = D >> 3;
  const int n_ctx = min(max(a.lens[b], 0), a.t_max);
  const int p0 = chunk * kCsSimPos, p1 = min(p0 + kCsSimPos, n_ctx);
  float* out = a.sim + ((long long)b * a.n_chunks + chunk) * K;
  if (p0 >= p1) {
    if (tid < K) out[tid] = -INFINITY;
    return;
  }
  for (int e = tid; e < K * nvec; e += kCsSimThreads) {
    const int j = e / nvec, c = e - j * nvec;
    *reinterpret_cast<uint4*>(s_h + j * D + c * 8) =
        *reinterpret_cast<const uint4*>(a.hc + ((long long)b * K + j) * a.ldh + c * 8);
  }
  for (int e = tid; e < (kCsSimThreads / 32) * kCsMaxK; e += kCsSimThreads) (&s_best[0][0])[e] = -INFINITY;
  __syncthreads();
  for (int j = warp; j < K; j += kCsSimThreads / 32) {
    const float nrm = warp_norm(s_h + j * D, D);
    if (lane == 0) s_hn[j] = nrm;
  }
  __syncthreads();
  for (int p = p0 + warp; p < p1; p += kCsSimThreads / 32) {
    const __nv_bfloat16* cv = a.ctx + ((long long)b * a.t_max + p) * D;
    float x[kCsMaxD / 256][8];
#pragma unroll
    for (int i = 0; i < kCsMaxD / 256; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(cv + c * 8), x[i]);
    }
    const float cn = a.ctx_norm[(long long)b * a.t_max + p];
    for (int j = 0; j < K; ++j) {
      float d = 0.f;
#pragma unroll
      for (int i = 0; i < kCsMaxD / 256; ++i) {
        const int c = lane + 32 * i;
        if (c < nvec) {
          float hv[8];
          unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(s_h + j * D + c * 8), hv);
#pragma unroll
          for (int e = 0; e < 8; ++e) d = fmaf(hv[e], x[i][e], d);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      const float hn = s_hn[j];
      const float cs = (hn == 0.f || cn == 0.f) ? 0.f : __fdiv_rn(d, __fmul_rn(hn, cn));
      if (lane == 0) s_best[warp][j] = fmaxf(s_best[warp][j], cs);
    }
  }
  __syncthreads();
  if (tid < K) {
    float s = s_best[0][tid];
#pragma unroll
    for (int w = 1; w < kCsSimThreads / 32; ++w) s = fmaxf(s, s_best[w][tid]);
    out[tid] = s;
  }
}

__global__ void __launch_bounds__(kCsSimThreads) cs_commit_kernel(const __grid_constant__ RerankArgs a) {
  __shared__ int s_w;
  const int b = blockIdx.x, tid = threadIdx.x, K = a.kq, D = a.D;
  const int L = a.lens[b];
  if (tid == 0) {
    const float alpha = a.alpha, keep = 1.f - alpha;
    int win = 0;
    bool found = false;
    float best = 0.f;
    for (int j = 0; j < K; ++j) {
      const long long r = (long long)b * K + j;
      if (a.cand_tok[r] < 0) continue;
      float s = -INFINITY;
      for (int c = 0; c < a.n_chunks; ++c) s = fmaxf(s, a.sim[((long long)b * a.n_chunks + c) * K + j]);
      if (!(s > -INFINITY)) s = 0.f;                  // an empty context (not reached: prompts hold >= 1 token)
      const float score = __fsub_rn(__fmul_rn(keep, a.cand_p[r]), __fmul_rn(alpha, s));
      if (!found || score > best) {
        best = score;
        win = j;
        found = true;
      }
    }
    const int id = found ? a.cand_tok[(long long)b * K + win] : 0;
    const int step = *a.step;
    long long col = -1;
    if (!a.done[b]) {
      bool is_stop = false;
      for (int q = 0; q < a.n_stop; ++q) is_stop |= a.stop[q] == id;
      if (is_stop)
        a.done[b] = 1;
      else
        col = id;
    }
    if (step >= 0 && step < a.max_new) a.tokens[(long long)b * a.max_new + step] = col;
    a.win_ids[b] = id;
    s_w = win;
  }
  __syncthreads();
  const long long r = (long long)b * K + s_w;
  const __nv_bfloat16* h = a.hc + r * a.ldh;
  const int nvec = D >> 3;
  for (int c = tid; c < nvec; c += kCsSimThreads)
    reinterpret_cast<uint4*>(a.win_h + (long long)b * D)[c] = reinterpret_cast<const uint4*>(h)[c];
  if (L >= 0 && L < a.t_max) {
    for (int c = tid; c < nvec; c += kCsSimThreads)
      reinterpret_cast<uint4*>(a.ctx + ((long long)b * a.t_max + L) * D)[c] = reinterpret_cast<const uint4*>(h)[c];
    if (tid < 32) {
      const float nrm = warp_norm(h, D);
      if (tid == 0) a.ctx_norm[(long long)b * a.t_max + L] = nrm;
    }
    const int dv = a.Dh >> 3, per = a.n_layer * 2 * a.H * dv;
    const long long BK = (long long)a.B * K;
    for (int e = tid; e < per; e += kCsSimThreads) {
      const int d = e % dv;
      int rest = e / dv;
      const int hh = rest % a.H;
      rest /= a.H;
      const int kv = rest & 1, l = rest >> 1;
      const uint4 x = reinterpret_cast<const uint4*>(a.side + ((l * 2 + kv) * BK + r) * D + hh * a.Dh)[d];
      __nv_bfloat16* cache = kv ? a.v_cache : a.k_cache;
      reinterpret_cast<uint4*>(cache + ((((long long)l * a.B + b) * a.H + hh) * a.t_max + L) * a.Dh)[d] = x;
    }
  }
  __syncthreads();
  if (tid == 0) a.lens[b] = L + 1;
}

__global__ void cs_incr_kernel(int* step) { *step += 1; }

// one warp per (position, row): ctx[b, p] = h[b, p] and its norm, for p < lens[b]
__global__ void __launch_bounds__(32) cs_context_init_kernel(const __nv_bfloat16* h, int T, int D, const int* lens,
                                                              __nv_bfloat16* ctx, float* ctx_norm, int t_max) {
  const int p = blockIdx.x, b = blockIdx.y, lane = threadIdx.x;
  if (p >= min(lens[b], t_max)) return;
  const __nv_bfloat16* x = h + ((long long)b * T + p) * D;
  for (int c = lane; c < D / 8; c += 32)
    reinterpret_cast<uint4*>(ctx + ((long long)b * t_max + p) * D)[c] = reinterpret_cast<const uint4*>(x)[c];
  const float nrm = warp_norm(x, D);
  if (lane == 0) ctx_norm[(long long)b * t_max + p] = nrm;
}

inline int cs_chunks(int t_max) { return (t_max + kCsSimPos - 1) / kCsSimPos; }

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// fp32 elements of the cs_rerank scratch (`sim`) for B rows of k candidates and a context of t_max positions
long long adapcc_cs_sim_numel(int B, int kq, int t_max) {
  if (B < 1 || kq < 1 || t_max < 1) return 0;
  return (long long)B * cs_chunks(t_max) * kq;
}

// logits fp32 [B, ld]; step int32 [1]; suppress int32 list (null when empty); done int32 [B]; next_ids int64, cand_tok
// int32, cand_p fp32 [B * kq]
int adapcc_cs_select(const float* logits, int ld, int vocab, int B, int kq, const int* step, int min_new,
                     const int* suppress, int n_suppress, const int* done, long long* next_ids, int* cand_tok,
                     float* cand_p, void* stream) {
  if (B < 1 || kq < 1 || kq > kCsMaxK || vocab < 1 || ld < vocab) {
    set_error("cs_select: need B >= 1, 1 <= kq <= %d, 1 <= vocab <= ld (B=%d kq=%d vocab=%d ld=%d)", kCsMaxK, B, kq,
              vocab, ld);
    return -1;
  }
  if (n_suppress < 0 || n_suppress > kCsMaxSuppress || (n_suppress && !suppress)) {
    set_error("cs_select: at most %d suppressed ids (got %d)", kCsMaxSuppress, n_suppress);
    return -1;
  }
  if (!logits || !step || !done || !next_ids || !cand_tok || !cand_p) {
    set_error("cs_select: null pointer");
    return -1;
  }
  const size_t bits = n_suppress > 0 && min_new > 0 ? (size_t)(vocab + 31) / 32 * sizeof(uint32_t) : 0;
  if (bits > 200 * 1024) {
    set_error("cs_select: suppression needs vocab <= %d (got %d)", 200 * 1024 * 8, vocab);
    return -1;
  }
  if (bits > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(cs_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bits));
  SelectArgs a{logits, ld, vocab, kq, step, min_new, suppress, n_suppress, done, next_ids, cand_tok, cand_p};
  cs_select_kernel<<<B, kBeamThreads, bits, (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// hc bf16 [B * kq, ldh]; cand_tok int32 / cand_p fp32 [B * kq]; ctx bf16 [B, t_max, D]; ctx_norm fp32 [B, t_max]; sim
// fp32 adapcc_cs_sim_numel elements; lens, done int32 [B]; stop int32 list; step int32 [1]; tokens int64 [B, max_new];
// win_ids int64 [B]; win_h bf16 [B, D]; side bf16 [n_layer, 2, B * kq, D]; k_cache / v_cache bf16
// [n_layer, B, H, t_max, Dh] with D = H * Dh
int adapcc_cs_rerank(const void* hc, int ldh, int B, int kq, int D, const int* cand_tok, const float* cand_p,
                     float alpha, void* ctx, float* ctx_norm, int t_max, float* sim, int* lens, int* done,
                     const int* stop, int n_stop, int* step, long long* tokens, int max_new, long long* win_ids,
                     void* win_h, const void* side, void* k_cache, void* v_cache, int n_layer, int H, int Dh,
                     void* stream) {
  if (B < 1 || B > 65535 || kq < 1 || kq > kCsMaxK || t_max < 1 || max_new < 1 || n_layer < 1 || H < 1 || Dh < 8 ||
      Dh % 8 != 0 || D != H * Dh || D > kCsMaxD || ldh < D || ldh % 8 != 0) {
    set_error("cs_rerank: need 1 <= B <= 65535, 1 <= kq <= %d, t_max, max_new, n_layer >= 1, Dh a positive multiple "
              "of 8, D = H * Dh <= %d, ldh >= D a multiple of 8 (B=%d kq=%d D=%d H=%d Dh=%d ldh=%d)", kCsMaxK, kCsMaxD,
              B, kq, D, H, Dh, ldh);
    return -1;
  }
  if (!(alpha >= 0.f && alpha <= 1.f) || n_stop < 0 || n_stop > kCsMaxStop || (n_stop && !stop)) {
    set_error("cs_rerank: need 0 <= alpha <= 1 and at most %d stop ids (got %g, %d)", kCsMaxStop, (double)alpha, n_stop);
    return -1;
  }
  if (!hc || !cand_tok || !cand_p || !ctx || !ctx_norm || !sim || !lens || !done || !step || !tokens || !win_ids ||
      !win_h || !side || !k_cache || !v_cache) {
    set_error("cs_rerank: null pointer");
    return -1;
  }
  if (((uintptr_t)hc | (uintptr_t)ctx | (uintptr_t)win_h | (uintptr_t)side | (uintptr_t)k_cache |
       (uintptr_t)v_cache) & 15) {
    set_error("cs_rerank: hidden states, context, side buffer and caches must be 16-byte aligned");
    return -1;
  }
  RerankArgs a{(const __nv_bfloat16*)hc, ldh, kq, D, B, cand_tok, cand_p, alpha, (__nv_bfloat16*)ctx, ctx_norm,
               t_max, cs_chunks(t_max), sim, lens, done, stop, n_stop, step, tokens, max_new, win_ids,
               (__nv_bfloat16*)win_h, (const __nv_bfloat16*)side, (__nv_bfloat16*)k_cache, (__nv_bfloat16*)v_cache,
               n_layer, H, Dh};
  cudaStream_t s = (cudaStream_t)stream;
  const size_t smem = (size_t)kq * D * sizeof(__nv_bfloat16);
  if (smem > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(cs_sim_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cs_sim_kernel<<<dim3(a.n_chunks, B), kCsSimThreads, smem, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  cs_commit_kernel<<<B, kCsSimThreads, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  cs_incr_kernel<<<1, 1, 0, s>>>(step);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// h bf16 [B, T, D] (the prefill's final hidden states); lens int32 [B] (the prompt lengths); ctx bf16 [B, t_max, D];
// ctx_norm fp32 [B, t_max]
int adapcc_cs_context_init(const void* h, int B, int T, int D, const int* lens, void* ctx, float* ctx_norm, int t_max,
                           void* stream) {
  if (B < 1 || B > 65535 || T < 1 || T > t_max || D < 8 || D % 8 != 0) {
    set_error("cs_context_init: need 1 <= B <= 65535, 1 <= T <= t_max, D a positive multiple of 8 (B=%d T=%d "
              "t_max=%d D=%d)", B, T, t_max, D);
    return -1;
  }
  if (!h || !lens || !ctx || !ctx_norm || (((uintptr_t)h | (uintptr_t)ctx) & 15)) {
    set_error("cs_context_init: null or misaligned pointer");
    return -1;
  }
  cs_context_init_kernel<<<dim3(T, B), 32, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)h, T, D, lens,
                                                                      (__nv_bfloat16*)ctx, ctx_norm, t_max);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
