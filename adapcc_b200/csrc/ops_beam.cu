// Beam search for GPT-2 generation: the per-token selection and the KV-cache reordering on the device, so a beam-search
// token is one CUDA graph replay (decode step, LM head, beam_step, kv_reorder), like a sampled token.
//
//   beam_rows   : one 512-thread CTA per beam row. Three passes over the row in global memory (no shared-memory copy,
//                 so any vocabulary size works): the maximum m, Z = sum_i expf(l_i - m), then every candidate's score
//                 c_i = s + ((l_i - m) - logf(Z)) as a 64-bit key (order-preserving float bits, then the inverted id, so
//                 a tie goes to the lower id), of which the row's N = K + n_stop best are kept (topk_rows.cuh, shared
//                 with contrastive search).
//   beam_select : one warp per item. The K rows' N best, re-keyed by the flat index j * V + i, are walked in rank order
//                 (rounds of a warp maximum): the first K non-stop candidates become the new beams, stop candidates
//                 ranked before the K-th are offered to the finished set, and the done rule is applied (DESIGN.md §4a).
//   kv_reorder  : cache[l, r, :, pos] = cache[l, parent[r], :, pos] for the generated positions, through a scratch
//                 buffer (gather, then scatter), so cycles and many-to-one parent maps come out right.
//
// Every fp32 sum runs in an order fixed by the thread layout (per-thread loops in id order, shuffle trees, warp partials
// added by a shuffle tree in warp order); an item's result depends only on its own rows. ops/beam.py evaluates the same
// definition in fp64.
#include <cuda_bf16.h>

#include <cmath>
#include <cstdint>

#include "common.h"
#include "topk_rows.cuh"

namespace adapcc {

constexpr int kBeamMaxK = 16;
constexpr int kBeamMaxStop = 8;
constexpr int kBeamMaxN = kBeamMaxK + kBeamMaxStop;   // candidates kept per row
constexpr int kBeamMaxSuppress = 1024;
constexpr int kReorderThreads = 256;

struct BeamArgs {
  const float* logits;         // [B * K, ld], the first `vocab` columns used
  int ld, vocab, B, K, N;      // N = K + n_stop candidates per row
  float* scores;               // [B * K] running log-probability sums of the beams (-inf: dead)
  int* step;                   // tokens selected so far (read here, incremented by beam_step_incr_kernel)
  int min_new;
  const int* suppress;         // ids removed while *step < min_new
  int n_suppress;
  const int* stop;             // ids that finish a hypothesis
  int n_stop;
  const float* pen;            // [max_new + 1]: fl32(L ^ length_penalty)
  int alpha_pos;               // length_penalty > 0
  int max_new;
  int* done;                   // [B]
  unsigned long long* cand;    // [B * K, N] scratch: each row's N best keys
  long long* next_ids;         // [B * K]: the new beams' tokens (the decode graph's input)
  int* parent;                 // [B * K]: row the new beam continues (absolute row index)
  long long* hist_tok;         // [max_new, B * K]: token of beam k at each step
  int* hist_back;              // [max_new, B * K]: its parent beam (0..K-1) at the previous step
  float* fin_score;            // [B, K] finished set, best first: normalised score
  int* fin_n;                  // [B, K] tokens of the hypothesis (the stop token excluded)
  int* fin_src;                // [B, K] beam whose history at step fin_n - 1 holds those tokens
  int* fin_count;              // [B]
};

__global__ void __launch_bounds__(kBeamThreads, 1) beam_rows_kernel(const __grid_constant__ BeamArgs a) {
  extern __shared__ uint32_t s_bits[];                // removed ids, one bit each (only while step < min_new)
  __shared__ float s_red[kBeamWarps];
  __shared__ unsigned long long s_top[kBeamWarps * kBeamMaxN];
  const int row = blockIdx.x, b = row / a.K, tid = threadIdx.x, N = a.N;
  unsigned long long* out = a.cand + (long long)row * N;
  const float s = a.scores[row];
  if (a.done[b] || !(s > -INFINITY)) {                // a finished item or a dead beam offers nothing
    if (tid < N) out[tid] = 0ull;
    return;
  }
  const int V = a.vocab;
  const bool sup = *a.step < a.min_new && a.n_suppress > 0;
  if (sup) {
    for (int w = tid; w < (V + 31) / 32; w += kBeamThreads) s_bits[w] = 0u;
    __syncthreads();
    for (int j = tid; j < a.n_suppress; j += kBeamThreads) {
      const int id = a.suppress[j];
      if (id >= 0 && id < V) atomicOr(&s_bits[id >> 5], 1u << (id & 31));
    }
  }
  for (int e = tid; e < kBeamWarps * N; e += kBeamThreads) s_top[e] = 0ull;
  __syncthreads();
  RowView rv{a.logits + (long long)row * a.ld, sup ? s_bits : nullptr, V, s, 0.f, 0.f};
  float m = -INFINITY;
  for (int i = tid; i < V; i += kBeamThreads)
    if (!rv.removed(i)) m = fmaxf(m, __ldg(rv.l + i));
  m = beam_block_max(s_red, m);
  if (!(m > -INFINITY)) {                             // every id removed or at -inf
    if (tid < N) out[tid] = 0ull;
    return;
  }
  float z = 0.f;
  for (int i = tid; i < V; i += kBeamThreads)
    if (!rv.removed(i)) z += expf(__ldg(rv.l + i) - m);
  z = beam_block_sum(s_red, z);
  rv.m = m;
  rv.lz = logf(z);
  row_top_keys<false>(rv, N, s_top, out);
}

struct FinishedSet {
  float score[kBeamMaxK];
  int n[kBeamMaxK], src[kBeamMaxK];
  int count, K;
  // keeps the K best by score; on a tie the earlier entry stays ahead
  __device__ void offer(float sh, int nn, int sc) {
    if (count == K && !(sh > score[K - 1])) return;
    int p = count < K ? count : K - 1;
    for (; p > 0 && score[p - 1] < sh; --p) {
      score[p] = score[p - 1];
      n[p] = n[p - 1];
      src[p] = src[p - 1];
    }
    score[p] = sh;
    n[p] = nn;
    src[p] = sc;
    if (count < K) ++count;
  }
};

__global__ void __launch_bounds__(32) beam_select_kernel(const __grid_constant__ BeamArgs a) {
  __shared__ unsigned long long s_c[kBeamMaxK * kBeamMaxN];
  __shared__ FinishedSet fs;
  __shared__ int s_tok[kBeamMaxK], s_par[kBeamMaxK];
  __shared__ float s_sc[kBeamMaxK];
  const int b = blockIdx.x, lane = threadIdx.x, K = a.K, N = a.N, V = a.vocab, BK = a.B * a.K;
  const int step = *a.step;
  if (a.done[b] || step >= a.max_new) {               // nothing moves: every row keeps its own cache
    if (lane < K) a.parent[b * K + lane] = b * K + lane;
    return;
  }
  for (int e = lane; e < K * N; e += 32) {
    const int j = e / N;
    const unsigned long long v = a.cand[(long long)(b * K + j) * N + (e - j * N)];
    const uint32_t flat = (uint32_t)j * (uint32_t)V + (0xFFFFFFFFu - (uint32_t)v);
    s_c[e] = v ? (v & 0xFFFFFFFF00000000ull) | (0xFFFFFFFFu - flat) : 0ull;
  }
  if (lane == 0) {
    fs.K = K;
    fs.count = a.fin_count[b];
    for (int k = 0; k < K; ++k) {
      fs.score[k] = a.fin_score[b * K + k];
      fs.n[k] = a.fin_n[b * K + k];
      fs.src[k] = a.fin_src[b * K + k];
    }
  }
  __syncwarp();
  // the walk: candidates in rank order until K non-stop ones are taken
  const int L = step + 1;                             // tokens of a hypothesis that ends at this step
  int nb = 0;
  unsigned long long bound = ~0ull;
  while (nb < K) {
    unsigned long long best = 0ull;
    for (int e = lane; e < K * N; e += 32) {
      const unsigned long long v = s_c[e];
      if (v < bound && v > best) best = v;
    }
    best = warp_max_u64(best);
    if (best == 0ull) break;
    bound = best;
    const uint32_t flat = 0xFFFFFFFFu - (uint32_t)best;
    const int j = (int)(flat / (uint32_t)V), i = (int)(flat - (uint32_t)j * (uint32_t)V);
    const float c = beam_key2f((uint32_t)(best >> 32));
    bool is_stop = false;
    for (int q = 0; q < a.n_stop; ++q) is_stop |= a.stop[q] == i;
    if (lane == 0) {
      if (is_stop) {
        fs.offer(c / a.pen[L], L - 1, j);
      } else {
        s_tok[nb] = i;
        s_par[nb] = j;
        s_sc[nb] = c;
      }
    }
    nb += !is_stop;
  }
  __syncwarp();
  if (lane < K) {
    const int r = b * K + lane;
    const long long h = (long long)step * BK + r;
    if (lane < nb) {
      a.next_ids[r] = s_tok[lane];
      a.parent[r] = b * K + s_par[lane];
      a.scores[r] = s_sc[lane];
      a.hist_tok[h] = s_tok[lane];
      a.hist_back[h] = s_par[lane];
    } else {                                          // fewer than K finite non-stop candidates: a dead beam
      a.next_ids[r] = 0;
      a.parent[r] = r;
      a.scores[r] = -INFINITY;
      a.hist_tok[h] = -1;
      a.hist_back[h] = lane;
    }
  }
  if (lane == 0) {
    int done = 0;
    if (step == a.max_new - 1) {                      // the last step: the live beams are offered in beam order
      for (int k = 0; k < nb; ++k) fs.offer(s_sc[k] / a.pen[a.max_new], a.max_new, k);
      done = 1;
    } else if (nb == 0) {
      done = 1;
    } else if (fs.count == K) {
      // a live sum can only fall: its best reachable normalised score is s / L_max^a (a > 0) or s / (L + 1)^a
      const float reach = s_sc[0] / a.pen[a.alpha_pos ? a.max_new : L + 1];
      done = !(reach > fs.score[K - 1]);
    }
    a.done[b] = done;
    a.fin_count[b] = fs.count;
  }
  __syncwarp();
  if (lane < K) {
    a.fin_score[b * K + lane] = fs.score[lane];
    a.fin_n[b * K + lane] = fs.n[lane];
    a.fin_src[b * K + lane] = fs.src[lane];
  }
}

__global__ void beam_step_incr_kernel(int* step) { *step += 1; }

// ---- KV-cache reordering -----------------------------------------------------------------------------------------
struct ReorderArgs {
  __nv_bfloat16* k;            // [L, R, H, t_max, Dh]
  __nv_bfloat16* v;
  int L, R, H, t_max, Dh, max_new;
  const int* parent;           // [R]
  const int* prompt_len;       // [R]: first generated position
  const int* lens;             // [R]: positions held
  uint4* scratch;              // [R, max_new, L, 2, H, Dh / 8]
};

// one CTA per (generated position t, row r): every layer, k and v, every head. A row that keeps its own parent, a
// parent out of range and positions at or past lens[r] are skipped.
template <bool kGather>
__global__ void __launch_bounds__(kReorderThreads) kv_reorder_kernel(const __grid_constant__ ReorderArgs a) {
  const int t = blockIdx.x, r = blockIdx.y;
  const int p = a.parent[r];
  if (p == r || p < 0 || p >= a.R) return;
  const int pos = a.prompt_len[r] + t;
  if (pos < 0 || pos >= a.lens[r] || pos >= a.t_max) return;
  const int nv = a.Dh / 8;
  const int per = a.L * 2 * a.H * nv;
  uint4* scr = a.scratch + ((long long)r * a.max_new + t) * per;
  const int src_row = kGather ? p : r;
  for (int e = threadIdx.x; e < per; e += kReorderThreads) {
    const int d = e % nv;
    int rest = e / nv;
    const int h = rest % a.H;
    rest /= a.H;
    const int kv = rest & 1, l = rest >> 1;
    __nv_bfloat16* base = kv ? a.v : a.k;
    uint4* cell = reinterpret_cast<uint4*>(base + ((((long long)l * a.R + src_row) * a.H + h) * a.t_max + pos) * a.Dh) + d;
    if (kGather)
      scr[e] = *cell;
    else
      *cell = scr[e];
  }
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// logits fp32 [B*K, ld]; scores fp32 [B*K]; step int32 [1]; suppress / stop int32 lists (may be null when empty);
// pen fp32 [max_new + 1]; done int32 [B]; cand uint64 [B*K, K + n_stop]; next_ids int64 [B*K]; parent int32 [B*K];
// hist_tok int64 [max_new, B*K]; hist_back int32 [max_new, B*K]; fin_score fp32 / fin_n, fin_src int32 [B, K];
// fin_count int32 [B]
int adapcc_beam_step(const float* logits, int ld, int vocab, int B, int K, float* scores, int* step, int min_new,
                     const int* suppress, int n_suppress, const int* stop, int n_stop, const float* pen, int alpha_pos,
                     int max_new, int* done, void* cand, long long* next_ids, int* parent, long long* hist_tok,
                     int* hist_back, float* fin_score, int* fin_n, int* fin_src, int* fin_count, void* stream) {
  if (B < 1 || K < 1 || K > kBeamMaxK || vocab < 1 || ld < vocab || max_new < 1 ||
      (unsigned long long)K * (unsigned long long)vocab > 0xFFFFFFFFull) {
    set_error("beam_step: need B >= 1, 1 <= K <= %d, vocab >= 1, ld >= vocab, K * vocab < 2^32, max_new >= 1 (B=%d "
              "K=%d vocab=%d ld=%d max_new=%d)", kBeamMaxK, B, K, vocab, ld, max_new);
    return -1;
  }
  if (n_suppress < 0 || n_suppress > kBeamMaxSuppress || n_stop < 0 || n_stop > kBeamMaxStop ||
      (n_suppress && !suppress) || (n_stop && !stop)) {
    set_error("beam_step: at most %d suppressed and %d stop ids (got %d, %d)", kBeamMaxSuppress, kBeamMaxStop,
              n_suppress, n_stop);
    return -1;
  }
  if (!logits || !scores || !step || !pen || !done || !cand || !next_ids || !parent || !hist_tok || !hist_back ||
      !fin_score || !fin_n || !fin_src || !fin_count) {
    set_error("beam_step: null pointer");
    return -1;
  }
  const size_t bits = n_suppress > 0 && min_new > 0 ? (size_t)(vocab + 31) / 32 * sizeof(uint32_t) : 0;
  if (bits > 200 * 1024) {
    set_error("beam_step: suppression needs vocab <= %d (got %d)", 200 * 1024 * 8, vocab);
    return -1;
  }
  if (bits > 48 * 1024) CUDA_TRY(cudaFuncSetAttribute(beam_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                      (int)bits));
  BeamArgs a{logits, ld, vocab, B, K, K + n_stop, scores, step, min_new, suppress, n_suppress, stop, n_stop, pen,
             alpha_pos, max_new, done, (unsigned long long*)cand, next_ids, parent, hist_tok, hist_back, fin_score,
             fin_n, fin_src, fin_count};
  cudaStream_t s = (cudaStream_t)stream;
  beam_rows_kernel<<<B * K, kBeamThreads, bits, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  beam_select_kernel<<<B, 32, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  beam_step_incr_kernel<<<1, 1, 0, s>>>(step);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// k / v bf16 [L, R, H, t_max, Dh] contiguous; parent, prompt_len, lens int32 [R]; scratch at least
// R * max_new * L * 2 * H * Dh bf16, 16-byte aligned
int adapcc_kv_reorder(void* k, void* v, int L, int R, int H, int t_max, int Dh, const int* parent,
                      const int* prompt_len, const int* lens, int max_new, void* scratch, void* stream) {
  if (L < 1 || R < 1 || R > 65535 || H < 1 || t_max < 1 || Dh < 8 || Dh % 8 != 0 || max_new < 1) {
    set_error("kv_reorder: need L, H, t_max, max_new >= 1, 1 <= R <= 65535, Dh a positive multiple of 8 (L=%d R=%d "
              "H=%d t_max=%d Dh=%d max_new=%d)", L, R, H, t_max, Dh, max_new);
    return -1;
  }
  if (!k || !v || !parent || !prompt_len || !lens || !scratch) {
    set_error("kv_reorder: null pointer");
    return -1;
  }
  if (((uintptr_t)k | (uintptr_t)v | (uintptr_t)scratch) & 15) {
    set_error("kv_reorder: k, v and scratch must be 16-byte aligned");
    return -1;
  }
  ReorderArgs a{(__nv_bfloat16*)k, (__nv_bfloat16*)v, L, R, H, t_max, Dh, max_new, parent, prompt_len, lens,
                (uint4*)scratch};
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid(max_new, R);
  kv_reorder_kernel<true><<<grid, kReorderThreads, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  kv_reorder_kernel<false><<<grid, kReorderThreads, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
