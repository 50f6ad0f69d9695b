// Beam search for GPT-2 generation: the per-token selection and the KV-cache reordering on the device, so a beam-search
// token is one CUDA graph replay (decode step, LM head, beam_step, kv_reorder), like a sampled token.
//
//   beam_rows   : one 512-thread CTA per beam row. Three passes over the row in global memory (no shared-memory copy,
//                 so any vocabulary size works): the maximum m, Z = sum_i expf(l_i - m), then every candidate's score
//                 c_i = s + ((l_i - m) - logf(Z)) as a 64-bit key (order-preserving float bits, then the inverted id, so
//                 a tie goes to the lower id), of which the row's N = K + n_stop best are kept (topk_rows.cuh, shared
//                 with contrastive search).
//   beam_select : one warp per item, its G groups of Kg = K / G beams in order (G = 1: plain beam search). A group's
//                 Kg rows' N best, re-keyed by the flat index j * V + i and by the Hamming penalty of the earlier
//                 groups' new tokens, are walked in rank order (rounds of a warp maximum): the first Kg non-stop
//                 candidates become the group's new beams, stop candidates ranked before the Kg-th are offered to the
//                 group's finished set, and the done rule is applied per group (DESIGN.md §4a).
//   kv_reorder  : cache[l, r, :, pos] = cache[l, parent[r], :, pos] for the generated positions, through a scratch
//                 buffer (gather, then scatter), so cycles and many-to-one parent maps come out right.
//
// Beam sampling (HuggingFace's do_sample=True with num_beams > 1) replaces the first two:
//   beam_sample_rows   : one 1024-thread CTA per beam row, the row's x_i = l_i / T in shared memory (the sampler's
//                        row_prologue, sample_filter.cuh). m and log Z of the unfiltered row as beam_rows computes
//                        them, then the sampler's top-h, top-k / top-p and truncation filters with a minimum keep
//                        count, then c_i = s + lp_i / T and the Gumbel key
//                        g_i = c_i + G_i of every kept id, G_i from the item's Philox stream (gumbel_row). The row's M
//                        best keys (a bisection for the M-th key, then a rank sort) are kept, with their c next to them.
//   beam_sample_select : one 512-thread CTA per item. Each key's place in the item's draw order is its place in its
//                        row plus, per other row, a binary search for the larger keys; the first M form the sample.
//                        The first K draws that finish are offered, and the K best-c draws that do not are the new
//                        beams (DESIGN.md §4a).
//
// Stochastic beam search (Kool et al. 2019; rules R1-R8 of ops/beam.py) replaces them too:
//   beam_stochastic_rows   : one 1024-thread CTA per beam row, x_i = l_i / T in shared memory (row_prologue). The
//                            sampler's filters (min_keep 1), log Z over the kept ids, then phi_i = phi + lp'_i and
//                            Gphi_i = phi_i + G_i of every kept id (gumbel_row, its own Philox counter word); the K + 1
//                            best Gphi (row_best_keys, shared with beam_sample_rows) are offered with their keys
//                            truncated at the beam's key G and their phi.
//   beam_stochastic_select : one 512-thread CTA per item. Every entry of the pool (finished set, offered children) is
//                            ranked by counting; the K first survive, entry K + 1 raises kappa.
//
// The three select kernels write their rows' outputs through one write_beam, and the three step entry points make
// their launches through one launch_beam_step.
//
// Every fp32 sum runs in an order fixed by the thread layout (per-thread loops in id order, shuffle trees, warp partials
// added by a shuffle tree in warp order); an item's result depends only on its own rows. ops/beam.py evaluates the same
// definition in fp64.
#include <cuda_bf16.h>

#include <cmath>
#include <cstdint>
#include <type_traits>

#include "common.h"
#include "sample_filter.cuh"
#include "topk_rows.cuh"

namespace adapcc {

constexpr int kBeamMaxK = 16;
constexpr int kBeamMaxStop = 8;
constexpr int kBeamMaxN = kBeamMaxK + kBeamMaxStop;   // candidates kept per row
constexpr int kBeamMaxSuppress = 1024;
constexpr int kBeamSampleMaxM = (kBeamMaxStop + 1) * kBeamMaxK;   // sampled candidates per item and per row
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
  float* fin_score;            // [B, G, Kg] finished sets, best first: normalised score
  int* fin_n;                  // [B, G, Kg] tokens of the hypothesis (the stop token excluded)
  int* fin_src;                // [B, G, Kg] beam whose history at step fin_n - 1 holds those tokens
  int* fin_count;              // [B * G]
  int G;                       // groups; group g owns the item's beams g * Kg .. (g + 1) * Kg - 1, Kg = K / G
  int* group_done;             // [B * G] (beam_select only)
  float lambda;                // diversity penalty (beam_select only)
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
  // the set of K = cap entries at fin_*[base ..] with its count at fin_count[ci]: thread t < cap loads entry t,
  // thread 0 the count as well
  __device__ void load(const BeamArgs& a, int base, int ci, int cap, int t) {
    if (t < cap) {
      score[t] = a.fin_score[base + t];
      n[t] = a.fin_n[base + t];
      src[t] = a.fin_src[base + t];
    }
    if (t == 0) {
      K = cap;
      count = a.fin_count[ci];
    }
  }
  // thread t < K stores entry t, thread 0 the count as well
  __device__ void store(const BeamArgs& a, int base, int ci, int t) const {
    if (t < K) {
      a.fin_score[base + t] = score[t];
      a.fin_n[base + t] = n[t];
      a.fin_src[base + t] = src[t];
    }
    if (t == 0) a.fin_count[ci] = count;
  }
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
  // the done rule after a step that is not the last, for the best live sum s of L = step + 1 tokens: the set is full
  // and s cannot reach its worst entry. A live sum can only fall, so its best reachable normalised score is
  // s / L_max^a (a > 0) or s / (L + 1)^a.
  __device__ bool done_rule(const BeamArgs& a, float s, int L) const {
    return count == K && !(s / a.pen[a.alpha_pos ? a.max_new : L + 1] > score[K - 1]);
  }
};

// Beam k of item b at this step. With `hist` its history slot records token tok from beam par (0..K-1), else -1 and
// the beam itself. With `live` (implies hist) the row continues beam par with tok and the score sc; else it is dead:
// token 0, its own cache, -inf.
__device__ __forceinline__ void write_beam(const BeamArgs& a, int b, int k, int step, bool hist, bool live, int tok,
                                           int par, float sc) {
  const int r = b * a.K + k;
  const long long h = (long long)step * (a.B * a.K) + r;
  a.hist_tok[h] = hist ? tok : -1;
  a.hist_back[h] = hist ? par : k;
  a.next_ids[r] = live ? tok : 0;
  a.parent[r] = live ? b * a.K + par : r;
  a.scores[r] = live ? sc : -INFINITY;
}

// One warp per item; the groups in order g = 0 .. G-1. A candidate whose token the earlier groups' new beams of this
// step took n > 0 times is re-keyed with c' = fl32(c - fl32(lambda * n)); n = 0 keeps c's key, so group 0 selects as
// plain beam search with K = Kg. The rows' N = K + n_stop unpenalised best suffice: at most K - Kg tokens are
// penalised (DESIGN.md §4a).
__global__ void __launch_bounds__(32) beam_select_kernel(const __grid_constant__ BeamArgs a) {
  __shared__ unsigned long long s_c[kBeamMaxK * kBeamMaxN];
  __shared__ FinishedSet fs;
  __shared__ int s_tok[kBeamMaxK], s_par[kBeamMaxK], s_taken[kBeamMaxK];
  __shared__ float s_sc[kBeamMaxK];
  const int b = blockIdx.x, lane = threadIdx.x, K = a.K, N = a.N, V = a.vocab, G = a.G, Kg = K / G;
  const int step = *a.step;
  // the done groups, one bit each, read next to the item's flag so that the loads overlap
  const unsigned g_done = __ballot_sync(0xffffffffu, lane < G && a.group_done[b * G + lane]);
  if (a.done[b] || step >= a.max_new) {               // nothing moves: every row keeps its own cache
    if (lane < K) a.parent[b * K + lane] = b * K + lane;
    return;
  }
  const int L = step + 1;                             // tokens of a hypothesis that ends at this step
  int n_taken = 0, all_done = 1;
  for (int g = 0; g < G; ++g) {
    const int j0 = g * Kg, fo = b * K + j0, gi = b * G + g;
    if (g_done >> g & 1u) {                           // a done group: dead rows that keep their own cache
      if (lane < Kg) a.parent[fo + lane] = fo + lane;
      continue;
    }
    for (int e = lane; e < Kg * N; e += 32) {
      const int j = j0 + e / N;
      const unsigned long long v = a.cand[(long long)(b * K + j) * N + (e - (j - j0) * N)];
      const uint32_t i = 0xFFFFFFFFu - (uint32_t)v, flat = (uint32_t)j * (uint32_t)V + i;
      uint32_t hi = (uint32_t)(v >> 32);
      int n = 0;
      for (int t = 0; t < n_taken; ++t) n += s_taken[t] == (int)i;
      if (v && n) {
        const float cp = __fsub_rn(beam_key2f(hi), __fmul_rn(a.lambda, (float)n));
        hi = cp > -INFINITY ? beam_f2key(cp) : 0u;
      }
      s_c[e] = v && hi ? ((unsigned long long)hi << 32) | (0xFFFFFFFFu - flat) : 0ull;
    }
    fs.load(a, fo, gi, Kg, lane);
    __syncwarp();
    // the walk: candidates in rank order until Kg non-stop ones are taken
    int nb = 0;
    unsigned long long bound = ~0ull;
    while (nb < Kg) {
      unsigned long long best = 0ull;
      for (int e = lane; e < Kg * N; e += 32) {
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
          s_taken[n_taken + nb] = i;
        }
      }
      nb += !is_stop;
    }
    __syncwarp();
    int done = 1;
    if (lane == 0) {
      if (step == a.max_new - 1) {                    // the last step: the live beams are offered in beam order
        for (int k = 0; k < nb; ++k) fs.offer(s_sc[k] / a.pen[a.max_new], a.max_new, j0 + k);
      } else {
        done = nb == 0 || fs.done_rule(a, s_sc[0], L);
      }
      if (G > 1) a.group_done[gi] = done;             // one group: a.done[b] is its flag
    }
    done = __shfl_sync(0xffffffffu, done, 0);
    all_done &= done;
    n_taken += nb;                                    // this step's new beams count, even if the group is now done
    __syncwarp();
    fs.store(a, fo, gi, lane);
    // fewer than Kg finite non-stop candidates leave dead beams; a done group's beams are dead from now on, and with
    // one group the item's done flag stops beam_rows_kernel
    if (lane < Kg)
      write_beam(a, b, j0 + lane, step, lane < nb, lane < nb, s_tok[lane], s_par[lane],
                 done && G > 1 ? -INFINITY : s_sc[lane]);
    __syncwarp();
  }
  if (lane == 0) a.done[b] = all_done;
}

__global__ void beam_step_incr_kernel(int* step) { *step += 1; }

// ---- beam sampling ---------------------------------------------------------------------------------------------------
struct BeamSampleArgs {
  BeamArgs a;                  // a.N = M = min_keep * K; a.cand [B * K, M]: each row's M best Gumbel keys, best first
  float temperature, top_p;
  int top_k;
  const long long* seeds;      // [B]: the item's Philox key
  float* cand_c;               // [B * K, M]: the candidate score c next to each key
  float top_h;                 // 0: off
  FilterArgs f;                // f.min_keep = max(2, 1 + n_stop), for every filter
};

// G = -log(-log u) for u = ((w >> 8) + 0.5) 2^-24: -log u is taken from u below 1/2 and from 1 - u above, and both
// are exact in fp32, so G is finite for every word
__device__ __forceinline__ float beam_gumbel(uint32_t w) {
  const uint32_t k = w >> 8;
  const float nlu = k < (1u << 23) ? -logf((float)(2u * k + 1u) * 0x1p-25f)
                                   : -log1pf(-(float)((1u << 25) - 2u * k - 1u) * 0x1p-25f);
  return -logf(nlu);
}

// The Gumbel pass of the sampled row kernels over the row x in s_x: each kept id (f2key(x_i) >= tau) becomes
// score(i) + G_i, every other id -inf. Ids 4q..4q+3 take the four words of Philox at counter (q, j, step, c3) under
// the item's seed, one call per four ids of which one is kept; c3 is 0 for beam sampling, 1 for stochastic beam
// search. Every x is read before the call; the row is complete for every thread after it.
template <class Score>
__device__ __forceinline__ void gumbel_row(float* s_x, int V, uint32_t tau, long long seed, int j, int step,
                                           uint32_t c3, Score score) {
  const uint32_t k0 = (uint32_t)(unsigned long long)seed, k1 = (uint32_t)((unsigned long long)seed >> 32);
  for (int q = threadIdx.x; q < (V + 3) / 4; q += kSampleThreads) {
    bool kept[4], any = false;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int i = 4 * q + e;
      kept[e] = i < V && f2key(s_x[i]) >= tau;
      any |= kept[e];
    }
    uint4 w = make_uint4(0u, 0u, 0u, 0u);
    if (any) w = philox4((uint32_t)q, (uint32_t)j, (uint32_t)step, c3, k0, k1);
    const uint32_t words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int i = 4 * q + e;
      if (i < V) s_x[i] = kept[e] ? score(i) + beam_gumbel(words[e]) : -INFINITY;
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kSampleThreads, 1) beam_sample_rows_kernel(const __grid_constant__ BeamSampleArgs p) {
  extern __shared__ float s_x[];                      // [vocab]: x_i = l_i / T, then g_i of the kept ids (-inf else)
  __shared__ SampleSmem sm;
  __shared__ float s_red[32];                         // beam_block_* with 1024 threads: warps 16-31 hold identities
  __shared__ unsigned long long s_sel[kBeamSampleMaxM];   // also top-h's kTopHN entries
  __shared__ int s_n;
  static_assert(kBeamSampleMaxM >= kTopHN, "top-h shares s_sel");
  const BeamArgs& a = p.a;
  const int row = blockIdx.x, b = row / a.K, j = row - b * a.K, tid = threadIdx.x, V = a.vocab, M = a.N;
  unsigned long long* out = a.cand + (long long)row * M;
  float* out_c = p.cand_c + (long long)row * M;
  const float s = a.scores[row];
  if (a.done[b] || !(s > -INFINITY)) {                // a finished item or a dead beam offers nothing
    for (int e = tid; e < M; e += kSampleThreads) out[e] = 0ull;
    return;
  }
  const int step = *a.step;
  const float* l = a.logits + (long long)row * a.ld;
  unsigned long long best;
  const int present = row_prologue(s_x, sm, l, V, p.temperature, step, a.min_new, a.suppress, a.n_suppress, best);
  // m and log Z over the remaining ids, by the first 512 threads in beam_rows' order (the same bits)
  float m = -INFINITY;
  if (tid < kBeamThreads)
    for (int i = tid; i < V; i += kBeamThreads)
      if (s_x[i] != -INFINITY) m = fmaxf(m, __ldg(l + i));
  m = beam_block_max(s_red, m);
  if (!(m > -INFINITY)) {                             // every id removed or at -inf
    for (int e = tid; e < M; e += kSampleThreads) out[e] = 0ull;
    return;
  }
  float z = 0.f;
  if (tid < kBeamThreads)
#pragma unroll 2                                      // the prologue's count and maximum stay live: 4 costs 2 registers
    for (int i = tid; i < V; i += kBeamThreads)
      if (s_x[i] != -INFINITY) z += expf(__ldg(l + i) - m);
  z = beam_block_sum(s_red, z);
  const float lz = logf(z);
  auto cand_score = [&](int i) { return s + __fdiv_rn((__ldg(l + i) - m) - lz, p.temperature); };
  // the sampler's filters on x, each keeping at least min_keep values; log Z above is the unfiltered row's
  const uint32_t mkey = (uint32_t)(best >> 32);
  const float mx = key2f(mkey);
  int kept = present;
  if (p.top_h > 0.f) kept = top_h_row(s_x, sm, V, present, mx, p.top_h, p.f.min_keep, s_sel, &s_n);
  uint32_t tau = row_tau(s_x, sm, V, p.top_k, p.top_p, p.f.min_keep, kept, mkey, mx);
  if (p.f.on()) {
    filter_row(s_x, sm, V, p.f, tau, mx, mkey);
    tau = kNegInfKey + 1;                             // the survivors are the finite ids
  }
  __syncthreads();                                    // every x is read before the row becomes the keys
  gumbel_row(s_x, V, tau, p.seeds[b], j, step, 0u, cand_score);   // g_i = c_i + G_i
  row_best_keys(s_x, sm, V, M, s_sel, &s_n, [&](int r, unsigned long long v) {
    out[r] = v;
    if (v) out_c[r] = cand_score((int)(0xFFFFFFFFu - (uint32_t)v));
  });
}

__global__ void __launch_bounds__(kBeamThreads) beam_sample_select_kernel(const __grid_constant__ BeamSampleArgs p) {
  __shared__ unsigned long long s_k[kBeamMaxK * kBeamSampleMaxM];   // the K rows' keys, re-keyed by the flat index
  __shared__ float s_c[kBeamMaxK * kBeamSampleMaxM];
  __shared__ int s_draw[kBeamSampleMaxM];             // draw d -> element j * M + place
  __shared__ unsigned char s_fin[kBeamSampleMaxM];    // draw d finishes
  __shared__ int s_beam[kBeamMaxK];                   // new beam k -> draw
  __shared__ FinishedSet fs;
  const BeamArgs& a = p.a;
  const int b = blockIdx.x, tid = threadIdx.x, K = a.K, M = a.N, V = a.vocab;
  const int step = *a.step;
  if (a.done[b] || step >= a.max_new) {               // nothing moves: every row keeps its own cache
    if (tid < K) a.parent[b * K + tid] = b * K + tid;
    return;
  }
  for (int e = tid; e < K * M; e += kBeamThreads) {
    const int j = e / M;
    const long long o = (long long)(b * K + j) * M + (e - j * M);
    const unsigned long long v = a.cand[o];
    const uint32_t flat = (uint32_t)j * (uint32_t)V + (0xFFFFFFFFu - (uint32_t)v);
    s_k[e] = v ? (v & 0xFFFFFFFF00000000ull) | (0xFFFFFFFFu - flat) : 0ull;
    s_c[e] = p.cand_c[o];
  }
  for (int d = tid; d < M; d += kBeamThreads) s_draw[d] = -1;
  if (tid < K) s_beam[tid] = -1;
  fs.load(a, b * K, b, K, tid);
  __syncthreads();
  // the draw order: a key's place in its (sorted) row plus the number of larger keys in each other row
  for (int e = tid; e < K * M; e += kBeamThreads) {
    const unsigned long long v = s_k[e];
    if (!v) continue;
    const int j = e / M;
    int r = e - j * M;
    for (int j2 = 0; j2 < K && r < M; ++j2) {
      if (j2 == j) continue;
      const unsigned long long* row = s_k + j2 * M;
      int lo = 0, hi = M;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (row[mid] > v) lo = mid + 1;
        else hi = mid;
      }
      r += lo;
    }
    if (r < M) s_draw[r] = e;
  }
  __syncthreads();
  const bool last = step == a.max_new - 1;
  auto token = [&](int e) { return (int)((0xFFFFFFFFu - (uint32_t)s_k[e]) - (uint32_t)(e / M) * (uint32_t)V); };
  for (int d = tid; d < M; d += kBeamThreads) {
    const int e = s_draw[d];
    bool f = last;
    if (e >= 0)
      for (int q = 0; q < a.n_stop; ++q) f |= a.stop[q] == token(e);
    s_fin[d] = f;
  }
  __syncthreads();
  // the new beams: the K best c among the drawn candidates that do not finish, ties to the earlier draw
  for (int d = tid; d < M; d += kBeamThreads) {
    const int e = s_draw[d];
    if (e < 0 || s_fin[d]) continue;
    const float c = s_c[e];
    int r = 0;
    for (int d2 = 0; d2 < M && r < K; ++d2) {
      const int e2 = s_draw[d2];
      if (e2 < 0 || s_fin[d2]) continue;
      const float c2 = s_c[e2];
      r += c2 > c || (c2 == c && d2 < d);
    }
    if (r < K) s_beam[r] = d;
  }
  __syncthreads();
  const int L = step + 1;                             // tokens of a hypothesis that ends at this step
  if (tid == 0) {                                     // the first K draws that finish are offered, in draw order
    for (int d = 0; d < K; ++d) {
      const int e = s_draw[d];
      if (e < 0) break;
      if (!s_fin[d]) continue;
      const int i = token(e);
      bool is_stop = false;
      for (int q = 0; q < a.n_stop; ++q) is_stop |= a.stop[q] == i;
      if (is_stop) fs.offer(s_c[e] / a.pen[L], L - 1, e / M);
      else fs.offer(s_c[e] / a.pen[a.max_new], a.max_new, d);
    }
  }
  if (tid < K) {
    const int e = last ? s_draw[tid] : (s_beam[tid] >= 0 ? s_draw[s_beam[tid]] : -1);
    // the last step has no live beams; its history slot k holds draw k, which an offer may point at
    if (e >= 0) write_beam(a, b, tid, step, true, !last, token(e), e / M, s_c[e]);
    else write_beam(a, b, tid, step, false, false, 0, 0, 0.f);
  }
  __syncthreads();
  if (tid == 0) a.done[b] = last || s_beam[0] < 0 || fs.done_rule(a, s_c[s_draw[s_beam[0]]], L);
  fs.store(a, b * K, b, tid);
}

// ---- stochastic beam search ------------------------------------------------------------------------------------------
struct BeamStochasticArgs {
  BeamArgs a;                  // a.N = K + 1; a.scores: the live beams' log-probabilities phi (-inf: dead); a.fin_score
                               // the finished entries' keys; a.cand [B * K, K + 1]: each row's offered children
  float temperature, top_p;
  int top_k;
  const long long* seeds;      // [B]: the item's Philox key
  float top_h;                 // 0: off
  FilterArgs f;                // min_keep 1, as in the sampler
  float* keys;                 // [B * K]: the live beams' keys G
  float* cand_key;             // [B * K, K + 1]: the truncated key of the child next to each cand entry
  float* cand_phi;             // [B * K, K + 1]: its log-probability phi
  float* fin_phi;              // [B, K]: the finished entries' log-probabilities
  float* kappa;                // [B]: the largest key pruned so far
};

// log(1 - exp(x)) for x <= 0 without cancellation on either side of -ln 2; -inf at x = 0
__device__ __forceinline__ float log1mexp(float x) {
  return x > -0.693147182f ? logf(-expm1f(x)) : log1pf(-expf(x));
}

__global__ void __launch_bounds__(kSampleThreads, 1)
beam_stochastic_rows_kernel(const __grid_constant__ BeamStochasticArgs p) {
  extern __shared__ float s_x[];                      // [vocab]: x_i = l_i / T, then Gphi_i of the kept ids (-inf else)
  __shared__ SampleSmem sm;
  __shared__ unsigned long long s_sel[kTopHN > kBeamMaxK + 1 ? kTopHN : kBeamMaxK + 1];   // top-h's too
  __shared__ unsigned long long s_ord[kBeamMaxK + 1];
  __shared__ int s_n;
  __shared__ float s_z;
  const BeamArgs& a = p.a;
  const int row = blockIdx.x, b = row / a.K, j = row - b * a.K, tid = threadIdx.x, V = a.vocab, N = a.N;
  unsigned long long* out = a.cand + (long long)row * N;
  const float phi = a.scores[row];
  if (a.done[b] || !(phi > -INFINITY)) {              // a finished item or a dead beam offers nothing
    if (tid < N) out[tid] = 0ull;
    return;
  }
  const int step = *a.step;
  const float* l = a.logits + (long long)row * a.ld;
  unsigned long long best;
  const int present = row_prologue(s_x, sm, l, V, p.temperature, step, a.min_new, a.suppress, a.n_suppress, best);
  if (present == 0) {                                 // every id removed or at -inf
    if (tid < N) out[tid] = 0ull;
    return;
  }
  // the sampler's filters (min_keep 1), then log Z over the kept ids: lp'_i = (x_i - m) - log Z
  const uint32_t mkey = (uint32_t)(best >> 32);
  const float m = key2f(mkey);
  int kept = present;
  if (p.top_h > 0.f) kept = top_h_row(s_x, sm, V, present, m, p.top_h, 1, s_sel, &s_n);
  uint32_t tau = row_tau(s_x, sm, V, p.top_k, p.top_p, 1, kept, mkey, m);
  if (p.f.on()) {
    filter_row(s_x, sm, V, p.f, tau, m, mkey);
    tau = kNegInfKey + 1;
  }
  float z = 0.f;
  int u0 = 0, u1 = 0, u2 = 0;
  for (int i = tid; i < V; i += kSampleThreads) {
    const float x = s_x[i];
    if (f2key(x) >= tau) z += expf(x - m);
  }
  block_sum(sm, z, u0, u1, u2);                       // its barriers order every read of x before the writes below
  const float lz = logf(z);
  auto child_phi = [&](int i) { return phi + ((__fdiv_rn(__ldg(l + i), p.temperature) - m) - lz); };
  gumbel_row(s_x, V, tau, p.seeds[b], j, step, 1u, child_phi);    // Gphi_i = phi_i + G_i
  // the K + 1 best children by Gphi, each with its key truncated at G: G - softplus(v),
  // v = G - Gphi + log1mexp(Gphi - Zj), Zj the row's largest Gphi (its child keeps G exactly)
  const float G = p.keys[row];
  float* out_key = p.cand_key + (long long)row * N;
  float* out_phi = p.cand_phi + (long long)row * N;
  const uint32_t zkey = row_best_keys(s_x, sm, V, N, s_sel, &s_n, [&](int r, unsigned long long v) {
    out[r] = v;
    s_ord[r] = v;
  });
  if (tid == 0) s_z = key2f(zkey);
  __syncthreads();
  if (tid < N && s_ord[tid]) {
    const unsigned long long v = s_ord[tid];
    const int i = (int)(0xFFFFFFFFu - (uint32_t)v);
    const float gphi = key2f((uint32_t)(v >> 32));
    const float u = (G - gphi) + log1mexp(gphi - s_z);
    out_key[tid] = (G - fmaxf(u, 0.f)) - log1pf(expf(-fabsf(u)));
    out_phi[tid] = child_phi(i);
  }
}

// One 512-thread CTA per item. The pool is the finished set (entries 0..K-1) and the rows' offered children; each
// entry's rank is the number of entries before it (descending key, then finished before children, the set's order,
// the lower flat index j * V + i), so the K + 1 first are known without a sort.
__global__ void __launch_bounds__(kBeamThreads) beam_stochastic_select_kernel(
    const __grid_constant__ BeamStochasticArgs p) {
  constexpr int kPool = kBeamMaxK + kBeamMaxK * (kBeamMaxK + 1);
  __shared__ unsigned long long s_k[kPool];           // (key bits << 32) | inverted order; 0: no entry
  __shared__ int s_at[kBeamMaxK + 1];                 // rank -> entry
  __shared__ FinishedSet old, nw;
  __shared__ float s_ophi[kBeamMaxK], s_nphi[kBeamMaxK];
  __shared__ int s_tok[kBeamMaxK], s_par[kBeamMaxK];
  __shared__ float s_phi[kBeamMaxK], s_key[kBeamMaxK];
  __shared__ int s_nb;
  const BeamArgs& a = p.a;
  const int b = blockIdx.x, tid = threadIdx.x, K = a.K, N = a.N, V = a.vocab, P = K + K * N;
  const int step = *a.step;
  if (a.done[b] || step >= a.max_new) {               // nothing moves: every row keeps its own cache
    if (tid < K) a.parent[b * K + tid] = b * K + tid;
    return;
  }
  old.load(a, b * K, b, K, tid);
  if (tid < K) {
    s_ophi[tid] = p.fin_phi[b * K + tid];
    nw.score[tid] = -INFINITY;
    nw.n[tid] = 0;
    nw.src[tid] = 0;
    s_nphi[tid] = -INFINITY;
  }
  if (tid <= K) s_at[tid] = -1;
  for (int e = tid; e < K * N; e += kBeamThreads) {
    const int j = e / N;
    const long long o = (long long)(b * K + j) * N + (e - j * N);
    const unsigned long long v = a.cand[o];
    const uint32_t key = v ? f2key(p.cand_key[o]) : 0u;
    const uint32_t flat = (uint32_t)j * (uint32_t)V + (0xFFFFFFFFu - (uint32_t)v);
    s_k[K + e] = key > kNegInfKey ? ((unsigned long long)key << 32) | (0xFFFFFFFFu - kBeamMaxK - flat) : 0ull;
  }
  __syncthreads();
  if (tid < K) {
    const uint32_t key = tid < old.count ? f2key(old.score[tid]) : 0u;
    s_k[tid] = key > kNegInfKey ? ((unsigned long long)key << 32) | (0xFFFFFFFFu - (uint32_t)tid) : 0ull;
  }
  __syncthreads();
  for (int e = tid; e < P; e += kBeamThreads) {
    const unsigned long long v = s_k[e];
    if (!v) continue;
    int r = 0;
    for (int f = 0; f < P && r <= K; ++f) r += s_k[f] > v;
    if (r <= K) s_at[r] = e;
  }
  __syncthreads();
  const bool last = step == a.max_new - 1;
  const int L = step + 1;                             // tokens of a hypothesis that ends at this step
  if (tid == 0) {                                     // the K first survive, in rank order
    nw.K = K;
    nw.count = 0;
    int nb = 0;
    auto finish = [&](float key, int n, int src, float ph) {
      nw.score[nw.count] = key;
      nw.n[nw.count] = n;
      nw.src[nw.count] = src;
      s_nphi[nw.count++] = ph;
    };
    for (int r = 0; r < K && s_at[r] >= 0; ++r) {
      const int e = s_at[r];
      const float key = key2f((uint32_t)(s_k[e] >> 32));
      if (e < K) {
        finish(key, old.n[e], old.src[e], s_ophi[e]);
        continue;
      }
      const int j = (e - K) / N;
      const long long o = (long long)(b * K + j) * N + (e - K - j * N);
      const int i = (int)(0xFFFFFFFFu - (uint32_t)a.cand[o]);
      bool is_stop = false;
      for (int q = 0; q < a.n_stop; ++q) is_stop |= a.stop[q] == i;
      if (is_stop) {
        finish(key, L - 1, j, p.cand_phi[o]);
        continue;
      }
      // a new beam takes history slot nb; at the last step it finishes there
      s_tok[nb] = i;
      s_par[nb] = j;
      s_phi[nb] = p.cand_phi[o];
      s_key[nb] = key;
      if (last) finish(key, a.max_new, nb, p.cand_phi[o]);
      ++nb;
    }
    if (s_at[K] >= 0) p.kappa[b] = fmaxf(p.kappa[b], key2f((uint32_t)(s_k[s_at[K]] >> 32)));
    s_nb = nb;
    a.done[b] = last || nb == 0;
  }
  __syncthreads();
  nw.store(a, b * K, b, tid);
  if (tid < K) {
    p.fin_phi[b * K + tid] = s_nphi[tid];
    const bool live = tid < s_nb && !last;
    write_beam(a, b, tid, step, tid < s_nb, live, s_tok[tid], s_par[tid], s_phi[tid]);
    p.keys[b * K + tid] = live ? s_key[tid] : -INFINITY;
  }
}

// ---- KV-cache reordering -----------------------------------------------------------------------------------------
struct ReorderArgs {
  __nv_bfloat16* k;            // [L, R, H, t_max, Dh]
  __nv_bfloat16* v;
  int L, R, H, t_max, Dh, max_new;
  const int* parent;           // [R]
  const int* prompt_len;       // [R]: first generated position
  const int* lens;             // [R]: positions held
  uint4* scratch;              // [R, max_new, L, 2, H, Dh / 8]; fp8: [R, max_new, L, 2, H, Dh / 16], then the scales
  float* k_scale;              // fp8 cache (k / v then hold e4m3 bytes): [L, R, H, t_max]; else null
  float* v_scale;
};

// one CTA per (generated position t, row r): every layer, k and v, every head. A row that keeps its own parent, a
// parent out of range and positions at or past lens[r] are skipped. kFp8: k / v are e4m3 bytes, and the scales move
// through float [R, max_new, L, 2, H] after the bytes in scratch.
template <bool kGather, bool kFp8>
__global__ void __launch_bounds__(kReorderThreads) kv_reorder_kernel(const __grid_constant__ ReorderArgs a) {
  using T = typename std::conditional<kFp8, uint8_t, __nv_bfloat16>::type;
  const int t = blockIdx.x, r = blockIdx.y;
  const int p = a.parent[r];
  if (p == r || p < 0 || p >= a.R) return;
  const int pos = a.prompt_len[r] + t;
  if (pos < 0 || pos >= a.lens[r] || pos >= a.t_max) return;
  const int nv = a.Dh / (16 / sizeof(T));
  const int per = a.L * 2 * a.H * nv;
  uint4* scr = a.scratch + ((long long)r * a.max_new + t) * per;
  const int src_row = kGather ? p : r;
  for (int e = threadIdx.x; e < per; e += kReorderThreads) {
    const int d = e % nv;
    int rest = e / nv;
    const int h = rest % a.H;
    rest /= a.H;
    const int kv = rest & 1, l = rest >> 1;
    T* base = reinterpret_cast<T*>(kv ? a.v : a.k);
    uint4* cell = reinterpret_cast<uint4*>(base + ((((long long)l * a.R + src_row) * a.H + h) * a.t_max + pos) * a.Dh) + d;
    if (kGather)
      scr[e] = *cell;
    else
      *cell = scr[e];
  }
  if constexpr (kFp8) {
    const int ns = a.L * 2 * a.H;
    float* sscr = reinterpret_cast<float*>(a.scratch + (long long)a.R * a.max_new * per) +
                  ((long long)r * a.max_new + t) * ns;
    for (int e = threadIdx.x; e < ns; e += kReorderThreads) {
      const int h = e % a.H, kv = (e / a.H) & 1, l = e / (2 * a.H);
      float* cell = (kv ? a.v_scale : a.k_scale) + (((long long)l * a.R + src_row) * a.H + h) * a.t_max + pos;
      if (kGather)
        sscr[e] = *cell;
      else
        *cell = sscr[e];
    }
  }
}

// the checks every step entry point makes; each then checks its own mode's arguments and sets a.N. alpha_pos < 0: no
// length penalty (stochastic beam search), so no pen
static int check_beam_args(const char* who, const BeamArgs& a) {
  if (a.B < 1 || a.K < 1 || a.K > kBeamMaxK || a.vocab < 1 || a.ld < a.vocab || a.max_new < 1) {
    set_error("%s: need B >= 1, 1 <= K <= %d, vocab >= 1, ld >= vocab, max_new >= 1 (B=%d K=%d vocab=%d ld=%d "
              "max_new=%d)", who, kBeamMaxK, a.B, a.K, a.vocab, a.ld, a.max_new);
    return -1;
  }
  if (a.n_suppress < 0 || a.n_suppress > kBeamMaxSuppress || a.n_stop < 0 || a.n_stop > kBeamMaxStop ||
      (a.n_suppress && !a.suppress) || (a.n_stop && !a.stop)) {
    set_error("%s: at most %d suppressed and %d stop ids (got %d, %d)", who, kBeamMaxSuppress, kBeamMaxStop,
              a.n_suppress, a.n_stop);
    return -1;
  }
  if (!a.logits || !a.scores || !a.step || (a.alpha_pos >= 0 && !a.pen) || !a.done || !a.cand || !a.next_ids || !a.parent || !a.hist_tok ||
      !a.hist_back || !a.fin_score || !a.fin_n || !a.fin_src || !a.fin_count) {
    set_error("%s: null pointer", who);
    return -1;
  }
  return 0;
}

// the sampled modes' scalars, and the vocabulary their row kernels hold in shared memory
static int check_sampling_args(const char* who, int vocab, float temperature, int top_k, float top_p) {
  if (vocab > kSampleMaxVocab || !(temperature > 0.f) || top_k < 0 || !(top_p > 0.f && top_p <= 1.f)) {
    set_error("%s: need vocab <= %d, temperature > 0, top_k >= 0, 0 < top_p <= 1 (got %d, %g, %d, %g)", who,
              kSampleMaxVocab, vocab, temperature, top_k, top_p);
    return -1;
  }
  return 0;
}

// the truncation filters of the sampled modes, each off at its neutral value
static int check_filter_args(const char* who, float min_p, float typical_p, float epsilon, float eta, float top_h) {
  if (!(min_p >= 0.f && min_p <= 1.f) || !(typical_p > 0.f && typical_p <= 1.f) || !(epsilon >= 0.f && epsilon < 1.f) ||
      !(eta >= 0.f && eta < 1.f) || !(top_h >= 0.f && top_h <= 1.f)) {
    set_error("%s: need 0 <= min_p <= 1, 0 < typical_p <= 1, 0 <= epsilon < 1, 0 <= eta < 1, 0 <= top_h <= 1 (got "
              "%g, %g, %g, %g, %g)", who, min_p, typical_p, epsilon, eta, top_h);
    return -1;
  }
  return 0;
}

// One step on the stream: `rows` with a CTA of `rows_threads` per beam row and `smem` bytes of dynamic shared memory
// (opted in above the default 48 KB), `select` with a CTA of `select_threads` per item, then the step increment.
template <class Args>
static int launch_beam_step(const BeamArgs& a, const Args& p, void (*rows)(Args), int rows_threads, size_t smem,
                            void (*select)(Args), int select_threads, void* stream) {
  if (smem > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(rows, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaStream_t s = (cudaStream_t)stream;
  rows<<<a.B * a.K, rows_threads, smem, s>>>(p);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  select<<<a.B, select_threads, 0, s>>>(p);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  beam_step_incr_kernel<<<1, 1, 0, s>>>(a.step);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// logits fp32 [B*K, ld]; scores fp32 [B*K]; step int32 [1]; suppress / stop int32 lists (may be null when empty);
// pen fp32 [max_new + 1]; done int32 [B]; group_done int32 [B*G] with the groups G dividing K (1: plain beam search);
// cand uint64 [B*K, K + n_stop]; next_ids int64 [B*K]; parent int32 [B*K]; hist_tok int64 / hist_back int32
// [max_new, B*K]; fin_score fp32 / fin_n, fin_src int32 [B, K]; fin_count int32 [B*G]; the diversity penalty lambda
// finite and >= 0
int adapcc_beam_step(const float* logits, int ld, int vocab, int B, int K, int G, float* scores, int* step, int min_new,
                     const int* suppress, int n_suppress, const int* stop, int n_stop, const float* pen, int alpha_pos,
                     int max_new, int* done, int* group_done, void* cand, long long* next_ids, int* parent,
                     long long* hist_tok, int* hist_back, float* fin_score, int* fin_n, int* fin_src, int* fin_count,
                     float lambda, void* stream) {
  BeamArgs a{logits, ld, vocab, B, K, 0, scores, step, min_new, suppress, n_suppress, stop, n_stop, pen, alpha_pos,
             max_new, done, (unsigned long long*)cand, next_ids, parent, hist_tok, hist_back, fin_score, fin_n,
             fin_src, fin_count, G, group_done, lambda};
  if (check_beam_args("beam_step", a)) return -1;
  if (G < 1 || K % G != 0 || (unsigned long long)K * (unsigned long long)vocab > 0xFFFFFFFFull || !group_done ||
      !(lambda >= 0.f && lambda < INFINITY)) {
    set_error("beam_step: need G >= 1 dividing K, K * vocab < 2^32, a finite diversity penalty >= 0 and group_done "
              "(K=%d G=%d vocab=%d lambda=%g)", K, G, vocab, lambda);
    return -1;
  }
  a.N = K + n_stop;
  const size_t bits = n_suppress > 0 && min_new > 0 ? (size_t)(vocab + 31) / 32 * sizeof(uint32_t) : 0;
  if (bits > 200 * 1024) {
    set_error("beam_step: suppression needs vocab <= %d (got %d)", 200 * 1024 * 8, vocab);
    return -1;
  }
  return launch_beam_step(a, a, beam_rows_kernel, kBeamThreads, bits, beam_select_kernel, 32, stream);
}

// adapcc_beam_step's arguments for one group (no G, group_done or lambda; fin_count int32 [B]), plus cand_c fp32
// [B*K, M] next to cand uint64 [B*K, M] (M = max(2, 1 + n_stop) * K), the sampling scalars (temperature > 0,
// top_k >= 0 with 0 off, 0 < top_p <= 1), seeds int64 [B] and the truncation filters (off at min_p = 0,
// typical_p = 1, epsilon = 0, eta = 0, top_h = 0); vocab <= 56 Ki
int adapcc_beam_sample_step(const float* logits, int ld, int vocab, int B, int K, float* scores, int* step,
                            int min_new, const int* suppress, int n_suppress, const int* stop, int n_stop,
                            const float* pen, int alpha_pos, int max_new, int* done, void* cand, float* cand_c,
                            long long* next_ids, int* parent, long long* hist_tok, int* hist_back, float* fin_score,
                            int* fin_n, int* fin_src, int* fin_count, float temperature, int top_k, float top_p,
                            const long long* seeds, float min_p, float typical_p, float epsilon, float eta,
                            float top_h, void* stream) {
  BeamSampleArgs p{BeamArgs{logits, ld, vocab, B, K, 0, scores, step, min_new, suppress, n_suppress, stop, n_stop,
                            pen, alpha_pos, max_new, done, (unsigned long long*)cand, next_ids, parent, hist_tok,
                            hist_back, fin_score, fin_n, fin_src, fin_count, 1, nullptr, 0.f},
                   temperature, top_p, top_k, seeds, cand_c, top_h, FilterArgs{min_p, typical_p, epsilon, eta, 0}};
  if (check_beam_args("beam_sample_step", p.a) ||
      check_sampling_args("beam_sample_step", vocab, temperature, top_k, top_p) ||
      check_filter_args("beam_sample_step", min_p, typical_p, epsilon, eta, top_h))
    return -1;
  if (!cand_c || !seeds) {
    set_error("beam_sample_step: null pointer");
    return -1;
  }
  p.f.min_keep = n_stop + 1 > 2 ? n_stop + 1 : 2;
  p.a.N = p.f.min_keep * K;
  return launch_beam_step(p.a, p, beam_sample_rows_kernel, kSampleThreads, (size_t)vocab * sizeof(float),
                          beam_sample_select_kernel, kBeamThreads, stream);
}

// stochastic beam search: adapcc_beam_sample_step's arguments without the length penalty, with scores the live beams'
// log-probabilities, keys fp32 [B*K] their keys, cand uint64 / cand_key, cand_phi fp32 [B*K, K + 1] the offered
// children, fin_score the finished entries' keys and fin_phi fp32 [B, K] their log-probabilities, kappa fp32 [B],
// then adapcc_beam_sample_step's truncation filters
int adapcc_beam_stochastic_step(const float* logits, int ld, int vocab, int B, int K, float* scores, float* keys,
                                int* step, int min_new, const int* suppress, int n_suppress, const int* stop, int n_stop,
                                int max_new, int* done, void* cand, float* cand_key, float* cand_phi,
                                long long* next_ids, int* parent, long long* hist_tok, int* hist_back,
                                float* fin_score, float* fin_phi, int* fin_n, int* fin_src, int* fin_count,
                                float* kappa, float temperature, int top_k, float top_p, const long long* seeds,
                                float min_p, float typical_p, float epsilon, float eta, float top_h, void* stream) {
  BeamStochasticArgs p{BeamArgs{logits, ld, vocab, B, K, 0, scores, step, min_new, suppress, n_suppress, stop, n_stop,
                                nullptr, -1, max_new, done, (unsigned long long*)cand, next_ids, parent, hist_tok,
                                hist_back, fin_score, fin_n, fin_src, fin_count, 1, nullptr, 0.f},
                       temperature, top_p, top_k, seeds, top_h, FilterArgs{min_p, typical_p, epsilon, eta, 1}, keys,
                       cand_key, cand_phi, fin_phi, kappa};
  if (check_beam_args("beam_stochastic_step", p.a) ||
      check_sampling_args("beam_stochastic_step", vocab, temperature, top_k, top_p) ||
      check_filter_args("beam_stochastic_step", min_p, typical_p, epsilon, eta, top_h))
    return -1;
  if (!keys || !cand_key || !cand_phi || !fin_phi || !kappa || !seeds) {
    set_error("beam_stochastic_step: null pointer");
    return -1;
  }
  p.a.N = K + 1;
  return launch_beam_step(p.a, p, beam_stochastic_rows_kernel, kSampleThreads, (size_t)vocab * sizeof(float),
                          beam_stochastic_select_kernel, kBeamThreads, stream);
}

// k / v bf16 [L, R, H, t_max, Dh] contiguous; parent, prompt_len, lens int32 [R]; scratch at least
// R * max_new * L * 2 * H * Dh bf16, 16-byte aligned. k_scale / v_scale: null for a bf16 cache; with an fp8 cache (k / v
// e4m3 bytes [L, R, H, t_max, Dh], Dh a multiple of 16) fp32 [L, R, H, t_max], and scratch at least
// R * max_new * L * 2 * H * (Dh + 4) bytes
int adapcc_kv_reorder(void* k, void* v, int L, int R, int H, int t_max, int Dh, const int* parent,
                      const int* prompt_len, const int* lens, int max_new, void* scratch, void* k_scale, void* v_scale,
                      void* stream) {
  if (L < 1 || R < 1 || R > 65535 || H < 1 || t_max < 1 || Dh < 8 || Dh % 8 != 0 || max_new < 1) {
    set_error("kv_reorder: need L, H, t_max, max_new >= 1, 1 <= R <= 65535, Dh a positive multiple of 8 (L=%d R=%d "
              "H=%d t_max=%d Dh=%d max_new=%d)", L, R, H, t_max, Dh, max_new);
    return -1;
  }
  if (!k_scale != !v_scale || (k_scale && Dh % 16 != 0) || ((uintptr_t)k_scale | (uintptr_t)v_scale) & 3) {
    set_error("kv_reorder: k_scale and v_scale must both be null, or both 4-byte aligned with Dh a multiple of 16 "
              "(Dh=%d)", Dh);
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
                (uint4*)scratch, (float*)k_scale, (float*)v_scale};
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid(max_new, R);
  if (k_scale)
    kv_reorder_kernel<true, true><<<grid, kReorderThreads, 0, s>>>(a);
  else
    kv_reorder_kernel<true, false><<<grid, kReorderThreads, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  if (k_scale)
    kv_reorder_kernel<false, true><<<grid, kReorderThreads, 0, s>>>(a);
  else
    kv_reorder_kernel<false, false><<<grid, kReorderThreads, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
