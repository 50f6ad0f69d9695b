// Speculative decoding for GPT-2 generation on the device, so a verify step is one CUDA graph replay: the drafts, the
// model on k + 1 slots per row, the LM head, then the slots' tokens and acceptance. The definitions are in
// ops/lookup.py, ops/assisted.py and DESIGN.md §4a. The slots' attention is adapcc_verify_attn in ops_decode.cu; this
// file finds prompt lookup's drafts, sets up a draft model's round, takes the arg-max of the slots (greedy
// verification) and accepts the drafts. adapcc_lookup_argmax launches lk_argmax and adapcc_lookup_accept lk_accept, so
// acceptance runs the same way on arg-maxes and on the draws of adapcc_sample_slots / adapcc_spec_slots
// (ops_sample.cu).
//
//   lk_argmax      : grid (slots, B), 512 threads: each real slot's arg-max (topk_rows.cuh with N = 1, ties to the lower
//                    id); suppress_ids are removed while emitted[b] + j < min_new.
//   lk_accept      : one thread per row: emits g_0, g_1, ... while the draft of the next slot equals the token just
//                    emitted, stopping at a stop id (sets done, not written), at max_new tokens (sets done) or at the
//                    first rejected draft; appends the emitted ids to the row's sequence, advances lens and emitted.
//                    With per-slot accepted flags (rejection sampling, spec_slots_kernel in ops_sample.cu) it emits
//                    the accepted drafts instead, then the token the slot of the first rejection holds.
//   lk_draft       : one CTA per row: the earliest earlier occurrence of the sequence's last m tokens (m from the
//                    n-gram size down to 1); the tokens after it are the drafts. Writes the next step's ids, positions
//                    and real-slot count.
//   lk_round       : one thread per row, assisted generation (a draft model proposes the drafts, ops/assisted.py): the
//                    start of a round from the target's state alone: slot 0, positions, real-slot count, the draft's
//                    first input and positions, and the draft cache's lengths. The drafts are drawn by
//                    sample_slots_kernel (ops_sample.cu).
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

constexpr int kLkMaxSlots = 16;                     // k + 1: the row's last token and up to 15 drafts
constexpr int kLkMaxNgram = 16;
constexpr int kLkMaxIds = 1024;                     // ids per suppress / stop list
constexpr int kLkDraftThreads = 256;

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
  const int* acc;              // [B * kq] or null: draft j + 1 accepted (rejection sampling); g then holds the token a
                               // round emits last if it ends at slot j
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
    const long long o = (long long)b * a.kq + j;
    const bool accepted = a.acc && j + 1 < nq && a.acc[o];
    const int t = accepted ? (int)a.ids[o + 1] : a.g[o];
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
    if (a.acc ? !accepted : j + 1 < nq && a.ids[o + 1] != t) break;   // draft j + 1 rejected
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

// ---- round set-up of assisted generation (a draft model proposes the drafts) ---------------------------------------
struct RoundArgs {
  const int* seq;              // [B, t_max]
  int t_max, B, kq, max_new, n_pos;
  const int* lens;             // [B]: the target cache's lengths
  const int* emitted;          // [B]
  const int* done;             // [B]
  long long* ids;              // [B * kq]: slot 0 the last token, the drafts' slots 0 (the draft draws fill them)
  long long* pos;              // [B * kq]: lens[b] + j, clamped to t_max - 1
  int* nq;                     // [B]: 1 + min(k, max_new - emitted - 1), 0 for a done row
  long long* d_in;             // [B]: the draft's first input, the last token
  int* d_lens;                 // [B]: the draft cache's lengths, set to the target's
  long long* d_pos;            // [kq, B]: the draft's positions at its step j, lens[b] + j clamped to n_pos - 1
};

__global__ void lk_round_kernel(const __grid_constant__ RoundArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  const int L = min(max(a.lens[b], 0), a.t_max - 1), K = a.kq - 1;
  const bool live = !a.done[b];
  const long long x = live ? a.seq[(long long)b * a.t_max + L] : 0;
  for (int j = 0; j < a.kq; ++j) {
    const long long o = (long long)b * a.kq + j;
    a.ids[o] = j == 0 ? x : 0;
    a.pos[o] = min(L + j, a.t_max - 1);
    a.d_pos[(long long)j * a.B + b] = min(L + j, a.n_pos - 1);
  }
  a.nq[b] = live ? 1 + max(0, min(K, a.max_new - a.emitted[b] - 1)) : 0;
  a.d_in[b] = x;
  a.d_lens[b] = L;
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// lk_argmax alone: logits fp32 [B * ls, ld]; suppress int32 list (null when empty); g int32 [B * kq]; nq, emitted,
// done int32 [B]
int adapcc_lookup_argmax(const float* logits, int ld, int vocab, int B, int kq, int ls, int min_new,
                         const int* suppress, int n_suppress, int* g, const int* nq, const int* emitted,
                         const int* done, void* stream) {
  if (B < 1 || B > 65535 || kq < 1 || kq > kLkMaxSlots || (ls != 1 && ls != kq) || vocab < 1 || ld < vocab) {
    set_error("lookup_argmax: need 1 <= B <= 65535, 1 <= kq <= %d, ls in {1, kq}, 1 <= vocab <= ld (B=%d kq=%d ls=%d "
              "vocab=%d ld=%d)", kLkMaxSlots, B, kq, ls, vocab, ld);
    return -1;
  }
  if (n_suppress < 0 || n_suppress > kLkMaxIds || (n_suppress && !suppress)) {
    set_error("lookup_argmax: at most %d suppressed ids (got %d)", kLkMaxIds, n_suppress);
    return -1;
  }
  if (!logits || !g || !nq || !emitted || !done) {
    set_error("lookup_argmax: null pointer");
    return -1;
  }
  const size_t bits = n_suppress > 0 && min_new > 0 ? (size_t)(vocab + 31) / 32 * sizeof(uint32_t) : 0;
  if (bits > 200 * 1024) {
    set_error("lookup_argmax: suppression needs vocab <= %d (got %d)", 200 * 1024 * 8, vocab);
    return -1;
  }
  if (bits > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(lk_argmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bits));
  AcceptArgs a{logits, ld, vocab, B, kq, ls, emitted, min_new, suppress, n_suppress, g, nullptr, nq, nullptr, 0,
               nullptr, nullptr, const_cast<int*>(done), nullptr, 0, nullptr, 0, nullptr, nullptr};
  lk_argmax_kernel<<<dim3(ls, B), kBeamThreads, bits, (cudaStream_t)stream>>>(a);
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

// lk_accept alone on the slots' tokens g (lk_argmax's arg-maxes, or adapcc_sample_slots' draws): g int32, ids int64
// [B * kq]; nq, lens, emitted, done int32 [B]; seq int32 [B, t_max]; stop int32 list (null when empty); tokens int64
// [B, max_new]; steps int32 [B] or null; acc int32 [B * kq] or null: the accepted flags and last tokens (g) of
// adapcc_spec_slots, null for the rule that a draft is accepted when it equals the token just emitted
int adapcc_lookup_accept(int B, int kq, const int* stop, int n_stop, const int* g, const long long* ids, const int* nq,
                         int* seq, int t_max, int* lens, int* emitted, int* done, long long* tokens, int max_new,
                         int* steps, const int* acc, void* stream) {
  if (B < 1 || B > 65535 || kq < 1 || kq > kLkMaxSlots || t_max < 1 || max_new < 1) {
    set_error("lookup_accept: need 1 <= B <= 65535, 1 <= kq <= %d, t_max, max_new >= 1 (B=%d kq=%d)", kLkMaxSlots, B,
              kq);
    return -1;
  }
  if (n_stop < 0 || n_stop > kLkMaxIds || (n_stop && !stop)) {
    set_error("lookup_accept: at most %d stop ids (got %d)", kLkMaxIds, n_stop);
    return -1;
  }
  if (!g || !ids || !nq || !seq || !lens || !emitted || !done || !tokens) {
    set_error("lookup_accept: null pointer");
    return -1;
  }
  AcceptArgs a{nullptr, 0, 0, B, kq, kq, emitted, 0, nullptr, 0, const_cast<int*>(g), ids, nq, seq, t_max, lens,
               emitted, done, stop, n_stop, tokens, max_new, steps, acc};
  lk_accept_kernel<<<(B + 63) / 64, 64, 0, (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// seq int32 [B, t_max]; lens, emitted, done int32 [B]; ids, pos int64 [B * kq]; nq int32 [B]; d_in int64 [B]; d_lens
// int32 [B]; d_pos int64 [kq, B]
int adapcc_assist_round(const int* seq, int t_max, int B, int kq, int max_new, int n_pos, const int* lens,
                        const int* emitted, const int* done, long long* ids, long long* pos, int* nq, long long* d_in,
                        int* d_lens, long long* d_pos, void* stream) {
  if (B < 1 || B > 65535 || kq < 1 || kq > kLkMaxSlots || t_max < 1 || max_new < 1 || n_pos < 1) {
    set_error("assist_round: need 1 <= B <= 65535, 1 <= kq <= %d, t_max, max_new, n_pos >= 1 (B=%d kq=%d t_max=%d "
              "n_pos=%d)", kLkMaxSlots, B, kq, t_max, n_pos);
    return -1;
  }
  if (!seq || !lens || !emitted || !done || !ids || !pos || !nq || !d_in || !d_lens || !d_pos) {
    set_error("assist_round: null pointer");
    return -1;
  }
  RoundArgs a{seq, t_max, B, kq, max_new, n_pos, lens, emitted, done, ids, pos, nq, d_in, d_lens, d_pos};
  lk_round_kernel<<<(B + 63) / 64, 64, 0, (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
