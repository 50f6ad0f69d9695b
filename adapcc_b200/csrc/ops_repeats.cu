// Repetition controls for GPT-2 generation on the device: the repetition penalty and no-repeat n-gram blocking applied
// to each row's fp32 logits between the LM head and the sampler or beam selection, inside the same CUDA graph replay.
//
//   repeats_kernel : one 512-thread CTA per group of `group` consecutive rows (a beam-search item; 1 row otherwise).
//                    With *step > 0 it first brings each row's device-resident sequence up to date: a row with a parent
//                    in its group takes the parent's generated region (every row of the group is read into shared
//                    memory before anything is written back, so cycles and many-to-one maps come out right), then the
//                    token the decode step just consumed goes at position lens[r] - 1. Then, per row, from the shared
//                    copy of the sequence:
//                      0. sequence bias (a table shared by all rows; null: off): one thread per distinct target id t
//                         walks t's entries in the defined order, sums the biases of those whose prefix ends the
//                         sequence (correctly rounded fp32 adds, the first term taken as is) and adds the sum to l_t
//                         once. Targets are distinct, so no two threads write one id; a barrier follows;
//                      1. penalty: every position reads its id's logit, a barrier, then every position writes the
//                         penalised value. Positions holding the same id read the same value and write the same bits, so
//                         each id is penalised exactly once without a de-duplication pass;
//                      2. n-grams: every start j whose n-1 ids match the sequence's last n-1 ids bans seq[j + n - 1]
//                         (-inf, also idempotent), after a barrier so no penalty write can land on a ban.
//
// The arithmetic is correctly rounded fp32 adds in a fixed order (__fadd_rn) and one multiply or divide per id
// (__fmul_rn / __fdiv_rn), so the result equals
// the definition in ops/repeats.py bit for bit and a row's result depends only on its own logits and sequence. The grid
// depends on R and group only, not on lens or step, so one capture serves every token.
#include <cmath>
#include <cstdint>

#include "common.h"

namespace adapcc {

constexpr int kRepThreads = 512;
constexpr int kRepMaxGroup = 16;
constexpr int kRepMaxLen = 1024;
constexpr int kBiasMaxEntries = 1024;

struct RepeatsArgs {
  float* logits;               // [R, ld], the first `vocab` columns used
  int ld, vocab, R;
  int* seq;                    // [R, t_max]: row r's sequence is seq[r, :lens[r]]
  int t_max;
  const int* prompt_len;       // [R]: first generated position (read only with a parent map)
  const int* lens;             // [R]
  const int* step;             // [1]: 0 on the prefill's call (the sequence is the prompt as stored)
  const long long* ids;        // [R]: the tokens the decode step just consumed
  const int* parent;           // [R] absolute row indices inside the row's group, or null
  int group;
  float penalty;               // 1: off
  int ngram;                   // 0: off
  // sequence bias: tab int32 [tgt U | start U + 1 | pre_off E | pre_len E | prefixes], val fp32 [E]; U = 0: off.
  // Target u's entries are [start[u], start[u + 1]); entry e applies when its pre_len[e] = m - 1 prefix ids
  // (tab[pre_off[e]...]) equal the sequence's last m - 1 ids and L >= m, or always when m = 1.
  const int* bias_tab;
  const float* bias_val;
  int bias_targets, bias_entries;
};

__global__ void __launch_bounds__(kRepThreads) repeats_kernel(const __grid_constant__ RepeatsArgs a) {
  extern __shared__ int s_seq[];                      // [group, t_max], then fp32 [t_max] values
  float* s_val = reinterpret_cast<float*>(s_seq + a.group * a.t_max);
  const int g0 = blockIdx.x * a.group, tid = threadIdx.x, T = a.t_max;
  const bool advance = *a.step > 0;
  for (int k = 0; k < a.group; ++k) {
    const int r = g0 + k;
    const int L = min(max(a.lens[r], 0), T);
    int src = r, lo = L;                              // positions [lo, L - 1) come from row src
    if (advance && a.parent) {
      const int p = a.parent[r];
      if (p >= g0 && p < g0 + a.group && p != r) {
        src = p;
        lo = max(a.prompt_len[r], 0);
      }
    }
    const int* own = a.seq + (long long)r * T;
    const int* from = a.seq + (long long)src * T;
    for (int j = tid; j < L; j += kRepThreads)
      s_seq[k * T + j] = (advance && j == L - 1) ? (int)a.ids[r] : (j >= lo ? from[j] : own[j]);
  }
  __syncthreads();
  if (advance) {                                      // write back what changed: the copied region and the new token
    for (int k = 0; k < a.group; ++k) {
      const int r = g0 + k;
      const int L = min(max(a.lens[r], 0), T);
      const int lo = a.parent ? min(max(a.prompt_len[r], 0), L) : max(L - 1, 0);
      int* own = a.seq + (long long)r * T;
      for (int j = lo + tid; j < L; j += kRepThreads) own[j] = s_seq[k * T + j];
    }
  }
  const float p = a.penalty;
  const int n = a.ngram, V = a.vocab;
  for (int k = 0; k < a.group; ++k) {
    const int r = g0 + k;
    const int L = min(max(a.lens[r], 0), T);
    const int* s = s_seq + k * T;
    float* l = a.logits + (long long)r * a.ld;
    if (a.bias_targets > 0) {
      const int U = a.bias_targets, E = a.bias_entries;
      const int* tgt = a.bias_tab;
      const int* start = tgt + U;
      const int* pre_off = start + U + 1;
      const int* pre_len = pre_off + E;
      for (int u = tid; u < U; u += kRepThreads) {
        float sum = 0.f;
        bool any = false;
        for (int e = start[u]; e < start[u + 1]; ++e) {
          const int m1 = pre_len[e];
          if (m1 > 0 && m1 >= L) continue;            // m > 1 and L < m: the entry cannot apply
          const int* pre = tgt + pre_off[e];
          const int* tail = s + L - m1;
          bool match = true;
          for (int q = 0; q < m1 && match; ++q) match = tail[q] == pre[q];
          if (match) {
            sum = any ? __fadd_rn(sum, a.bias_val[e]) : a.bias_val[e];
            any = true;
          }
        }
        const int t = tgt[u];
        if (any && t >= 0 && t < V) l[t] = __fadd_rn(l[t], sum);
      }
      __syncthreads();                                // biased values before the penalty reads them
    }
    if (p != 1.f) {
      for (int j = tid; j < L; j += kRepThreads) {
        const int id = s[j];
        if (id >= 0 && id < V) s_val[j] = l[id];
      }
      __syncthreads();
      for (int j = tid; j < L; j += kRepThreads) {
        const int id = s[j];
        if (id >= 0 && id < V) {
          const float v = s_val[j];
          l[id] = v < 0.f ? __fmul_rn(v, p) : __fdiv_rn(v, p);
        }
      }
    }
    __syncthreads();                                  // penalty writes before bans; s_val free for the next row
    if (n > 0 && L >= n) {
      const int tail = L - n + 1;                     // the sequence's last n - 1 ids start here
      for (int j = tid; j + n - 1 < L; j += kRepThreads) {
        bool match = true;
        for (int q = 0; q < n - 1 && match; ++q) match = s[j + q] == s[tail + q];
        const int id = s[j + n - 1];
        if (match && id >= 0 && id < V) l[id] = -INFINITY;
      }
    }
  }
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// logits fp32 [R, ld]; seq int32 [R, t_max]; prompt_len, lens int32 [R]; step int32 [1]; ids int64 [R]; parent int32
// [R] or null; group rows per parent group (R a multiple of it); bias_tab int32 / bias_val fp32 the sequence-bias table
// of RepeatsArgs, or null with bias_targets = 0 (off)
int adapcc_penalize_repeats(float* logits, int ld, int vocab, int R, int* seq, int t_max, const int* prompt_len,
                            const int* lens, const int* step, const long long* ids, const int* parent, int group,
                            float penalty, int ngram, const int* bias_tab, const float* bias_val, int bias_targets,
                            int bias_entries, void* stream) {
  if (R < 1 || vocab < 1 || ld < vocab || t_max < 1 || t_max > kRepMaxLen || group < 1 || group > kRepMaxGroup ||
      R % group != 0 || R / group > 65535) {
    set_error("penalize_repeats: need R >= 1, 1 <= vocab <= ld, 1 <= t_max <= %d, 1 <= group <= %d dividing R (R=%d "
              "vocab=%d ld=%d t_max=%d group=%d)", kRepMaxLen, kRepMaxGroup, R, vocab, ld, t_max, group);
    return -1;
  }
  if (!(penalty > 0.f) || !std::isfinite(penalty) || ngram < 0) {
    set_error("penalize_repeats: need a finite penalty > 0 and ngram >= 0 (got %g, %d)", (double)penalty, ngram);
    return -1;
  }
  if (!logits || !seq || !prompt_len || !lens || !step || !ids) {
    set_error("penalize_repeats: null pointer");
    return -1;
  }
  if (bias_targets < 0 || bias_entries < bias_targets || bias_entries > kBiasMaxEntries ||
      (bias_targets > 0 && (!bias_tab || !bias_val))) {
    set_error("penalize_repeats: need 0 <= bias targets <= bias entries <= %d and a table when on (got %d, %d)",
              kBiasMaxEntries, bias_targets, bias_entries);
    return -1;
  }
  const size_t smem = (size_t)(group + 1) * t_max * sizeof(int);
  if (smem > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(repeats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  RepeatsArgs a{logits, ld,    vocab,   R,     seq,      t_max,    prompt_len,   lens,        step,
                ids,    parent, group, penalty, ngram, bias_tab, bias_val, bias_targets, bias_entries};
  repeats_kernel<<<R / group, kRepThreads, smem, (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
