// SynthID Text (Dathathri et al., Nature 2024; HuggingFace's SynthIDTextWatermarkLogitsProcessor): the int64 hash and
// the g-value table lookup shared by the sampler's tournament (ops_sample.cu) and the detector (ops_synthid.cu). The
// definition is in ops/synthid.py.
//
// All arithmetic is uint64 with wrap-around: acc(h, x) = (h + x) * 6364136223846793005 + 1. The hash of a context c
// (n - 1 ids) is acc folded over c from 1; layer l's key for a candidate v is acc(acc(hash(c), v), k_l) and its g-value
// table[signed(key) mod S], with Python's non-negative floor-mod. The table is a bitset of ceil(S / 32) words (bit
// i & 31 of word i >> 5), read from global memory through the read-only path.
#pragma once

#include <cstdint>

namespace adapcc {

constexpr int kSynthIDMaxDepth = 64;          // watermarking layers m
constexpr int kSynthIDMaxNgram = 16;          // n-gram length n
constexpr int kSynthIDMaxTable = 1 << 24;     // table entries S
constexpr unsigned long long kSynthIDMult = 6364136223846793005ull;

struct SynthIDArgs {
  const uint32_t* table;                      // ceil(S / 32) words
  long long size;                             // S
  long long mask;                             // S - 1 when S is a power of two, else -1
  int depth, ngram, history, skip;            // m, n, H, s0 (n - 1 with skip_first_ngram_calls, else 0)
  unsigned long long keys[kSynthIDMaxDepth];
};

__host__ __device__ __forceinline__ unsigned long long synthid_acc(unsigned long long h, unsigned long long x) {
  return (h + x) * kSynthIDMult + 1ull;
}

// table[floor-mod(signed(key), S)]; for a power-of-two S the floor-mod is the low bits of the two's complement
__device__ __forceinline__ uint32_t synthid_g(const SynthIDArgs& s, unsigned long long key) {
  long long r;
  if (s.mask >= 0) {
    r = (long long)(key & (unsigned long long)s.mask);
  } else {
    r = (long long)key % s.size;
    if (r < 0) r += s.size;
  }
  return (__ldg(s.table + (r >> 5)) >> (r & 31)) & 1u;
}

// the hash of the n - 1 ids before generated step t of a row whose generated ids are gen[0, t); ids before the first
// generated one are 0 (the processor's state starts as zeros; the prompt does not enter)
__device__ __forceinline__ unsigned long long synthid_context_hash(const long long* gen, int t, int ngram) {
  unsigned long long h = 1ull;
  for (int j = t - ngram + 1; j < t; ++j) h = synthid_acc(h, j < 0 ? 0ull : (unsigned long long)gen[j]);
  return h;
}

// Fills `w` from the host-side parameters (keys: a host array of `depth` words), or sets the error naming `who`:
// 1 <= S <= 2^24, 1 <= depth <= 64, 2 <= ngram <= 16, history >= 1, skip 0 or ngram - 1. Returns 0 or -1.
int synthid_args(const char* who, const unsigned* table, long long table_size, int depth, int ngram, int history,
                 int skip, const unsigned long long* keys, SynthIDArgs& w);

}  // namespace adapcc
