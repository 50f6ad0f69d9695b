// SynthID Text watermarking for GPT-2 generation (Dathathri et al., Nature 2024; HuggingFace's
// SynthIDTextWatermarkLogitsProcessor): the sampler's SynthID instantiation and the detector's counts. The definition
// is in ops/synthid.py (DESIGN.md §4a); the hash and the table lookup are synthid.cuh.
//
//   sample_tokens_synthid_kernel : sample_tokens_kernel (ops_sample.cu) with the tournament of step 6b between the
//                                  truncation filters and the draw (draw_row<true>, sample_row.cuh). One CTA of 1024
//                                  threads per row. The row's context is hashed from its own reply columns, so there
//                                  is no per-row state and the kernel replays from the decode graph like the plain
//                                  sampler. It lives here, not in ops_sample.cu: a second caller of the __noinline__
//                                  filters in that translation unit would change their register allocation and so the
//                                  SASS of the existing sampling kernels.
//   synthid_count_kernel         : one CTA per row of a right-padded [B, T] id matrix. Each context's hash goes to
//                                  shared memory; a position is scored when its context is not repeated (HuggingFace's
//                                  compute_context_repetition_mask over every context of the row), it lies in
//                                  [max(n - 1, scored_from), L) and before the row's first EOS. The number scored and
//                                  the g-value count of every layer are integer sums reduced in a fixed shuffle /
//                                  shared-memory tree, no atomics; optionally the g-values and the mask are written in
//                                  HuggingFace's layout.
#include <climits>
#include <cstdint>
#include <mutex>

#include "common.h"
#include "sample_row.cuh"
#include "synthid.cuh"

namespace adapcc {

constexpr int kSynthCountThreads = 512;
constexpr int kSynthCountMaxLen = 4096;                // ids per row of the detector: 32 KiB of context hashes
constexpr int kSynthMaxDevices = 64;

struct SynthIDSampleArgs {
  SampleArgs s;
  SynthIDArgs w;
};

// The row of sample_tokens_kernel with SynthID. Step t is watermarked unless t < s0 (skip_first_ngram_calls), or the
// context hash of t equals that of a step in [max(s0, t - H), t), or is 0 while t - s0 < H (the processor's history
// starts as zeros). Every thread hashes some earlier steps from the row's reply columns and __syncthreads_or combines
// them, so nothing depends on order. On a step that is not watermarked the row is draw_row<true> without a tournament,
// the same bits as sample_tokens_kernel.
__global__ void __launch_bounds__(kSampleThreads, 1)
sample_tokens_synthid_kernel(const __grid_constant__ SynthIDSampleArgs args) {
  extern __shared__ float s_x[];                    // [vocab]
  __shared__ SampleSmem sm;
  const SampleArgs& a = args.s;
  const SynthIDArgs& w = args.w;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int step = *a.step;                         // incremented by the next kernel on the stream, after every CTA
  long long* gen = a.tokens + (long long)b * a.max_new;
  if (a.done[b]) {                                  // a finished row keeps done set and pads its reply with -1
    if (tid == 0) {
      if (step < a.max_new) gen[step] = -1;
      a.next_ids[b] = 0;
    }
    return;
  }
  const SynthIDArgs* sid = nullptr;
  unsigned long long hc = 0ull;
  const int t = min(step, a.max_new);
  if (t >= w.skip) {
    hc = synthid_context_hash(gen, t, w.ngram);
    int rep = hc == 0ull && t - w.skip < w.history;
    for (int j = max(w.skip, t - w.history) + tid; j < t && !rep; j += kSampleThreads)
      rep = synthid_context_hash(gen, j, w.ngram) == hc;
    if (!__syncthreads_or(rep)) sid = &w;
  }
  const int token = draw_row<true>(s_x, sm, a, a.logits + (long long)b * a.ld, step, a.pos[b], a.seeds[b], nullptr,
                                   sid, hc);
  if (tid == 0) {
    bool stopped = false;
    for (int j = 0; j < a.n_stop; ++j) stopped |= a.stop[j] == token;
    a.next_ids[b] = token;
    if (step < a.max_new) gen[step] = stopped ? -1 : token;
    if (stopped) a.done[b] = 1;
  }
}

struct SynthIDCountArgs {
  const int* ids;              // [B, T]
  int T;
  const int* lens;             // [B]
  const int* scored_from;      // [B]
  long long eos;               // the EOS id; -1: none
  int* counts;                 // [B, 1 + m]: scored, then the g-value count of each layer
  unsigned char* g;            // optional [B, T - n + 1, m]
  unsigned char* mask;         // optional [B, T - n + 1]
  SynthIDArgs w;
};

// every thread gets the block's result of op: a shuffle tree per warp, then each thread folds the warp partials in
// warp order
template <class Op>
__device__ __forceinline__ int count_reduce(int v, int* s_part, Op op) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();                                  // the previous reduction's readers are done with s_part
  if (lane == 0) s_part[warp] = v;
  __syncthreads();
  v = s_part[0];
  for (int q = 1; q < kSynthCountThreads / 32; ++q) v = op(v, s_part[q]);
  return v;
}

__global__ void __launch_bounds__(kSynthCountThreads)
synthid_count_kernel(const __grid_constant__ SynthIDCountArgs a) {
  extern __shared__ unsigned long long s_hash[];    // [T - n + 1] context hashes, then [T - n + 1] scored flags
  __shared__ int s_part[kSynthCountThreads / 32];
  const SynthIDArgs& w = a.w;
  const int b = blockIdx.x, tid = threadIdx.x, n = w.ngram, T = a.T;
  const int nc = T - n + 1;                         // contexts (and n-grams) of the row
  unsigned char* s_ok = reinterpret_cast<unsigned char*>(s_hash + nc);
  const int* row = a.ids + (long long)b * T;
  const int L = min(max(a.lens[b], 0), T);
  int eos = INT_MAX;                                // the row's first EOS position
  if (a.eos >= 0)
    for (int j = tid; j < T; j += kSynthCountThreads)
      if ((long long)row[j] == a.eos) eos = min(eos, j);
  eos = count_reduce(eos, s_part, [](int x, int y) { return min(x, y); });
  for (int i = tid; i < nc; i += kSynthCountThreads) {
    unsigned long long h = 1ull;
    for (int q = 0; q < n - 1; ++q) h = synthid_acc(h, (unsigned long long)(long long)row[i + q]);
    s_hash[i] = h;
  }
  __syncthreads();
  const int from = a.scored_from[b];
  int scored = 0;
  for (int i = tid; i < nc; i += kSynthCountThreads) {
    const unsigned long long h = s_hash[i];
    bool rep = h == 0ull && i < w.history;          // the history starts as zeros
    for (int e = max(0, i - w.history); e < i && !rep; ++e) rep = s_hash[e] == h;
    const int j = i + n - 1;                        // the n-gram's last position
    const bool ok = !rep && j < L && j >= from && j < eos;
    s_ok[i] = ok;
    scored += ok;
    if (a.mask) a.mask[(long long)b * nc + i] = ok;
  }
  scored = count_reduce(scored, s_part, [](int x, int y) { return x + y; });
  const int m = w.depth;
  int* out = a.counts + (long long)b * (1 + m);
  if (tid == 0) out[0] = scored;
  for (int l = 0; l < m; ++l) {
    const unsigned long long key = w.keys[l];
    int c = 0;
    for (int i = tid; i < nc; i += kSynthCountThreads) {
      if (!s_ok[i] && !a.g) continue;
      const unsigned long long hv = synthid_acc(s_hash[i], (unsigned long long)(long long)row[i + n - 1]);
      const uint32_t g = synthid_g(w, synthid_acc(hv, key));
      if (a.g) a.g[((long long)b * nc + i) * m + l] = (unsigned char)g;
      c += s_ok[i] ? (int)g : 0;
    }
    c = count_reduce(c, s_part, [](int x, int y) { return x + y; });
    if (tid == 0) out[1 + l] = c;
  }
}

int synthid_args(const char* who, const unsigned* table, long long table_size, int depth, int ngram, int history,
                 int skip, const unsigned long long* keys, SynthIDArgs& w) {
  if (!table || !keys || table_size < 1 || table_size > kSynthIDMaxTable || depth < 1 || depth > kSynthIDMaxDepth ||
      ngram < 2 || ngram > kSynthIDMaxNgram || history < 1 || (skip != 0 && skip != ngram - 1)) {
    set_error("%s: need a table and keys, 1 <= S <= %d, 1 <= depth <= %d, 2 <= ngram <= %d, history >= 1 and skip 0 "
              "or ngram - 1 (S=%lld depth=%d ngram=%d history=%d skip=%d)", who, kSynthIDMaxTable, kSynthIDMaxDepth,
              kSynthIDMaxNgram, table_size, depth, ngram, history, skip);
    return -1;
  }
  w.table = (const uint32_t*)table;
  w.size = table_size;
  w.mask = (table_size & (table_size - 1)) == 0 ? table_size - 1 : -1;
  w.depth = depth;
  w.ngram = ngram;
  w.history = history;
  w.skip = skip;
  for (int l = 0; l < kSynthIDMaxDepth; ++l) w.keys[l] = l < depth ? keys[l] : 0ull;
  return 0;
}

int sample_tokens_synthid_launch(const SampleArgs& s, const SynthIDArgs& w, int B, cudaStream_t stream) {
  static std::once_flag once[kSynthMaxDevices];
  static cudaError_t setup[kSynthMaxDevices];
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kSynthMaxDevices) { set_error("sample_tokens_synthid: device %d out of range", dev); return -1; }
  std::call_once(once[dev], [&] {
    setup[dev] = cudaFuncSetAttribute(sample_tokens_synthid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kSampleMaxVocab * (int)sizeof(float));
  });
  CUDA_TRY(setup[dev]);
  const SynthIDSampleArgs a{s, w};
  sample_tokens_synthid_kernel<<<B, kSampleThreads, (size_t)s.vocab * sizeof(float), stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// ids int32 [B, T] (T >= ngram); lens, scored_from int32 [B]; eos the EOS id (-1: none); counts int32 [B, 1 + depth]
// out; g uint8 [B, T - ngram + 1, depth] and mask uint8 [B, T - ngram + 1] out, both or neither; the table and keys as
// in adapcc_sample_tokens_synthid.
int adapcc_synthid_count(const int* ids, int T, int B, const int* lens, const int* scored_from, long long eos,
                         const unsigned* table, long long table_size, int depth, int ngram, int history,
                         const unsigned long long* keys, int* counts, unsigned char* g, unsigned char* mask,
                         void* stream) {
  SynthIDCountArgs a{ids, T, lens, scored_from, eos, counts, g, mask, {}};
  if (synthid_args("synthid_count", table, table_size, depth, ngram, history, 0, keys, a.w)) return -1;
  if (B < 1 || B > 65535 || T < ngram || T > kSynthCountMaxLen) {
    set_error("synthid_count: need 1 <= B <= 65535 and ngram <= T <= %d (B=%d T=%d ngram=%d)", kSynthCountMaxLen, B, T,
              ngram);
    return -1;
  }
  if (!ids || !lens || !scored_from || !counts || !g != !mask) {
    set_error("synthid_count: null pointer, or only one of g and mask");
    return -1;
  }
  const int nc = T - ngram + 1;
  const size_t smem = (size_t)nc * (sizeof(unsigned long long) + 1);
  synthid_count_kernel<<<B, kSynthCountThreads, smem, (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
