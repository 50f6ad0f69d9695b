// Token sampling for GPT-2 generation: the tied LM head in bf16 and one seeded top-k / top-p draw per row, both on the
// device, so a whole generation step (decode, head, sample) can be replayed from one CUDA graph without a host sync.
//
//   lm_head : out[b, i] = sum_d h[b, d] * W[i, d] (bf16 in, fp32 out). Memory bound at GPT-2's batch sizes, so W is
//             streamed once per call for all rows: the h rows sit in shared memory, a warp holds kHeadRows rows of W in
//             registers and forms their dot products with every h row. Lane l owns the 8-element chunks l, l + 32, ...
//             of d; each lane adds its chunks in order and a shuffle tree adds the lanes. The order depends on D only,
//             so a row's bits do not depend on B, on the other rows or on which warp handles which rows of W.
//   sample  : one CTA of 1024 threads per row; the row's x_i = l_i / temperature stay in shared memory for all passes.
//             Top-h, the top-k threshold, the top-p cut-off and the truncation filters are those of sample_filter.cuh
//             (shared with sampled beam search). The draw is an inclusive scan over the surviving weights in index
//             order.
//   slots   : the draws of assisted generation, one CTA per verify slot or draft (grid (slots, B)), through the same
//             row body as `sample`, with a per-slot Philox counter and step (DESIGN.md §4a). A draft draw can also
//             write the draft's filtered weights, which rejection-sampling verification reads.
//   spec    : rejection-sampling verification of a round, one CTA per verify slot (grid (k + 1, B)): the slot's draw,
//             the acceptance of its draft and the residual draw, each from its own Philox word (DESIGN.md §4a).
//
// Every floating-point sum runs in fp32 in an order fixed by the thread layout (per-thread loops in index order,
// shuffle trees, warp partials added in warp order), never by arrival. A row's token depends on its logits, its seed,
// its position and the scalars only: not on B, nor on graph replay versus eager launch. DESIGN.md §4a has the
// definition the kernel implements; ops/sampling.py evaluates the same definition in fp64.
#include <cuda_bf16.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <mutex>

#include "common.h"
#include "device_prims.cuh"
#include "sample_filter.cuh"
#include "sample_row.cuh"

namespace adapcc {

constexpr int kHeadThreads = 256;
constexpr int kHeadRows = 4;                 // rows of W per warp and iteration
constexpr int kHeadMaxChunks = 4;            // 8-element chunks of d per lane: D <= 32 * 8 * 4 = 1024
constexpr int kHeadMaxD = 32 * 8 * kHeadMaxChunks;
constexpr int kHeadMaxB = 64;                // h in shared memory: 64 x 1024 x 2 B = 128 KB at most
constexpr int kSampleMaxList = 1024;
constexpr int kOpsMaxDevices = 64;
constexpr int kSlotMaxSlots = 16;            // verify slots per row (LOOKUP_MAX_TOKENS + 1)

__global__ void __launch_bounds__(kHeadThreads)
lm_head_logits_kernel(const __nv_bfloat16* __restrict__ h, int ld_h, const __nv_bfloat16* __restrict__ W, int V, int D,
                      float* __restrict__ out, int B) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  __nv_bfloat16* s_h = reinterpret_cast<__nv_bfloat16*>(s_raw);   // [B, D]
  const int nvec = D >> 3;
  for (int i = threadIdx.x; i < B * nvec; i += kHeadThreads) {
    const int b = i / nvec, c = i - b * nvec;
    *reinterpret_cast<uint4*>(s_h + (long long)b * D + c * 8) =
        *reinterpret_cast<const uint4*>(h + (long long)b * ld_h + c * 8);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = blockIdx.x * (kHeadThreads / 32) + (threadIdx.x >> 5);
  const int stride = gridDim.x * (kHeadThreads / 32) * kHeadRows;
  for (int r0 = warp * kHeadRows; r0 < V; r0 += stride) {
    uint4 w[kHeadRows][kHeadMaxChunks];
#pragma unroll
    for (int r = 0; r < kHeadRows; ++r)
#pragma unroll
      for (int j = 0; j < kHeadMaxChunks; ++j) {
        const int c = lane + 32 * j;
        w[r][j] = (r0 + r < V && c < nvec) ? __ldg(reinterpret_cast<const uint4*>(W + (long long)(r0 + r) * D + c * 8))
                                           : make_uint4(0u, 0u, 0u, 0u);
      }
    for (int b = 0; b < B; ++b) {
      float acc[kHeadRows];
#pragma unroll
      for (int r = 0; r < kHeadRows; ++r) acc[r] = 0.f;
#pragma unroll
      for (int j = 0; j < kHeadMaxChunks; ++j) {
        const int c = lane + 32 * j;
        if (c < nvec) {
          float hv[8];
          unpack<__nv_bfloat16>(*reinterpret_cast<const uint4*>(s_h + (long long)b * D + c * 8), hv);
#pragma unroll
          for (int r = 0; r < kHeadRows; ++r) {
            float wv[8];
            unpack<__nv_bfloat16>(w[r][j], wv);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[r] = fmaf(hv[e], wv[e], acc[r]);
          }
        }
      }
#pragma unroll
      for (int r = 0; r < kHeadRows; ++r)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
      float v = acc[0];
#pragma unroll
      for (int r = 1; r < kHeadRows; ++r) v = lane == r ? acc[r] : v;
      if (lane < kHeadRows && r0 + lane < V) out[(long long)b * V + r0 + lane] = v;
    }
  }
}

// ---- sampling --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSampleThreads, 1)
sample_tokens_kernel(const __grid_constant__ SampleArgs a) {
  extern __shared__ float s_x[];                    // [vocab]
  __shared__ SampleSmem sm;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int step = *a.step;                         // incremented by the next kernel on the stream, after every CTA
  long long* tok_out = a.tokens + (long long)b * a.max_new + step;
  if (a.done[b]) {                                  // a finished row keeps done set and pads its reply with -1
    if (tid == 0) {
      if (step < a.max_new) *tok_out = -1;
      a.next_ids[b] = 0;
    }
    return;
  }
  const int token = draw_row(s_x, sm, a, a.logits + (long long)b * a.ld, step, a.pos[b], a.seeds[b]);
  if (tid == 0) {
    bool stopped = false;
    for (int j = 0; j < a.n_stop; ++j) stopped |= a.stop[j] == token;
    a.next_ids[b] = token;
    if (step < a.max_new) *tok_out = stopped ? -1 : token;
    if (stopped) a.done[b] = 1;
  }
}

__global__ void step_incr_kernel(int* step) { *step += 1; }

// ---- per-slot draws of speculative decoding (DESIGN.md §4a, assisted generation) -------------------------------------
struct SlotArgs {
  SampleArgs s;              // logits [B * kq, ld], the scalars, suppress list and seeds [B]; the rest unused
  int B, kq, S, slot0;       // kq logits rows per row b; CTA x draws slot j = slot0 + x of S slots per row
  const int* lens;           // [B]: the row's cached tokens; slot j draws the token at sequence index lens + j + 1
  const int* emitted;        // [B]: tokens emitted so far; slot j is generated step emitted + j
  const int* done;           // [B]
  const int* nq;             // [B]: the row's real verify slots
  int* g;                    // verify: g[b * S + j] (slot j real iff j < nq)
  long long* ids;            // draft: ids[b * S + j + 1] and next[b] (draft j + 1 real iff j + 1 < nq; else 0)
  long long* next;
  float* q;                  // draft, optional: the filtered weights of draft step j, q[(b * (S - 1) + j) * vocab + i]
  float* zq;                 // ... (0 off the survivors) and their total zq[b * (S - 1) + j]
};

__global__ void __launch_bounds__(kSampleThreads, 1)
sample_slots_kernel(const __grid_constant__ SlotArgs a) {
  extern __shared__ float s_x[];                    // [vocab]
  __shared__ SampleSmem sm;
  const int x = blockIdx.x, b = blockIdx.y, j = a.slot0 + x;
  const bool draft = a.ids != nullptr;
  if (a.done[b] || j + (draft ? 1 : 0) >= a.nq[b]) {   // a done row or a pad slot: nothing is drawn
    if (draft && threadIdx.x == 0) {
      a.ids[(long long)b * a.S + j + 1] = 0;
      a.next[b] = 0;
    }
    return;
  }
  RowCut cut;
  const int token = draw_row(s_x, sm, a.s, a.s.logits + ((long long)b * a.kq + x) * a.s.ld, a.emitted[b] + j,
                             a.lens[b] + j + 1, a.s.seeds[b], &cut);
  if (threadIdx.x == 0) {
    if (draft) {
      a.ids[(long long)b * a.S + j + 1] = token;
      a.next[b] = token;
    } else {
      a.g[(long long)b * a.S + j] = token;
    }
  }
  if (a.q) {                                        // the draft's distribution at this step, for rejection sampling
    const long long r = (long long)b * (a.S - 1) + j;
    float* q = a.q + r * a.s.vocab;
    for (int i = threadIdx.x; i < a.s.vocab; i += kSampleThreads) {
      const float v = s_x[i];
      q[i] = f2key(v) >= cut.tau ? expf(v - cut.m) : 0.f;
    }
    if (threadIdx.x == 0) a.zq[r] = cut.zp;
  }
}

// ---- rejection-sampling verification (DESIGN.md §4a) ------------------------------------------------------------------
struct SpecArgs {
  SlotArgs t;                // the model's slots: logits [B * S, ld] (kq = S, slot0 = 0), g [B * S]; ids, q unused
  const long long* ids;      // [B * S]: draft j + 1 in slot j + 1
  const float* q;            // [B, S - 1, vocab] and [B, S - 1]: the draft's weights and totals (sample_slots_kernel)
  const float* zq;
  int* acc;                  // [B * S]: draft j + 1 accepted, for j < nq - 1
  int* last;                 // [B * S]: the round's last token if it ends at slot j: t_j for j < nq - 1, else g_j
};

// CTA (j, b): draws g_j as sample_slots_kernel does; for a slot with a real draft d = d_{j+1} it also decides d
// (accepted iff v Q_j(d) < P_j(d), v from Philox word 1 at lens + j + 1) and draws the residual t_j from
// max(0, P_j - Q_j) with rho_d = 0 (word 2 at lens + j + 1; g_j when no weight is left). No slot depends on another.
__global__ void __launch_bounds__(kSampleThreads, 1)
spec_slots_kernel(const __grid_constant__ SpecArgs a) {
  extern __shared__ float s_x[];                    // [vocab]
  __shared__ SampleSmem sm;
  const SlotArgs& t = a.t;
  const int j = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, V = t.s.vocab;
  const int nq = t.nq[b];
  if (t.done[b] || j >= nq) return;
  const int L = t.lens[b];
  const long long seed = t.s.seeds[b];
  const long long o = (long long)b * t.S + j;
  RowCut cut;
  const int token = draw_row(s_x, sm, t.s, t.s.logits + o * t.s.ld, t.emitted[b] + j, L + j + 1, seed, &cut);
  if (j + 1 >= nq) {                                // the last real slot: a round that gets here emits g_j
    if (tid == 0) {
      t.g[o] = token;
      a.last[o] = token;
    }
    return;
  }
  const long long r = (long long)b * (t.S - 1) + j;
  const float* wq = a.q + r * V;
  const float zq = a.zq[r];
  const long long dl = a.ids[o + 1];
  const int d = dl >= 0 && dl < V ? (int)dl : -1;
  const uint4 w = philox4((uint32_t)(L + j + 1), (uint32_t)(unsigned long long)seed,
                          (uint32_t)((unsigned long long)seed >> 32));
  if (tid == 0) {
    const float pd = d >= 0 ? cut_prob(s_x[d], cut) : 0.f;
    const float qd = d >= 0 && zq > 0.f ? wq[d] / zq : 0.f;
    t.g[o] = token;
    a.acc[o] = philox_uniform(w.y) * qd < pd;       // strict: an id with P = 0 is never accepted
  }
  __syncthreads();                                  // s_x[d] is read before the row becomes the residual
  for (int i = tid; i < V; i += kSampleThreads) {
    const float p = cut_prob(s_x[i], cut), q = zq > 0.f ? wq[i] / zq : 0.f;
    s_x[i] = i == d ? 0.f : fmaxf(0.f, p - q);
  }
  __syncthreads();
  float zr;
  const int res = scan_pick(s_x, sm, V, [](float x) { return x > 0.f; }, [](float x) { return x; },
                            philox_uniform(w.z), zr);
  if (tid == 0) a.last[o] = res >= 0 ? res : token;
}

// The checks and set-up shared by adapcc_sample_slots and adapcc_spec_slots; fills `s` or sets the error.
static int slot_args(const char* who, const float* logits, int ld, int vocab, int B, int kq, int S, int slot0,
                     bool draft, float temperature, int top_k, float top_p, float min_p, float typical_p,
                     float epsilon, float eta, float top_h, const long long* seeds, const int* lens, const int* emitted,
                     const int* done, const int* nq, int min_new, const int* suppress, int n_suppress, SampleArgs& s) {
  if (B < 1 || B > 65535 || S < 1 || S > kSlotMaxSlots || kq < 1 || (draft && kq != 1) || slot0 < 0 ||
      slot0 + kq + (draft ? 1 : 0) > S || vocab < 1 || vocab > kSampleMaxVocab || ld < vocab) {
    set_error("%s: need 1 <= B <= 65535, 1 <= S <= %d, kq >= 1 (1 for drafts), 0 <= slot0, slot0 + kq (+ 1 for "
              "drafts) <= S, 1 <= vocab <= %d, ld >= vocab (B=%d S=%d kq=%d slot0=%d vocab=%d ld=%d)", who,
              kSlotMaxSlots, kSampleMaxVocab, B, S, kq, slot0, vocab, ld);
    return -1;
  }
  if (!(temperature >= 0.f) || top_k < 0 || !(top_p > 0.f && top_p <= 1.f) || !(min_p >= 0.f && min_p <= 1.f) ||
      !(typical_p > 0.f && typical_p <= 1.f) || !(epsilon >= 0.f && epsilon < 1.f) || !(eta >= 0.f && eta < 1.f) ||
      !(top_h >= 0.f && top_h <= 1.f)) {
    set_error("%s: need temperature >= 0, top_k >= 0, 0 < top_p <= 1, 0 <= min_p <= 1, 0 < typical_p <= 1, 0 <= "
              "epsilon < 1, 0 <= eta < 1, 0 <= top_h <= 1 (got %g, %d, %g, %g, %g, %g, %g, %g)", who, temperature,
              top_k, top_p, min_p, typical_p, epsilon, eta, top_h);
    return -1;
  }
  if (n_suppress < 0 || n_suppress > kSampleMaxList || (n_suppress && !suppress)) {
    set_error("%s: a suppress list of at most %d ids (got %d)", who, kSampleMaxList, n_suppress);
    return -1;
  }
  if (!logits || !seeds || !lens || !emitted || !done || !nq) {
    set_error("%s: null pointer", who);
    return -1;
  }
  s = SampleArgs{logits, ld, vocab, temperature, top_p, top_k, seeds, nullptr, nullptr, min_new, suppress, n_suppress,
                 nullptr, 0, nullptr, nullptr, nullptr, 1, top_h, FilterArgs{min_p, typical_p, epsilon, eta, 1}};
  return 0;
}

// the row of a sampling kernel in shared memory, once per device
template <class Kernel>
static int allow_row_smem(const char* who, Kernel kernel, std::once_flag* once, cudaError_t* setup) {
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kOpsMaxDevices) { set_error("%s: device %d out of range", who, dev); return -1; }
  std::call_once(once[dev], [&] {
    setup[dev] = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kSampleMaxVocab * (int)sizeof(float));
  });
  CUDA_TRY(setup[dev]);
  return 0;
}

// The checks of adapcc_sample_tokens_filtered and adapcc_sample_tokens_synthid; fills `a` or sets the error.
static int sample_args(const char* who, const float* logits, int ld, int vocab, int B, float temperature, int top_k,
                       float top_p, float min_p, float typical_p, float epsilon, float eta, const long long* seeds,
                       const int* pos, int* step, int min_new, const int* suppress, int n_suppress, const int* stop,
                       int n_stop, int* done, long long* next_ids, long long* tokens, int max_new, float top_h,
                       SampleArgs& a) {
  if (B < 1 || vocab < 1 || vocab > kSampleMaxVocab || ld < vocab || max_new < 1) {
    set_error("%s: need B >= 1, 1 <= vocab <= %d, ld >= vocab, max_new >= 1 (B=%d vocab=%d ld=%d max_new=%d)", who,
              kSampleMaxVocab, B, vocab, ld, max_new);
    return -1;
  }
  if (!(temperature >= 0.f) || top_k < 0 || !(top_p > 0.f && top_p <= 1.f)) {
    set_error("%s: need temperature >= 0, top_k >= 0, 0 < top_p <= 1 (got %g, %d, %g)", who, temperature, top_k,
              top_p);
    return -1;
  }
  if (!(min_p >= 0.f && min_p <= 1.f) || !(typical_p > 0.f && typical_p <= 1.f) || !(epsilon >= 0.f && epsilon < 1.f) ||
      !(eta >= 0.f && eta < 1.f) || !(top_h >= 0.f && top_h <= 1.f)) {
    set_error("%s: need 0 <= min_p <= 1, 0 < typical_p <= 1, 0 <= epsilon < 1, 0 <= eta < 1, 0 <= top_h <= 1 (got "
              "%g, %g, %g, %g, %g)", who, min_p, typical_p, epsilon, eta, top_h);
    return -1;
  }
  if (n_suppress < 0 || n_stop < 0 || n_suppress > kSampleMaxList || n_stop > kSampleMaxList ||
      (n_suppress && !suppress) || (n_stop && !stop)) {
    set_error("%s: suppress / stop lists of at most %d ids (got %d, %d)", who, kSampleMaxList, n_suppress, n_stop);
    return -1;
  }
  if (!logits || !seeds || !pos || !step || !done || !next_ids || !tokens) {
    set_error("%s: null pointer", who);
    return -1;
  }
  a = SampleArgs{logits, ld, vocab, temperature, top_p, top_k, seeds, pos, step, min_new, suppress, n_suppress,
                 stop, n_stop, done, next_ids, tokens, max_new, top_h, FilterArgs{min_p, typical_p, epsilon, eta, 1}};
  return 0;
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// h: bf16 [B, ld_h] (the first D columns used); w: bf16 [V, D] contiguous; out: fp32 [B, V] contiguous
int adapcc_lm_head_logits(const void* h, int ld_h, const void* w, int V, int D, void* out, int B, void* stream) {
  if (B < 1 || B > kHeadMaxB || V < 1 || D < 8 || D > kHeadMaxD || D % 8 != 0 || ld_h < D || ld_h % 8 != 0) {
    set_error("lm_head_logits: need 1 <= B <= %d, V >= 1, D a multiple of 8 in [8, %d], ld_h >= D and a multiple of "
              "8 (B=%d V=%d D=%d ld_h=%d)", kHeadMaxB, kHeadMaxD, B, V, D, ld_h);
    return -1;
  }
  if (((uintptr_t)h | (uintptr_t)w) & 15 || (uintptr_t)out & 3) {
    set_error("lm_head_logits: h and w must be 16-byte aligned, out 4-byte aligned");
    return -1;
  }
  static std::once_flag once[kOpsMaxDevices];
  static cudaError_t setup[kOpsMaxDevices];
  static int sms[kOpsMaxDevices];
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kOpsMaxDevices) { set_error("lm_head_logits: device %d out of range", dev); return -1; }
  std::call_once(once[dev], [&] {
    setup[dev] = cudaFuncSetAttribute(lm_head_logits_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kHeadMaxB * kHeadMaxD * 2);
    if (setup[dev] == cudaSuccess) setup[dev] = cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
  });
  CUDA_TRY(setup[dev]);
  const size_t smem = (size_t)B * D * 2;
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lm_head_logits_kernel, kHeadThreads, smem));
  const int rows_per_cta = (kHeadThreads / 32) * kHeadRows;
  const int grid = std::max(1, std::min((V + rows_per_cta - 1) / rows_per_cta, std::max(1, per_sm) * sms[dev]));
  lm_head_logits_kernel<<<grid, kHeadThreads, smem, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)h, ld_h, (const __nv_bfloat16*)w, V, D, (float*)out, B);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// logits: fp32 [B, ld]; seeds int64 [B]; pos int32 [B]; step: int32 [1] on the device; suppress / stop: int32 lists
// on the device (may be null when empty); done int32 [B]; next_ids int64 [B]; tokens int64 [B, max_new]; the
// filters are off at min_p = 0, typical_p = 1, epsilon = 0, eta = 0 and top_h = 0
int adapcc_sample_tokens_filtered(const float* logits, int ld, int vocab, int B, float temperature, int top_k,
                                  float top_p, float min_p, float typical_p, float epsilon, float eta,
                                  const long long* seeds, const int* pos, int* step, int min_new, const int* suppress,
                                  int n_suppress, const int* stop, int n_stop, int* done, long long* next_ids,
                                  long long* tokens, int max_new, float top_h, void* stream) {
  SampleArgs a;
  if (sample_args("sample_tokens", logits, ld, vocab, B, temperature, top_k, top_p, min_p, typical_p, epsilon, eta,
                  seeds, pos, step, min_new, suppress, n_suppress, stop, n_stop, done, next_ids, tokens, max_new,
                  top_h, a))
    return -1;
  static std::once_flag once[kOpsMaxDevices];
  static cudaError_t setup[kOpsMaxDevices];
  if (allow_row_smem("sample_tokens", sample_tokens_kernel, once, setup)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  sample_tokens_kernel<<<B, kSampleThreads, (size_t)vocab * sizeof(float), s>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  step_incr_kernel<<<1, 1, 0, s>>>(step);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// adapcc_sample_tokens_filtered with SynthID's tournament (DESIGN.md §4a, step 6b) on the steps it watermarks: table
// uint32 [ceil(S / 32)] on the device (the g-value bitset of S = table_size entries, S in [1, 2^24]); depth m in [1,
// 64] keys (host array), ngram n in [2, 16], history H >= 1, skip s0 in {0, n - 1}. A row's context comes from its
// reply columns tokens[b, 0, step), so there is no other per-row state.
int adapcc_sample_tokens_synthid(const float* logits, int ld, int vocab, int B, float temperature, int top_k,
                                 float top_p, float min_p, float typical_p, float epsilon, float eta,
                                 const long long* seeds, const int* pos, int* step, int min_new, const int* suppress,
                                 int n_suppress, const int* stop, int n_stop, int* done, long long* next_ids,
                                 long long* tokens, int max_new, float top_h, const unsigned* table,
                                 long long table_size, int depth, int ngram, int history, int skip,
                                 const unsigned long long* keys, void* stream) {
  SampleArgs a;
  if (sample_args("sample_tokens_synthid", logits, ld, vocab, B, temperature, top_k, top_p, min_p, typical_p, epsilon,
                  eta, seeds, pos, step, min_new, suppress, n_suppress, stop, n_stop, done, next_ids, tokens, max_new,
                  top_h, a))
    return -1;
  SynthIDArgs w;
  if (synthid_args("sample_tokens_synthid", table, table_size, depth, ngram, history, skip, keys, w)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  if (sample_tokens_synthid_launch(a, w, B, s)) return -1;
  step_incr_kernel<<<1, 1, 0, s>>>(step);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// logits fp32 [B * kq, ld]; seeds int64 [B]; lens, emitted, done, nq int32 [B]; suppress: int32 list (null when
// empty). Verify draws: g int32 [B * S], ids = next = q = zq = null. Draft draws (kq = 1: draft j + 1 needs draft j):
// ids int64 [B * S] and next int64 [B], g null; optionally (temperature > 0) the draft's weights q fp32
// [B, S - 1, vocab] and totals zq fp32 [B, S - 1] of step slot0, both or neither.
int adapcc_sample_slots(const float* logits, int ld, int vocab, int B, int kq, int S, int slot0, float temperature,
                        int top_k, float top_p, float min_p, float typical_p, float epsilon, float eta,
                        const long long* seeds, const int* lens, const int* emitted, const int* done, const int* nq,
                        int min_new, const int* suppress, int n_suppress, int* g, long long* ids, long long* next,
                        float* q, float* zq, float top_h, void* stream) {
  const bool draft = ids != nullptr;
  SampleArgs s;
  if (slot_args("sample_slots", logits, ld, vocab, B, kq, S, slot0, draft, temperature, top_k, top_p, min_p,
                typical_p, epsilon, eta, top_h, seeds, lens, emitted, done, nq, min_new, suppress, n_suppress, s))
    return -1;
  if ((draft ? (!next || g) : (!g || next)) || !q != !zq || (q && (!draft || !(temperature > 0.f)))) {
    set_error("sample_slots: not exactly one of g and (ids, next), or q / zq without the other, or not with a draft "
              "draw at temperature > 0");
    return -1;
  }
  static std::once_flag once[kOpsMaxDevices];
  static cudaError_t setup[kOpsMaxDevices];
  if (allow_row_smem("sample_slots", sample_slots_kernel, once, setup)) return -1;
  SlotArgs a{s, B, kq, S, slot0, lens, emitted, done, nq, g, ids, next, q, zq};
  sample_slots_kernel<<<dim3(kq, B), kSampleThreads, (size_t)vocab * sizeof(float), (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// Rejection-sampling verification of a round, one CTA per slot: logits fp32 [B * S, ld]; seeds int64 [B]; lens,
// emitted, done, nq int32 [B]; suppress int32 list (null when empty); ids int64 [B * S] (the drafts); q fp32
// [B, S - 1, vocab] and zq fp32 [B, S - 1] (sample_slots' draft weights); g, acc, last int32 [B * S]. temperature > 0.
int adapcc_spec_slots(const float* logits, int ld, int vocab, int B, int S, float temperature, int top_k, float top_p,
                      float min_p, float typical_p, float epsilon, float eta, const long long* seeds, const int* lens,
                      const int* emitted, const int* done, const int* nq, int min_new, const int* suppress,
                      int n_suppress, const long long* ids, const float* q, const float* zq, int* g, int* acc,
                      int* last, float top_h, void* stream) {
  SampleArgs s;
  if (slot_args("spec_slots", logits, ld, vocab, B, S, S, 0, false, temperature, top_k, top_p, min_p, typical_p,
                epsilon, eta, top_h, seeds, lens, emitted, done, nq, min_new, suppress, n_suppress, s))
    return -1;
  if (S < 2 || !(temperature > 0.f)) {
    set_error("spec_slots: need S >= 2 and temperature > 0 (got %d, %g)", S, temperature);
    return -1;
  }
  if (!ids || !q || !zq || !g || !acc || !last) {
    set_error("spec_slots: null pointer");
    return -1;
  }
  static std::once_flag once[kOpsMaxDevices];
  static cudaError_t setup[kOpsMaxDevices];
  if (allow_row_smem("spec_slots", spec_slots_kernel, once, setup)) return -1;
  SlotArgs t{s, B, S, S, 0, lens, emitted, done, nq, g, nullptr, nullptr, nullptr, nullptr};
  SpecArgs a{t, ids, q, zq, acc, last};
  spec_slots_kernel<<<dim3(S, B), kSampleThreads, (size_t)vocab * sizeof(float), (cudaStream_t)stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// adapcc_sample_tokens_filtered with every filter off
int adapcc_sample_tokens(const float* logits, int ld, int vocab, int B, float temperature, int top_k, float top_p,
                         const long long* seeds, const int* pos, int* step, int min_new, const int* suppress,
                         int n_suppress, const int* stop, int n_stop, int* done, long long* next_ids, long long* tokens,
                         int max_new, void* stream) {
  return adapcc_sample_tokens_filtered(logits, ld, vocab, B, temperature, top_k, top_p, 0.f, 1.f, 0.f, 0.f, seeds, pos,
                                       step, min_new, suppress, n_suppress, stop, n_stop, done, next_ids, tokens,
                                       max_new, 0.f, stream);
}

}  // extern "C"
