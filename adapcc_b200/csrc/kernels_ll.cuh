// Low-latency ("LL") one-shot all-reduce for small messages (numerics incl. odd tails and back-to-back ops mixed with
// barrier-protocol ops: tests/gpu_collectives_worker.py, which needs at least 2 GPUs); AUTO picks it for all-rank
// messages <= 32 KB (CommContext::allreduce).
//
// The direct one-shot kernel (kernels_direct.cuh) costs two flag barriers per op: publish, barrier, pull,
// barrier — four NVLink latencies. Here the
// flag travels WITH the data, the way NCCL's LL protocol does it (third-party/nccl/src/device/prims_ll.h in the
// reference tree), but push-based over NVSwitch peer memory:
//
//   every rank stores its message into a private slot inside EVERY peer's LL buffer as 16-byte lines
//   {word0, flag, word1, flag}; the receiver polls its OWN memory (no NVLink round trip) until both flags of a
//   line carry this op's number, sums the lines of all ranks in rank order (bitwise identical result everywhere)
//   and writes the output. One NVLink store latency end to end, no barrier.
//
// Slot reuse: lines are double-buffered by the parity of an LL-only op counter. A rank can only start LL op
// k+2 after finishing op k+1, which needed the k+1 lines of every peer, which a peer only sends after it has
// consumed op k — so a slot is never overwritten while its owner still reads it. That argument needs every LL
// op to involve ALL ranks, hence: all-active ops only (relay-control subsets use the barrier kernels).
#pragma once
#include "device_prims.cuh"

namespace adapcc {

constexpr int kLLMaxBytes = 32768;                       // payload per rank per op
constexpr int kLLSlotBytes = 2 * kLLMaxBytes;            // 8 payload bytes per 16-byte line
constexpr size_t kLLBufferBytes = (size_t)2 * kMaxRanks * kLLSlotBytes;   // 2 parities x sources = 2 MB

struct LLArgs {
  char* ll[kMaxRanks];            // ll[r]: rank r's LL buffer in my address space
  unsigned long long* ll_seq;     // local: number of LL ops completed
};

__device__ __forceinline__ void st_ll_line(void* p, uint32_t w0, uint32_t w1, uint32_t flag) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %2};" ::"l"(p), "r"(w0), "r"(flag), "r"(w1) : "memory");
}
__device__ __forceinline__ uint4 ld_ll_line(const void* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

template <typename U> struct LLWord;                     // one 32-bit wire word <-> fp32 lanes
template <> struct LLWord<float> {
  static constexpr int kElems = 1;
  __device__ static void unpack(uint32_t w, float* f) { f[0] = __uint_as_float(w); }
  __device__ static uint32_t pack(const float* f) { return __float_as_uint(f[0]); }
};
template <> struct LLWord<__nv_bfloat16> {
  static constexpr int kElems = 2;
  __device__ static void unpack(uint32_t w, float* f) {
    const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
    f[0] = t.x; f[1] = t.y;
  }
  __device__ static uint32_t pack(const float* f) {
    __nv_bfloat162 t = __floats2bfloat162_rn(f[0], f[1]);
    return *reinterpret_cast<uint32_t*>(&t);
  }
};
template <> struct LLWord<__half> {
  static constexpr int kElems = 2;
  __device__ static void unpack(uint32_t w, float* f) {
    const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w));
    f[0] = t.x; f[1] = t.y;
  }
  __device__ static uint32_t pack(const float* f) {
    __half2 t = __floats2half2_rn(f[0], f[1]);
    return *reinterpret_cast<uint32_t*>(&t);
  }
};

// n elements of U, in/out 4-byte aligned, all ranks active. OP: SUM or MAX; scale applied to the result (AVG).
template <typename U, int OP>
__global__ void __launch_bounds__(256)
allreduce_ll_kernel(const __grid_constant__ DevComm c, const __grid_constant__ LLArgs a, const U* __restrict__ in,
                    U* __restrict__ out, long long n, float scale) {
  constexpr int E = LLWord<U>::kElems;                   // elements per word
  const uint32_t flag = (uint32_t)(*a.ll_seq) + 1u;      // never 0 (the buffer's initial state)
  const size_t parity_off = (size_t)(flag & 1u) * kMaxRanks * kLLSlotBytes;
  const int me = c.rank, world = c.world;
  const long long nwords = (n + E - 1) / E;
  const long long nlines = (nwords + 1) / 2;
  const uint32_t* in_w = reinterpret_cast<const uint32_t*>(in);

  for (long long line = blockIdx.x * (long long)blockDim.x + threadIdx.x; line < nlines;
       line += (long long)gridDim.x * blockDim.x) {
    // ---- my two words (zero padded past the end; a trailing odd element is loaded alone) ----
    uint32_t w[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const long long wi = 2 * line + k;
      if ((wi + 1) * E <= n) w[k] = in_w[wi];
      else if (wi * E < n) {                             // E == 2 and n odd: last element only
        const unsigned short h = reinterpret_cast<const unsigned short*>(in)[wi * E];
        w[k] = (uint32_t)h;
      } else w[k] = 0u;
    }
    // ---- push to every peer's slot for source `me` ----
    for (int p = 0; p < world; ++p) {
      if (p == me) continue;
      st_ll_line(a.ll[p] + parity_off + (size_t)me * kLLSlotBytes + (size_t)line * 16, w[0], w[1], flag);
    }
    // ---- gather + reduce in rank order ----
    float acc[2][E];
    bool first = true;
    unsigned long long t0 = 0;
    for (int p = 0; p < world; ++p) {
      uint32_t v[2];
      if (p == me) { v[0] = w[0]; v[1] = w[1]; }
      else {
        const char* src = a.ll[me] + parity_off + (size_t)p * kLLSlotBytes + (size_t)line * 16;
        uint4 l = ld_ll_line(src);
        unsigned spins = 0;
        while (l.y != flag || l.w != flag) {
          if ((++spins & 0xff) == 0 && c.timeout_ns) {
            if (t0 == 0) t0 = globaltimer_ns();
            else if (globaltimer_ns() - t0 > c.timeout_ns) { atomicExch(c.err, 3u); break; }
          }
          l = ld_ll_line(src);
        }
        v[0] = l.x; v[1] = l.z;
      }
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        float f[E];
        LLWord<U>::unpack(v[k], f);
#pragma unroll
        for (int e = 0; e < E; ++e) acc[k][e] = first ? f[e] : (OP == MAX ? fmaxf(acc[k][e], f[e]) : acc[k][e] + f[e]);
      }
      first = false;
    }
    // ---- result ----
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const long long wi = 2 * line + k;
#pragma unroll
      for (int e = 0; e < E; ++e) acc[k][e] *= scale;
      if ((wi + 1) * E <= n) reinterpret_cast<uint32_t*>(out)[wi] = LLWord<U>::pack(acc[k]);
      else if (wi * E < n) {
        const uint32_t pw = LLWord<U>::pack(acc[k]);
        reinterpret_cast<unsigned short*>(out)[wi * E] = (unsigned short)(pw & 0xffffu);
      }
    }
  }
  // last block out: advance both counters (op sequence stays in step with the other kernels)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const uint32_t t = atomicAdd(c.ticket, 1u);
    if (t == gridDim.x - 1) {
      *c.ticket = 0;
      *c.seq = *c.seq + 1;
      *a.ll_seq = *a.ll_seq + 1;
    }
  }
}

}  // namespace adapcc
