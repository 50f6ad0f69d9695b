// Device-side building blocks shared by every collective kernel:
//   * system-scope release/acquire flag protocol on symmetric signal pads (replaces the
//     reference's per-chunk cudaIpc events + SysV shm bool + CPU spin,
//     /root/reference/csrc/trans.cu:58-100),
//   * 16-byte "pack" load/store/convert helpers (fp32 / bf16 / fp16 wire formats),
//   * NVLS multimem.ld_reduce / multimem.st wrappers (sm_90+; we build sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.h"

namespace adapcc {

// ----------------------------------------------------------------------------------
// Kernel-visible communicator state (passed by value as a __grid_constant__ param).
// ----------------------------------------------------------------------------------
struct DevComm {
  int rank;                        // my world rank
  int world;
  int n_active;                    // participants of this op
  int my_index;                    // my position in active_ranks, -1 if not a participant
  int active_ranks[kMaxRanks];     // sorted world ranks taking part
  char* data[kMaxRanks];           // data[r]: rank r's symmetric data window, my VA space
  char* mc_data;                   // multicast alias of the same window (or nullptr)
  uint32_t* pad[kMaxRanks];        // pad[r]: rank r's barrier pad  [kMaxBlocks][kMaxRanks]
  unsigned long long* flag[kMaxRanks];  // flag[r]: rank r's chunk flags [3][kMaxBlocks]
  uint32_t* bar_epoch;             // local, [kMaxBlocks][kMaxRanks]: barrier epoch per (block, peer)
  unsigned long long* seq;         // local: op sequence number of this context
  uint32_t* ticket;                // local: last-block ticket
  uint32_t* err;                   // local: sticky error word (timeouts)
  unsigned long long timeout_ns;   // spin timeout (0 = wait forever)
  // A logical op larger than the staging window runs as back-to-back pieces (one launch each). The op
  // sequence number must move exactly ONCE per logical op on every rank (a rank that sits an op out runs one
  // skip_op), so only the last piece advances it; tree tokens stay monotonic through `item_base`.
  int op_advance;                  // 1 on the last (or only) piece of an op, 0 on earlier pieces
  unsigned long long item_base;    // tree kernels: pipeline items consumed by earlier pieces of this op
};

// ----------------------------------------------------------------------------------
// flags
// ----------------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// Spin until *p >= want (wrap-safe). Gives up after c.timeout_ns and latches c.err so
// the host can fail loudly instead of hanging the GPU.
__device__ __forceinline__ bool wait_flag32(const DevComm& c, const uint32_t* p, uint32_t want) {
  if ((int32_t)(ld_acquire_sys(p) - want) >= 0) return true;
  unsigned long long t0 = globaltimer_ns();
  unsigned spins = 0;
  while ((int32_t)(ld_acquire_sys(p) - want) < 0) {
    if ((++spins & 0x3ff) == 0 && c.timeout_ns) {
      if (globaltimer_ns() - t0 > c.timeout_ns) { atomicExch(c.err, 1u); return false; }
    }
  }
  return true;
}
__device__ __forceinline__ bool wait_flag64(const DevComm& c, const unsigned long long* p,
                                            unsigned long long want) {
  if (ld_acquire_sys64(p) >= want) return true;
  unsigned long long t0 = globaltimer_ns();
  unsigned spins = 0;
  while (ld_acquire_sys64(p) < want) {
    if ((++spins & 0x3ff) == 0 && c.timeout_ns) {
      if (globaltimer_ns() - t0 > c.timeout_ns) { atomicExch(c.err, 2u); return false; }
    }
  }
  return true;
}

// Per-block barrier across the participants of the op. Block b of every participant
// synchronises only with block b of the others, so different blocks pipeline freely
// through the phases of a collective (no grid-wide sync). The release/acquire pair makes
// every write the block did before the barrier (local, peer or multicast) visible to the
// peers' block b after it.
//
// Epochs are kept PER PAIR (block, peer): with relay control different ranks execute
// different numbers of barriers (a rank skips the ops it is not active in), but any barrier
// that involves both r and p is executed by both, so the pairwise counters stay equal.
// Thread t < n_active owns the pair (this rank, active_ranks[t]) for the whole kernel.
struct BarrierState {
  uint32_t epoch;    // value of the last barrier with my peer (threads >= n_active: unused)
  int peer;
};

__device__ __forceinline__ BarrierState barrier_begin(const DevComm& c) {
  BarrierState b;
  b.peer = (int)threadIdx.x < c.n_active ? c.active_ranks[threadIdx.x] : -1;
  b.epoch = b.peer >= 0 ? c.bar_epoch[blockIdx.x * kMaxRanks + b.peer] : 0u;
  return b;
}

__device__ __forceinline__ void block_barrier(const DevComm& c, BarrierState& b) {
  __syncthreads();
  if (b.peer >= 0) {
    b.epoch += 1;
    st_release_sys(c.pad[b.peer] + blockIdx.x * kMaxRanks + c.rank, b.epoch);
    wait_flag32(c, c.pad[c.rank] + blockIdx.x * kMaxRanks + b.peer, b.epoch);
  }
  __syncthreads();
}

// Every kernel ends with this: persist the pair epochs and let the last block to finish
// advance the context's op sequence number (device-side, so the kernels stay CUDA-graph
// capturable: no host-computed epoch is baked into the launch).
__device__ __forceinline__ void finish_op(const DevComm& c, const BarrierState& b, int advance = -1) {
  if (advance < 0) advance = c.op_advance;
  if (b.peer >= 0) c.bar_epoch[blockIdx.x * kMaxRanks + b.peer] = b.epoch;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const uint32_t t = atomicAdd(c.ticket, 1u);
    if (t == gridDim.x - 1) {
      *c.ticket = 0;
      *c.seq = *c.seq + (unsigned long long)advance;
    }
  }
}

// ----------------------------------------------------------------------------------
// packs: 16 bytes of wire data
// ----------------------------------------------------------------------------------
template <typename T> struct WireTraits;
template <> struct WireTraits<float> { static constexpr int kEpp = 4; };
template <> struct WireTraits<__nv_bfloat16> { static constexpr int kEpp = 8; };
template <> struct WireTraits<__half> { static constexpr int kEpp = 8; };

__device__ __forceinline__ uint4 ld16(const void* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st16(void* p, uint4 v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w) : "memory");
}

template <typename W> __device__ __forceinline__ void unpack(uint4 v, float* f);
template <> __device__ __forceinline__ void unpack<float>(uint4 v, float* f) {
  f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y);
  f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
}
template <> __device__ __forceinline__ void unpack<__nv_bfloat16>(uint4 v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}
template <> __device__ __forceinline__ void unpack<__half>(uint4 v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
    float2 t = __half22float2(h);
    f[2 * i] = t.x; f[2 * i + 1] = t.y;
  }
}
template <typename W> __device__ __forceinline__ uint4 pack(const float* f);
template <> __device__ __forceinline__ uint4 pack<float>(const float* f) {
  return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                    __float_as_uint(f[3]));
}
template <> __device__ __forceinline__ uint4 pack<__nv_bfloat16>(const float* f) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 b = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<uint32_t*>(&b);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
template <> __device__ __forceinline__ uint4 pack<__half>(const float* f) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

template <typename U> __device__ __forceinline__ float to_float(U v);
template <> __device__ __forceinline__ float to_float<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_float<__half>(__half v) { return __half2float(v); }
template <typename U> __device__ __forceinline__ U from_float(float v);
template <> __device__ __forceinline__ float from_float<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }

// Load kEpp user elements starting at element e0 into fp32 registers (zero padded past
// n). `vec_ok` = user pointer is 16-byte aligned, so full packs use 128-bit accesses.
template <typename U, int kEpp>
__device__ __forceinline__ void load_user(const U* __restrict__ base, long long e0, long long n,
                                          bool vec_ok, float* f) {
  if (vec_ok && e0 + kEpp <= n) {
    constexpr int kVecs = (int)(sizeof(U) * kEpp / 16);
    const uint4* p = reinterpret_cast<const uint4*>(base + e0);
#pragma unroll
    for (int v = 0; v < kVecs; ++v) {
      uint4 q = ld16(p + v);
      unpack<U>(q, f + v * (kEpp / kVecs));
    }
  } else {
#pragma unroll
    for (int i = 0; i < kEpp; ++i) f[i] = (e0 + i < n) ? to_float<U>(base[e0 + i]) : 0.f;
  }
}
template <typename U, int kEpp>
__device__ __forceinline__ void store_user(U* __restrict__ base, long long e0, long long n,
                                           bool vec_ok, const float* f) {
  if (vec_ok && e0 + kEpp <= n) {
    constexpr int kVecs = (int)(sizeof(U) * kEpp / 16);
    uint4* p = reinterpret_cast<uint4*>(base + e0);
#pragma unroll
    for (int v = 0; v < kVecs; ++v) st16(p + v, pack<U>(f + v * (kEpp / kVecs)));
  } else {
#pragma unroll
    for (int i = 0; i < kEpp; ++i)
      if (e0 + i < n) base[e0 + i] = from_float<U>(f[i]);
  }
}

template <int OP> __device__ __forceinline__ float red_identity() { return OP == MAX ? -INFINITY : 0.f; }
template <int OP> __device__ __forceinline__ float red_apply(float a, float b) {
  return OP == MAX ? fmaxf(a, b) : a + b;
}

// ----------------------------------------------------------------------------------
// NVLS (in-switch reduction / broadcast through the multicast mapping)
// ----------------------------------------------------------------------------------
template <typename W, int OP> __device__ __forceinline__ uint4 mc_ld_reduce(const void* mc);
template <> __device__ __forceinline__ uint4 mc_ld_reduce<float, SUM>(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}
template <> __device__ __forceinline__ uint4 mc_ld_reduce<__nv_bfloat16, SUM>(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}
template <> __device__ __forceinline__ uint4 mc_ld_reduce<__half, SUM>(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}
template <> __device__ __forceinline__ uint4 mc_ld_reduce<__nv_bfloat16, MAX>(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.max.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}
template <> __device__ __forceinline__ uint4 mc_ld_reduce<__half, MAX>(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.max.v4.f16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}
// fp32 max has no NVLS form; the host never selects NVLS for it.
template <> __device__ __forceinline__ uint4 mc_ld_reduce<float, MAX>(const void* mc) {
  return make_uint4(0, 0, 0, 0);
}

__device__ __forceinline__ void mc_st16(void* mc, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

}  // namespace adapcc
