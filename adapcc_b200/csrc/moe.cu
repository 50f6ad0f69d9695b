// Expert-parallel MoE exchange kernels over symmetric memory (dispatch / combine all-to-all).
//
// The reference's MoE workload uses the vendored fastmoe (/root/reference/models/moe/train_moe.py;
// third-party/fastmoe/cuda/local_exchange.cuh:5-69 count/assign-pos kernels,
// global_exchange.h:11-98 grouped ncclSend/ncclRecv all-to-all-v, parallel_linear.cuh per-expert
// cuBLAS GEMMs). GPU-first equivalent: the token exchange is NOT a collective library call — each
// rank's kernel stores token rows straight into the destination rank's expert buffer over NVLink
// (dispatch) and loads result rows straight out of it (combine); slot assignment is a device-side
// stable rank per expert (token order); ranks only meet at per-CTA flag barriers on the signal pad.
//
// Buffer layout on every rank (symmetric heap): [E_local][world][capacity][d]  — expert-major, so
// the expert MLP is one batched GEMM over [E_local, world*capacity, d] with static shapes (CUDA
// graph friendly); rows past a (expert, source) pair's count stay zero.
#include <cuda_bf16.h>

#include "comm_context.h"
#include "device_prims.cuh"

namespace adapcc {

struct MoePeers {
  char* buf[kMaxRanks];      // rank r's buffer in MY address space
};

// slot assignment by STABLE rank: pos[i] = #{j < i : expert[j] == expert[i]}, or -1 when that rank is >= capacity or
// the expert id is invalid; counts[e] = the uncapped number of assignments to e. An expert keeps its first `capacity`
// assignments in token order (the drop rule of MoEMLP._local), and the buffer's row order, hence the bits of the
// expert GEMMs' weight gradients, is the same on every run (an atomic counter hands out slots in arrival order).
// One CTA per expert scans all assignments in chunks of blockDim: ballot + popc within a warp, warp totals through
// shared memory. No host-visible sizes, so it stays CUDA-graph capturable.
constexpr int kMoeAssignThreads = 1024;
__global__ void __launch_bounds__(kMoeAssignThreads)
moe_assign_kernel(const int* __restrict__ expert, int n_assign, int n_expert, int capacity, int* __restrict__ counts,
                  int* __restrict__ pos) {
  __shared__ int warp_hits[kMoeAssignThreads / 32];
  const int e = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  int base = 0;                                       // hits of expert e before this chunk
  for (int i0 = 0; i0 < n_assign; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    const int x = i < n_assign ? expert[i] : -1;
    const bool hit = x == e;
    const unsigned int b = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) warp_hits[warp] = __popc(b);
    __syncthreads();
    int before = base, total = 0;
    for (int w = 0; w < nwarps; ++w) {
      const int h = warp_hits[w];
      if (w < warp) before += h;
      total += h;
    }
    if (hit) {
      const int r = before + __popc(b & ((1u << lane) - 1u));
      pos[i] = r < capacity ? r : -1;
    } else if (e == 0 && i < n_assign && (x < 0 || x >= n_expert)) {
      pos[i] = -1;
    }
    base += total;
    __syncthreads();                                  // warp_hits is rewritten by the next chunk
  }
  if (threadIdx.x == 0) counts[e] = base;
}

// push: row i of src ([n_assign, d] bf16) -> buffer of rank (e / E_local), slot (e % E_local, me, pos).
// One warp per row, 128-bit stores over NVLink. `scale` (optional, fp32 per row) is fused.
__global__ void __launch_bounds__(256)
moe_push_kernel(const __nv_bfloat16* __restrict__ src, const int* __restrict__ expert, const int* __restrict__ pos,
                const float* __restrict__ scale, MoePeers peers, int me, int world, int e_local, int capacity,
                int d, int n_assign) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_assign) return;
  const int p = pos[warp];
  if (p < 0) return;
  const int e = expert[warp];
  const int dst = e / e_local, le = e % e_local;
  char* out = peers.buf[dst] + ((size_t)((le * world + me) * (size_t)capacity + p)) * d * 2;
  const uint4* in = reinterpret_cast<const uint4*>(src + (size_t)warp * d);
  const float s = scale ? scale[warp] : 1.f;
  for (int v = lane; v < d / 8; v += 32) {
    uint4 q = in[v];
    if (scale) {
      float f[8];
      unpack<__nv_bfloat16>(q, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] *= s;
      q = pack<__nv_bfloat16>(f);
    }
    st16(out + (size_t)v * 16, q);
  }
}

// pull: dst row i <- buffer of rank (e / E_local), slot (e % E_local, me, pos); dropped rows -> 0.
__global__ void __launch_bounds__(256)
moe_pull_kernel(__nv_bfloat16* __restrict__ dst_rows, const int* __restrict__ expert, const int* __restrict__ pos,
                MoePeers peers, int me, int world, int e_local, int capacity, int d, int n_assign) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_assign) return;
  const int p = pos[warp];
  uint4* out = reinterpret_cast<uint4*>(dst_rows + (size_t)warp * d);
  if (p < 0) {
    for (int v = lane; v < d / 8; v += 32) out[v] = make_uint4(0, 0, 0, 0);
    return;
  }
  const int e = expert[warp];
  const int src = e / e_local, le = e % e_local;
  const char* in = peers.buf[src] + ((size_t)((le * world + me) * (size_t)capacity + p)) * d * 2;
  for (int v0 = lane; v0 < d / 8; v0 += 32 * 4) {
    uint4 q[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (v0 + u * 32 < d / 8) q[u] = ld16(in + (size_t)(v0 + u * 32) * 16);
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (v0 + u * 32 < d / 8) out[v0 + u * 32] = q[u];
  }
}

// all participants meet (one CTA): orders "my pushes are visible" before "peers read their buffers"
__global__ void barrier_kernel(const __grid_constant__ DevComm c) {
  BarrierState b = barrier_begin(c);
  block_barrier(c, b);
  finish_op(c, b);
}

namespace adapcc_detail {
void launch_barrier(const DevComm& dc, cudaStream_t s) { barrier_kernel<<<1, 64, 0, s>>>(dc); }
}  // namespace adapcc_detail

}  // namespace adapcc

using namespace adapcc;

extern "C" {

int adapcc_barrier(void* h, const int* active, int n_active, void* stream) {
  CommContext* c = static_cast<CommContext*>(h);
  std::vector<int> act(active, active + n_active);
  return c->device_barrier(act, (cudaStream_t)stream);
}

// expert: int32 [n_assign]; pos: int32 [n_assign] (stable rank within the expert, -1 = dropped); counts: int32
// [n_expert], overwritten with the uncapped totals.
int adapcc_moe_assign(const int* expert, int n_assign, int n_expert, int capacity, int* counts, int* pos,
                      void* stream) {
  if (n_expert <= 0) { set_error("moe_assign: n_expert must be positive"); return -1; }
  if (n_assign <= 0) return 0;
  moe_assign_kernel<<<n_expert, kMoeAssignThreads, 0, (cudaStream_t)stream>>>(expert, n_assign, n_expert, capacity,
                                                                             counts, pos);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// `heap_offset`: byte offset of the [E_local][world][capacity][d] buffer inside the symmetric heap
// (same on every rank). direction 0 = push (src -> remote buffers), 1 = pull (remote buffers -> dst).
int adapcc_moe_exchange(void* h, int direction, void* rows, const int* expert, const int* pos, const float* scale,
                        unsigned long long heap_offset, int e_local, int capacity, int d, int n_assign,
                        void* stream) {
  CommContext* c = static_cast<CommContext*>(h);
  if (d % 8 != 0) { set_error("moe_exchange: d must be a multiple of 8"); return -1; }
  if (!c->heap_ptr()) { set_error("moe_exchange: context has no symmetric heap"); return -1; }
  const size_t need = (size_t)e_local * c->world() * capacity * d * 2;
  if (heap_offset + need > c->heap_bytes()) { set_error("moe_exchange: buffer exceeds the symmetric heap"); return -1; }
  if (n_assign <= 0) return 0;
  MoePeers peers;
  for (int r = 0; r < c->world(); ++r) peers.buf[r] = (char*)c->peer_heap_ptr(r) + heap_offset;
  const int blocks = (n_assign * 32 + 255) / 256;
  if (direction == 0)
    moe_push_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)rows, expert, pos, scale, peers,
                                                              c->rank(), c->world(), e_local, capacity, d, n_assign);
  else
    moe_pull_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)rows, expert, pos, peers, c->rank(),
                                                              c->world(), e_local, capacity, d, n_assign);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
