// Pipelined staged all-reduce for LARGE tensors that are not in the symmetric heap.
//
// The plain staged kernel (kernels_direct.cuh) runs stage-in -> NVLink phase -> stage-out with all
// CTAs in lockstep, so HBM copies and link traffic never overlap, and large staged tensors fall well
// behind the zero-copy path. Here the message is cut into pieces and the grid into two sub-grids,
// the same idea as the tree kernel's reduce/broadcast split (and the reference's thread pair per
// tree, /root/reference/csrc/allreduce.cu:735-742):
//
//   stager CTAs [0, S)   : stage-in(piece p+2) / stage-out(piece p)      — local HBM traffic
//   link CTAs   [S, S+L) : barrier, NVLS or two-shot phase on piece p+1, barrier — NVLink traffic
//
// hand-off through two device-local counters per piece (in_ready / out_ready, gpu scope); only the
// link CTAs take part in the cross-GPU flag barriers. A link CTA signals its peers for piece p only
// after ALL local stagers finished piece p, so after the barrier every rank's piece p is fully
// staged; out_ready[p] reaches L only after every link CTA passed the post-phase barrier, i.e. all
// peers finished writing piece p into this window.
#pragma once
#include "kernels_direct.cuh"

namespace adapcc {

constexpr int kMaxPieces = 64;

struct PipeState {            // device memory, zeroed; reset by the last CTA of every op
  unsigned in_ready[kMaxPieces];
  unsigned out_ready[kMaxPieces];
};

__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu(unsigned* p) {
  asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p) : "memory");
}

__device__ __forceinline__ bool wait_local(const DevComm& c, const unsigned* p, unsigned want) {
  if (threadIdx.x == 0) {
    unsigned long long t0 = globaltimer_ns();
    unsigned spins = 0;
    while (ld_acquire_gpu(p) < want) {
      if ((++spins & 0x3ff) == 0 && c.timeout_ns && globaltimer_ns() - t0 > c.timeout_ns) {
        atomicExch(c.err, 3u);
        break;
      }
    }
  }
  __syncthreads();
  return true;
}

template <typename U, typename W, int OP, int ALGO, int NR>
__global__ void __launch_bounds__(kThreads, 1)
allreduce_pipelined_kernel(const __grid_constant__ DevComm c, PipeState* __restrict__ ps, const U* __restrict__ in,
                           U* __restrict__ out, long long n, float scale, int n_stagers, int n_pieces) {
  constexpr int kEpp = WireTraits<W>::kEpp;
  BarrierState epoch = barrier_begin(c);
  const int na = c.n_active, me = c.my_index;
  const int S = n_stagers, L = (int)gridDim.x - n_stagers;
  const bool in_vec = (reinterpret_cast<uintptr_t>(in) & 15) == 0;
  const bool out_vec = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  char* const local = c.data[c.rank];
  const long long npacks = (n + kEpp - 1) / kEpp;
  const long long ppp = (npacks + n_pieces - 1) / n_pieces;     // packs per piece

  auto piece = [&](int p) {
    Partition P;
    P.pack0 = (long long)p * ppp;
    long long cnt = npacks - P.pack0;
    P.npacks = cnt < 0 ? 0 : (cnt > ppp ? ppp : cnt);
    P.nslices = na;
    P.pps = (P.npacks + na - 1) / na;
    return P;
  };

  if ((int)blockIdx.x < S) {
    // ------------------------------- stager sub-grid -----------------------------------------
    const SubGrid g((int)blockIdx.x, S);
    for (int i = 0; i < n_pieces + 2; ++i) {
      if (i < n_pieces) {
        stage_in<U, W>(piece(i), in, n, in_vec, local, g);
        __syncthreads();
        if (threadIdx.x == 0) red_release_gpu(&ps->in_ready[i]);
      }
      if (i >= 2) {
        const int p = i - 2;
        wait_local(c, &ps->out_ready[p], (unsigned)L);
        stage_out<U, W>(piece(p), out, n, out_vec, local, scale, g);
      }
    }
  } else {
    // -------------------------------- link sub-grid ------------------------------------------
    const SubGrid g((int)blockIdx.x - S, L);
    for (int p = 0; p < n_pieces; ++p) {
      const Partition P = piece(p);
      wait_local(c, &ps->in_ready[p], (unsigned)S);
      block_barrier(c, epoch);                       // every rank's piece p is staged
      const long long base = P.slice_begin(me), cnt = P.slice_count(me);
      if (ALGO == TWO_SHOT) two_shot_phase1<W, OP, NR>(c, base, cnt, false, scale, false, 0, g);
      else nvls_phase1<W, OP>(c, base, cnt, false, scale, false, 0, g);
      block_barrier(c, epoch);                       // every rank's piece p is complete in all windows
      if (threadIdx.x == 0) red_release_gpu(&ps->out_ready[p]);
    }
  }
  // last CTA out resets the hand-off counters for the next op (everybody is done with them)
  if (epoch.peer >= 0) c.bar_epoch[blockIdx.x * kMaxRanks + epoch.peer] = epoch.epoch;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const uint32_t t = atomicAdd(c.ticket, 1u);
    if (t == gridDim.x - 1) {
      for (int i = 0; i < kMaxPieces; ++i) { ps->in_ready[i] = 0; ps->out_ready[i] = 0; }
      __threadfence();
      *c.ticket = 0;
      *c.seq = *c.seq + (unsigned long long)c.op_advance;
    }
  }
}

}  // namespace adapcc
