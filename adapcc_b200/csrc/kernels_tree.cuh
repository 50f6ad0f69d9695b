// Strategy-driven tree collectives: one kernel executes the synthesised set of parallel
// reduction / broadcast trees ("transmissions"), chunk-pipelined, entirely on the device.
//
// Behavioural parity with the reference's allreduce/reduce/boardcast contexts
// (/root/reference/csrc/allreduce.cu:201-666, reduce.cu:153-367, boardcast.cu:152-318):
//   * the tensor is cut into one contiguous slice per tree, each slice into chunks,
//   * reduce runs leaf -> root, broadcast root -> leaf on the same tree, and a chunk starts
//     its way down as soon as the root has reduced it (reduce/broadcast pipelining),
//   * relay control: ranks that are not active contribute nothing but still forward.
// What is different (GPU-first): no pthread per tree, no copy engine, no IPC events, no
// host sync per chunk. A parent PULLS its children's partial sums with 128-bit peer loads
// over NVLink straight out of the child's symmetric window (so there is no per-child
// staging slot), reduces in fp32 registers and publishes the chunk with one
// st.release.sys flag. Tails are handled (reference defect: dropped by integer division).
#pragma once
#include "device_prims.cuh"
#include "kernels_direct.cuh"

namespace adapcc {

struct TreeRole {
  int parent;                    // effective parent (world rank) or -1 when root
  int n_children;                // children pulled from in the reduce phase
  int children[kMaxChildren];
  int flags;
};

struct TreePlan {
  int n_trees;
  int do_reduce, do_bcast;
  int zero_copy;                 // the tensors live at the same heap offset on every rank: reduce / broadcast in place
  long long chunk_packs;
  long long slice_begin[kMaxTrees + 1];   // in packs; slice t = [begin[t], begin[t+1])
  TreeRole role[kMaxTrees];
};

// One chunk of the reduce phase: acc = (own data) (+) children's partial sums. Children are
// pulled NCB at a time with UN packs each, i.e. NCB x UN independent 128-bit peer loads in
// flight per thread on top of the UN local loads.
template <typename U, typename W, int OP, int NCB, int UN>
__device__ __forceinline__ void reduce_chunk(const DevComm& c, const TreeRole& role, long long p0, long long pc,
                                             const U* __restrict__ in, U* __restrict__ out, long long n,
                                             bool in_vec, bool out_vec, char* __restrict__ local, bool has_local,
                                             bool is_root, bool to_window, bool to_user, float scale) {
  constexpr int kEpp = WireTraits<W>::kEpp;
  const int nc = role.n_children;
  for (long long j0 = threadIdx.x; j0 < pc; j0 += (long long)kThreads * UN) {
    float acc[UN][kEpp];
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const long long j = j0 + (long long)u * kThreads;
      if (j < pc && has_local) {
        load_user<U, kEpp>(in, (p0 + j) * kEpp, n, in_vec, acc[u]);
      } else {
#pragma unroll
        for (int i = 0; i < kEpp; ++i) acc[u][i] = red_identity<OP>();
      }
    }
    for (int a0 = 0; a0 < nc; a0 += NCB) {
      uint4 v[UN][NCB];
#pragma unroll
      for (int b = 0; b < NCB; ++b) {
        if (a0 + b < nc) {
          const char* kid = c.data[role.children[a0 + b]];
#pragma unroll
          for (int u = 0; u < UN; ++u) {
            const long long j = j0 + (long long)u * kThreads;
            if (j < pc) v[u][b] = ld16(kid + (p0 + j) * 16);
          }
        }
      }
#pragma unroll
      for (int b = 0; b < NCB; ++b) {
        if (a0 + b < nc) {
#pragma unroll
          for (int u = 0; u < UN; ++u) {
            const long long j = j0 + (long long)u * kThreads;
            if (j < pc) {
              float f[kEpp];
              unpack<W>(v[u][b], f);
#pragma unroll
              for (int i = 0; i < kEpp; ++i) acc[u][i] = red_apply<OP>(acc[u][i], f[i]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const long long j = j0 + (long long)u * kThreads;
      if (j < pc) {
        if (is_root) {
#pragma unroll
          for (int i = 0; i < kEpp; ++i) acc[u][i] *= scale;
        }
        if (to_window) st16(local + (p0 + j) * 16, pack<W>(acc[u]));
        if (to_user) store_user<U, kEpp>(out, (p0 + j) * kEpp, n, out_vec, acc[u]);
      }
    }
  }
}

// The grid is split in two halves, like the reference's reduce thread + broadcast thread per
// tree (/root/reference/csrc/allreduce.cu:735-742): CTAs [0, G/2) run the reduce pipeline over
// the (tree, chunk) items, CTAs [G/2, G) run the broadcast pipeline over the same items. The
// root's reduce CTA b hands chunk after chunk to the broadcast side through bflag[b] — the
// device-side equivalent of the reference's bcstCount mailbox (allreduce.cu:651-653) — so a
// chunk travels down while later chunks are still being reduced and neither pipeline ever
// idles waiting for the other phase.
template <typename U, typename W, int OP>
__device__ __forceinline__ void tree_collective_body(const DevComm& c, const TreePlan& plan,
                                                     const U* __restrict__ in, U* __restrict__ out, long long n,
                                                     float scale, unsigned long long q, BarrierState& epoch,
                                                     int lanes) {
  constexpr int kEpp = WireTraits<W>::kEpp;
  const bool in_vec = (reinterpret_cast<uintptr_t>(in) & 15) == 0;
  const bool out_vec = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  char* const local = c.data[c.rank];
  const int half = lanes;                       // CTAs [0, lanes) reduce, [lanes, 2*lanes) broadcast
  if ((int)blockIdx.x >= 2 * lanes) return;     // persistent relay grids may be wider than this op
  const bool bcast_side = (int)blockIdx.x >= half;
  const int lane = bcast_side ? blockIdx.x - half : blockIdx.x;   // pipeline lane 0..half-1
  unsigned long long* const my_rflag = c.flag[c.rank] + lane;
  // three single-writer flag words per lane: partial sum ready (reduce CTA), result ready at
  // the root (root's reduce CTA), result forwarded (broadcast CTA)
  unsigned long long* const my_root_bflag = c.flag[c.rank] + kMaxBlocks + lane;
  unsigned long long* const my_fwd_bflag = c.flag[c.rank] + 2 * kMaxBlocks + lane;

  long long max_k = 0;
  for (int t = 0; t < plan.n_trees; ++t) {
    const long long len = plan.slice_begin[t + 1] - plan.slice_begin[t];
    const long long nk = (len + plan.chunk_packs - 1) / plan.chunk_packs;
    max_k = nk > max_k ? nk : max_k;
  }
  const long long n_items = max_k * plan.n_trees;

  unsigned long long m = 0;
  for (long long item = lane; item < n_items; item += half, ++m) {
    const int t = (int)(item % plan.n_trees);
    const long long k = item / plan.n_trees;
    const long long p0 = plan.slice_begin[t] + k * plan.chunk_packs;
    long long pc = plan.slice_begin[t + 1] - p0;
    if (pc <= 0) continue;
    if (pc > plan.chunk_packs) pc = plan.chunk_packs;
    const unsigned long long token = (q << 24) | (c.item_base + m + 1);
    const TreeRole& role = plan.role[t];
    const bool is_root = role.parent < 0;
    const int nc = role.n_children;

    if (!bcast_side) {
      // ------------------------------ reduce pipeline ------------------------------
      if (plan.do_reduce && (role.flags & TR_IN_REDUCE)) {
        if (nc > 0) {
          if ((int)threadIdx.x < nc) wait_flag64(c, c.flag[role.children[threadIdx.x]] + lane, token);
          __syncthreads();
        }
        const bool has_local = role.flags & TR_HAS_LOCAL;
        const bool to_window = !is_root || (plan.do_bcast && (role.flags & TR_PUBLISH));
        // in place the window IS the user tensor: one store
        const bool to_user = is_root && (role.flags & TR_WANT_RESULT) && !(plan.zero_copy && to_window);
        reduce_chunk<U, W, OP, 2, 4>(c, role, p0, pc, in, out, n, in_vec, out_vec, local, has_local, is_root,
                                     to_window, to_user, scale);
        __syncthreads();
        if (threadIdx.x == 0) st_release_sys64(is_root ? my_root_bflag : my_rflag, token);
      } else if (!plan.do_reduce && plan.do_bcast && is_root) {
        // pure broadcast: the root publishes its tensor chunk by chunk (in place there is nothing to copy)
        for (long long j0 = threadIdx.x; j0 < pc && !plan.zero_copy; j0 += (long long)kThreads * kUnroll) {
          float f[kUnroll][kEpp];
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            const long long j = j0 + (long long)u * kThreads;
            if (j < pc) load_user<U, kEpp>(in, (p0 + j) * kEpp, n, in_vec, f[u]);
          }
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            const long long j = j0 + (long long)u * kThreads;
            if (j < pc) st16(local + (p0 + j) * 16, pack<W>(f[u]));
          }
        }
        __syncthreads();
        if (threadIdx.x == 0) st_release_sys64(my_root_bflag, token);
      }
    } else {
      // ----------------------------- broadcast pipeline ----------------------------
      if (plan.do_bcast && !is_root && (role.flags & TR_IN_BCAST)) {
        if (threadIdx.x == 0)
          wait_flag64(c, c.flag[role.parent] + ((role.flags & TR_PARENT_IS_ROOT) ? 1 : 2) * kMaxBlocks + lane, token);
        __syncthreads();
        const bool publish = role.flags & TR_PUBLISH;
        const bool want = (role.flags & TR_WANT_RESULT) && !(plan.zero_copy && publish);
        const char* src = c.data[role.parent];
        constexpr int UB = 8;
        for (long long j0 = threadIdx.x; j0 < pc; j0 += (long long)kThreads * UB) {
          uint4 v[UB];
#pragma unroll
          for (int u = 0; u < UB; ++u) {
            const long long j = j0 + (long long)u * kThreads;
            if (j < pc) v[u] = ld16(src + (p0 + j) * 16);
          }
#pragma unroll
          for (int u = 0; u < UB; ++u) {
            const long long j = j0 + (long long)u * kThreads;
            if (j < pc) {
              if (publish) st16(local + (p0 + j) * 16, v[u]);
              if (want) {
                float f[kEpp];
                unpack<W>(v[u], f);
                store_user<U, kEpp>(out, (p0 + j) * kEpp, n, out_vec, f);
              }
            }
          }
        }
        if (publish) {
          __syncthreads();
          if (threadIdx.x == 0) st_release_sys64(my_fwd_bflag, token);
        }
      }
    }
  }
  // windows are reused by the next op: nobody leaves while a peer may still be pulling
  block_barrier(c, epoch);
}

template <typename U, typename W, int OP>
__global__ void __launch_bounds__(kThreads, 1)
tree_collective_kernel(const __grid_constant__ DevComm c, const __grid_constant__ TreePlan plan,
                       const U* __restrict__ in, U* __restrict__ out, long long n, float scale) {
  BarrierState epoch = barrier_begin(c);
  tree_collective_body<U, W, OP>(c, plan, in, out, n, scale, *c.seq, epoch, (int)(gridDim.x >> 1));
  finish_op(c, epoch);
}

// Persistent relay kernel: ONE launch serves every gradient bucket of a training step on a rank
// that is not active in it (a straggler). The rank contributes no data; where the strategy routes
// other ranks' chunks through it, its CTAs pull them from the children's windows, (re-)reduce, and
// publish them for the parent, bucket after bucket, without the host re-launching anything and
// without touching the training stream. `work[i]` describes bucket i (same plans the active ranks
// run, with this rank's relay roles); op sequence numbers advance exactly as if the buckets had
// been launched one by one, so relays and active ranks stay in step.
struct RelayWork {
  TreePlan plan;
  long long n;
  float scale;
  int skip;        // 1: this rank holds no role in this bucket -> only the sequence number moves
  int lanes;       // pipeline lanes the active ranks use for this bucket (grid = 2 * lanes there)
};

template <typename W, int OP>
__global__ void __launch_bounds__(kThreads, 1)
tree_relay_persistent_kernel(const __grid_constant__ DevComm c, const RelayWork* __restrict__ work, int n_work) {
  BarrierState epoch = barrier_begin(c);
  const unsigned long long q0 = *c.seq;
  for (int i = 0; i < n_work; ++i) {
    if (work[i].skip) continue;
    tree_collective_body<W, W, OP>(c, work[i].plan, (const W*)nullptr, (W*)nullptr, work[i].n, work[i].scale,
                                   q0 + (unsigned long long)i, epoch, work[i].lanes);
  }
  finish_op(c, epoch, n_work);
}

// Keeps a non-participating rank's op sequence number in step with the others.
__global__ void skip_op_kernel(const __grid_constant__ DevComm c) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *c.seq = *c.seq + 1;
}

}  // namespace adapcc
