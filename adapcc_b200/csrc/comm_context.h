// Host-side communicator context: symmetric windows, signal pads, device-resident op
// state, strategy, and the launchers for every collective kernel.
//
// One context == one "transmission context" of the reference
// (allreduceContext/reduceContext/boardcastContext, /root/reference/csrc/include/trans.h:219-255)
// but without threads or queues: a collective is one kernel launch on the caller's stream.
#pragma once
#include <memory>
#include <string>
#include <vector>

#include "schedule.h"
#include "symm_mem.h"

namespace adapcc {

struct Tunables {
  int max_blocks = 64;                 // CTAs per collective kernel (same on all ranks)
  long long one_shot_max_bytes = 256 << 10;   // wire bytes: <= -> one-shot
  long long nvls_min_bytes = 0;        // wire bytes: >= -> NVLS when available
  long long ll_max_bytes = 32768;      // AUTO: all-rank messages up to this size use the LL kernel (0 = never)
  int nvls_min_ranks = 3;              // NVLS only pays off when >2 ranks share the switch reduction
  int relay_mode = RELAY_FORWARD;
  long long timeout_ms = 30000;
  long long pipe_min_bytes = 32ll << 20;   // staged ops at least this large use the pipelined kernel (0 = never)
  int pipe_nvls = 0;                        // also pipeline staged NVLS ops (HBM-bound on an NVSwitch box)
  int pipe_stagers = 48, pipe_links = 48;   // CTAs of its two sub-grids
  long long pipe_piece_bytes = 16ll << 20;
  int force_kernel = 0;                // run kernels even for a single participant (smoke / ncu)
  int tree_blocks = 128;                // CTAs of the tree kernel (half reduce, half broadcast)
  long long tree_chunk_max_bytes = 256 << 10;  // device pipelining granularity (wire bytes)
};

class CommContext {
 public:
  ~CommContext();
  int init(const std::string& name, int rank, int world, int device, size_t staging_bytes,
           size_t heap_bytes);
  void destroy();

  int load_strategy_text(const std::string& xml);
  int load_strategy_file(const std::string& path);

  // Direct collectives. `active`: sorted world ranks taking part (must contain rank_ to
  // launch anything but a sequence bump). In-place allowed (in == out).
  int allreduce(const void* in, void* out, long long count, int dtype, int wire, int op, int algo,
                const std::vector<int>& active, cudaStream_t stream);
  int reduce(const void* in, void* out, long long count, int dtype, int wire, int op, int algo,
             int root, const std::vector<int>& active, cudaStream_t stream);
  int broadcast(void* buf, long long count, int dtype, int root, const std::vector<int>& active,
                cudaStream_t stream);
  // Dense all-to-all, `per_peer` elements to/from every active rank (in != out).
  int alltoall(const void* in, void* out, long long per_peer, int dtype, const std::vector<int>& active,
               cudaStream_t stream);
  // Strategy-driven tree collective (prim = ALLREDUCE / REDUCE / BOARDCAST).
  int tree_collective(int prim, const void* in, void* out, long long count, int dtype, int wire,
                      int op, long long chunk_bytes, const std::vector<int>& active,
                      cudaStream_t stream);
  // Relay duty for a whole training step in ONE persistent kernel: bucket i has counts[i] elements
  // of `wire` dtype and chunk_bytes[i]; this rank must NOT be in `active`. Falls back to per-bucket
  // launches when a bucket does not fit the staging window.
  int tree_relay_persistent(int n_buckets, const long long* counts, const long long* chunk_bytes, int wire, int op,
                            const std::vector<int>& active, cudaStream_t stream);
  // Low-latency one-shot all-reduce (kernels_ll.cuh): all ranks active, <= 32 KB, flag-in-data, no barrier.
  // Available unless the context was created with ADAPCC_LL=0 (the 2 MB LL buffer is allocated by default).
  int allreduce_ll(const void* in, void* out, long long count, int dtype, int op, cudaStream_t stream);
  bool has_ll() const { return ll_.size != 0; }
  int skip_op(cudaStream_t stream);
  // One-CTA device barrier among `active` (orders peer stores before peer loads across kernels).
  int device_barrier(const std::vector<int>& active, cudaStream_t stream);

  // Reads (and clears) the sticky device error word; synchronises the stream.
  int check(cudaStream_t stream);

  void* heap_ptr() const { return heap_.size ? heap_.peers[rank_] : nullptr; }
  size_t heap_bytes() const { return heap_.size; }
  size_t staging_bytes() const { return staging_.size; }
  bool has_multicast() const { return staging_.mc != nullptr; }
  bool heap_multicast() const { return heap_.mc != nullptr; }
  int symm_backend() const { return staging_.backend; }
  int rank() const { return rank_; }
  int world() const { return world_; }
  const Strategy& strategy() const { return strategy_; }
  Tunables tun;
  int last_algo = 0;                   // algorithm picked by the last allreduce (for tests)
  SymmContext& symm() { return symm_; }
  void* peer_heap_ptr(int r) const { return heap_.peers[r]; }
  void* peer_staging_ptr(int r) const { return staging_.peers[r]; }
  void* staging_mc_ptr() const { return staging_.mc; }
  void* heap_mc_ptr() const { return heap_.mc; }
  // 2*kMaxRanks u64 ping-pong slots of rank r (inside its signal window)
  void* profile_flag_ptr(int r) const { return (char*)sig_.peers[r] + 32768; }

 private:
  struct Window { char* data[kMaxRanks]; char* mc; size_t capacity; bool zero_copy; };
  // Resolve where the op's data lives: inside the heap (zero copy) or the staging window.
  Window resolve(const void* in, const void* out, size_t bytes_wire, bool same_dtype);
  int fill_comm(const std::vector<int>& participants, const Window& w, void* dc_out);
  int pick_algo(int algo, long long wire_bytes, int op, int wire, bool all_active, const Window& w);

  SymmContext symm_;
  SymmBuffer staging_, heap_, sig_, ll_;
  char* d_state_ = nullptr;            // bar_epoch[], ticket, err, seq
  void* d_pipe_ = nullptr;             // PipeState of the pipelined staged kernel
  void* d_relay_work_[2] = {nullptr, nullptr};   // RelayWork[] of the persistent relay kernel, double-buffered:
  void* h_relay_work_[2] = {nullptr, nullptr};   // pinned host copies + one event per slot, so a step's descriptors are
  cudaEvent_t relay_ev_[2] = {nullptr, nullptr}; // uploaded asynchronously (no stream sync on the relay path)
  size_t relay_work_cap_ = 0;
  int relay_slot_ = 0;
  Strategy strategy_;
  int rank_ = 0, world_ = 1, device_ = 0;
  bool inited_ = false;
};

}  // namespace adapcc
