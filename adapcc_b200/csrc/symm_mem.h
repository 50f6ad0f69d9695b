// Symmetric-memory manager: every rank allocates the same-sized buffer, all buffers are
// mapped into every rank's address space (direct ld/st over NVLink from inside kernels)
// and, where the NVSwitch supports it, bound to one multicast object (NVLS
// multimem.ld_reduce / multimem.st).
//
// This is the native replacement for the reference's POSIX/SysV shared-memory
// tables of cudaIpcMemHandle_t / cudaIpcEventHandle_t and the receiver-allocated 1.6 GB
// per-child staging buffers (/root/reference/csrc/shm_ipc.cpp:5-96,
// /root/reference/csrc/allreduce.cu:442-495): one VMM allocation per rank, no IPC events,
// no host-visible flags.
#pragma once
#include <vector>

#include "bootstrap.h"
#include "common.h"

namespace adapcc {

enum SymmBackend : int { SYMM_VMM = 0, SYMM_CUDA_IPC = 1, SYMM_EXTERNAL = 2 };

struct SymmBuffer {
  size_t size = 0;                 // bytes usable (>= requested)
  void* peers[kMaxRanks] = {0};    // peers[r]: rank r's buffer in MY address space
  void* mc = nullptr;              // multicast mapping (nullptr if unavailable)
  int backend = SYMM_VMM;
  // teardown bookkeeping
  CUmemGenericAllocationHandle handles[kMaxRanks] = {0};
  CUmemGenericAllocationHandle mc_handle = 0;
  bool mc_bound = false;
};

class SymmContext {
 public:
  int init(const std::string& name, int rank, int world, int device);
  void destroy();

  // Collective: every rank must call with the same `bytes`/`want_mc`.
  int alloc(size_t bytes, bool want_mc, SymmBuffer* out);
  int free(SymmBuffer* buf);

  int rank() const { return rank_; }
  int world() const { return world_; }
  int device() const { return device_; }
  bool vmm_ok() const { return vmm_ok_; }
  bool multicast_ok() const { return mc_ok_; }
  Bootstrap& boot() { return boot_; }

 private:
  int alloc_vmm(size_t bytes, bool want_mc, SymmBuffer* out);
  int alloc_ipc(size_t bytes, SymmBuffer* out);
  int setup_multicast(size_t bytes, SymmBuffer* out);
  bool all_agree(bool mine);

  Bootstrap boot_;
  int rank_ = 0, world_ = 1, device_ = 0;
  bool vmm_ok_ = false, mc_ok_ = false;
};

}  // namespace adapcc
