// adapcc_b200 native runtime — shared definitions.
//
// Replaces the reference's csrc/include/init.h limits (MAX_DEVICES 16, MAX_TRANS 8,
// MAX_CHUNK_NUM 512, 1.6 GB/child staging; /root/reference/csrc/include/init.h:14-25)
// with a design sized for one 8-GPU NVSwitch box: no per-child staging slots, no
// per-chunk IPC events, sizes are 64-bit.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

namespace adapcc {

constexpr int kMaxRanks   = 16;    // ranks in one NVLink domain handled by one kernel
constexpr int kMaxTrees   = 8;     // parallel "transmissions" (strategy trees)
constexpr int kMaxBlocks  = 160;   // upper bound on CTAs of any collective kernel
constexpr int kMaxChildren = kMaxRanks - 1;

// Primitive ids: identical numbering to /root/reference/commu.py:28-35 and
// csrc/include/trans.h:27-36.
enum Primitive : int {
  ALLREDUCE = 0, REDUCE = 1, BOARDCAST = 2, ALLGATHER = 3,
  ALLTOALL = 4, REDUCESCATTER = 5, DETECT = 6, PROFILE = 7,
};

enum DType : int { F32 = 0, BF16 = 1, F16 = 2 };
enum RedOp : int { SUM = 0, AVG = 1, MAX = 2 };
enum Algo  : int { AUTO = 0, ONE_SHOT = 1, TWO_SHOT = 2, NVLS = 3, TREE = 4 };

// Role of one rank in one strategy tree for one op (see schedule.h / kernels_tree.cuh).
enum TreeRoleFlags : int {
  TR_HAS_LOCAL = 1,     // contributes its own data to the reduction (rank is active)
  TR_IN_REDUCE = 2,     // takes part in the reduce phase (has data and/or active subtree)
  TR_IN_BCAST = 4,      // must pull the result from its parent in the broadcast phase
  TR_WANT_RESULT = 8,   // writes the result into its user tensor
  TR_PUBLISH = 16,      // other ranks pull the result from this rank (has bcast children)
  TR_PARENT_IS_ROOT = 32,  // my effective parent is the tree's root (selects which flag to wait on)
};

inline size_t dtype_size(int dt) { return dt == F32 ? 4 : 2; }

// thread-local last-error string surfaced to Python (ops fail loudly, never silently
// fall back).
void set_error(const char* fmt, ...);
const char* get_error();
int log_level();

#define ADAPCC_LOG(lvl, ...)                                   \
  do { if (::adapcc::log_level() >= (lvl)) {                   \
    fprintf(stderr, "[adapcc] " __VA_ARGS__); fprintf(stderr, "\n"); } } while (0)

#define CUDA_TRY(expr)                                                         \
  do { cudaError_t _e = (expr); if (_e != cudaSuccess) {                       \
    ::adapcc::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr,           \
                        cudaGetErrorString(_e)); return -1; } } while (0)

#define CU_TRY(expr)                                                           \
  do { CUresult _e = (expr); if (_e != CUDA_SUCCESS) {                         \
    const char* _s = ::adapcc::cu_error_string(_e);                            \
    ::adapcc::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, _s);      \
    return -1; } } while (0)

const char* cu_error_string(CUresult r);

// Number of kernels this library has launched (bench.py reports it as gpu_launches).
void count_launch(int n = 1);
long long launch_count();

}  // namespace adapcc
