#include "comm_context.h"

#include <algorithm>

#include "kernels_direct.cuh"
#include "kernels_ll.cuh"
#include "kernels_pipelined.cuh"
#include "kernels_tree.cuh"

namespace adapcc {

namespace {
constexpr size_t kPadBytes = 16384;                       // barrier pad region
constexpr size_t kFlagOffset = kPadBytes;                 // chunk flags follow
constexpr size_t kSigBytes = 65536;
constexpr size_t kStateEpoch = 0, kStateTicket = 12288, kStateErr = 12292, kStateSeq = 12296,
                 kStateLLSeq = 12304, kStateBytes = 16384;
static_assert(kMaxBlocks * kMaxRanks * 4 <= kStateTicket, "epoch table too small");
static_assert(kMaxBlocks * kMaxRanks * 4 <= kPadBytes, "pad too small");
static_assert(3 * kMaxBlocks * 8 + kFlagOffset <= 32768, "flag region too small");

int epp_of(int wire) { return wire == F32 ? 4 : 8; }

bool combo_ok(int dtype, int wire) {
  return (dtype == F32 && (wire == F32 || wire == BF16 || wire == F16)) ||
         (dtype == BF16 && wire == BF16) || (dtype == F16 && wire == F16);
}

// dispatch helpers --------------------------------------------------------------------
#define ADAPCC_DISPATCH_TYPES(dtype, wire, ...)                                            \
  [&]() -> int {                                                                           \
    if (dtype == F32 && wire == F32) { using U = float; using W = float; __VA_ARGS__ }     \
    if (dtype == F32 && wire == BF16) { using U = float; using W = __nv_bfloat16; __VA_ARGS__ } \
    if (dtype == F32 && wire == F16) { using U = float; using W = __half; __VA_ARGS__ }    \
    if (dtype == BF16 && wire == BF16) { using U = __nv_bfloat16; using W = __nv_bfloat16; __VA_ARGS__ } \
    if (dtype == F16 && wire == F16) { using U = __half; using W = __half; __VA_ARGS__ }   \
    set_error("unsupported dtype/wire combination %d/%d", dtype, wire);                    \
    return -1;                                                                             \
  }()

template <typename U, typename W, int OP, int NR>
int launch_direct_nr(int algo, int blocks, cudaStream_t s, const DevComm& dc, const U* i, U* o, long long n,
                     float scale, int flags, int root) {
  switch (algo) {
    case ONE_SHOT:
      allreduce_direct_kernel<U, W, OP, ONE_SHOT, NR><<<blocks, kThreads, 0, s>>>(dc, i, o, n, scale, flags, root);
      break;
    case TWO_SHOT:
      allreduce_direct_kernel<U, W, OP, TWO_SHOT, NR><<<blocks, kThreads, 0, s>>>(dc, i, o, n, scale, flags, root);
      break;
    default:
      set_error("launch_direct: bad algo %d", algo);
      return -1;
  }
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

template <typename U, typename W, int OP>
int launch_direct(int algo, int blocks, cudaStream_t s, const DevComm& dc, const void* in, void* out,
                  long long n, float scale, int flags, int root) {
  const U* i = static_cast<const U*>(in);
  U* o = static_cast<U*>(out);
  if (algo == NVLS) {
    allreduce_direct_kernel<U, W, OP, NVLS, 2><<<blocks, kThreads, 0, s>>>(dc, i, o, n, scale, flags, root);
    CUDA_TRY(cudaGetLastError());
    count_launch();
    return 0;
  }
  const int na = dc.n_active;
  if (na <= 2) return launch_direct_nr<U, W, OP, 2>(algo, blocks, s, dc, i, o, n, scale, flags, root);
  if (na <= 4) return launch_direct_nr<U, W, OP, 4>(algo, blocks, s, dc, i, o, n, scale, flags, root);
  if (na <= 8) return launch_direct_nr<U, W, OP, 8>(algo, blocks, s, dc, i, o, n, scale, flags, root);
  return launch_direct_nr<U, W, OP, 16>(algo, blocks, s, dc, i, o, n, scale, flags, root);
}
template <typename U, typename W, int OP>
int launch_pipelined(int algo, int stagers, int links, int pieces, cudaStream_t s, const DevComm& dc, PipeState* ps,
                     const void* in, void* out, long long n, float scale) {
  const U* i = static_cast<const U*>(in);
  U* o = static_cast<U*>(out);
  const int blocks = stagers + links;
  const int na = dc.n_active;
#define PIPE_LAUNCH(ALGO_, NR_) \
  allreduce_pipelined_kernel<U, W, OP, ALGO_, NR_><<<blocks, kThreads, 0, s>>>(dc, ps, i, o, n, scale, stagers, pieces)
  if (algo == NVLS) PIPE_LAUNCH(NVLS, 2);
  else if (na <= 2) PIPE_LAUNCH(TWO_SHOT, 2);
  else if (na <= 4) PIPE_LAUNCH(TWO_SHOT, 4);
  else if (na <= 8) PIPE_LAUNCH(TWO_SHOT, 8);
  else PIPE_LAUNCH(TWO_SHOT, 16);
#undef PIPE_LAUNCH
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}
}  // namespace

CommContext::~CommContext() { destroy(); }

int CommContext::init(const std::string& name, int rank, int world, int device, size_t staging_bytes,
                      size_t heap_bytes) {
  rank_ = rank;
  world_ = world;
  device_ = device;
  if (symm_.init(name, rank, world, device)) return -1;
  if (symm_.alloc(kSigBytes, false, &sig_)) return -1;
  if (staging_bytes < (1u << 20)) staging_bytes = 1u << 20;
  if (symm_.alloc(staging_bytes, true, &staging_)) return -1;
  if (heap_bytes) {
    if (symm_.alloc(heap_bytes, true, &heap_)) return -1;
  }
  {
    // low-latency buffer (2 MB): on by default since its first multi-GPU run (round 2: 4.2 us at 1 KB on 2 GPUs vs
    // 9.3 us for the barrier kernels, 332 numerics checks); ADAPCC_LL=0 turns it off — alike on every rank
    const char* ll = getenv("ADAPCC_LL");
    if (!(ll && atoi(ll) == 0) && world > 1) {
      if (symm_.alloc(kLLBufferBytes, false, &ll_)) return -1;
    }
  }
  CUDA_TRY(cudaMalloc(&d_state_, kStateBytes));
  CUDA_TRY(cudaMemset(d_state_, 0, kStateBytes));
  CUDA_TRY(cudaMalloc(&d_pipe_, sizeof(PipeState)));
  CUDA_TRY(cudaMemset(d_pipe_, 0, sizeof(PipeState)));
  CUDA_TRY(cudaDeviceSynchronize());
  const char* e = getenv("ADAPCC_MAX_BLOCKS");
  if (e && atoi(e) > 0) tun.max_blocks = std::min(atoi(e), kMaxBlocks);
  e = getenv("ADAPCC_TIMEOUT_MS");
  if (e) tun.timeout_ms = atoll(e);
  if (world > 1 && symm_.boot().barrier()) return -1;
  inited_ = true;
  return 0;
}

void CommContext::destroy() {
  if (!inited_) return;
  inited_ = false;
  cudaSetDevice(device_);
  cudaDeviceSynchronize();
  if (ll_.size) symm_.free(&ll_);
  symm_.free(&heap_);
  symm_.free(&staging_);
  symm_.free(&sig_);
  if (d_state_) cudaFree(d_state_);
  d_state_ = nullptr;
  if (d_pipe_) cudaFree(d_pipe_);
  d_pipe_ = nullptr;
  for (int i = 0; i < 2; ++i) {
    if (d_relay_work_[i]) cudaFree(d_relay_work_[i]);
    if (h_relay_work_[i]) cudaFreeHost(h_relay_work_[i]);
    if (relay_ev_[i]) cudaEventDestroy(relay_ev_[i]);
    d_relay_work_[i] = h_relay_work_[i] = nullptr;
    relay_ev_[i] = nullptr;
  }
  relay_work_cap_ = 0;
  symm_.destroy();
}

int CommContext::load_strategy_text(const std::string& xml) { return strategy_.load(xml, world_) ? 0 : -1; }
int CommContext::load_strategy_file(const std::string& path) {
  return strategy_.load_file(path, world_) ? 0 : -1;
}

CommContext::Window CommContext::resolve(const void* in, const void* out, size_t bytes, bool same_dtype) {
  Window w{};
  const char* hb = heap_.size ? (const char*)heap_.peers[rank_] : nullptr;
  const char* p = (const char*)in;
  if (hb && same_dtype && in == out && p >= hb && p + bytes <= hb + heap_.size &&
      ((p - hb) & 15) == 0) {
    const size_t off = (size_t)(p - hb);
    for (int r = 0; r < world_; ++r) w.data[r] = (char*)heap_.peers[r] + off;
    w.mc = heap_.mc ? (char*)heap_.mc + off : nullptr;
    w.capacity = heap_.size - off;
    w.zero_copy = true;
    return w;
  }
  for (int r = 0; r < world_; ++r) w.data[r] = (char*)staging_.peers[r];
  w.mc = (char*)staging_.mc;
  w.capacity = staging_.size;
  w.zero_copy = false;
  return w;
}

int CommContext::fill_comm(const std::vector<int>& parts, const Window& w, void* out) {
  DevComm& dc = *static_cast<DevComm*>(out);
  memset(&dc, 0, sizeof(dc));
  dc.rank = rank_;
  dc.world = world_;
  dc.n_active = (int)parts.size();
  dc.my_index = -1;
  for (int i = 0; i < (int)parts.size(); ++i) {
    if (parts[i] < 0 || parts[i] >= world_) { set_error("active rank %d out of range", parts[i]); return -1; }
    if (i && parts[i] <= parts[i - 1]) { set_error("active list must be sorted and unique"); return -1; }
    dc.active_ranks[i] = parts[i];
    if (parts[i] == rank_) dc.my_index = i;
  }
  for (int r = 0; r < world_; ++r) {
    dc.data[r] = w.data[r];
    dc.pad[r] = (uint32_t*)sig_.peers[r];
    dc.flag[r] = (unsigned long long*)((char*)sig_.peers[r] + kFlagOffset);
  }
  dc.mc_data = w.mc;
  dc.bar_epoch = (uint32_t*)(d_state_ + kStateEpoch);
  dc.ticket = (uint32_t*)(d_state_ + kStateTicket);
  dc.err = (uint32_t*)(d_state_ + kStateErr);
  dc.seq = (unsigned long long*)(d_state_ + kStateSeq);
  dc.timeout_ns = tun.timeout_ms > 0 ? (unsigned long long)tun.timeout_ms * 1000000ull : 0ull;
  dc.op_advance = 1;
  dc.item_base = 0;
  return 0;
}

int CommContext::pick_algo(int algo, long long wire_bytes, int op, int wire, bool all_active,
                           const Window& w) {
  const bool nvls_ok = w.mc != nullptr && all_active && !(op == MAX && wire == F32);
  if (algo == NVLS && !nvls_ok) {
    set_error("NVLS requested but unavailable (multicast=%d all_active=%d op=%d)", (int)(w.mc != nullptr),
              (int)all_active, op);
    return -1;
  }
  if (algo == ONE_SHOT || algo == TWO_SHOT || algo == NVLS) return algo;
  if (algo != AUTO) { set_error("bad algo %d", algo); return -1; }
  const bool nvls_pref = nvls_ok && wire_bytes >= tun.nvls_min_bytes && world_ >= tun.nvls_min_ranks;
  // zero-copy tensors never need the staging pass a one-shot would add, so the in-place NVLS / two-shot
  // kernels are taken at every size (not yet re-measured on an 8-GPU H100 system)
  if (w.zero_copy) return nvls_pref ? NVLS : TWO_SHOT;
  if (wire_bytes <= tun.one_shot_max_bytes) return ONE_SHOT;
  return nvls_pref ? NVLS : TWO_SHOT;
}

int CommContext::allreduce_ll(const void* in, void* out, long long count, int dtype, int op, cudaStream_t stream) {
  if (!inited_) { set_error("context not initialised"); return -1; }
  if (count <= 0) return skip_op(stream);
  const size_t esize = dtype_size(dtype);
  if (world_ == 1) {
    if (in != out) CUDA_TRY(cudaMemcpyAsync(out, in, (size_t)count * esize, cudaMemcpyDeviceToDevice, stream));
    return skip_op(stream);
  }
  if (!ll_.size) { set_error("allreduce_ll: no LL buffer (the context was created with ADAPCC_LL=0 or world size 1)"); return -1; }
  if ((size_t)count * esize > (size_t)kLLMaxBytes) { set_error("allreduce_ll: message larger than %d bytes", kLLMaxBytes); return -1; }
  if (((uintptr_t)in | (uintptr_t)out) & 3) { set_error("allreduce_ll: tensors must be 4-byte aligned"); return -1; }
  std::vector<int> all(world_);
  for (int r = 0; r < world_; ++r) all[r] = r;
  DevComm dc;
  Window w = resolve(nullptr, nullptr, 0, false);
  if (fill_comm(all, w, &dc)) return -1;
  LLArgs a{};
  for (int r = 0; r < world_; ++r) a.ll[r] = (char*)ll_.peers[r];
  a.ll_seq = (unsigned long long*)(d_state_ + kStateLLSeq);
  const float scale = (op == AVG) ? 1.f / (float)world_ : 1.f;
  const long long words = ((long long)count * (long long)esize + 3) / 4, lines = (words + 1) / 2;
  const int blocks = (int)std::max<long long>(1, std::min<long long>(8, (lines + 255) / 256));
#define LL_LAUNCH(U)                                                                                         \
  do {                                                                                                       \
    if (op == MAX) allreduce_ll_kernel<U, MAX><<<blocks, 256, 0, stream>>>(dc, a, (const U*)in, (U*)out, count, scale); \
    else allreduce_ll_kernel<U, SUM><<<blocks, 256, 0, stream>>>(dc, a, (const U*)in, (U*)out, count, scale); \
  } while (0)
  if (dtype == F32) LL_LAUNCH(float);
  else if (dtype == BF16) LL_LAUNCH(__nv_bfloat16);
  else if (dtype == F16) LL_LAUNCH(__half);
  else { set_error("allreduce_ll: unsupported dtype %d", dtype); return -1; }
#undef LL_LAUNCH
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

int CommContext::skip_op(cudaStream_t stream) {
  DevComm dc;
  Window w = resolve(nullptr, nullptr, 0, false);
  if (fill_comm({}, w, &dc)) return -1;
  skip_op_kernel<<<1, 32, 0, stream>>>(dc);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

int CommContext::reduce(const void* in, void* out, long long count, int dtype, int wire, int op, int algo,
                        int root, const std::vector<int>& active, cudaStream_t stream) {
  if (!inited_) { set_error("context not initialised"); return -1; }
  if (!combo_ok(dtype, wire)) { set_error("unsupported dtype/wire %d/%d", dtype, wire); return -1; }
  if (count < 0) { set_error("negative count"); return -1; }
  const bool mine = std::find(active.begin(), active.end(), rank_) != active.end();
  if (!mine || count == 0) return skip_op(stream);
  const int na = (int)active.size();
  int root_index = -1;
  int flags = 0;
  if (root >= 0) {
    for (int i = 0; i < na; ++i)
      if (active[i] == root) root_index = i;
    if (root_index < 0) { set_error("reduce root %d is not in the active list", root); return -1; }
    flags |= F_ROOT_ONLY;
  }
  const size_t esize = dtype_size(dtype), wsize = dtype_size(wire);
  if (na == 1 && !tun.force_kernel) {
    if (in != out) CUDA_TRY(cudaMemcpyAsync(out, in, (size_t)count * esize, cudaMemcpyDeviceToDevice, stream));
    return skip_op(stream);
  }
  const float scale = (op == AVG) ? 1.f / (float)na : 1.f;
  const int kop = (op == MAX) ? MAX : SUM;
  const bool root_only_op = root >= 0;
  Window w = resolve(in, out, (size_t)count * esize, dtype == wire);
  int a = pick_algo(algo, count * (long long)wsize, kop, wire, na == world_, w);
  if (a < 0) return -1;
  if (a == ONE_SHOT && w.zero_copy) {      // in-place one-shot would race with peers' reads
    w = Window{};
    for (int r = 0; r < world_; ++r) w.data[r] = (char*)staging_.peers[r];
    w.mc = (char*)staging_.mc;
    w.capacity = staging_.size;
    w.zero_copy = false;
  }
  last_algo = a;
  if (w.zero_copy) flags |= F_ZERO_COPY;
  const int epp = epp_of(wire);
  // staged ops larger than the window run as back-to-back pieces
  const long long cap_elems = w.zero_copy ? count : (long long)(w.capacity / 16) * epp;
  DevComm dc;
  if (fill_comm(active, w, &dc)) return -1;
  long long done = 0;
  while (done < count) {
    const long long n = std::min(count - done, cap_elems);
    const long long npacks = (n + epp - 1) / epp;
    dc.op_advance = (done + n >= count) ? 1 : 0;      // the op sequence number moves once per logical op
    int blocks = (int)std::min<long long>((npacks + (long long)kThreads * kUnroll - 1) / ((long long)kThreads * kUnroll),
                                          (long long)std::min(tun.max_blocks, kMaxBlocks));
    if (blocks < 1) blocks = 1;
    const char* pin = (const char*)in + (size_t)done * esize;
    char* pout = (char*)out + (size_t)done * esize;
    if (w.zero_copy && done) { set_error("internal: zero-copy op split into pieces"); return -1; }
    const long long wire_bytes = n * (long long)wsize;
    // splitting the grid into stager and link CTAs overlaps the staged two-shot's HBM copies with its link
    // traffic; staged NVLS is bound by local HBM traffic (6 bytes moved per payload byte) and gains nothing
    // from the split, so NVLS opts in only when asked to
    const bool pipe_algo = a == TWO_SHOT || (a == NVLS && tun.pipe_nvls);
    const bool pipelined = !w.zero_copy && !root_only_op && pipe_algo && tun.pipe_min_bytes > 0 &&
                           wire_bytes >= tun.pipe_min_bytes &&
                           tun.pipe_stagers + tun.pipe_links <= kMaxBlocks && tun.pipe_stagers > 0 && tun.pipe_links > 0;
    if (pipelined) {
      int pieces = (int)std::min<long long>(kMaxPieces, std::max<long long>(4, (wire_bytes + tun.pipe_piece_bytes - 1) /
                                                                                  std::max<long long>(1, tun.pipe_piece_bytes)));
      int rc = ADAPCC_DISPATCH_TYPES(dtype, wire, {
        if (kop == MAX)
          return launch_pipelined<U, W, MAX>(a, tun.pipe_stagers, tun.pipe_links, pieces, stream, dc, (PipeState*)d_pipe_, pin, pout, n, scale);
        return launch_pipelined<U, W, SUM>(a, tun.pipe_stagers, tun.pipe_links, pieces, stream, dc, (PipeState*)d_pipe_, pin, pout, n, scale);
      });
      if (rc) return rc;
      done += n;
      continue;
    }
    int rc = ADAPCC_DISPATCH_TYPES(dtype, wire, {
      if (kop == MAX) return launch_direct<U, W, MAX>(a, blocks, stream, dc, pin, pout, n, scale, flags, root_index);
      return launch_direct<U, W, SUM>(a, blocks, stream, dc, pin, pout, n, scale, flags, root_index);
    });
    if (rc) return rc;
    done += n;
  }
  return 0;
}

int CommContext::allreduce(const void* in, void* out, long long count, int dtype, int wire, int op, int algo,
                           const std::vector<int>& active, cudaStream_t stream) {
  // AUTO: small all-rank messages take the flag-in-data LL kernel (one NVLink store latency, no barrier)
  if (algo == AUTO && ll_.size && tun.ll_max_bytes > 0 && count > 0 && (int)active.size() == world_ && world_ > 1 &&
      dtype == wire && (long long)count * (long long)dtype_size(dtype) <= std::min<long long>(tun.ll_max_bytes, kLLMaxBytes) &&
      ((((uintptr_t)in) | ((uintptr_t)out)) & 3) == 0) {
    last_algo = 5;
    return allreduce_ll(in, out, count, dtype, op, stream);
  }
  return reduce(in, out, count, dtype, wire, op, algo, -1, active, stream);
}

int CommContext::broadcast(void* buf, long long count, int dtype, int root, const std::vector<int>& active,
                           cudaStream_t stream) {
  if (!inited_) { set_error("context not initialised"); return -1; }
  const bool mine = std::find(active.begin(), active.end(), rank_) != active.end();
  if (!mine || count == 0) return skip_op(stream);
  const int na = (int)active.size();
  int root_index = -1;
  for (int i = 0; i < na; ++i)
    if (active[i] == root) root_index = i;
  if (root_index < 0) { set_error("broadcast root %d is not in the active list", root); return -1; }
  if (na == 1 && !tun.force_kernel) return skip_op(stream);
  const size_t esize = dtype_size(dtype);
  Window w = resolve(buf, buf, (size_t)count * esize, true);
  const int wire = dtype;
  const int epp = epp_of(wire);
  const long long cap_elems = w.zero_copy ? count : (long long)(w.capacity / 16) * epp;
  const int use_mc = (w.mc != nullptr && na == world_) ? 1 : 0;
  DevComm dc;
  if (fill_comm(active, w, &dc)) return -1;
  long long done = 0;
  while (done < count) {
    const long long n = std::min(count - done, cap_elems);
    const long long npacks = (n + epp - 1) / epp;
    dc.op_advance = (done + n >= count) ? 1 : 0;
    int blocks = (int)std::min<long long>((npacks + (long long)kThreads * kUnroll - 1) / ((long long)kThreads * kUnroll),
                                          (long long)std::min(tun.max_blocks, kMaxBlocks));
    if (blocks < 1) blocks = 1;
    char* p = (char*)buf + (size_t)done * esize;
    const int flags = w.zero_copy ? F_ZERO_COPY : 0;
    int rc = ADAPCC_DISPATCH_TYPES(dtype, wire, {
      broadcast_direct_kernel<U, W><<<blocks, kThreads, 0, stream>>>(dc, (U*)p, n, root_index, use_mc, flags);
      CUDA_TRY(cudaGetLastError());
      count_launch();
      return 0;
    });
    if (rc) return rc;
    done += n;
  }
  return 0;
}

int CommContext::alltoall(const void* in, void* out, long long per_peer, int dtype, const std::vector<int>& active,
                          cudaStream_t stream) {
  if (!inited_) { set_error("context not initialised"); return -1; }
  if (in == out) { set_error("alltoall must be out of place"); return -1; }
  const bool mine = std::find(active.begin(), active.end(), rank_) != active.end();
  if (!mine || per_peer == 0) return skip_op(stream);
  const int na = (int)active.size();
  const size_t esize = dtype_size(dtype);
  if (na == 1 && !tun.force_kernel) {
    CUDA_TRY(cudaMemcpyAsync(out, in, (size_t)per_peer * esize, cudaMemcpyDeviceToDevice, stream));
    return skip_op(stream);
  }
  const int epp = epp_of(dtype);
  const long long ppacks = (per_peer + epp - 1) / epp;
  if ((size_t)ppacks * 16 * na > staging_.size) {
    set_error("alltoall: %lld bytes per peer exceed the staging window; raise staging_mb", ppacks * 16);
    return -1;
  }
  Window w{};
  for (int r = 0; r < world_; ++r) w.data[r] = (char*)staging_.peers[r];
  w.mc = (char*)staging_.mc;
  w.capacity = staging_.size;
  DevComm dc;
  if (fill_comm(active, w, &dc)) return -1;
  int blocks = (int)std::min<long long>((ppacks + kThreads - 1) / kThreads, (long long)std::min(tun.max_blocks, kMaxBlocks));
  if (blocks < 1) blocks = 1;
  if (dtype == F32) alltoall_kernel<float><<<blocks, kThreads, 0, stream>>>(dc, (const float*)in, (float*)out, per_peer);
  else if (dtype == BF16) alltoall_kernel<__nv_bfloat16><<<blocks, kThreads, 0, stream>>>(dc, (const __nv_bfloat16*)in, (__nv_bfloat16*)out, per_peer);
  else if (dtype == F16) alltoall_kernel<__half><<<blocks, kThreads, 0, stream>>>(dc, (const __half*)in, (__half*)out, per_peer);
  else { set_error("alltoall: bad dtype %d", dtype); return -1; }
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

int CommContext::tree_collective(int prim, const void* in, void* out, long long count, int dtype, int wire,
                                 int op, long long chunk_bytes, const std::vector<int>& active,
                                 cudaStream_t stream) {
  if (!inited_) { set_error("context not initialised"); return -1; }
  if (strategy_.trees.empty()) { set_error("tree collective without a loaded strategy"); return -1; }
  if (!combo_ok(dtype, wire)) { set_error("unsupported dtype/wire %d/%d", dtype, wire); return -1; }
  if (prim != ALLREDUCE && prim != REDUCE && prim != BOARDCAST) { set_error("bad tree primitive %d", prim); return -1; }
  std::vector<bool> act(world_, false);
  for (int r : active) {
    if (r < 0 || r >= world_) { set_error("active rank %d out of range", r); return -1; }
    act[r] = true;
  }
  const int nt = (int)strategy_.trees.size();
  // roles of every rank (participants must agree everywhere), then mine
  std::vector<int> participants;
  std::vector<HostTreeRole> mine(nt);
  for (int r = 0; r < world_; ++r) {
    bool any = false;
    for (int t = 0; t < nt; ++t) {
      HostTreeRole role = tree_role(strategy_.trees[t], r, act, prim, tun.relay_mode);
      any |= role.any();
      if (r == rank_) mine[t] = role;
    }
    if (any) participants.push_back(r);
  }
  const bool me_in = std::find(participants.begin(), participants.end(), rank_) != participants.end();
  if (!me_in || count == 0) return skip_op(stream);

  const size_t esize = dtype_size(dtype);
  const int epp = epp_of(wire);
  int n_contrib = 0;
  for (int r : active) (void)r, ++n_contrib;
  const float scale = (op == AVG && n_contrib > 0) ? 1.f / (float)n_contrib : 1.f;
  const int kop = (op == MAX) ? MAX : SUM;

  // Tensors inside the symmetric heap are reduced IN PLACE (no staging pass in either direction): a rank's chunk region
  // goes own data -> partial sum (pulled by its parent) -> final result (pulled from its parent), and the flag chain
  // orders every overwrite after the last read of the previous content. Needs every rank active (a relay has no tensor
  // at that offset) and a whole number of 16-byte packs.
  Window w = resolve(in, out, (size_t)count * esize, dtype == wire);
  // (REDUCE keeps the staged path: in place it would leave partial sums in the non-root ranks' tensors)
  const bool zc = w.zero_copy && prim != REDUCE && (int)active.size() == world_ && (((size_t)count * esize) & 15) == 0 &&
                  in != nullptr;
  if (!zc) {
    w = Window{};
    for (int r = 0; r < world_; ++r) w.data[r] = (char*)staging_.peers[r];
    w.mc = (char*)staging_.mc;
    w.capacity = staging_.size;
    w.zero_copy = false;
  }
  DevComm dc;
  if (fill_comm(participants, w, &dc)) return -1;

  TreePlan plan;
  memset(&plan, 0, sizeof(plan));
  plan.n_trees = nt;
  plan.zero_copy = zc ? 1 : 0;
  plan.do_reduce = prim != BOARDCAST;
  plan.do_bcast = prim != REDUCE;
  // the API's chunk size is an upper bound; the device pipelines at a finer granularity so
  // that enough (tree, chunk) items exist to keep every CTA busy
  if (tun.tree_chunk_max_bytes >= 16 && chunk_bytes > tun.tree_chunk_max_bytes) chunk_bytes = tun.tree_chunk_max_bytes;
  if (chunk_bytes < 16) chunk_bytes = 16;
  plan.chunk_packs = chunk_bytes / 16;
  for (int t = 0; t < nt; ++t) {
    TreeRole& tr = plan.role[t];
    tr.parent = mine[t].parent;
    tr.flags = mine[t].flags;
    tr.n_children = (int)mine[t].children.size();
    if (tr.n_children > kMaxChildren) { set_error("too many children in tree %d", t); return -1; }
    for (int i = 0; i < tr.n_children; ++i) tr.children[i] = mine[t].children[i];
  }
  const long long cap_elems = zc ? count : (long long)(w.capacity / 16) * epp;
  long long done = 0;
  while (done < count) {
    const long long n = std::min(count - done, cap_elems);
    const long long npacks = (n + epp - 1) / epp;
    const long long per = (npacks + nt - 1) / nt;
    long long max_chunks = 0;
    for (int t = 0; t <= nt; ++t) plan.slice_begin[t] = std::min<long long>((long long)t * per, npacks);
    max_chunks = (per + plan.chunk_packs - 1) / plan.chunk_packs;
    const long long items = max_chunks * nt;
    // two CTAs per pipeline lane: one on the reduce side, one on the broadcast side
    int lanes = (int)std::min<long long>(items, (long long)std::min(tun.tree_blocks, kMaxBlocks) / 2);
    if (lanes < 1) lanes = 1;
    const int blocks = 2 * lanes;
    dc.op_advance = (done + n >= count) ? 1 : 0;
    if (dc.item_base + (unsigned long long)((items + lanes - 1) / lanes) >= (1ull << 24)) {
      set_error("tree collective: more than 2^24 pipeline items in one op (raise the chunk size or staging_mb)");
      return -1;
    }
    const char* pin = (const char*)in + (size_t)done * esize;
    char* pout = (char*)out + (size_t)done * esize;
    int rc = ADAPCC_DISPATCH_TYPES(dtype, wire, {
      if (kop == MAX)
        tree_collective_kernel<U, W, MAX><<<blocks, kThreads, 0, stream>>>(dc, plan, (const U*)pin, (U*)pout, n, scale);
      else
        tree_collective_kernel<U, W, SUM><<<blocks, kThreads, 0, stream>>>(dc, plan, (const U*)pin, (U*)pout, n, scale);
      CUDA_TRY(cudaGetLastError());
      count_launch();
      return 0;
    });
    if (rc) return rc;
    done += n;
    dc.item_base += (unsigned long long)((items + lanes - 1) / lanes);   // later pieces: strictly larger tokens
  }
  return 0;
}

int CommContext::tree_relay_persistent(int n_buckets, const long long* counts, const long long* chunk_bytes_in,
                                       int wire, int op, const std::vector<int>& active, cudaStream_t stream) {
  if (!inited_) { set_error("context not initialised"); return -1; }
  if (strategy_.trees.empty()) { set_error("relay without a loaded strategy"); return -1; }
  if (n_buckets <= 0) return 0;
  if (std::find(active.begin(), active.end(), rank_) != active.end()) {
    set_error("tree_relay_persistent: rank %d is active; relays only", rank_);
    return -1;
  }
  std::vector<bool> act(world_, false);
  for (int r : active) {
    if (r < 0 || r >= world_) { set_error("active rank %d out of range", r); return -1; }
    act[r] = true;
  }
  const int nt = (int)strategy_.trees.size();
  const int epp = epp_of(wire);
  const long long cap_elems = (long long)(staging_.size / 16) * epp;
  bool fits = true;
  for (int i = 0; i < n_buckets; ++i) fits &= counts[i] <= cap_elems;
  std::vector<int> participants;
  std::vector<HostTreeRole> mine(nt);
  for (int r = 0; r < world_; ++r) {
    bool any = false;
    for (int t = 0; t < nt; ++t) {
      HostTreeRole role = tree_role(strategy_.trees[t], r, act, ALLREDUCE, tun.relay_mode);
      any |= role.any();
      if (r == rank_) mine[t] = role;
    }
    if (any) participants.push_back(r);
  }
  const bool me_in = std::find(participants.begin(), participants.end(), rank_) != participants.end();
  if (!me_in || !fits) {
    // nothing routes through this rank (or a bucket needs several pieces): plain per-bucket path
    for (int i = 0; i < n_buckets; ++i) {
      int rc = me_in ? tree_collective(ALLREDUCE, nullptr, nullptr, counts[i], wire, wire, op, chunk_bytes_in[i],
                                       active, stream)
                     : skip_op(stream);
      if (rc) return rc;
    }
    return 0;
  }
  std::vector<RelayWork> works(n_buckets);
  int max_lanes = 1;
  for (int i = 0; i < n_buckets; ++i) {
    RelayWork& w = works[i];
    memset(&w, 0, sizeof(w));
    TreePlan& plan = w.plan;
    plan.n_trees = nt;
    plan.do_reduce = 1;
    plan.do_bcast = 1;
    long long chunk_bytes = chunk_bytes_in[i];
    if (tun.tree_chunk_max_bytes >= 16 && chunk_bytes > tun.tree_chunk_max_bytes) chunk_bytes = tun.tree_chunk_max_bytes;
    if (chunk_bytes < 16) chunk_bytes = 16;
    plan.chunk_packs = chunk_bytes / 16;
    for (int t = 0; t < nt; ++t) {
      TreeRole& tr = plan.role[t];
      tr.parent = mine[t].parent;
      tr.flags = mine[t].flags;
      tr.n_children = (int)mine[t].children.size();
      for (int k = 0; k < tr.n_children; ++k) tr.children[k] = mine[t].children[k];
    }
    const long long n = counts[i];
    const long long npacks = (n + epp - 1) / epp;
    const long long per = (npacks + nt - 1) / nt;
    for (int t = 0; t <= nt; ++t) plan.slice_begin[t] = std::min<long long>((long long)t * per, npacks);
    const long long items = ((per + plan.chunk_packs - 1) / plan.chunk_packs) * nt;
    int lanes = (int)std::min<long long>(items, (long long)std::min(tun.tree_blocks, kMaxBlocks) / 2);
    if (lanes < 1) lanes = 1;
    w.lanes = lanes;
    w.n = n;
    w.scale = (op == AVG && !active.empty()) ? 1.f / (float)active.size() : 1.f;
    w.skip = n == 0;
    max_lanes = std::max(max_lanes, lanes);
  }
  const size_t bytes = sizeof(RelayWork) * works.size();
  if (bytes > relay_work_cap_) {
    CUDA_TRY(cudaStreamSynchronize(stream));            // (re)allocation only: first step / more buckets than before
    for (int i = 0; i < 2; ++i) {
      if (d_relay_work_[i]) cudaFree(d_relay_work_[i]);
      if (h_relay_work_[i]) cudaFreeHost(h_relay_work_[i]);
      CUDA_TRY(cudaMalloc(&d_relay_work_[i], bytes));
      CUDA_TRY(cudaMallocHost(&h_relay_work_[i], bytes));
      if (!relay_ev_[i]) CUDA_TRY(cudaEventCreateWithFlags(&relay_ev_[i], cudaEventDisableTiming));
    }
    relay_work_cap_ = bytes;
  }
  // asynchronous upload through a pinned slot; a slot is rewritten only after the copy issued from it two steps ago
  // has executed (the event wait is a no-op in steady state) — no stream synchronisation on the relay path
  const int slot = relay_slot_;
  relay_slot_ ^= 1;
  CUDA_TRY(cudaEventSynchronize(relay_ev_[slot]));
  memcpy(h_relay_work_[slot], works.data(), bytes);
  CUDA_TRY(cudaMemcpyAsync(d_relay_work_[slot], h_relay_work_[slot], bytes, cudaMemcpyHostToDevice, stream));
  CUDA_TRY(cudaEventRecord(relay_ev_[slot], stream));
  Window win{};
  for (int r = 0; r < world_; ++r) win.data[r] = (char*)staging_.peers[r];
  win.mc = (char*)staging_.mc;
  win.capacity = staging_.size;
  DevComm dc;
  if (fill_comm(participants, win, &dc)) return -1;
  const int kop = (op == MAX) ? MAX : SUM;
  const int blocks = 2 * max_lanes;
  const RelayWork* dw = static_cast<const RelayWork*>(d_relay_work_[slot]);
#define RELAY_LAUNCH(W_)                                                                              \
  do {                                                                                                \
    if (kop == MAX) tree_relay_persistent_kernel<W_, MAX><<<blocks, kThreads, 0, stream>>>(dc, dw, n_buckets); \
    else tree_relay_persistent_kernel<W_, SUM><<<blocks, kThreads, 0, stream>>>(dc, dw, n_buckets);   \
  } while (0)
  if (wire == F32) RELAY_LAUNCH(float);
  else if (wire == BF16) RELAY_LAUNCH(__nv_bfloat16);
  else if (wire == F16) RELAY_LAUNCH(__half);
  else { set_error("relay: bad wire dtype %d", wire); return -1; }
#undef RELAY_LAUNCH
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

namespace adapcc_detail { void launch_barrier(const DevComm& dc, cudaStream_t s); }

int CommContext::device_barrier(const std::vector<int>& active, cudaStream_t stream) {
  if (!inited_) { set_error("context not initialised"); return -1; }
  const bool mine = std::find(active.begin(), active.end(), rank_) != active.end();
  if (!mine || active.size() <= 1) return skip_op(stream);
  std::vector<int> act(active);
  std::sort(act.begin(), act.end());
  DevComm dc;
  Window w = resolve(nullptr, nullptr, 0, false);
  if (fill_comm(act, w, &dc)) return -1;
  adapcc_detail::launch_barrier(dc, stream);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

int CommContext::check(cudaStream_t stream) {
  CUDA_TRY(cudaStreamSynchronize(stream));
  uint32_t err = 0;
  CUDA_TRY(cudaMemcpy(&err, d_state_ + kStateErr, sizeof(err), cudaMemcpyDeviceToHost));
  if (err) {
    CUDA_TRY(cudaMemset(d_state_ + kStateErr, 0, sizeof(err)));
    set_error("device-side wait timed out (code %u): a peer did not arrive within %lld ms", err,
              tun.timeout_ms);
    return (int)err;
  }
  return 0;
}

}  // namespace adapcc
