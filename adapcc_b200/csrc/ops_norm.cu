// Fused LayerNorm forward / backward and column-sum (bias-gradient) kernels for the transformer
// workloads (GPT-2, ViT). The reference trains stock HF / vit-pytorch modules
// (/root/reference/models/gpt2/train_gpt2_ddp.py:157-159, models/vit/train_vit.py:30-40), whose eager
// LayerNorm backward (GammaBetaBackward + grad_input kernels) and bias-gradient reductions are
// separate multi-pass kernels. These kernels are memory-bound single-pass replacements:
//   ln_fwd : one warp per row, row held in registers (D = 256*VPL, VPL<=4), writes y, mean, rstd
//   ln_bwd : one warp per row for dx; per-lane fp32 accumulators for dgamma/dbeta, reduced per CTA
//            into a [grid, D] partial buffer, finalised by colsum_finalize
//   colsum : column sums of a [rows, cols] bf16 matrix in fp32 (bias gradients), two-stage
#include <cuda_bf16.h>

#include <algorithm>

#include "common.h"
#include "device_prims.cuh"
#include "dropout.cuh"

namespace adapcc {

constexpr int kLnWarps = 8;   // warps (rows in flight) per CTA

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// lane l owns vectors l, l+32, ... (VPL of them), each 8 bf16.
// RES: the row is x + res (the transformer's residual add); the bf16-rounded sum is written to
// `sum_out` (the new residual stream) and normalised in the same pass, so the separate add kernel
// and its re-read disappear.
// DROP (with RES): the row is x + drop(res), the dropout of a transformer's residual branch (dropout.cuh): res is
// masked and scaled in fp32 as it is read, the mask being recomputed from (seed, step, site, row, vector).
template <int VPL, bool RES, bool DROP = false>
__global__ void __launch_bounds__(kLnWarps * 32, VPL <= 3 ? 3 : 2)
ln_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
              const __nv_bfloat16* __restrict__ gamma, const __nv_bfloat16* __restrict__ beta,
              __nv_bfloat16* __restrict__ sum_out, __nv_bfloat16* __restrict__ y, float* __restrict__ mean,
              float* __restrict__ rstd, int rows, float eps, const DropArgs drop) {
  static_assert(RES || !DROP, "dropout acts on the residual branch");
  constexpr int D = VPL * 256;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  DropKey dkey{};
  if constexpr (DROP) dkey = drop_key(drop);
  uint4 gp[VPL], bp[VPL];                       // packed; unpacked at use (registers buy occupancy here)
#pragma unroll
  for (int v = 0; v < VPL; ++v) {
    gp[v] = reinterpret_cast<const uint4*>(gamma)[lane + 32 * v];
    bp[v] = reinterpret_cast<const uint4*>(beta)[lane + 32 * v];
  }
  for (int r = blockIdx.x * kLnWarps + warp; r < rows; r += gridDim.x * kLnWarps) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)r * D);
    float f[VPL][8];
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      unpack<__nv_bfloat16>(ld16(xr + lane + 32 * v), f[v]);
      if constexpr (RES) {
        float fr[8];
        unpack<__nv_bfloat16>(ld16(reinterpret_cast<const uint4*>(res + (size_t)r * D) + lane + 32 * v), fr);
        if constexpr (DROP) drop_apply(fr, drop_keep8(r, lane + 32 * v, drop, dkey), drop.scale);
#pragma unroll
        for (int i = 0; i < 8; ++i) f[v][i] += fr[i];
        const uint4 packed = pack<__nv_bfloat16>(f[v]);      // statistics are taken of the ROUNDED sum,
        st16(reinterpret_cast<uint4*>(sum_out + (size_t)r * D) + lane + 32 * v, packed);
        unpack<__nv_bfloat16>(packed, f[v]);                 // exactly what add-then-LayerNorm would see
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) s += f[v][i];
    }
    const float mu = warp_sum(s) * (1.f / D);
    float q = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
      for (int i = 0; i < 8; ++i) { const float d = f[v][i] - mu; q += d * d; }
    const float rs = rsqrtf(warp_sum(q) * (1.f / D) + eps);
    uint4* yr = reinterpret_cast<uint4*>(y + (size_t)r * D);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      float o[8], g[8], b[8];
      unpack<__nv_bfloat16>(gp[v], g);
      unpack<__nv_bfloat16>(bp[v], b);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = (f[v][i] - mu) * rs * g[i] + b[i];
      st16(yr + lane + 32 * v, pack<__nv_bfloat16>(o));
    }
    if (lane == 0) { mean[r] = mu; rstd[r] = rs; }
  }
}

// RES: dx += dres (the gradient arriving on the residual stream), fused into the same pass.
// DROP: the forward was s = x + drop(res), so the two inputs' gradients differ: dx as before, and a second output
// ddrop = mask * scale * dx (taken of the fp32 dx, rounded to bf16 once) for the dropped branch, with the forward's mask.
// A DROP instantiation is compiled on its own: which fp32 multiplies and adds become FFMAs can differ from the
// DROP = false one, so its dx / dgamma / dbeta agree with it to rounding, not bit for bit. p = 0 runs DROP = false.
template <int VPL, bool RES, bool DROP = false>
__global__ void __launch_bounds__(kLnWarps * 32, VPL <= 3 ? 2 : 1)
ln_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
              const __nv_bfloat16* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
              const __nv_bfloat16* __restrict__ dres, __nv_bfloat16* __restrict__ dx,
              float* __restrict__ part_dgamma, float* __restrict__ part_dbeta, int rows,
              __nv_bfloat16* __restrict__ ddrop, const DropArgs drop) {
  constexpr int D = VPL * 256;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // gamma stays packed (bf16x8 per register quad) and is unpacked at use: 12 instead of 24 registers
  // at D = 768, which is what lets two CTAs (16 rows in flight) share an SM
  uint4 gp[VPL];
  float dg[VPL][8], db[VPL][8];
#pragma unroll
  for (int v = 0; v < VPL; ++v) {
    gp[v] = reinterpret_cast<const uint4*>(gamma)[lane + 32 * v];
#pragma unroll
    for (int i = 0; i < 8; ++i) dg[v][i] = db[v][i] = 0.f;
  }
  for (int r = blockIdx.x * kLnWarps + warp; r < rows; r += gridDim.x * kLnWarps) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)r * D);
    const uint4* dr = reinterpret_cast<const uint4*>(dy + (size_t)r * D);
    const float mu = mean[r], rs = rstd[r];
    float xh[VPL][8], gy[VPL][8];
    float c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      float fx[8], fd[8], g[8];
      unpack<__nv_bfloat16>(ld16(xr + lane + 32 * v), fx);
      unpack<__nv_bfloat16>(ld16(dr + lane + 32 * v), fd);
      unpack<__nv_bfloat16>(gp[v], g);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        xh[v][i] = (fx[i] - mu) * rs;
        gy[v][i] = fd[i] * g[i];
        c1 += gy[v][i];
        c2 += gy[v][i] * xh[v][i];
        dg[v][i] += fd[i] * xh[v][i];
        db[v][i] += fd[i];
      }
    }
    c1 = warp_sum(c1) * (1.f / D);
    c2 = warp_sum(c2) * (1.f / D);
    uint4* ox = reinterpret_cast<uint4*>(dx + (size_t)r * D);
    DropKey dkey{};                               // read per row: held across the loop it would cost the registers
    if constexpr (DROP) dkey = drop_key(drop);    // that keep two CTAs on an SM at D = 768
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = rs * (gy[v][i] - c1 - xh[v][i] * c2);
      if constexpr (RES) {
        float fr[8];
        unpack<__nv_bfloat16>(ld16(reinterpret_cast<const uint4*>(dres + (size_t)r * D) + lane + 32 * v), fr);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] += fr[i];
      }
      st16(ox + lane + 32 * v, pack<__nv_bfloat16>(o));
      if constexpr (DROP) {
        drop_apply(o, drop_keep8(r, lane + 32 * v, drop, dkey), drop.scale);
        st16(reinterpret_cast<uint4*>(ddrop + (size_t)r * D) + lane + 32 * v, pack<__nv_bfloat16>(o));
      }
    }
  }
  // CTA reduction of the per-warp column accumulators -> one partial row per CTA
  __shared__ float sm[kLnWarps][D];
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
      for (int i = 0; i < 8; ++i) sm[warp][(lane + 32 * v) * 8 + i] = pass == 0 ? dg[v][i] : db[v][i];
    __syncthreads();
    float* out = (pass == 0 ? part_dgamma : part_dbeta) + (size_t)blockIdx.x * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < kLnWarps; ++w) s += sm[w][c];
      out[c] = s;
    }
    __syncthreads();
  }
}

// out[c] (bf16 or fp32) = sum_p part[p][c]. Block = 32 columns x 32 row lanes: every row lane sums
// a strided subset of the partial rows (128-byte coalesced row segments), then the 32 lanes are
// combined through shared memory (one thread per column walking all partial rows leaves most of the
// memory bandwidth unused).
template <typename O>
__global__ void __launch_bounds__(1024)
colsum_finalize_kernel(const float* __restrict__ part, int nparts, int cols, O* __restrict__ out) {
  __shared__ float sm[32][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  if (c < cols)
    for (int p = threadIdx.y; p < nparts; p += 32) s += part[(size_t)p * cols + c];
  sm[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 32; ++r) t += sm[r][threadIdx.x];
    out[c] = from_float<O>(t);
  }
}

// Two independent reductions of the same shape in one launch (LayerNorm's dgamma and dbeta):
// blockIdx.y picks the pair. These kernels are ~2.5 us of pure launch latency each, 50 per GPT-2 step.
template <typename O>
__global__ void __launch_bounds__(1024)
colsum_finalize_pair_kernel(const float* __restrict__ part_a, const float* __restrict__ part_b, int nparts, int cols,
                            O* __restrict__ out_a, O* __restrict__ out_b) {
  __shared__ float sm[32][33];
  const float* part = blockIdx.y == 0 ? part_a : part_b;
  O* out = blockIdx.y == 0 ? out_a : out_b;
  const int c = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  if (c < cols)
    for (int p = threadIdx.y; p < nparts; p += 32) s += part[(size_t)p * cols + c];
  sm[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 32; ++r) t += sm[r][threadIdx.x];
    out[c] = from_float<O>(t);
  }
}

// partial column sums: grid (col tiles of 256 columns, row splits); thread handles 8 columns x
// a strided set of rows; 32 row-groups per CTA combine through shared memory.
__global__ void __launch_bounds__(256)
colsum_partial_kernel(const __nv_bfloat16* __restrict__ a, int rows, int cols, float* __restrict__ part) {
  // blockDim = (32 vectors of 8 cols, 8 row lanes)
  const int vcol = blockIdx.x * 32 + threadIdx.x;          // vector column index
  const int nvec = cols / 8;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  if (vcol < nvec) {
    for (int r = blockIdx.y * 8 + threadIdx.y; r < rows; r += gridDim.y * 8) {
      float f[8];
      unpack<__nv_bfloat16>(ld16(reinterpret_cast<const uint4*>(a + (size_t)r * cols) + vcol), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += f[i];
    }
  }
  __shared__ float sm[8][32][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) sm[threadIdx.y][threadIdx.x][i] = acc[i];
  __syncthreads();
  if (threadIdx.y == 0 && vcol < nvec) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += sm[w][threadIdx.x][i];
      part[(size_t)blockIdx.y * cols + vcol * 8 + i] = s;
    }
  }
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// SMs of the current device (132 on an H100 SXM), read once.
static int sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
      (void)cudaGetLastError();
      sms = 132;
    }
  }
  return sms;
}

// Persistent grid: at most `per_sm` CTAs per SM (what the launch bounds make resident), shrunk so that
// every CTA runs the same number of row-group iterations (8192 rows, 396 slots on 132 SMs -> 342 CTAs x 3).
static int ln_grid(int rows, int per_sm) {
  const int groups = std::max(1, (rows + kLnWarps - 1) / kLnWarps);
  const int cap = sm_count() * per_sm;
  const int iters = (groups + cap - 1) / cap;
  return (groups + iters - 1) / iters;
}
static int ln_fwd_ctas_per_sm(int d) { return d <= 768 ? 3 : 2; }   // = the kernels' __launch_bounds__
static int ln_bwd_ctas_per_sm(int d) { return d <= 768 ? 2 : 1; }
int adapcc_ln_partials(int rows) { return ln_grid(rows, 2); }       // upper bound of the backward grid

// y = LayerNorm(x [+ res]); when res != nullptr the bf16 sum x + res is also written to sum_out.
// drop (with res): the sum is x + drop(res).
static int ln_fwd_launch(const void* x, const void* res, const void* gamma, const void* beta, void* sum_out, void* y,
                         float* mean, float* rstd, int rows, int d, float eps, void* stream,
                         const DropArgs* drop = nullptr) {
  cudaStream_t s = (cudaStream_t)stream;
  if (rows <= 0) return 0;
  const int grid = ln_grid(rows, ln_fwd_ctas_per_sm(d));
#define LN_FWD(V)                                                                                                  \
  do {                                                                                                             \
    if (drop)                                                                                                      \
      ln_fwd_kernel<V, true, true><<<grid, kLnWarps * 32, 0, s>>>((const __nv_bfloat16*)x,                         \
          (const __nv_bfloat16*)res, (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta,                      \
          (__nv_bfloat16*)sum_out, (__nv_bfloat16*)y, mean, rstd, rows, eps, *drop);                               \
    else if (res)                                                                                                  \
      ln_fwd_kernel<V, true><<<grid, kLnWarps * 32, 0, s>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)res,    \
          (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta, (__nv_bfloat16*)sum_out, (__nv_bfloat16*)y,     \
          mean, rstd, rows, eps, DropArgs{});                                                                      \
    else                                                                                                           \
      ln_fwd_kernel<V, false><<<grid, kLnWarps * 32, 0, s>>>((const __nv_bfloat16*)x, nullptr,                     \
          (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta, nullptr, (__nv_bfloat16*)y, mean, rstd, rows,   \
          eps, DropArgs{});                                                                                        \
  } while (0)
  switch (d) {
    case 256: LN_FWD(1); break;
    case 512: LN_FWD(2); break;
    case 768: LN_FWD(3); break;
    case 1024: LN_FWD(4); break;
    default: set_error("ln_fwd: unsupported width %d (256/512/768/1024)", d); return -1;
  }
#undef LN_FWD
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

int adapcc_ln_fwd(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd, int rows,
                  int d, float eps, void* stream) {
  return ln_fwd_launch(x, nullptr, gamma, beta, nullptr, y, mean, rstd, rows, d, eps, stream);
}

int adapcc_add_ln_fwd(const void* x, const void* res, const void* gamma, const void* beta, void* sum_out, void* y,
                      float* mean, float* rstd, int rows, int d, float eps, void* stream) {
  if (!res || !sum_out) { set_error("add_ln_fwd: res and sum_out are required"); return -1; }
  return ln_fwd_launch(x, res, gamma, beta, sum_out, y, mean, rstd, rows, d, eps, stream);
}

// part: fp32 scratch of 2 * adapcc_ln_partials(rows) * d floats. dgamma/dbeta: bf16 [d].
// dres (optional, bf16 [rows, d]): gradient of the residual stream, added to dx in the same pass.
// drop (optional): ddrop (bf16 [rows, d]) = mask * scale * dx is written as well.
static int ln_bwd_launch(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd,
                         const void* dres, void* dx, void* dgamma, void* dbeta, float* part, int rows, int d,
                         void* stream, void* ddrop = nullptr, const DropArgs* drop = nullptr) {
  cudaStream_t s = (cudaStream_t)stream;
  if (rows <= 0) return 0;
  const int grid = ln_grid(rows, ln_bwd_ctas_per_sm(d));
  float* pg = part;
  float* pb = part + (size_t)grid * d;
#define LN_BWD(V)                                                                                                  \
  do {                                                                                                             \
    const __nv_bfloat16 *dy_ = (const __nv_bfloat16*)dy, *x_ = (const __nv_bfloat16*)x;                            \
    const __nv_bfloat16 *g_ = (const __nv_bfloat16*)gamma, *dr_ = (const __nv_bfloat16*)dres;                      \
    __nv_bfloat16 *dx_ = (__nv_bfloat16*)dx, *dd_ = (__nv_bfloat16*)ddrop;                                         \
    if (drop && dres)                                                                                              \
      ln_bwd_kernel<V, true, true><<<grid, kLnWarps * 32, 0, s>>>(dy_, x_, g_, mean, rstd, dr_, dx_, pg, pb, rows, \
                                                                  dd_, *drop);                                     \
    else if (drop)                                                                                                 \
      ln_bwd_kernel<V, false, true><<<grid, kLnWarps * 32, 0, s>>>(dy_, x_, g_, mean, rstd, nullptr, dx_, pg, pb,  \
                                                                   rows, dd_, *drop);                              \
    else if (dres)                                                                                                 \
      ln_bwd_kernel<V, true><<<grid, kLnWarps * 32, 0, s>>>(dy_, x_, g_, mean, rstd, dr_, dx_, pg, pb, rows,       \
                                                            nullptr, DropArgs{});                                  \
    else                                                                                                           \
      ln_bwd_kernel<V, false><<<grid, kLnWarps * 32, 0, s>>>(dy_, x_, g_, mean, rstd, nullptr, dx_, pg, pb, rows,  \
                                                             nullptr, DropArgs{});                                 \
  } while (0)
  switch (d) {
    case 256: LN_BWD(1); break;
    case 512: LN_BWD(2); break;
    case 768: LN_BWD(3); break;
    case 1024: LN_BWD(4); break;
    default: set_error("ln_bwd: unsupported width %d (256/512/768/1024)", d); return -1;
  }
#undef LN_BWD
  CUDA_TRY(cudaGetLastError());
  colsum_finalize_pair_kernel<__nv_bfloat16><<<dim3((d + 31) / 32, 2), dim3(32, 32), 0, s>>>(
      pg, pb, grid, d, (__nv_bfloat16*)dgamma, (__nv_bfloat16*)dbeta);
  CUDA_TRY(cudaGetLastError());
  count_launch(2);
  return 0;
}

int adapcc_ln_bwd(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd, void* dx,
                  void* dgamma, void* dbeta, float* part, int rows, int d, void* stream) {
  return ln_bwd_launch(dy, x, gamma, mean, rstd, nullptr, dx, dgamma, dbeta, part, rows, d, stream);
}

int adapcc_add_ln_bwd(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd,
                      const void* dres, void* dx, void* dgamma, void* dbeta, float* part, int rows, int d,
                      void* stream) {
  return ln_bwd_launch(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, part, rows, d, stream);
}

// The residual branch under dropout (dropout.cuh): seed int64 [1] and step int32 [1] on the device, site / thr / scale
// of the definition. thr == 0 (p = 0) keeps everything with scale 1: the bits of adapcc_add_ln_fwd / _bwd.
// sum_out = x + drop(res), y = LayerNorm(sum_out)
int adapcc_add_ln_drop_fwd(const void* x, const void* res, const void* gamma, const void* beta, void* sum_out, void* y,
                           float* mean, float* rstd, int rows, int d, float eps, const void* seed, const void* step,
                           int site, unsigned int thr, float scale, void* stream) {
  DropArgs a;
  if (!res || !sum_out) { set_error("add_ln_drop_fwd: res and sum_out are required"); return -1; }
  if (!drop_args("add_ln_drop_fwd", seed, step, site, thr, scale, &a)) return -1;
  return ln_fwd_launch(x, res, gamma, beta, sum_out, y, mean, rstd, rows, d, eps, stream, &a);
}

// dx = LayerNorm backward [+ dsum], ddrop = mask * scale * dx: the gradients of x and of res
int adapcc_add_ln_drop_bwd(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd,
                           const void* dsum, void* dx, void* ddrop, void* dgamma, void* dbeta, float* part, int rows,
                           int d, const void* seed, const void* step, int site, unsigned int thr, float scale,
                           void* stream) {
  DropArgs a;
  if (!ddrop) { set_error("add_ln_drop_bwd: ddrop is required"); return -1; }
  if (!drop_args("add_ln_drop_bwd", seed, step, site, thr, scale, &a)) return -1;
  return ln_bwd_launch(dy, x, gamma, mean, rstd, dsum, dx, dgamma, dbeta, part, rows, d, stream, ddrop, &a);
}

int adapcc_colsum_splits(int rows) { return std::max(1, std::min(64, rows / 64)); }

// out (bf16 [cols]) = column sums of a (bf16 [rows, cols]); part: fp32 scratch [splits, cols].
int adapcc_colsum(const void* a, int rows, int cols, void* out, float* part, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (cols % 8 != 0) { set_error("colsum: cols must be a multiple of 8"); return -1; }
  if (rows <= 0) return 0;
  const int splits = adapcc_colsum_splits(rows);
  dim3 grid((cols / 8 + 31) / 32, splits), block(32, 8);
  colsum_partial_kernel<<<grid, block, 0, s>>>((const __nv_bfloat16*)a, rows, cols, part);
  colsum_finalize_kernel<__nv_bfloat16><<<(cols + 31) / 32, dim3(32, 32), 0, s>>>(part, splits, cols, (__nv_bfloat16*)out);
  CUDA_TRY(cudaGetLastError());
  count_launch(2);
  return 0;
}

}  // extern "C"
