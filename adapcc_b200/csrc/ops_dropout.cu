// Stand-alone dropout y = mask * scale * x with the mask of dropout.cuh: what the unfused paths use (fp32 parameters,
// widths the fused add-LayerNorm does not take, the multiple-choice head's summary input). Out of place; the backward is
// the same launch on dY, since the mask is recomputed from (seed, step, site, row, column) rather than stored.
#include <cuda_bf16.h>

#include "common.h"
#include "device_prims.cuh"
#include "dropout.cuh"

namespace adapcc {

// one thread per 8 consecutive columns of a row (one Philox call); cols % 8 == 0
template <typename T>
__global__ void __launch_bounds__(256)
dropout_kernel(const T* __restrict__ x, T* __restrict__ y, int rows, int nvec, const DropArgs drop) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)rows * nvec) return;
  const int row = (int)(i / nvec), vec = (int)(i - (long long)row * nvec);
  const uint32_t keep = drop_keep8(row, vec, drop, drop_key(drop));
  float f[8];
  if constexpr (sizeof(T) == 2) {
    unpack<__nv_bfloat16>(ld16(reinterpret_cast<const uint4*>(x) + i), f);
    drop_apply(f, keep, drop.scale);
    st16(reinterpret_cast<uint4*>(y) + i, pack<__nv_bfloat16>(f));
  } else {
    const float4 a = reinterpret_cast<const float4*>(x)[2 * i], b = reinterpret_cast<const float4*>(x)[2 * i + 1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
    f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    drop_apply(f, keep, drop.scale);
    reinterpret_cast<float4*>(y)[2 * i] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4*>(y)[2 * i + 1] = make_float4(f[4], f[5], f[6], f[7]);
  }
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

// x, y: contiguous [rows, cols] bf16 (dtype_bytes 2) or fp32 (4), 16-byte aligned, cols % 8 == 0;
// seed int64 [1] and step int32 [1] on the device
int adapcc_dropout(const void* x, void* y, int rows, int cols, int dtype_bytes, const void* seed, const void* step,
                   int site, unsigned int thr, float scale, void* stream) {
  if (rows <= 0 || cols <= 0) return 0;
  if (cols % 8 != 0 || (dtype_bytes != 2 && dtype_bytes != 4)) { set_error("dropout: cols %% 8 == 0, bf16 or fp32"); return -1; }
  if (((uintptr_t)x | (uintptr_t)y) & 15) { set_error("dropout: x / y must be 16-byte aligned"); return -1; }
  DropArgs d;
  if (!drop_args("dropout", seed, step, site, thr, scale, &d)) return -1;
  const int nvec = cols / 8;
  const long long total = (long long)rows * nvec;
  const unsigned grid = (unsigned)((total + 255) / 256);
  if (dtype_bytes == 2)
    dropout_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, rows, nvec, d);
  else
    dropout_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)x, (float*)y, rows, nvec, d);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
