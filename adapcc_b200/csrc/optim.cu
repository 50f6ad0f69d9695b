// Fused optimizer kernels for the flat-buffer data-parallel engine (adapcc_b200/parallel/engine.py).
//
// The reference's workloads step torch/apex optimizers parameter by parameter after a blocking
// gradient hook (/root/reference/train_ddp.py:37-54, /root/reference/models/gpt2/train_gpt2_ddp.py:160-195:
// AdamW + clip_grad_norm_ 1.0). With all parameters and (all-reduced) gradients living in two flat
// buffers the whole update is two launches: a sum-of-squares reduction (global grad norm, no host
// sync) and one AdamW pass that applies the clip coefficient, updates fp32 master / m / v and
// writes the bf16 parameters back — memory bound, 128-bit accesses, graph capturable. With gradient accumulation two
// more passes per bucket, both launched from the engine's bucket-ready events: accumulate a micro-batch's gradient into
// an fp32 buffer, and fold the last one in with the 1/M mean before the bucket's collective.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "common.h"

namespace adapcc {

template <typename T> __device__ __forceinline__ float ldf(const T* p, long long i);
template <> __device__ __forceinline__ float ldf<float>(const float* p, long long i) { return p[i]; }
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p, long long i) { return __bfloat162float(p[i]); }

// ---- sum of squares ---------------------------------------------------------------------------
// DETERMINISTIC: every block writes its partial sum to a slot, the last block to finish adds the slots in index order
// and does ONE read-modify-write of `out`. (A float atomicAdd per block made the grad norm — and through the clip
// coefficient every parameter — depend on block scheduling: data-parallel replicas drifted apart by one bf16 ulp on
// ~1e-6 of the elements per step although their gradients were bit-identical; found with tools/replica_debug_worker.py.)
constexpr int kSumsqMaxBlocks = 592;
__device__ float g_sumsq_partials[kSumsqMaxBlocks];
__device__ unsigned int g_sumsq_ticket = 0;

template <typename T>
__global__ void __launch_bounds__(512) sumsq_kernel(const T* __restrict__ g, long long n, float* __restrict__ out) {
  constexpr int kVec = 16 / sizeof(T);
  float acc = 0.f;
  const long long nv = n / kVec;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const uint4* gv = reinterpret_cast<const uint4*>(g);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += stride) {
    uint4 q = gv[i];
    const T* e = reinterpret_cast<const T*>(&q);
#pragma unroll
    for (int k = 0; k < kVec; ++k) { float f = ldf<T>(e, k); acc += f * f; }
  }
  if (blockIdx.x == 0)
    for (long long i = nv * kVec + threadIdx.x; i < n; i += blockDim.x) { float f = ldf<T>(g, i); acc += f * f; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float warp_sum[16];
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? warp_sum[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) {
      g_sumsq_partials[blockIdx.x] = v;
      __threadfence();
      const unsigned int t = atomicAdd(&g_sumsq_ticket, 1u);
      if (t == gridDim.x - 1) {                       // last block: fixed-order total
        __threadfence();
        float total = 0.f;
        for (unsigned int b = 0; b < gridDim.x; ++b) total += *((volatile float*)&g_sumsq_partials[b]);
        *out += total;                                // launches of one stream are serialised: a plain RMW is enough
        g_sumsq_ticket = 0;
      }
    }
  }
}

// ---- fused AdamW --------------------------------------------------------------------------------
// G: gradient dtype, P: parameter dtype (bf16 params keep an fp32 master copy).
struct AdamArgs {
  float lr, beta1, beta2, eps, weight_decay;
  float bias1, bias2;          // 1 - beta^t
  float max_norm;              // <= 0: no clipping
  float grad_scale;            // extra multiplier on gradients (e.g. 1/accumulation steps)
};

template <typename P, typename G>
__global__ void __launch_bounds__(512)
adamw_kernel(P* __restrict__ param, const G* __restrict__ grad, float* __restrict__ master, float* __restrict__ m,
             float* __restrict__ v, long long n, AdamArgs a, const float* __restrict__ sumsq,
             const int* __restrict__ step_ptr, const float* __restrict__ lr_ptr) {
  if (lr_ptr != nullptr) a.lr = *lr_ptr;   // device-resident learning rate: schedules work under CUDA-graph replay
  if (step_ptr != nullptr) {   // device-resident step counter: keeps the launch CUDA-graph replayable
    const float t = (float)(*step_ptr);
    a.bias1 = 1.f - powf(a.beta1, t);
    a.bias2 = 1.f - powf(a.beta2, t);
  }
  float coef = a.grad_scale;
  if (a.max_norm > 0.f && sumsq != nullptr) {
    const float norm = sqrtf(*sumsq) * a.grad_scale;
    coef *= fminf(1.f, a.max_norm / (norm + 1e-6f));
  }
  const long long stride = (long long)gridDim.x * blockDim.x;
  constexpr int kV = 4;
  const long long nv = n / kV;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += stride) {
    const long long e0 = i * kV;
    float4 w = *reinterpret_cast<const float4*>(master + e0);
    float4 mm = *reinterpret_cast<const float4*>(m + e0);
    float4 vv = *reinterpret_cast<const float4*>(v + e0);
    float g[kV];
#pragma unroll
    for (int k = 0; k < kV; ++k) g[k] = ldf<G>(grad, e0 + k) * coef;
    float* wp = &w.x; float* mp = &mm.x; float* vp = &vv.x;
#pragma unroll
    for (int k = 0; k < kV; ++k) {
      mp[k] = a.beta1 * mp[k] + (1.f - a.beta1) * g[k];
      vp[k] = a.beta2 * vp[k] + (1.f - a.beta2) * g[k] * g[k];
      const float mhat = mp[k] / a.bias1;
      const float vhat = vp[k] / a.bias2;
      wp[k] = wp[k] * (1.f - a.lr * a.weight_decay) - a.lr * mhat / (sqrtf(vhat) + a.eps);
    }
    *reinterpret_cast<float4*>(master + e0) = w;
    *reinterpret_cast<float4*>(m + e0) = mm;
    *reinterpret_cast<float4*>(v + e0) = vv;
    if (sizeof(P) == 2) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(w.x, w.y), hi = __floats2bfloat162_rn(w.z, w.w);
      uint2 pk = make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(param) + e0) = pk;
    } else {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(param) + e0) = w;
    }
  }
  if (blockIdx.x == 0) {
    for (long long e = nv * kV + threadIdx.x; e < n; e += blockDim.x) {
      const float gg = ldf<G>(grad, e) * coef;
      float mm = a.beta1 * m[e] + (1.f - a.beta1) * gg;
      float vv = a.beta2 * v[e] + (1.f - a.beta2) * gg * gg;
      float w = master[e] * (1.f - a.lr * a.weight_decay) - a.lr * (mm / a.bias1) / (sqrtf(vv / a.bias2) + a.eps);
      m[e] = mm; v[e] = vv; master[e] = w;
      if (sizeof(P) == 2) reinterpret_cast<__nv_bfloat16*>(param)[e] = __float2bfloat16_rn(w);
      else reinterpret_cast<float*>(param)[e] = w;
    }
  }
}

// plain SGD (the reference's VGG16 template uses optim.SGD(lr=0.001), train_ddp.py:37)
template <typename P, typename G>
__global__ void __launch_bounds__(512)
sgd_kernel(P* __restrict__ param, const G* __restrict__ grad, float* __restrict__ master, long long n, float lr,
           float grad_scale) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
    const float w = master[e] - lr * ldf<G>(grad, e) * grad_scale;
    master[e] = w;
    if (sizeof(P) == 2) reinterpret_cast<__nv_bfloat16*>(param)[e] = __float2bfloat16_rn(w);
    else reinterpret_cast<float*>(param)[e] = w;
  }
}

// ---- gradient accumulation over micro-batches ---------------------------------------------------------------------
// The engine's fp32 accumulator acc of the micro-batch gradients g_1..g_M (bf16 or fp32, whatever the flat buffer
// holds): acc = f32(g_1), acc = f32(acc + f32(g_m)), and on the last micro-batch g = round(f32(f32(acc + f32(g_M)) *
// scale)) with scale = f32(1/M). Every add and multiply is rounded on its own (__fadd_rn / __fmul_rn: never contracted
// into an FMA), so the result is the same bits as that definition in torch. One thread per 8 elements per iteration:
// 16-byte loads and stores, no atomics. n % 8 == 0 and 16-byte aligned pointers (checked by the entry points).
template <typename T> struct Vec8;
template <> struct Vec8<__nv_bfloat16> {
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, long long i, float (&f)[8]) {
    const uint4 q = reinterpret_cast<const uint4*>(p)[i];
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
    for (int k = 0; k < 4; ++k) { const float2 t = __bfloat1622float2(h[k]); f[2 * k] = t.x; f[2 * k + 1] = t.y; }
  }
  static __device__ __forceinline__ void store(__nv_bfloat16* p, long long i, const float (&f)[8]) {
    uint4 q;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&q);
#pragma unroll
    for (int k = 0; k < 4; ++k) h[k] = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
    reinterpret_cast<uint4*>(p)[i] = q;
  }
};
template <> struct Vec8<float> {
  static __device__ __forceinline__ void load(const float* p, long long i, float (&f)[8]) {
    const float4 a = reinterpret_cast<const float4*>(p)[2 * i], b = reinterpret_cast<const float4*>(p)[2 * i + 1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
  static __device__ __forceinline__ void store(float* p, long long i, const float (&f)[8]) {
    reinterpret_cast<float4*>(p)[2 * i] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4*>(p)[2 * i + 1] = make_float4(f[4], f[5], f[6], f[7]);
  }
};

// acc = f32(g) (FIRST) or acc = acc + f32(g)
template <typename T, bool FIRST>
__global__ void __launch_bounds__(256) grad_accum_kernel(const T* __restrict__ g, float* __restrict__ acc, long long nv) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += stride) {
    float f[8];
    Vec8<T>::load(g, i, f);
    if (!FIRST) {
      float a[8];
      Vec8<float>::load(acc, i, a);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] = __fadd_rn(a[k], f[k]);
    }
    Vec8<float>::store(acc, i, f);
  }
}

// g = round(f32(acc + f32(g)) * scale)
template <typename T>
__global__ void __launch_bounds__(256) grad_fold_kernel(T* __restrict__ g, const float* __restrict__ acc, long long nv,
                                                        float scale) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += stride) {
    float f[8], a[8];
    Vec8<T>::load(g, i, f);
    Vec8<float>::load(acc, i, a);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = __fmul_rn(__fadd_rn(a[k], f[k]), scale);
    Vec8<T>::store(g, i, f);
  }
}

// blocks of 256 threads for n / 8 vectors: at most 8 resident blocks on each of the H100's 132 SMs
inline unsigned grad_accum_grid(long long n) { return (unsigned)std::min<long long>(132 * 8, (n / 8 + 255) / 256); }

inline bool grad_accum_args(const char* who, const void* g, const float* acc, long long n, int dtype) {
  if (dtype != BF16 && dtype != F32) { set_error("%s: gradient dtype must be bf16 or fp32, got %d", who, dtype); return false; }
  if (n % 8 != 0) { set_error("%s: n = %lld must be a multiple of 8", who, n); return false; }
  if ((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(acc)) & 15) {
    set_error("%s: gradient and accumulator must be 16-byte aligned", who);
    return false;
  }
  return true;
}

}  // namespace adapcc

using namespace adapcc;

extern "C" {

int adapcc_fused_adamw_lr(void* param, const void* grad, float* master, float* m, float* v, long long n,
                          int param_dtype, int grad_dtype, float lr, float beta1, float beta2, float eps,
                          float weight_decay, int step, float max_norm, float grad_scale, const float* sumsq,
                          const int* step_ptr, const float* lr_ptr, void* stream);

// out must be zeroed by the caller (cudaMemsetAsync on the same stream); accumulates.
int adapcc_sumsq(const void* g, long long n, int dtype, float* out, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (n <= 0) return 0;
  if (reinterpret_cast<uintptr_t>(g) & 15) { set_error("sumsq: pointer must be 16-byte aligned"); return -1; }
  int blocks = (int)std::min<long long>(kSumsqMaxBlocks, (n / 8 + 511) / 512);
  if (blocks < 1) blocks = 1;
  if (dtype == F32) sumsq_kernel<float><<<blocks, 512, 0, s>>>((const float*)g, n, out);
  else if (dtype == BF16) sumsq_kernel<__nv_bfloat16><<<blocks, 512, 0, s>>>((const __nv_bfloat16*)g, n, out);
  else { set_error("sumsq: unsupported dtype %d", dtype); return -1; }
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// param dtype / grad dtype in {F32, BF16}. master/m/v are fp32 (master may alias param when fp32).
int adapcc_fused_adamw(void* param, const void* grad, float* master, float* m, float* v, long long n,
                       int param_dtype, int grad_dtype, float lr, float beta1, float beta2, float eps,
                       float weight_decay, int step, float max_norm, float grad_scale, const float* sumsq,
                       const int* step_ptr, void* stream) {
  return adapcc_fused_adamw_lr(param, grad, master, m, v, n, param_dtype, grad_dtype, lr, beta1, beta2, eps, weight_decay,
                               step, max_norm, grad_scale, sumsq, step_ptr, nullptr, stream);
}

// Same, with an optional device-resident learning rate (lr_ptr != NULL overrides `lr`).
int adapcc_fused_adamw_lr(void* param, const void* grad, float* master, float* m, float* v, long long n,
                          int param_dtype, int grad_dtype, float lr, float beta1, float beta2, float eps,
                          float weight_decay, int step, float max_norm, float grad_scale, const float* sumsq,
                          const int* step_ptr, const float* lr_ptr, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (n <= 0) return 0;
  if ((reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(master) |
       reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) {
    set_error("adamw: buffers must be 16-byte aligned");
    return -1;
  }
  AdamArgs a;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.weight_decay = weight_decay;
  a.bias1 = 1.f - powf(beta1, (float)step);
  a.bias2 = 1.f - powf(beta2, (float)step);
  a.max_norm = max_norm; a.grad_scale = grad_scale;
  int blocks = (int)std::min<long long>(1184, (n / 4 + 511) / 512);
  if (blocks < 1) blocks = 1;
  if (param_dtype == BF16 && grad_dtype == BF16)
    adamw_kernel<__nv_bfloat16, __nv_bfloat16><<<blocks, 512, 0, s>>>((__nv_bfloat16*)param, (const __nv_bfloat16*)grad, master, m, v, n, a, sumsq, step_ptr, lr_ptr);
  else if (param_dtype == F32 && grad_dtype == F32)
    adamw_kernel<float, float><<<blocks, 512, 0, s>>>((float*)param, (const float*)grad, master, m, v, n, a, sumsq, step_ptr, lr_ptr);
  else if (param_dtype == BF16 && grad_dtype == F32)
    adamw_kernel<__nv_bfloat16, float><<<blocks, 512, 0, s>>>((__nv_bfloat16*)param, (const float*)grad, master, m, v, n, a, sumsq, step_ptr, lr_ptr);
  else if (param_dtype == F32 && grad_dtype == BF16)
    adamw_kernel<float, __nv_bfloat16><<<blocks, 512, 0, s>>>((float*)param, (const __nv_bfloat16*)grad, master, m, v, n, a, sumsq, step_ptr, lr_ptr);
  else { set_error("adamw: unsupported dtypes %d/%d", param_dtype, grad_dtype); return -1; }
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// Micro-batch accumulate: acc = f32(g) when `first`, else acc = f32(acc + f32(g)). g: n elements of `dtype` (F32 or
// BF16), acc: n fp32; both 16-byte aligned, n % 8 == 0.
int adapcc_grad_accum(const void* g, float* acc, long long n, int dtype, int first, void* stream) {
  if (!grad_accum_args("grad_accum", g, acc, n, dtype)) return -1;
  if (n <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grad_accum_grid(n);
  if (dtype == BF16) {
    if (first) grad_accum_kernel<__nv_bfloat16, true><<<grid, 256, 0, s>>>((const __nv_bfloat16*)g, acc, n / 8);
    else grad_accum_kernel<__nv_bfloat16, false><<<grid, 256, 0, s>>>((const __nv_bfloat16*)g, acc, n / 8);
  } else {
    if (first) grad_accum_kernel<float, true><<<grid, 256, 0, s>>>((const float*)g, acc, n / 8);
    else grad_accum_kernel<float, false><<<grid, 256, 0, s>>>((const float*)g, acc, n / 8);
  }
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

// Last micro-batch: g = round(f32(f32(acc + f32(g)) * scale)), in place; scale is 1/M.
int adapcc_grad_fold(void* g, const float* acc, long long n, int dtype, float scale, void* stream) {
  if (!grad_accum_args("grad_fold", g, acc, n, dtype)) return -1;
  if (n <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grad_accum_grid(n);
  if (dtype == BF16) grad_fold_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((__nv_bfloat16*)g, acc, n / 8, scale);
  else grad_fold_kernel<float><<<grid, 256, 0, s>>>((float*)g, acc, n / 8, scale);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

__global__ void incr_int_kernel(int* p) { if (threadIdx.x == 0 && blockIdx.x == 0) *p += 1; }

int adapcc_incr_int(int* p, void* stream) {
  incr_int_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(p);
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

int adapcc_fused_sgd(void* param, const void* grad, float* master, long long n, int param_dtype, int grad_dtype,
                     float lr, float grad_scale, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (n <= 0) return 0;
  int blocks = (int)std::min<long long>(1184, (n + 511) / 512);
  if (param_dtype == BF16 && grad_dtype == BF16)
    sgd_kernel<__nv_bfloat16, __nv_bfloat16><<<blocks, 512, 0, s>>>((__nv_bfloat16*)param, (const __nv_bfloat16*)grad, master, n, lr, grad_scale);
  else if (param_dtype == F32 && grad_dtype == F32)
    sgd_kernel<float, float><<<blocks, 512, 0, s>>>((float*)param, (const float*)grad, master, n, lr, grad_scale);
  else { set_error("sgd: unsupported dtypes %d/%d", param_dtype, grad_dtype); return -1; }
  CUDA_TRY(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
