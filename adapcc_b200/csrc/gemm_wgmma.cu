// Hopper GEMM with a fused epilogue: TMA -> mbarrier ring -> wgmma, accumulator in registers.
//
//   out[M, N] = act(A[M, K] . W[N, K]^T + bias[N])          bf16 in / out, fp32 accumulation
//   ACT 0: identity          1: GELU(tanh)       (both optionally also write pre = A.W^T + bias, for the backward)
//       2: dGELU: out = (A.W^T) * gelu'(aux) — the MLP backward dH = (dY.W2) (.) gelu'(pre) — and, optionally,
//          colsum[N] += column sums of `out` (the bias gradient of the up-projection, accumulated in fp32). The sums
//          are deterministic: every CTA writes its tile's column sums (its 8 warps added in a fixed order) to row
//          `m_blk` of an fp32 [tiles_m, N] work buffer, and a second kernel adds the rows in ascending order.
//       3: residual: out = A.W^T + bias + aux    (projection + residual add)
//   For ACT >= 2 the `pre` argument is an INPUT (aux, same shape as out).
//
// The bias and the activation are applied to the accumulator registers before anything goes to HBM: a GEMM + bias
// followed by a stand-alone GELU kernel writes the [M, N] tensor, reads it back and writes it again.
//
// One CTA = 384 threads, a 128 x BN output tile at a time (BN = 256 when N % 256 == 0, else 128):
//   warpgroup 0, one thread : TMA producer — cp.async.bulk.tensor.2d of the A (128 x 64) and W (BN x 64) K slabs,
//                             128-byte swizzled, into a ring of 4 (BN 256) or 6 (BN 128) stages; `full[s]` completes
//                             on the transferred bytes
//   warpgroups 1, 2         : 64 rows each — 4 x wgmma.m64nBNk16 per slab, one wgmma group kept in flight; a slab is
//                             released (`empty[s]`) once the group that read it has retired; then the epilogue
//                             (bias + activation in fp32, bf16 stores) straight from the accumulator registers
// Grid policies (the `variant` argument):
//   0: one tile per CTA.   1: persistent CTAs (grid = SMs) — the producer streams the next tile's slabs while the
//   consumers run the epilogue.   2 / 3: clusters of two CTAs on vertically adjacent tiles that share W: each CTA
//   loads half of the W slab and multicasts it to both (half the W traffic out of L2); `empty[s]` then counts the
//   consumers of both CTAs, because the peer's multicast writes into this CTA's stage. 2 = one pair tile per cluster,
//   3 = persistent clusters (the variant the GPT-2 MLP uses; the only one with the colsum output).
// Every mbarrier wait is bounded by wall clock (trap after 2 s instead of hanging the GPU on a protocol bug).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <mutex>

#include "common.h"

namespace adapcc {
namespace wg {

constexpr int kBM = 128;           // tile rows: two consumer warpgroups x wgmma M = 64
constexpr int kBK = 64;            // K slab: 64 bf16 = 128 B = one swizzle-128B row
constexpr int kMmaK = 16;          // K per wgmma for 16-bit inputs
constexpr int kThreads = 384;
constexpr int kMaxDevices = 64;    // per-device launch setup slots

template <int BN>
struct Cfg {
  static constexpr int kStages = BN == 256 ? 4 : 6;                  // 192 KB of operand ring either way
  static constexpr uint32_t kABytes = kBM * kBK * 2;                 // 16 KB
  static constexpr uint32_t kBBytes = BN * kBK * 2;                  // 16 / 32 KB
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  static constexpr uint32_t kColsumOffset = kStages * kStageBytes;   // fp32 [8 warps][BN]: column sums (ACT 2)
  static constexpr uint32_t kBarOffset = kColsumOffset + 8 * BN * 4; // full[S], empty[S]
  static constexpr uint32_t kDynamic = kBarOffset + 2 * kStages * 8 + 1024;   // + slack for the 1024-B alignment
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded by WALL CLOCK (%globaltimer), not by poll count: how long one try_wait may suspend is
// implementation-defined. A protocol bug traps after 2 s instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  unsigned long long t0;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
#pragma unroll 1
  for (;;) {
    if (mbar_try_wait(bar, parity)) return;
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    if (t - t0 > 2000000000ull) __trap();
  }
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive on the barrier at `bar`'s offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(bar), "r"(cta));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire;" ::: "memory");
}

// ---- TMA -----------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c_inner, int c_outer,
                                            uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c_inner), "r"(c_outer) : "memory");
}
// the same box lands at `dst` in every CTA of `mask`, and completes bytes on the barrier at `bar`'s offset in each
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t dst, const CUtensorMap* map, int c_inner, int c_outer,
                                                      uint32_t bar, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c_inner), "r"(c_outer), "h"(mask) : "memory");
}

// ---- wgmma ---------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major operand, 128-byte swizzle: rows of 128 B, 8-row groups 1024 B apart
// (stride byte offset); the leading byte offset is unused for swizzled K-major layouts (canonical value 1).
__device__ __forceinline__ uint64_t smem_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);          // [0,14)  start address / 16
  d |= (uint64_t)1 << 16;                              // [16,30) leading byte offset / 16
  d |= (uint64_t)(1024u >> 4) << 32;                   // [32,46) stride byte offset / 16
  d |= (uint64_t)1 << 62;                              // [62,64) SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] += A[64 x 16] . B[N x 16]^T, both operands K-major in shared memory; D in registers in the wgmma
// fragment layout: d[4 i + 2 h + j] = D[16 warp + lane / 4 + 8 h][8 i + 2 (lane % 4) + j]
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t}\n"
      :
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db));
}

__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}\n"
      :
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db));
}
template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 256) wgmma_m64n256k16(d, da, db);
  else wgmma_m64n128k16(d, da, db);
}

// ---- epilogue math -------------------------------------------------------------------------------
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 0.5 x (1 + tanh(k (x + c x^3)))
__device__ __forceinline__ float gelu_tanh(float x) {
  const float u = x * fmaf(0.0356774081f, x * x, 0.7978845608f);      // k x + k c x^3
  const float hx = 0.5f * x;
  return fmaf(hx, tanh_fast(u), hx);
}
// d/dx: 0.5 (1 + t) + 0.5 x (1 - t^2) k (1 + 3 c x^2)
__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float x2 = x * x;
  const float t = tanh_fast(x * fmaf(0.0356774081f, x2, 0.7978845608f));
  const float du = fmaf(0.1070322243f, x2, 0.7978845608f);             // k (1 + 3 c x^2)
  return fmaf(0.5f * x * (1.f - t * t), du, 0.5f + 0.5f * t);
}
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t w) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
}

// CLUSTER = 1: CTAs walk tiles t = blockIdx.x, blockIdx.x + gridDim.x, ...  CLUSTER = 2: clusters walk pair tiles
// (256 x BN) the same way and CTA r of the cluster owns rows 128 r .. 128 r + 127 of the pair tile.
// colsum_rows (ACT 2, optional): fp32 [tiles_m, N], row m_blk receives the column sums of row tile m_blk.
template <int BN, int ACT, int CLUSTER>
__global__ void __launch_bounds__(kThreads, 1)
gemm_bias_act_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w,
                           const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ out,
                           __nv_bfloat16* __restrict__ pre, float* __restrict__ colsum_rows, int M, int N, int K,
                           int tiles_n, int num_tiles) {
  using C = Cfg<BN>;
  constexpr int S = C::kStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;                   // swizzle-128B tiles need 1024-B alignment
  float* colbuf = reinterpret_cast<float*>(smem_raw + (base - raw) + C::kColsumOffset);
  const uint32_t bar0 = base + C::kBarOffset;
  auto full = [&](int s) { return bar0 + 8u * s; };
  auto empty = [&](int s) { return bar0 + 8u * (S + s); };
  auto smem_a = [&](int s) { return base + (uint32_t)s * C::kStageBytes; };
  auto smem_b = [&](int s) { return base + (uint32_t)s * C::kStageBytes + C::kABytes; };

  const int wgi = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const uint32_t rank = CLUSTER > 1 ? cluster_ctarank() : 0u;
  const int group = blockIdx.x / CLUSTER, num_groups = gridDim.x / CLUSTER;
  const int num_kb = K / kBK;
  const int tiles_m = (M + kBM - 1) / kBM;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    for (int s = 0; s < S; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), 2 * CLUSTER);                          // one arrive per consumer warpgroup of each CTA
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (CLUSTER > 1) cluster_sync_all();                            // the peer's barriers exist before anyone signals them

  if (wgi == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (tid == 0) {
      // ===== TMA producer: one continuous slab stream over all tiles of this CTA =====
      uint32_t it = 0;
      for (int t = group; t < num_tiles; t += num_groups) {
        const int m_blk = (t / tiles_n) * CLUSTER + (int)rank, n_blk = t % tiles_n;
        // a CTA whose rows lie wholly below M still feeds its peer's multicast: it loads an in-range A box and
        // writes nothing
        const int a_row = min(m_blk, tiles_m - 1) * kBM;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = (int)(it % S);
          const uint32_t ph = (it / S) & 1u;
          mbar_wait(empty(s), ph ^ 1u);                           // first pass over the ring falls through
          mbar_expect_tx(full(s), C::kStageBytes);
          tma_load_2d(smem_a(s), &map_a, kb * kBK, a_row, full(s));
          if (CLUSTER == 1)
            tma_load_2d(smem_b(s), &map_w, kb * kBK, n_blk * BN, full(s));
          else
            tma_load_2d_multicast(smem_b(s) + rank * (C::kBBytes / 2), &map_w, kb * kBK, n_blk * BN + (int)rank * (BN / 2),
                                  full(s), (uint16_t)0x3);
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ===== consumers: warpgroup c owns rows 64 c .. 64 c + 63 of the tile =====
    const int c = wgi - 1, warp = tid >> 5, lane = tid & 31;
    auto release = [&](int s) {
      if (tid == 0) {
        if (CLUSTER == 1) {
          mbar_arrive(empty(s));
        } else {
#pragma unroll
          for (int r = 0; r < CLUSTER; ++r) mbar_arrive_cluster(empty(s), (uint32_t)r);
        }
      }
    };
    uint32_t it = 0;
    for (int t = group; t < num_tiles; t += num_groups) {
      const int m_blk = (t / tiles_n) * CLUSTER + (int)rank, n_blk = t % tiles_n;
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int s = (int)(it % S);
        const uint32_t ph = (it / S) & 1u;
        mbar_wait(full(s), ph);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / kMmaK; ++k) {
          // advancing K inside the 128-B swizzle atom = advancing the start address (32 B per wgmma K)
          const uint64_t da = smem_desc_k_sw128(smem_a(s) + (uint32_t)(c * 64 * kBK * 2 + k * kMmaK * 2));
          const uint64_t db = smem_desc_k_sw128(smem_b(s) + (uint32_t)(k * kMmaK * 2));
          wgmma_tile<BN>(acc, da, db);
        }
        wgmma_commit();
        wgmma_wait<1>();                                          // the previous slab's group has retired
        if (prev >= 0) release(prev);
        prev = s;
      }
      wgmma_wait<0>();
      if (prev >= 0) release(prev);

      // ===== epilogue from the accumulator registers =====
      const int row_a = m_blk * kBM + c * 64 + warp * 16 + (lane >> 2);
      const bool valid[2] = {row_a < M, row_a + 8 < M};
      const int col_base = n_blk * BN + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int col = col_base + 8 * i;
        float2 bv = make_float2(0.f, 0.f);
        if (ACT != 2 && bias != nullptr) bv = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(bias + col)));
        float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const size_t off = (size_t)(row_a + 8 * h) * (size_t)N + (size_t)col;
          const float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
          uint32_t o;
          if (ACT >= 2) {
            const float2 ax = valid[h] ? unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(pre + off)))
                                       : make_float2(0.f, 0.f);
            if (ACT == 2) {
              o = pack_bf16x2(v0 * gelu_tanh_grad(ax.x), v1 * gelu_tanh_grad(ax.y));
              if (valid[h]) {                                     // sums of the bf16 values written
                const float2 r = unpack_bf16x2(o);
                cs0 += r.x;
                cs1 += r.y;
              }
            } else {
              // bf16-round the projection first, then add: what `x + linear(h)` computes on bf16 tensors
              const float2 pr = unpack_bf16x2(pack_bf16x2(v0 + bv.x, v1 + bv.y));
              o = pack_bf16x2(pr.x + ax.x, pr.y + ax.y);
            }
          } else {
            const uint32_t u = pack_bf16x2(v0 + bv.x, v1 + bv.y);
            if (ACT == 1) {
              // the activation sees the bf16-rounded pre-activation, exactly like gelu(linear(x)) on bf16 tensors
              const float2 r = unpack_bf16x2(u);
              o = pack_bf16x2(gelu_tanh(r.x), gelu_tanh(r.y));
            } else {
              o = u;
            }
            if (pre != nullptr && valid[h]) *reinterpret_cast<uint32_t*>(pre + off) = u;
          }
          if (valid[h]) *reinterpret_cast<uint32_t*>(out + off) = o;
        }
        if (ACT == 2 && colsum_rows != nullptr) {
          // the 8 lanes of a column pair (lane / 4 = 0..7), then this warp's slot of the shared buffer
#pragma unroll
          for (int x = 4; x < 32; x <<= 1) {
            cs0 += __shfl_xor_sync(0xffffffffu, cs0, x);
            cs1 += __shfl_xor_sync(0xffffffffu, cs1, x);
          }
          if (lane < 4) {
            float* slot = colbuf + (c * 4 + warp) * BN + 8 * i + 2 * lane;
            slot[0] = cs0;
            slot[1] = cs1;
          }
        }
      }
      if (ACT == 2 && colsum_rows != nullptr) {
        // the tile's column sums, warps added in a fixed order; the second barrier keeps the next tile's writes out
        // of the buffer until it has been read
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (m_blk < tiles_m) {
          for (int j = c * 128 + tid; j < BN; j += 256) {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) v += colbuf[w * BN + j];
            colsum_rows[(size_t)m_blk * N + n_blk * BN + j] = v;
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
    }
  }
  if (CLUSTER > 1) cluster_sync_all();                            // no CTA leaves while its peer may still signal it
}

// colsum[j] += sum over m of rows[m, j], m ascending
__global__ void colsum_rows_add_kernel(const float* __restrict__ rows, float* __restrict__ colsum, int tiles_m, int N) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  float v = 0.f;
  for (int m = 0; m < tiles_m; ++m) v += rows[(size_t)m * N + j];
  colsum[j] += v;
}

// ---- host ----------------------------------------------------------------------------------------
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    else
      (void)cudaGetLastError();
  });
  return fn;
}

// row-major [rows, cols] bf16 matrix, box = (64 columns, box_rows rows), 128-byte swizzle
static int make_map(CUtensorMap* map, const void* ptr, int rows, int cols, int box_rows) {
  EncodeTiledFn enc = encode_tiled();
  if (!enc) { set_error("gemm: cuTensorMapEncodeTiled unavailable"); return -1; }
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  const cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("gemm: cuTensorMapEncodeTiled failed (%d)", (int)r); return -1; }
  return 0;
}

// persistent: grid = min(tiles, SMs); otherwise one (pair) tile per CTA (cluster)
template <int BN, int ACT, int CLUSTER>
static int launch(const void* a, const void* w, const void* bias, void* out, void* pre, float* colsum,
                  float* colsum_work, int M, int N, int K, bool persistent, cudaStream_t s) {
  auto kern = gemm_bias_act_wgmma_kernel<BN, ACT, CLUSTER>;
  // the shared-memory opt-in is a per-device function attribute: set it once for every device this process uses
  static std::once_flag once[kMaxDevices];
  static int sms[kMaxDevices];
  static cudaError_t setup[kMaxDevices];
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDevices) { set_error("gemm: device %d out of range", dev); return -1; }
  std::call_once(once[dev], [&] {
    setup[dev] = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg<BN>::kDynamic);
    if (setup[dev] == cudaSuccess) setup[dev] = cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
  });
  CUDA_TRY(setup[dev]);
  CUtensorMap ma, mw;
  if (make_map(&ma, a, M, K, kBM)) return -1;
  if (make_map(&mw, w, N, K, BN / CLUSTER)) return -1;          // in a cluster each CTA loads half of the W slab
  const int tiles_n = N / BN, tiles_m = (M + kBM - 1) / kBM;
  const int num_tiles = tiles_n * ((tiles_m + CLUSTER - 1) / CLUSTER);
  const int groups = persistent ? std::min(num_tiles, sms[dev] / CLUSTER) : num_tiles;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(groups * CLUSTER));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = Cfg<BN>::kDynamic;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CLUSTER;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, ma, mw, (const __nv_bfloat16*)bias, (__nv_bfloat16*)out,
                              (__nv_bfloat16*)pre, colsum != nullptr ? colsum_work : nullptr, M, N, K, tiles_n,
                              num_tiles));
  count_launch();
  if (colsum != nullptr) {
    colsum_rows_add_kernel<<<(N + 255) / 256, 256, 0, s>>>(colsum_work, colsum, tiles_m, N);
    CUDA_TRY(cudaGetLastError());
    count_launch();
  }
  return 0;
}

}  // namespace wg
}  // namespace adapcc

using namespace adapcc;

extern "C" {

// out = act(a[M,K] @ w[N,K]^T + bias); pre (optional) = the pre-activation. bf16 row-major, 16-byte aligned.
// act 2: out = (a @ w^T) * gelu'(aux); act 3: out = a @ w^T + bias + aux — aux is passed in `pre` (an input then).
// K % 64 == 0, N % 128 == 0 (256-wide tiles when N % 256 == 0).
// variant 0: one tile per CTA; 1: persistent CTAs; 2: two-CTA clusters sharing W by TMA multicast (N % 256 == 0).
int adapcc_gemm_bias_act_v(const void* a, const void* w, const void* bias, void* out, void* pre, int M, int N, int K,
                           int act, int variant, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if (K % wg::kBK != 0 || N % 128 != 0) { set_error("gemm: need K %% 64 == 0 and N %% 128 == 0 (got K=%d N=%d)", K, N); return -1; }
  if (act < 0 || act > 3) { set_error("gemm: act must be 0 (none), 1 (gelu_tanh), 2 (dgelu * aux) or 3 (+ aux)"); return -1; }
  if (act >= 2 && pre == nullptr) { set_error("gemm: act %d needs the aux tensor (passed as `pre`)", act); return -1; }
  if (act >= 2 && variant != 0) { set_error("gemm: act %d is only built for variant 0", act); return -1; }
  if (variant < 0 || variant > 2) { set_error("gemm: variant must be 0, 1 or 2"); return -1; }
  if (variant == 2 && (N % 256 != 0 || act > 1)) { set_error("gemm: variant 2 (CTA pairs) needs N %% 256 == 0 and act 0/1"); return -1; }
  if (((uintptr_t)a | (uintptr_t)w | (uintptr_t)out | (uintptr_t)pre | (uintptr_t)bias) & 15) { set_error("gemm: operands must be 16-byte aligned"); return -1; }
  cudaStream_t s = (cudaStream_t)stream;
  if (variant == 2)
    return act ? wg::launch<256, 1, 2>(a, w, bias, out, pre, nullptr, nullptr, M, N, K, false, s)
               : wg::launch<256, 0, 2>(a, w, bias, out, pre, nullptr, nullptr, M, N, K, false, s);
  const bool persistent = variant == 1;
#define WG_LAUNCH(BN_)                                                                              \
  switch (act) {                                                                                    \
    case 0: return wg::launch<BN_, 0, 1>(a, w, bias, out, pre, nullptr, nullptr, M, N, K, persistent, s);    \
    case 1: return wg::launch<BN_, 1, 1>(a, w, bias, out, pre, nullptr, nullptr, M, N, K, persistent, s);    \
    case 2: return wg::launch<BN_, 2, 1>(a, w, bias, out, pre, nullptr, nullptr, M, N, K, persistent, s);    \
    default: return wg::launch<BN_, 3, 1>(a, w, bias, out, pre, nullptr, nullptr, M, N, K, persistent, s);   \
  }
  if (N % 256 == 0) { WG_LAUNCH(256) }
  WG_LAUNCH(128)
#undef WG_LAUNCH
}

int adapcc_gemm_bias_act(const void* a, const void* w, const void* bias, void* out, void* pre, int M, int N, int K,
                         int act, void* stream) {
  return adapcc_gemm_bias_act_v(a, w, bias, out, pre, M, N, K, act, 0, stream);
}

// Variant 3, the one the GPT-2 MLP uses: persistent two-CTA clusters, 256 x 256 per cluster.
// act 0 / 1: out = act(a @ w^T + bias), pre (optional output) = a @ w^T + bias.
// act 2: out = (a @ w^T) * gelu'(pre)  (pre = aux INPUT), colsum (optional, fp32 [N], accumulated into) += column sums;
// colsum_work: fp32 [ceil(M / 128), N] scratch, needed with colsum.
// bf16 row-major operands, 16-byte aligned; K % 64 == 0, N % 256 == 0.
int adapcc_gemm_pp(const void* a, const void* w, const void* bias, void* out, void* pre, float* colsum,
                   float* colsum_work, int M, int N, int K, int act, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if (K % wg::kBK != 0 || N % 256 != 0) { set_error("gemm_pp: need K %% 64 == 0 and N %% 256 == 0 (got K=%d N=%d)", K, N); return -1; }
  if (act < 0 || act > 2) { set_error("gemm_pp: act must be 0 (none), 1 (gelu) or 2 (dgelu)"); return -1; }
  if (act == 2 && pre == nullptr) { set_error("gemm_pp: act 2 needs the saved pre-activation"); return -1; }
  if (colsum != nullptr && (act != 2 || colsum_work == nullptr)) { set_error("gemm_pp: colsum needs act 2 and the [ceil(M/128), N] work buffer"); return -1; }
  if (((uintptr_t)a | (uintptr_t)w | (uintptr_t)out | (uintptr_t)pre | (uintptr_t)bias) & 15) { set_error("gemm_pp: operands must be 16-byte aligned"); return -1; }
  cudaStream_t s = (cudaStream_t)stream;
  switch (act) {
    case 0: return wg::launch<256, 0, 2>(a, w, bias, out, pre, nullptr, nullptr, M, N, K, true, s);
    case 1: return wg::launch<256, 1, 2>(a, w, bias, out, pre, nullptr, nullptr, M, N, K, true, s);
    default: return wg::launch<256, 2, 2>(a, w, bias, out, pre, colsum, colsum_work, M, N, K, true, s);
  }
}

}  // extern "C"
