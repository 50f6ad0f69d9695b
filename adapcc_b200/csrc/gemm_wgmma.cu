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
//                             128-byte swizzled, into a ring of Cfg::kStages stages; `full[s]` completes on the
//                             transferred bytes
//   warpgroups 1, 2         : 64 rows each — 4 x wgmma.m64nBNk16 per slab, one wgmma group kept in flight; a slab is
//                             released (`empty[s]`) once the group that read it has retired; then the epilogue
//                             (bias + activation in fp32 on the accumulator registers, as before any bf16 rounding)
// Epilogue: each consumer warp owns 16 rows and a ring of Cfg::kEpiBufs 16 x 64 bf16 staging buffers (2 KB,
// 128-byte swizzled). Per 64-column sub-tile it packs its results to bf16, writes them with stmatrix, fences the
// generic proxy against the async one and one lane issues a TMA store (cp.async.bulk.tensor, bulk_group) of the
// sub-tile; the tensor map's bounds clip rows >= M. A buffer is written again only once the store that last read it
// has (cp.async.bulk.wait_group.read), so the stores drain to HBM under the next tile's wgmmas. ACT 2 / 3 read `aux`
// the same way in reverse: a TMA load into the staging buffer (issued during the tile's middle slab, completing on a
// per-buffer mbarrier), ldmatrix into the fragment layout, and the result is stored back in place.
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
constexpr int kEpiRows = 16;       // rows of one consumer warp's staging sub-tile (its wgmma fragment rows)
constexpr uint32_t kEpiBytes = kEpiRows * kBK * 2;   // 2 KB: 16 rows x 64 bf16, 128-byte swizzled
constexpr uint32_t kSmemOptIn = 232448;               // sm_90 per-block dynamic shared memory limit

template <int BN>
struct Cfg {
  static constexpr int kStages = BN == 256 ? 3 : 5;
  static constexpr uint32_t kABytes = kBM * kBK * 2;                 // 16 KB
  static constexpr uint32_t kBBytes = BN * kBK * 2;                  // 16 / 32 KB
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  // what the ring, the column-sum buffer, the ring's barriers and the alignment slack leave, in staging buffers per
  // consumer warp (each with its aux mbarrier); more than BN / 64 would never be used
  static constexpr uint32_t kFixed = kStages * kStageBytes + 8 * BN * 4 + 2 * kStages * 8 + 1024;
  static constexpr int kEpiBufs = (int)std::min<uint32_t>(BN / 64, (kSmemOptIn - kFixed) / (8 * (kEpiBytes + 8)));
  static_assert(kEpiBufs >= 1, "no shared memory left for the epilogue staging buffers");
  static constexpr uint32_t kEpiOffset = kStages * kStageBytes;      // [8 warps][kEpiBufs] staging buffers
  static constexpr uint32_t kColsumOffset = kEpiOffset + 8 * kEpiBufs * kEpiBytes;   // fp32 [8 warps][BN] (ACT 2)
  static constexpr uint32_t kBarOffset = kColsumOffset + 8 * BN * 4; // full[S], empty[S], aux[8 warps][kEpiBufs]
  static constexpr uint32_t kDynamic = kBarOffset + (2 * kStages + 8 * kEpiBufs) * 8 + 1024;   // + alignment slack
  static_assert(kDynamic <= kSmemOptIn, "shared memory over the opt-in limit");
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
// arrive on the barrier at `bar`'s offset in CTA `cta` of the cluster. Default (.release.cta) semantics: the arrival
// only has to follow the wgmmas that read the stage, which wgmma.wait_group has already retired. A .release.cluster
// arrive compiles to MEMBAR.ALL.GPU, which waits for this thread's outstanding global stores and held every stage
// refill of the pair up behind it.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(bar), "r"(cta));
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
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
// shared -> global; the box's rows past the tensor map's bounds are not written
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c_inner, int c_outer) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(src), "r"(c_inner), "r"(c_outer) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's most recent bulk groups may still be reading their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// generic-proxy shared-memory writes become visible to the async proxy (a following TMA store)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- staging sub-tiles: 8 x 8 b16 matrices between the wgmma fragment layout and shared memory ---------------------
// x4: matrix q's row r is addressed by lane 8 q + r; a thread's register q holds row lane / 4, columns 2 (lane % 4)
// and + 1 of matrix q — for the accumulator, the pair d[4 i + 2 h], d[4 i + 2 h + 1].
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};"
               ::"r"(addr), "r"(r0), "r"(r1), "r"(r2), "r"(r3) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr) : "memory");
}
// A warp's 16 x 64 sub-tile as 4 x4 groups: group p holds the column groups 2p, 2p + 1 (8 columns = one 16-B chunk
// each) of rows 0-7 and 8-15, i.e. matrices (h 0, 2p), (h 1, 2p), (h 0, 2p + 1), (h 1, 2p + 1); registers
// v[4p .. 4p + 3] in that order. The buffer is in the TMA's 128-byte swizzled layout: chunk c of row r sits at
// r * 128 + ((c ^ (r % 8)) * 16), so the 8 rows of a matrix fall on 8 different bank groups.
__device__ __forceinline__ uint32_t stage_addr(uint32_t buf, int lane, int p) {
  const int r = (lane & 7) + 8 * ((lane >> 3) & 1), chunk = 2 * p + (lane >> 4);
  return buf + (uint32_t)(r * 128 + ((chunk ^ (r & 7)) << 4));
}
__device__ __forceinline__ void stage_write(uint32_t buf, int lane, const uint32_t (&v)[16]) {
#pragma unroll
  for (int p = 0; p < 4; ++p) stmatrix_x4(stage_addr(buf, lane, p), v[4 * p], v[4 * p + 1], v[4 * p + 2], v[4 * p + 3]);
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
// map_out / map_pre: [M, N] bf16, 64 x 16 boxes, 128-byte swizzle (map_pre is unused when has_pre == 0).
// colsum_rows (ACT 2, optional): fp32 [tiles_m, N], row m_blk receives the column sums of row tile m_blk.
template <int BN, int ACT, int CLUSTER>
__global__ void __launch_bounds__(kThreads, 1)
gemm_bias_act_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w,
                           const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_pre,
                           const __nv_bfloat16* __restrict__ bias, int has_pre, float* __restrict__ colsum_rows, int M,
                           int N, int K, int tiles_n, int num_tiles) {
  using C = Cfg<BN>;
  constexpr int S = C::kStages, NB = C::kEpiBufs, J = BN / 64;   // J: 64-column sub-tiles per tile
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
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_out) : "memory");
    if (has_pre) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_pre) : "memory");
    for (int s = 0; s < S; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), 2 * CLUSTER);                          // one arrive per consumer warpgroup of each CTA
    }
    for (int b = 0; b < 8 * NB; ++b) mbar_init(bar0 + 8u * (2 * S + b), 1);   // aux loads: expect_tx + bytes
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
    // this warp's 16 rows: staging ring buf(b), aux barrier abar(b) (parity bit b of aux_phase)
    const int gw = c * 4 + warp;
    const uint32_t epi0 = base + C::kEpiOffset + (uint32_t)(gw * NB) * kEpiBytes;
    auto buf = [&](int b) { return epi0 + (uint32_t)b * kEpiBytes; };
    auto abar = [&](int b) { return bar0 + 8u * (2 * S + gw * NB + b); };
    uint32_t aux_phase = 0, epi_it = 0;
    uint32_t it = 0;
    for (int t = group; t < num_tiles; t += num_groups) {
      const int m_blk = (t / tiles_n) * CLUSTER + (int)rank, n_blk = t % tiles_n;
      const int row_w = m_blk * kBM + c * 64 + warp * 16;       // first row of this warp's sub-tiles
      // a warp whose rows lie wholly below M (always so in a cluster CTA past the last row tile) moves no data
      const bool rows_in = row_w < M;
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
        if (ACT >= 2 && kb == num_kb / 2 && rows_in && lane == 0) {
          // under the wgmmas of the middle slab: once the previous tile's stores have read the ring, load this tile's
          // first NB aux sub-tiles into it — half a mainloop after those stores were issued, half a mainloop before the
          // epilogue needs the loads
          bulk_wait_read<0>();
#pragma unroll
          for (int b = 0; b < NB; ++b) {
            mbar_expect_tx(abar(b), kEpiBytes);
            tma_load_2d(buf(b), &map_pre, n_blk * BN + 64 * b, row_w, abar(b));
          }
        }
        wgmma_wait<1>();                                          // the previous slab's group has retired
        if (prev >= 0) release(prev);
        prev = s;
      }
      wgmma_wait<0>();
      if (prev >= 0) release(prev);

      // ===== epilogue: fp32 math on the accumulator registers, bf16 sub-tiles out through shared memory + TMA =====
      const int row_a = row_w + (lane >> 2);
      const bool valid[2] = {row_a < M, row_a + 8 < M};
      const int col_base = n_blk * BN + 2 * (lane & 3);
      // TMA-store sub-tile j of this warp's rows from staging buffer b, once every lane's writes to it are fenced
      auto store_sub = [&](uint32_t b, const CUtensorMap* map, int j) {
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
          tma_store_2d(map, buf((int)b), n_blk * BN + 64 * j, row_w);
          bulk_commit();
        }
      };
#pragma unroll
      for (int j = 0; j < J; ++j) {
        // ov: the result, v[2 ii + h]. For ACT 2 / 3 the aux sub-tile in buffer j % NB is read one x4 group (column
        // groups 2p, 2p + 1) at a time into the same registers and the group's results are written back in place.
        uint32_t ov[16], uv[16];
        const int ab = j % NB;
        if (ACT >= 2 && rows_in) {
          mbar_wait(abar(ab), (aux_phase >> ab) & 1u);
          aux_phase ^= 1u << ab;
        }
#pragma unroll
        for (int ii = 0; ii < 8; ++ii) {
          const int i = 8 * j + ii;
          if (ACT >= 2 && (ii & 1) == 0) {
            if (rows_in)
              ldmatrix_x4(stage_addr(buf(ab), lane, ii / 2), ov[2 * ii], ov[2 * ii + 1], ov[2 * ii + 2], ov[2 * ii + 3]);
            else
              ov[2 * ii] = ov[2 * ii + 1] = ov[2 * ii + 2] = ov[2 * ii + 3] = 0u;
          }
          const int col = col_base + 8 * i;
          float2 bv = make_float2(0.f, 0.f);
          if (ACT != 2 && bias != nullptr) bv = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(bias + col)));
          float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
            uint32_t o;
            if (ACT >= 2) {
              const float2 ax = valid[h] ? unpack_bf16x2(ov[2 * ii + h]) : make_float2(0.f, 0.f);
              if (ACT == 2) {
                o = pack_bf16x2(v0 * gelu_tanh_grad(ax.x), v1 * gelu_tanh_grad(ax.y));
                if (valid[h]) {                                   // sums of the bf16 values written
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
              uv[2 * ii + h] = u;
            }
            ov[2 * ii + h] = o;
          }
          if (ACT >= 2 && (ii & 1) == 1 && rows_in)
            stmatrix_x4(stage_addr(buf(ab), lane, ii / 2), ov[2 * ii - 2], ov[2 * ii - 1], ov[2 * ii], ov[2 * ii + 1]);
          if (ACT == 2 && colsum_rows != nullptr) {
            // the 8 lanes of a column pair (lane / 4 = 0..7), then this warp's slot of the shared buffer
#pragma unroll
            for (int x = 4; x < 32; x <<= 1) {
              cs0 += __shfl_xor_sync(0xffffffffu, cs0, x);
              cs1 += __shfl_xor_sync(0xffffffffu, cs1, x);
            }
            if (lane < 4) {
              float* slot = colbuf + gw * BN + 8 * i + 2 * lane;
              slot[0] = cs0;
              slot[1] = cs1;
            }
          }
        }
        if (!rows_in) continue;
        if (ACT >= 2) {
          store_sub(ab, &map_out, j);
          if (j + NB < J && lane == 0) {
            bulk_wait_read<0>();                                  // the store has read the buffer: refill it
            mbar_expect_tx(abar(ab), kEpiBytes);
            tma_load_2d(buf(ab), &map_pre, n_blk * BN + 64 * (j + NB), row_w, abar(ab));
          }
        } else {
          // ring reuse: with one commit per buffer use, <= NB - 1 groups still reading means the next buffer is free
          if (has_pre) {
            if (lane == 0) bulk_wait_read<NB - 1>();
            __syncwarp();
            stage_write(buf(epi_it % NB), lane, uv);
            store_sub(epi_it++ % NB, &map_pre, j);
          }
          if (lane == 0) bulk_wait_read<NB - 1>();
          __syncwarp();
          stage_write(buf(epi_it % NB), lane, ov);
          store_sub(epi_it++ % NB, &map_out, j);
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
    if (lane == 0) bulk_wait_all();                               // the staging buffers outlive every store
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
  CUtensorMap ma, mw, mo, mp = {};
  if (make_map(&ma, a, M, K, kBM)) return -1;
  if (make_map(&mw, w, N, K, BN / CLUSTER)) return -1;          // in a cluster each CTA loads half of the W slab
  if (make_map(&mo, out, M, N, kEpiRows)) return -1;            // one consumer warp's 16 x 64 staging sub-tile
  if (pre != nullptr && make_map(&mp, pre, M, N, kEpiRows)) return -1;
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
  CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, ma, mw, mo, mp, (const __nv_bfloat16*)bias, pre != nullptr ? 1 : 0,
                              colsum != nullptr ? colsum_work : nullptr, M, N, K, tiles_n, num_tiles));
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
