// Thin inline-PTX wrappers for the sm_90a primitives used by the tensor-core kernels:
// mbarrier, TMA (cp.async.bulk[.tensor]), wgmma.mma_async and its shared-memory matrix descriptors.
// Descriptor bit layouts follow the PTX ISA "warpgroup-level matrix shared memory layout" tables; nothing here is
// library code.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <type_traits>

namespace b200 {
namespace tc {

// f(std::integral_constant<int, I>) for I = B .. E-1: the index is a constant expression inside f (wgmma widths and
// register offsets must be known at compile time)
template <int B, int E, typename F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (B < E) {
    f(std::integral_constant<int, B>{});
    static_for<B + 1, E>(f);
  }
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// 128-byte aligned start of the dynamic shared memory, derived by pointer arithmetic so the compiler keeps the address space
__device__ __forceinline__ uint8_t* align_smem128(uint8_t* raw) { return raw + ((128u - (smem_u32(raw) & 127u)) & 127u); }

// ---- mbarrier -------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// one lane of a CONVERGED warp (elect.sync): lets a whole warp run the loop control of a single-thread role, so the
// compiler keeps descriptors / addresses on the uniform datapath instead of emitting per-instruction waterfall loops
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// the retry loop stays inside the asm block: a C++ loop around try_wait is a divergent path to ptxas, which then
// serialises the wgmma instructions that follow it
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra WAIT_%=;\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}

// ---- TMA ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// global -> L2 prefetch of a contiguous range (16-byte granules); no completion mechanism, a hint for a later bulk_load
__device__ __forceinline__ void bulk_prefetch_l2(const void* gsrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gsrc), "r"(bytes) : "memory");
}

// ---- wgmma (warpgroup MMA, accumulators in registers) --------------------------------------------------
// A warpgroup = four consecutive warps 4k .. 4k+3.  Every wgmma instruction below is executed by all 128 threads.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across a wgmma.wait_group
template <int K>
__device__ __forceinline__ void wg_fence_acc(float* d) {
#pragma unroll
  for (int i = 0; i < K; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// named barrier of the 128 threads of one warpgroup (ids 8.. are free for this)
__device__ __forceinline__ void wg_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
// named barrier of `threads` threads (a multiple of 32)
__device__ __forceinline__ void named_bar(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

#include "wgmma_shapes.inc"

// D[64 x N] (+)= A[64 x 16] * B[16 x N] for any N that is a multiple of 8: one instruction when a specialisation exists,
// otherwise the N range is split (the B descriptor of a K-major / no-swizzle image advances by SBO per 8 columns).
template <int N, int TB = 0>
__device__ __forceinline__ void wg_mma_ss(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate, uint32_t b_sbo) {
  constexpr int kDirect = (N == 8 || N == 16 || N == 32 || N == 48 || N == 64 || N == 96 || N == 128 || N == 192 || N == 256);
  if constexpr (kDirect) {
    Mma<N>::template ss<TB>(d, adesc, bdesc, accumulate);
  } else {
    constexpr int P = N > 256 ? 256 : N > 192 ? 192 : N > 128 ? 128 : N > 96 ? 96 : N > 64 ? 64 : N > 48 ? 48 : N > 32 ? 32 : N > 16 ? 16 : 8;
    Mma<P>::template ss<TB>(d, adesc, bdesc, accumulate);
    wg_mma_ss<N - P, TB>(d + P / 2, adesc, bdesc + (uint64_t)(((P / 8) * b_sbo) >> 4), accumulate, b_sbo);
  }
}

// Shared-memory matrix descriptor, no swizzle ("interleave"): core matrix = 8 rows x 16 bytes stored contiguously (128 B).
// K-major: lbo = byte distance between the two K-adjacent core matrices of one K=16 step, sbo = byte distance between
// consecutive 8-row groups.  Bits: [0,14) addr>>4, [16,30) lbo>>4, [32,46) sbo>>4, [62,64) layout type = 0 (no swizzle).
__device__ __forceinline__ uint64_t make_desc_kmajor_noswz(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

// ---- accumulator fragment -> one row per thread ---------------------------------------------------------
// The fp32 accumulator of an m64nN wgmma is spread over the warpgroup: thread (warp w, lane l) holds, for every 8-column
// block i, d[4i + {0,1}] = D[16w + l/4][8i + 2(l%4) + {0,1}] and d[4i + {2,3}] = the same columns of row 16w + 8 + l/4.
// The epilogues want one output row per thread and 8 consecutive columns, so the warpgroup passes 16-column slices of its
// 64 rows through a small shared-memory buffer (kStageFloats floats per warpgroup): afterwards warp w reads row
// 32 (w & 1) + l and columns 8 (w >> 1) .. + 8 of the slice.
constexpr int kStageLd = 20;                      // padded row stride (floats) of the slice buffer
constexpr int kStageFloats = 64 * kStageLd;
template <int C0>
__device__ __forceinline__ void wg_stage16(const float* d, float* buf, int wid, int lane) {
  const int r = 16 * wid + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int j = (C0 / 8 + i) * 4;
    *reinterpret_cast<float2*>(buf + r * kStageLd + 8 * i + c) = make_float2(d[j], d[j + 1]);
    *reinterpret_cast<float2*>(buf + (r + 8) * kStageLd + 8 * i + c) = make_float2(d[j + 2], d[j + 3]);
  }
}
__device__ __forceinline__ void wg_read8(const float* buf, int wid, int lane, float (&v)[8]) {
  const float4* s = reinterpret_cast<const float4*>(buf + (32 * (wid & 1) + lane) * kStageLd + 8 * (wid >> 1));
  const float4 a = s[0], b = s[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

}  // namespace tc

// cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda link dependency).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_tiled();

}  // namespace b200
