// Global multi-head self-attention of the ViT encoder (UNETR) on Hopper wgmma tensor cores.
//
// Reference: SABlock.forward (monai/networks/blocks/selfattention.py:170-217): per batch item and head (head_dim 64, no bias,
// no mask) out = softmax(q k^T * scale) v over all S tokens.
//
// One persistent CTA per SM works on tiles = (batch item, head, 128-query row tile), ordered so that the tiles of one
// (item, head) -- which read the same K / V -- are neighbours and mostly land on the same CTA.  Two consumer warpgroups take
// 64 query rows each and walk the keys in blocks of 64 (flash-attention style, online softmax):
//   S[64 x 64] = Q K^T                        4 wgmma m64n64k16 (SS form: Q and K both from shared memory)
//   softmax: running row maximum m and row sum l in registers, scores in log2 units (the caller folds
//            dim_head^-0.5 * log2(e) into the q rows of the qkv projection, so the kernel uses exp2 only);
//            keys >= S of the last block get -inf before the row maximum;
//            P = 2^(S - m) rounded to fp16 -- the S accumulator fragment, packed to fp16 pairs, is the register A operand of
//   O[64 x 64] += P V                         4 wgmma m64n64k16 (RS form), V read in place as an MN-major B operand (NC8
//            rows are 16-byte vectors of 8 dims); l sums the same fp16-rounded P values the MMA consumes;
//   epilogue: O / l -> fp16 NC8 (query rows >= S are not stored).
// Every 8-dim chunk of Q, K, V is contiguous over tokens in NC8, i.e. already a K-major core-matrix column: all operand
// traffic is 1-D bulk copies clamped to the valid rows.  K / V stream through a ring of kMhStages blocks, so any S >= 1 works.
// The summation order is fixed: two runs give bit-identical output.
//
// Warp roles (384 threads): warp 0 = copy producer, warps 4-7 / 8-11 = the two consumer warpgroups.
#include "common.cuh"
#include "tc90.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

constexpr int kMhDim = 64;                                    // head_dim
constexpr int kMhChunks = kMhDim / 8;                         // 8-dim NC8 chunks per head
constexpr int kMhKeys = 64;                                   // keys per block
constexpr int kMhStages = 4;                                  // K / V ring depth
constexpr int kMhQChunk = 128 * 16;                           // one chunk of a 128-row Q tile (bytes)
constexpr int kMhQBytes = kMhChunks * kMhQChunk;              // 16 KB per Q buffer (two are kept)
constexpr int kMhKChunk = kMhKeys * 16;                       // one chunk of a 64-key block (bytes)
constexpr int kMhKvBytes = 2 * kMhChunks * kMhKChunk;         // K and V of one block: 16 KB per stage
constexpr int kMhThreads = 384;
constexpr int kMhSmem = 2 * kMhQBytes + kMhStages * kMhKvBytes + 2 * 2 * tc::kStageFloats * 4 + 256 + 128;

struct MhsaTcParams {
  const __half* qkv; __half* out;
  int C8, heads, nqt, nkb;
  long long S, total;
};

__device__ __forceinline__ float mh_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 2^(a - m), 2^(b - m) as packed fp16; `sum` accumulates the two ROUNDED values (what the PV MMA multiplies)
__device__ __forceinline__ uint32_t mh_exp2_pack(float a, float b, float m, float& sum) {
  const __half2 h = __floats2half2_rn(mh_ex2(a - m), mh_ex2(b - m));
  const float2 r = __half22float2(h);
  sum += r.x + r.y;
  return *reinterpret_cast<const uint32_t*>(&h);
}

__global__ void __launch_bounds__(kMhThreads, 1) mhsa_tc_kernel(MhsaTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = tc::align_smem128(smem_raw);   // keeps the shared address space (LDS/STS, not generic LD/ST)
  uint8_t* s_q = smem;                                   // [2 buffers][8 chunks][128 rows][16 B]
  uint8_t* s_kv = s_q + 2 * kMhQBytes;                   // [stage][K chunks 0-7, V chunks 0-7][64 keys][16 B]
  float* s_stage = reinterpret_cast<float*>(s_kv + kMhStages * kMhKvBytes);   // [2 warpgroups][2][kStageFloats]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stage + 2 * 2 * tc::kStageFloats);
  uint64_t* q_full = bars + 0;                  // [2]  the Q tile of buffer b has landed
  uint64_t* q_empty = bars + 2;                 // [2]  the S MMAs that read Q buffer b are done (one arrival per warpgroup)
  uint64_t* kv_full = bars + 4;                 // [kMhStages]
  uint64_t* kv_empty = bars + 4 + kMhStages;    // [kMhStages]  the PV MMAs that read stage s are done

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const long long S = p.S;
  const long long lo = p.total * blockIdx.x / gridDim.x, hi = p.total * (blockIdx.x + 1) / gridDim.x;

  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { tc::mbar_init(&q_full[i], 1); tc::mbar_init(&q_empty[i], 2); }
    for (int i = 0; i < kMhStages; ++i) { tc::mbar_init(&kv_full[i], 1); tc::mbar_init(&kv_empty[i], 2); }
    tc::fence_barrier_init();
  }
  // zero Q / K / V: rows the clamped bulk copies never write must hold finite values (masked keys multiply V by P = 0)
  {
    const uint4 z = make_uint4(0, 0, 0, 0);
    uint4* zq = reinterpret_cast<uint4*>(s_q);
    const int nz = (2 * kMhQBytes + kMhStages * kMhKvBytes) / 16;
    for (int i = threadIdx.x; i < nz; i += blockDim.x) zq[i] = z;
  }
  tc::fence_proxy_async();
  __syncthreads();

  if (warp == 0) {
    // ===================== copy producer =====================
    if (lane == 0) {
      int ks = 0; uint32_t kph = 0;
      int it = 0;
      for (long long f = lo; f < hi; ++f, ++it) {
        const int qt = (int)(f % p.nqt);
        const long long bh = f / p.nqt;
        const int h = (int)(bh % p.heads), b = (int)(bh / p.heads);
        const __half* base = p.qkv + (long long)b * (3 * p.C8) * S * 8;
        const int qb = it & 1;
        const int rows = (int)min(128LL, S - (long long)qt * 128);
        tc::mbar_wait(&q_empty[qb], (uint32_t)(((it >> 1) & 1) ^ 1));   // the S MMAs that read this buffer two tiles ago are done
        tc::mbar_arrive_expect_tx(&q_full[qb], (uint32_t)(kMhChunks * rows * 16));
        for (int c = 0; c < kMhChunks; ++c)
          tc::bulk_load(s_q + qb * kMhQBytes + c * kMhQChunk, base + (((long long)h * kMhChunks + c) * S + (long long)qt * 128) * 8,
                        rows * 16, &q_full[qb]);
        for (int kb = 0; kb < p.nkb; ++kb) {
          const int keys = (int)min((long long)kMhKeys, S - (long long)kb * kMhKeys);
          tc::mbar_wait(&kv_empty[ks], kph ^ 1u);
          tc::mbar_arrive_expect_tx(&kv_full[ks], (uint32_t)(2 * kMhChunks * keys * 16));
          uint8_t* dst = s_kv + ks * kMhKvBytes;
          for (int c = 0; c < 2 * kMhChunks; ++c) {   // K chunks then V chunks
            const long long chunk = (long long)(c < kMhChunks ? p.heads + h : 2 * p.heads + h) * kMhChunks + (c % kMhChunks);
            tc::bulk_load(dst + c * kMhKChunk, base + (chunk * S + (long long)kb * kMhKeys) * 8, keys * 16, &kv_full[ks]);
          }
          if (++ks == kMhStages) { ks = 0; kph ^= 1u; }
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    // ===================== consumers: warpgroup g owns query rows 64 g .. 64 g + 63 of every tile =====================
    const int g = (warp >> 2) - 1, wid = warp & 3;
    const uint32_t q_a = tc::smem_u32(s_q), kv_a = tc::smem_u32(s_kv);
    float* stage = s_stage + g * 2 * tc::kStageFloats;
    const int tail = (int)(S - (long long)(p.nkb - 1) * kMhKeys);   // valid keys of the last block (1 .. 64)
    int ks = 0; uint32_t kph = 0;
    int sl = 0;
    int it = 0;
    for (long long f = lo; f < hi; ++f, ++it) {
      const int qb = it & 1;
      float o[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) o[j] = 0.f;
      float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows 16 wid + lane/4 and + 8 of the warpgroup
      tc::mbar_wait(&q_full[qb], (uint32_t)((it >> 1) & 1));
      const uint32_t qbase = q_a + qb * kMhQBytes + g * 1024;
#pragma unroll 1
      for (int kb = 0; kb < p.nkb; ++kb) {
        tc::mbar_wait(&kv_full[ks], kph);
        const uint32_t kbase = kv_a + ks * kMhKvBytes, vbase = kbase + kMhChunks * kMhKChunk;
        // ---- S = Q K^T for 64 keys: K = 64 dims in four k16 steps (two 8-dim chunks each) ----
        float sc[32];
        tc::wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          tc::Mma<64>::ss<0>(sc, tc::make_desc_kmajor_noswz(qbase + 2 * k * kMhQChunk, kMhQChunk, 128),
                             tc::make_desc_kmajor_noswz(kbase + 2 * k * kMhKChunk, kMhKChunk, 128), k > 0 ? 1u : 0u);
        tc::wg_commit();
        tc::wg_wait<0>();
        tc::wg_fence_acc<32>(sc);
        if (kb == p.nkb - 1 && wid == 0 && lane == 0) tc::mbar_arrive(&q_empty[qb]);   // this warpgroup is done with Q
        if (kb == p.nkb - 1 && tail < kMhKeys) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int c = 8 * i + 2 * (lane & 3);
            if (c >= tail) { sc[4 * i] = -INFINITY; sc[4 * i + 2] = -INFINITY; }
            if (c + 1 >= tail) { sc[4 * i + 1] = -INFINITY; sc[4 * i + 3] = -INFINITY; }
          }
        }
        // ---- online softmax (the 4 lanes of a quad share a row) ----
        float x0 = sc[0], x1 = sc[2];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          x0 = fmaxf(x0, fmaxf(sc[4 * i], sc[4 * i + 1]));
          x1 = fmaxf(x1, fmaxf(sc[4 * i + 2], sc[4 * i + 3]));
        }
        x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 1)); x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 2));
        x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 1)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 2));
        const float n0 = fmaxf(m0, x0), n1 = fmaxf(m1, x1);   // finite: every block holds at least one valid key
        const float a0 = mh_ex2(m0 - n0), a1 = mh_ex2(m1 - n1);
        m0 = n0; m1 = n1;
        l0 *= a0; l1 *= a1;
#pragma unroll
        for (int i = 0; i < 8; ++i) { o[4 * i] *= a0; o[4 * i + 1] *= a0; o[4 * i + 2] *= a1; o[4 * i + 3] *= a1; }
        uint32_t pa[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          pa[kk][0] = mh_exp2_pack(sc[8 * kk + 0], sc[8 * kk + 1], m0, l0);
          pa[kk][1] = mh_exp2_pack(sc[8 * kk + 2], sc[8 * kk + 3], m1, l1);
          pa[kk][2] = mh_exp2_pack(sc[8 * kk + 4], sc[8 * kk + 5], m0, l0);
          pa[kk][3] = mh_exp2_pack(sc[8 * kk + 6], sc[8 * kk + 7], m1, l1);
        }
        // ---- O += P V (MN-major B: 8 keys x 16 B (8 dims) per core matrix, next 8 keys +128 B (LBO), next 8 dims +chunk (SBO)) ----
        tc::wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          tc::Mma<64>::rs<1>(o, pa[kk], tc::make_desc_kmajor_noswz(vbase + kk * 256, 128, kMhKChunk), 1u);
        tc::wg_commit();
        tc::wg_wait<0>();
        tc::wg_fence_acc<32>(o);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
          for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(pa[kk][j])::"memory");   // A registers stay live until the wait
        if (wid == 0 && lane == 0) tc::mbar_arrive(&kv_empty[ks]);
        if (++ks == kMhStages) { ks = 0; kph ^= 1u; }
      }
      // ---- epilogue: O / l -> fp16 NC8 (one row and 8 dims per thread after each 16-dim slice exchange) ----
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
      for (int i = 0; i < 8; ++i) { o[4 * i] *= i0; o[4 * i + 1] *= i0; o[4 * i + 2] *= i1; o[4 * i + 3] *= i1; }
      const int qt = (int)(f % p.nqt);
      const long long bh = f / p.nqt;
      const int h = (int)(bh % p.heads), b = (int)(bh / p.heads);
      const long long r = (long long)qt * 128 + 64 * g + 32 * (wid & 1) + lane;
      __half* ob = p.out + (((long long)b * p.C8 + (long long)h * kMhChunks) * S + r) * 8;
#pragma unroll
      for (int c16 = 0; c16 < kMhDim / 16; ++c16, ++sl) {
        float* buf = stage + (sl & 1) * tc::kStageFloats;
        tc::wg_stage16<0>(o + c16 * 8, buf, wid, lane);
        tc::wg_bar(8 + g);
        float v[8];
        tc::wg_read8(buf, wid, lane, v);
        if (r < S) {
          uint4 hv;
          __half2* hp = reinterpret_cast<__half2*>(&hv);
#pragma unroll
          for (int j = 0; j < 4; ++j) hp[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
          *reinterpret_cast<uint4*>(ob + (long long)(2 * c16 + (wid >> 1)) * S * 8) = hv;
        }
      }
    }
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_mhsa_tc(const void* qkv, int N, int C, int heads, long long S, void* out, void* stream) {
  B200_REQUIRE(qkv && out, "mhsa_tc: null pointer");
  B200_REQUIRE(N > 0 && heads > 0 && S > 0, "mhsa_tc: empty problem (N = %d, heads = %d, S = %lld)", N, heads, S);
  if (C != heads * kMhDim)
    return set_err(B200_ERR_UNSUPPORTED, "mhsa_tc: head_dim must be 64 (C = %d, heads = %d)", C, heads);
  B200_REQUIRE(S <= (1LL << 30), "mhsa_tc: %lld tokens exceed the supported sequence length", S);
  MhsaTcParams p;
  p.qkv = (const __half*)qkv; p.out = (__half*)out;
  p.C8 = C / 8; p.heads = heads; p.S = S;
  p.nqt = (int)ceil_div(S, 128); p.nkb = (int)ceil_div(S, kMhKeys);
  p.total = (long long)N * heads * p.nqt;
  dim3 grid((unsigned)std::min<long long>(p.total, num_sms()));
  // per-device attribute: set on every call (cheap), so a second GPU in the same process works
  B200_CUDA(cudaFuncSetAttribute(mhsa_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMhSmem));
  mhsa_tc_kernel<<<grid, kMhThreads, kMhSmem, (cudaStream_t)stream>>>(p);
  B200_LAUNCH_CHECK("mhsa_tc_kernel");
  return B200_OK;
}
