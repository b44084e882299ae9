// Fused transformer MLP on Hopper wgmma tensor cores (SURVEY.md §8 rows a12, a13):
//     out = x + W2 * gelu(W1 * LayerNorm(x) + b1) + b2
// i.e. norm2 + MLPBlock + the residual add of SwinTransformerBlock.forward (monai/networks/nets/swin_unetr.py:675-698 with
// monai/networks/blocks/mlp.py:75-80) in ONE kernel for C = 48 tokens (stage 1 of SwinUNETR fs48).
//
// Why: as separate launches the 4C-wide hidden tensor is written by fc1 and read again by fc2 (768 of the 1 344 bytes the MLP
// moves per token) and LayerNorm is a pass of its own.  Here a 128-token tile flows through
//   bulk copy X (NC8 rows: one contiguous 2 KB piece per 8-channel chunk)  ->  LayerNorm in place in shared memory (a thread
//   per token)  ->  GEMM1 [64 x 48] x W1^T per warpgroup into registers (192 fp32 columns)  ->  + b1, GELU, fp16 -- the
//   accumulator fragment of GEMM1 IS the register A operand of GEMM2 (same row / column ownership), so the hidden activations
//   never leave the registers  ->  GEMM2 [64 x 192] x W2^T (48 columns)  ->  + b2 + x  ->  NC8.
// Both weight matrices (2 x 18 KB as wgmma B images, the same packing as gemm_tc.cu) stay resident in shared memory.
//
// Warp roles (384 threads, one persistent CTA per SM):
//   warp 0      producer: weights once, then one X tile per iteration (2-stage ring);
//   warps 4-11  two consumer warpgroups, rows 0-63 / 64-127 of every tile: LayerNorm, GEMM1, GELU, GEMM2, epilogue.
#include "common.cuh"
#include "tc90.cuh"
#include "gelu.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

constexpr int kMlpC = 48, kMlpH = 192;
constexpr int kMlpXBytes = (kMlpC / 8) * 2048;        // one X tile: 6 chunks of 128 rows x 16 B
constexpr int kMlpW1Bytes = kMlpH * kMlpC * 2, kMlpW2Bytes = kMlpC * kMlpH * 2;
constexpr int kMlpParFloats = 3 * kMlpC + kMlpH;     // gamma, beta, b2, b1
constexpr int kMlpSmem = 2 * kMlpXBytes + kMlpW1Bytes + kMlpW2Bytes + 256 + kMlpParFloats * 4 + 2 * 2 * tc::kStageFloats * 4 + 128;
constexpr int kMlpThreads = 384;

struct MlpParams {
  const __half* x; __half* y; const __half* w1; const __half* w2;
  const float* b1; const float* b2; const float* gamma; const float* beta;
  float eps;
  int Nb, S;            // batch items, tokens per item
  int x_ctot, y_ctot;   // channel counts of the NC8 buffers (== 48)
};

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(kMlpThreads, 1) mlp_fused_tc_kernel(MlpParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = tc::align_smem128(smem_raw);   // keeps the shared address space (LDS/STS, not generic LD/ST)
  uint8_t* s_x = smem;                                  // [2] X tiles (raw, then normalised in place)
  uint8_t* s_w1 = s_x + 2 * kMlpXBytes;
  uint8_t* s_w2 = s_w1 + kMlpW1Bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_w2 + kMlpW2Bytes);
  uint64_t* x_full = bars;          // [2] tx
  uint64_t* x_free = bars + 2;      // [2] one arrival per consumer warpgroup (GEMM1 has read its half of the tile)
  uint64_t* w_full = bars + 4;      // tx
  float* s_gamma = reinterpret_cast<float*>(bars + 32);   // 256 bytes of barrier space precede the parameter table
  float* s_beta = s_gamma + kMlpC;
  float* s_b2 = s_beta + kMlpC;
  float* s_b1 = s_b2 + kMlpC;
  float* s_stage = s_b1 + kMlpH;                         // [2 warpgroups][2][kStageFloats]

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int row_tiles = (p.S + 127) / 128;
  const long long total = (long long)p.Nb * row_tiles;

  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { tc::mbar_init(&x_full[i], 1); tc::mbar_init(&x_free[i], 2); }
    tc::mbar_init(w_full, 1);
    tc::fence_barrier_init();
  }
  {  // rows a clamped bulk copy never writes must hold finite values
    const uint4 z = make_uint4(0, 0, 0, 0);
    uint4* zx = reinterpret_cast<uint4*>(s_x);
    for (int i = threadIdx.x; i < 2 * kMlpXBytes / 16; i += blockDim.x) zx[i] = z;
  }
  for (int i = threadIdx.x; i < kMlpC; i += blockDim.x) {
    s_gamma[i] = p.gamma ? p.gamma[i] : 1.f; s_beta[i] = p.beta ? p.beta[i] : 0.f; s_b2[i] = p.b2[i];
  }
  for (int i = threadIdx.x; i < kMlpH; i += blockDim.x) s_b1[i] = p.b1[i];
  tc::fence_proxy_async();
  __syncthreads();

  if (warp == 0) {
    // ===================== producer =====================
    if (lane == 0) {
      tc::mbar_arrive_expect_tx(w_full, kMlpW1Bytes + kMlpW2Bytes);
      tc::bulk_load(s_w1, p.w1, kMlpW1Bytes, w_full);
      tc::bulk_load(s_w2, p.w2, kMlpW2Bytes, w_full);
      int it = 0;
      for (long long t = blockIdx.x; t < total; t += gridDim.x, ++it) {
        const int b = it & 1;
        const uint32_t ph = (uint32_t)((it >> 1) & 1);
        const int n = (int)(t / row_tiles), rt = (int)(t % row_tiles);
        const int rows = min(128, p.S - rt * 128);
        tc::mbar_wait(&x_free[b], ph ^ 1);
        tc::mbar_arrive_expect_tx(&x_full[b], (kMlpC / 8) * rows * 16);
        const __half* src = p.x + ((long long)n * (p.x_ctot / 8) * p.S + rt * 128) * 8;
        for (int c = 0; c < kMlpC / 8; ++c) tc::bulk_load(s_x + b * kMlpXBytes + c * 2048, src + (long long)c * p.S * 8, rows * 16, &x_full[b]);
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    const int g = (warp >> 2) - 1, wid = warp & 3;
    const uint32_t x_a = tc::smem_u32(s_x), w1_a = tc::smem_u32(s_w1), w2_a = tc::smem_u32(s_w2);
    float* stage = s_stage + g * 2 * tc::kStageFloats;
    const int c_lane = 2 * (lane & 3);        // first fragment column of this thread inside each 8-column block
    int sl = 0;
    tc::mbar_wait(w_full, 0u);
    int it = 0;
    for (long long t = blockIdx.x; t < total; t += gridDim.x, ++it) {
      const int b = it & 1;
      const uint32_t ph = (uint32_t)((it >> 1) & 1);
      const int n = (int)(t / row_tiles), rt = (int)(t % row_tiles);
      tc::mbar_wait(&x_full[b], ph);
      // ---- LayerNorm of the warpgroup's 64 rows, in place (warps 0-1 of the group, one row per thread) ----
      if (wid < 2) {
        uint8_t* xr = s_x + b * kMlpXBytes + (64 * g + 32 * wid + lane) * 16;
        float f[kMlpC];
#pragma unroll
        for (int c = 0; c < kMlpC / 8; ++c) {
          const uint4 raw = *reinterpret_cast<const uint4*>(xr + c * 2048);
          const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
          for (int j = 0; j < 4; ++j) { const float2 v = __half22float2(h2[j]); f[c * 8 + 2 * j] = v.x; f[c * 8 + 2 * j + 1] = v.y; }
        }
        float sum = 0.f;
#pragma unroll
        for (int c = 0; c < kMlpC; ++c) sum += f[c];
        const float mean = sum * (1.f / kMlpC);
        float var = 0.f;
#pragma unroll
        for (int c = 0; c < kMlpC; ++c) { const float d = f[c] - mean; var = fmaf(d, d, var); }
        const float rstd = 1.f / sqrtf(var * (1.f / kMlpC) + p.eps);
#pragma unroll
        for (int c = 0; c < kMlpC / 8; ++c) {
          uint4 o;
          __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int k = c * 8 + 2 * j;
            oh[j] = __floats2half2_rn((f[k] - mean) * rstd * s_gamma[k] + s_beta[k], (f[k + 1] - mean) * rstd * s_gamma[k + 1] + s_beta[k + 1]);
          }
          *reinterpret_cast<uint4*>(xr + c * 2048) = o;
        }
        tc::fence_proxy_async();   // generic-proxy stores -> visible to the wgmma operand reads
      }
      tc::wg_bar(8 + g);
      // ---- GEMM1: D1 = LN(X) * W1^T (64 x 192) ----
      float d1[kMlpH / 2];
      tc::wg_fence();
#pragma unroll
      for (int k = 0; k < kMlpC / 16; ++k) {
        const uint64_t ad = tc::make_desc_kmajor_noswz(x_a + b * kMlpXBytes + k * 4096 + g * 1024, 2048, 128);
        const uint64_t bd = tc::make_desc_kmajor_noswz(w1_a + k * kMlpH * 32, kMlpH * 16, 128);
        tc::wg_mma_ss<kMlpH>(d1, ad, bd, k != 0 ? 1u : 0u, 128);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc<kMlpH / 2>(d1);
      if (wid == 0 && lane == 0) tc::mbar_arrive(&x_free[b]);
      // ---- + b1, GELU, fp16: the D1 fragment of columns 16k .. 16k+15 is the A fragment of K-step k of GEMM2 ----
      uint32_t a[kMlpH / 16][4];
#pragma unroll
      for (int k = 0; k < kMlpH / 16; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = 16 * k + 8 * (j >> 1) + c_lane;
          const float* dv = d1 + 8 * k + 2 * j;
          a[k][j] = pack_half2(gelu_erf(dv[0] + s_b1[col]), gelu_erf(dv[1] + s_b1[col + 1]));
        }
      // ---- GEMM2: D2 = H * W2^T (64 x 48) ----
      float d2[kMlpC / 2];
      tc::wg_fence();
#pragma unroll
      for (int k = 0; k < kMlpH / 16; ++k) {
        const uint64_t bd = tc::make_desc_kmajor_noswz(w2_a + k * kMlpC * 32, kMlpC * 16, 128);
        tc::Mma<kMlpC>::rs<0>(d2, a[k], bd, k != 0 ? 1u : 0u);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc<kMlpC / 2>(d2);
#pragma unroll
      for (int k = 0; k < kMlpH / 16; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(a[k][j])::"memory");   // A registers stay live until the wait
      // ---- epilogue: + b2 + x (the raw row, re-read from global memory: an L2 hit), NC8 store ----
      const int r = rt * 128 + 64 * g + 32 * (wid & 1) + lane;
      const bool ok = r < p.S;
#pragma unroll
      for (int c16 = 0; c16 < kMlpC / 16; ++c16, ++sl) {
        float* buf = stage + (sl & 1) * tc::kStageFloats;
        tc::wg_stage16<0>(d2 + c16 * 8, buf, wid, lane);
        tc::wg_bar(8 + g);
        float v[8];
        tc::wg_read8(buf, wid, lane, v);
        const int c = 2 * c16 + (wid >> 1);
        if (ok) {
          const uint4 res = __ldg(reinterpret_cast<const uint4*>(p.x + ((long long)n * (p.x_ctot / 8) * p.S + r) * 8 + (long long)c * p.S * 8));
          const __half2* rh = reinterpret_cast<const __half2*>(&res);
          uint4 o;
          __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 rr = __half22float2(rh[j]);
            const int k = c * 8 + 2 * j;
            oh[j] = __floats2half2_rn(v[2 * j] + s_b2[k] + rr.x, v[2 * j + 1] + s_b2[k + 1] + rr.y);
          }
          *reinterpret_cast<uint4*>(p.y + ((long long)n * (p.y_ctot / 8) * p.S + r) * 8 + (long long)c * p.S * 8) = o;
        }
      }
    }
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_mlp_fused_tc(const void* x, int x_ctot, int Nb, int S, int C, int hidden, const void* packed_w1, const float* b1,
                                 const void* packed_w2, const float* b2, const float* gamma, const float* beta, float eps, void* y,
                                 int y_ctot, void* stream) {
  B200_REQUIRE(x && y && packed_w1 && packed_w2 && b1 && b2, "mlp_fused_tc: null pointer");
  B200_REQUIRE(C == kMlpC && hidden == kMlpH, "mlp_fused_tc: implemented for C = 48, hidden = 192 (got %d, %d)", C, hidden);
  B200_REQUIRE(x_ctot == C && y_ctot == C, "mlp_fused_tc: the token buffers must hold exactly C channels");
  B200_REQUIRE(Nb > 0 && S > 0, "mlp_fused_tc: empty problem");
  MlpParams p;
  p.x = (const __half*)x; p.y = (__half*)y; p.w1 = (const __half*)packed_w1; p.w2 = (const __half*)packed_w2;
  p.b1 = b1; p.b2 = b2; p.gamma = gamma; p.beta = beta; p.eps = eps; p.Nb = Nb; p.S = S; p.x_ctot = x_ctot; p.y_ctot = y_ctot;
  B200_CUDA(cudaFuncSetAttribute(mlp_fused_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMlpSmem));
  const long long total = (long long)Nb * ((S + 127) / 128);
  dim3 grid((unsigned)std::min<long long>(total, num_sms()));
  mlp_fused_tc_kernel<<<grid, kMlpThreads, kMlpSmem, (cudaStream_t)stream>>>(p);
  B200_LAUNCH_CHECK("mlp_fused_tc_kernel");
  return B200_OK;
}
