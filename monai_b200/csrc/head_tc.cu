// Output head on Hopper wgmma tensor cores (SURVEY.md §8 rows a9, a14): the tail of the last residual block fused with UnetOutBlock,
//     logits = W_out * lrelu(instnorm(y2) + instnorm(res)) + b_out
// (monai/networks/blocks/dynunet_block.py:104-111 followed by 247-267: norm2 + residual (norm3 of the 1x1x1 branch, or the block
// input) + LeakyReLU, then the 1x1x1 convolution to <= 16 classes) for C = 48 input channels.
//
// Why: the CUDA-core version (swin.cu: head_conv_norm_nc8_kernel) spends 2 100 instructions per voxel -- 14 x 48 FMAs plus the
// weight reads -- and runs at 1.8 TB/s (ncu: 49 % issue-active with 24 resident warps).  Here the 48 -> 16 contraction is one
// MMA (M = 128 voxels, N = 16, K = 48) and the threads only normalise: per 128-voxel tile
//   bulk copies of the y2 and residual tiles (NC8 rows: 2 KB per 8-channel chunk)  ->  t = lrelu(y2 * sc + sh + res * rsc + rsh),
//   fp16, written in place over the y2 tile = the K-major core-matrix image of the A operand  ->  wgmma into registers  ->
//   + bias  ->  NCDHW logits (fp16 / fp32).
// The per-(batch item, channel) scale / shift tables of ALL batch items are built once per CTA in shared memory.
//
// Warp roles (384 threads, one persistent CTA per SM): warp 0 = copy producer, warps 4-7 and 8-11 = two "row" warpgroups that
// alternate tiles (transform of the tile, its two m64 wgmma chains, output); four operand stages keep ~96 KB of loads in
// flight per SM.
#include "common.cuh"
#include "tc90.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

constexpr int kHdC = 48, kHdN = 16;
constexpr int kHdTile = (kHdC / 8) * 2048;            // one operand tile: 6 chunks of 128 rows x 16 B
constexpr int kHdWBytes = kHdN * kHdC * 2;
constexpr int kHdMaxTab = 64 * 1024;                  // scale / shift tables: N * C * 16 bytes
constexpr int kHdStages = 4;                          // operand tiles in flight per SM (4 x 24 KB: the HBM latency-bandwidth product)

struct HeadTcParams {
  const __half* x; const __half* res; const float* stats; const float* res_stats; const float* wgt; const float* bias;
  void* y;
  int N, Cout, res_ctot, res_coff;
  long long S;
  float eps, slope;
};

template <typename TO>
__global__ void __launch_bounds__(384, 1) head_conv_norm_tc_kernel(HeadTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = tc::align_smem128(smem_raw);
  uint8_t* s_x = smem;                                  // [kHdStages] y2 tiles (raw, then t in place)
  uint8_t* s_r = s_x + kHdStages * kHdTile;             // [kHdStages] residual tiles
  uint8_t* s_w = s_r + kHdStages * kHdTile;             // B image of W_out (16 x 48)
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_w + kHdWBytes);
  uint64_t* x_full = bars;                      // [kHdStages] tx
  uint64_t* x_free = bars + kHdStages;          // [kHdStages] one arrival: the MMAs of the stage have completed
  float* s_bias = reinterpret_cast<float*>(bars + 3 * kHdStages + 6);  // [16]
  float* s_out = s_bias + 16;                   // [2 row groups][16 cout][128 rows] accumulator transpose
  float4* s_tab = reinterpret_cast<float4*>(s_out + 2 * 16 * 128);   // [N][48] {sc, sh, rsc, rsh}

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int row_tiles = (int)((p.S + 127) / 128);
  const long long total = (long long)p.N * row_tiles;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kHdStages; ++i) { tc::mbar_init(&x_full[i], 1); tc::mbar_init(&x_free[i], 1); }
    tc::fence_barrier_init();
  }
  {  // rows a clamped bulk copy never writes must hold finite values
    const uint4 z = make_uint4(0, 0, 0, 0);
    uint4* zx = reinterpret_cast<uint4*>(s_x);
    for (int i = threadIdx.x; i < 2 * kHdStages * kHdTile / 16; i += blockDim.x) zx[i] = z;
  }
  {  // B image [k16][khalf][2 groups][8 cout][8 k] (the gemm_tc packing with NT = 16); rows >= Cout are zero
    __half* sb = reinterpret_cast<__half*>(s_w);
    for (int i = threadIdx.x; i < kHdN * kHdC; i += blockDim.x) {
      int r = i;
      const int kk = r % 8; r /= 8;
      const int rw = r % 8; r /= 8;
      const int g = r % 2; r /= 2;
      const int khalf = r % 2; r /= 2;
      const int k16 = r;
      const int co = g * 8 + rw, k = k16 * 16 + khalf * 8 + kk;
      sb[i] = __float2half_rn(co < p.Cout ? p.wgt[co * kHdC + k] : 0.f);
    }
    for (int i = threadIdx.x; i < 16; i += blockDim.x) s_bias[i] = (i < p.Cout && p.bias) ? p.bias[i] : 0.f;
    const float invS = 1.f / (float)p.S;
    for (int i = threadIdx.x; i < p.N * kHdC; i += blockDim.x) {
      // same statistics arithmetic as norm_act_nc8_kernel
      const float s = p.stats[2 * i], q = p.stats[2 * i + 1];
      const float mean = s * invS, var = fmaxf(q * invS - mean * mean, 0.f), rstd = 1.f / sqrtf(var + p.eps);
      float4 t = make_float4(rstd, -mean * rstd, 1.f, 0.f);
      if (p.res_stats) {
        const float rs = p.res_stats[2 * i], rq = p.res_stats[2 * i + 1];
        const float rmean = rs * invS, rvar = fmaxf(rq * invS - rmean * rmean, 0.f), rrstd = 1.f / sqrtf(rvar + p.eps);
        t.z = rrstd; t.w = -rmean * rrstd;
      }
      s_tab[i] = t;
    }
  }
  tc::fence_proxy_async();
  __syncthreads();

  if (warp == 0) {
    // ===================== producer =====================
    if (lane == 0) {
      int it = 0;
      for (long long t = blockIdx.x; t < total; t += gridDim.x, ++it) {
        const int b = it % kHdStages;
        const uint32_t ph = (uint32_t)((it / kHdStages) & 1);
        const int n = (int)(t / row_tiles), rt = (int)(t % row_tiles);
        const int rows = (int)min((long long)128, p.S - (long long)rt * 128);
        tc::mbar_wait(&x_free[b], ph ^ 1);
        tc::mbar_arrive_expect_tx(&x_full[b], 2 * (kHdC / 8) * rows * 16);
        const __half* xs = p.x + ((long long)n * (kHdC / 8) * p.S + (long long)rt * 128) * 8;
        const __half* rs = p.res + (((long long)n * (p.res_ctot / 8) + p.res_coff / 8) * p.S + (long long)rt * 128) * 8;
        for (int c = 0; c < kHdC / 8; ++c) {
          tc::bulk_load(s_x + b * kHdTile + c * 2048, xs + (long long)c * p.S * 8, rows * 16, &x_full[b]);
          tc::bulk_load(s_r + b * kHdTile + c * 2048, rs + (long long)c * p.S * 8, rows * 16, &x_full[b]);
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    // ===================== row groups: group g (a warpgroup) takes every other tile: transform, MMA, output =====================
    const int g = (warp >> 2) - 1;            // 0 / 1 = tile parity
    const int wid = warp & 3;
    const int row = wid * 32 + lane;
    const float slope = p.slope;
    const uint32_t x_a = tc::smem_u32(s_x), w_a = tc::smem_u32(s_w);
    float* so = s_out + g * 16 * 128;
    int it = g;
    for (long long t = (long long)blockIdx.x + (long long)g * gridDim.x; t < total; t += 2LL * gridDim.x, it += 2) {
      const int st = it % kHdStages;
      const int n = (int)(t / row_tiles), rt = (int)(t % row_tiles);
      tc::mbar_wait(&x_full[st], (uint32_t)((it / kHdStages) & 1));
      uint8_t* xr = s_x + st * kHdTile + row * 16;
      const uint8_t* rr = s_r + st * kHdTile + row * 16;
      const float4* tab = s_tab + n * kHdC;
#pragma unroll
      for (int c = 0; c < kHdC / 8; ++c) {
        const uint4 xv = *reinterpret_cast<const uint4*>(xr + c * 2048), rv = *reinterpret_cast<const uint4*>(rr + c * 2048);
        const __half2* xh = reinterpret_cast<const __half2*>(&xv);
        const __half2* rh = reinterpret_cast<const __half2*>(&rv);
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 a = __half22float2(xh[j]), b = __half22float2(rh[j]);
          const float4 k0 = tab[c * 8 + 2 * j], k1 = tab[c * 8 + 2 * j + 1];
          float f0 = fmaf(a.x, k0.x, k0.y) + fmaf(b.x, k0.z, k0.w);
          float f1 = fmaf(a.y, k1.x, k1.y) + fmaf(b.y, k1.z, k1.w);
          f0 = f0 >= 0.f ? f0 : f0 * slope;
          f1 = f1 >= 0.f ? f1 : f1 * slope;
          oh[j] = __floats2half2_rn(f0, f1);
        }
        *reinterpret_cast<uint4*>(xr + c * 2048) = o;
      }
      tc::fence_proxy_async();   // generic-proxy stores -> visible to the wgmma operand reads
      tc::wg_bar(8 + g);         // the whole 128-row A image is written (and the previous tile's s_out reads are done)
      float acc[2][kHdN / 2];
      tc::wg_fence();
#pragma unroll
      for (int k = 0; k < kHdC / 16; ++k) {
        const uint64_t bd = tc::make_desc_kmajor_noswz(w_a + k * kHdN * 32, kHdN * 16, 128);
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          const uint64_t ad = tc::make_desc_kmajor_noswz(x_a + st * kHdTile + k * 4096 + m * 1024, 2048, 128);
          tc::wg_mma_ss<kHdN>(acc[m], ad, bd, k != 0 ? 1u : 0u, 128);
        }
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc<kHdN / 2>(acc[0]);
      tc::wg_fence_acc<kHdN / 2>(acc[1]);
      if (wid == 0 && lane == 0) tc::mbar_arrive(&x_free[st]);
      // fragment (rows 64 m + 16 wid + lane/4 (+8), columns 8 i + 2 (lane%4) (+1)) -> [cout][row] -> one row per thread
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int i = 0; i < kHdN / 8; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int r = 64 * m + 16 * wid + (lane >> 2) + 8 * (e >> 1), c = 8 * i + 2 * (lane & 3) + (e & 1);
            so[c * 128 + r] = acc[m][4 * i + e];
          }
      tc::wg_bar(8 + g);
      const long long r = (long long)rt * 128 + row;
      if (r < p.S) {
        TO* yo = (TO*)p.y + (long long)n * p.Cout * p.S + r;
#pragma unroll
        for (int o = 0; o < 16; ++o)
          if (o < p.Cout) io<TO>::st(yo + (long long)o * p.S, so[o * 128 + row] + s_bias[o]);
      }
    }
  }
}

// host side: launch if the shape is covered (C = 48, a residual, tables fit); returns B200_ERR_UNSUPPORTED otherwise
int launch_head_conv_norm_tc(const void* x, int N, int C, long long S, const float* stats, float eps, const void* res, int res_ctot,
                             int res_coff, const float* res_stats, float slope, const float* weight, const float* bias, int Cout,
                             void* y, int out_dtype, cudaStream_t st) {
  if (C != kHdC || !res || (long long)N * C * 16 > kHdMaxTab || Cout > 16) return B200_ERR_UNSUPPORTED;
  HeadTcParams p{(const __half*)x, (const __half*)res, stats, res_stats, weight, bias, y, N, Cout, res_ctot, res_coff, S, eps, slope};
  const int smem = 2 * kHdStages * kHdTile + kHdWBytes + (3 * kHdStages + 6) * 8 + 64 + 2 * 16 * 128 * 4 + N * C * 16 + 128;
  const long long total = (long long)N * ((S + 127) / 128);
  dim3 grid((unsigned)std::min<long long>(total, num_sms()));
  if (out_dtype == B200_DT_F16) {
    B200_CUDA(cudaFuncSetAttribute(head_conv_norm_tc_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    head_conv_norm_tc_kernel<__half><<<grid, 384, smem, st>>>(p);
  } else {
    B200_CUDA(cudaFuncSetAttribute(head_conv_norm_tc_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    head_conv_norm_tc_kernel<float><<<grid, 384, smem, st>>>(p);
  }
  B200_LAUNCH_CHECK("head_conv_norm_tc_kernel");
  return B200_OK;
}

}  // namespace b200
