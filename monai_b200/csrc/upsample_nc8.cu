// Decoder join of SegResNet on NC8 buffers: y = up(x) + skip, with optional deterministic InstanceNorm / GroupNorm statistics of y
// (monai/networks/nets/segresnet.py decode: `up(x) + down_x[i + 1]`, where up = 1x1x1 conv + nn.Upsample(trilinear,
// align_corners=False) or a transposed convolution k2 s2).
//
// scale 2: trilinear x2 with align_corners=False -- along each axis the source coordinate of output o is o / 2 - 0.25, clamped at 0,
// so the stencil is fixed: output 2i = 0.75 x[i] + 0.25 x[max(i - 1, 0)], output 2i + 1 = 0.75 x[i] + 0.25 x[min(i + 1, n - 1)]
// (what F.interpolate computes), evaluated in fp32 as nested lerps, W innermost.  scale 1: a plain add (the transposed-convolution
// upsample already ran on gemm_tc).  The kernel is bound by HBM: x once (the eight corner reads of a voxel hit L1 / L2), skip and y
// once each.
//
// Statistics (stats.cuh): one block per (batch item, 8-channel chunk, slice of voxels); a thread walks a fixed strided subset of the
// voxels, the block combines its threads in a fixed order and writes one partial row, and launch_stats_finish adds the rows in fp64.
// No floating-point atomics: the sums are the same bits on every run.
//
// Also here: the 2x max pool of BasicUNet's encoder (basic_unet.py Down: nn.MaxPool3d(2)) on NC8 channel slices.  One thread per
// (output voxel, 8-channel chunk) makes eight 16-byte loads and one 16-byte store; like the decoder join it is bound by HBM.
#include "common.cuh"
#include "stats.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

struct UpAddP {
  const __half* x; const __half* skip; __half* y;
  int x_ctot, x_coff, s_ctot, s_coff, y_ctot, y_coff;
  int C, D, H, W;             // x: low resolution
  int Do, Ho, Wo;             // skip / y
  float* part;                // [N][C/8][gridDim.x][16] {sum, sumsq} per channel, or NULL
};

__device__ __forceinline__ void ld8(const __half* p, float (&v)[8]) {
  const uint4 r = __ldg(reinterpret_cast<const uint4*>(p));
  const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
  for (int k = 0; k < 4; ++k) { const float2 f = __half22float2(h[k]); v[2 * k] = f.x; v[2 * k + 1] = f.y; }
}

// the two source indices of output o along an axis of n source voxels (weights 0.75, 0.25)
__device__ __forceinline__ int2 up2_src(int o, int n) {
  const int i = o >> 1;
  return make_int2(i, (o & 1) ? min(i + 1, n - 1) : max(i - 1, 0));
}

template <int SCALE>
__global__ void __launch_bounds__(256) upsample_add_nc8_kernel(UpAddP p) {
  const int chunk = blockIdx.y, n = blockIdx.z;
  const long long Si = (long long)p.D * p.H * p.W, So = (long long)p.Do * p.Ho * p.Wo;
  const __half* xs = p.x + (((long long)n * (p.x_ctot / 8) + p.x_coff / 8 + chunk) * Si) * 8;
  const __half* ss = p.skip + (((long long)n * (p.s_ctot / 8) + p.s_coff / 8 + chunk) * So) * 8;
  __half* ys = p.y + (((long long)n * (p.y_ctot / 8) + p.y_coff / 8 + chunk) * So) * 8;
  float bs[8], bq[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { bs[j] = 0.f; bq[j] = 0.f; }
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < So; s += (long long)gridDim.x * blockDim.x) {
    float v[8], k[8];
    if constexpr (SCALE == 1) {
      ld8(xs + s * 8, v);
    } else {
      const int ow = (int)(s % p.Wo);
      const long long t = s / p.Wo;
      const int oh = (int)(t % p.Ho), od = (int)(t / p.Ho);
      const int2 sd = up2_src(od, p.D), sh = up2_src(oh, p.H), sw = up2_src(ow, p.W);
      float pl[2][8];   // the two D planes, each already interpolated along W and H
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const long long base = (long long)(a ? sd.y : sd.x) * p.H;
        float row[2][8];
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const long long r = (base + (b ? sh.y : sh.x)) * p.W;
          float u[8], w1[8];
          ld8(xs + (r + sw.x) * 8, u);
          ld8(xs + (r + sw.y) * 8, w1);
#pragma unroll
          for (int j = 0; j < 8; ++j) row[b][j] = 0.75f * u[j] + 0.25f * w1[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) pl[a][j] = 0.75f * row[0][j] + 0.25f * row[1][j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.75f * pl[0][j] + 0.25f * pl[1][j];
    }
    ld8(ss + s * 8, k);
    uint4 hv;
    __half2* hp = reinterpret_cast<__half2*>(&hv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[j] += k[j];
      bs[j] += v[j];
      bq[j] = fmaf(v[j], v[j], bq[j]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) hp[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
    *reinterpret_cast<uint4*>(ys + s * 8) = hv;
  }
  if (!p.part) return;
  // fixed-order block reduction: butterfly within each warp, then the warps in index order
  __shared__ float s_red[8][16];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float a = warp_sum(bs[j]), b = warp_sum(bq[j]);
    if (lane == 0) { s_red[wid][2 * j] = a; s_red[wid][2 * j + 1] = b; }
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w][threadIdx.x];
    p.part[(((long long)n * gridDim.y + chunk) * gridDim.x + blockIdx.x) * 16 + threadIdx.x] = t;
  }
}

// blocks per (batch item, chunk): enough for eight 256-thread blocks per SM in all, never more than the voxels need (also sizes
// the max pool's grid)
static int upsample_add_blocks(int N, int C, long long So) {
  const long long planes = (long long)N * (C / 8);
  const long long want = ((long long)num_sms() * 8 + planes - 1) / planes;
  return (int)std::max<long long>(1, std::min<long long>(want, (So + 255) / 256));
}

// y = max over the 2x2x2 cell of x, per channel; __hmax2_nan keeps a NaN, as torch's max pooling does
__global__ void __launch_bounds__(256) maxpool2_nc8_kernel(const __half* __restrict__ x, int x_ctot, int x_coff, __half* __restrict__ y,
                                                           int y_ctot, int y_coff, int D, int H, int W) {
  const int chunk = blockIdx.y, n = blockIdx.z;
  const int Do = D >> 1, Ho = H >> 1, Wo = W >> 1;
  const long long Si = (long long)D * H * W, So = (long long)Do * Ho * Wo;
  const __half* xs = x + (((long long)n * (x_ctot / 8) + x_coff / 8 + chunk) * Si) * 8;
  __half* ys = y + (((long long)n * (y_ctot / 8) + y_coff / 8 + chunk) * So) * 8;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < So; s += (long long)gridDim.x * blockDim.x) {
    const int ow = (int)(s % Wo);
    const long long t = s / Wo;
    const int oh = (int)(t % Ho), od = (int)(t / Ho);
    const __half* p = xs + (((long long)(2 * od) * H + 2 * oh) * W + 2 * ow) * 8;
    uint4 m = __ldg(reinterpret_cast<const uint4*>(p));
    __half2* mh = reinterpret_cast<__half2*>(&m);
#pragma unroll
    for (int k = 1; k < 8; ++k) {
      const long long off = ((long long)((k >> 2) & 1) * H * W + (long long)((k >> 1) & 1) * W + (k & 1)) * 8;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(p + off));
      const __half2* vh = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) mh[j] = __hmax2_nan(mh[j], vh[j]);
    }
    *reinterpret_cast<uint4*>(ys + s * 8) = m;
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_maxpool2_nc8(const void* x, int x_ctot, int x_coff, int N, int C, int D, int H, int W, void* y, int y_ctot, int y_coff,
                                 void* stream) {
  B200_REQUIRE(x && y, "maxpool2_nc8: null pointer");
  B200_REQUIRE(N > 0 && C > 0 && D > 0 && H > 0 && W > 0, "maxpool2_nc8: empty problem");
  B200_REQUIRE(C % 8 == 0 && x_ctot % 8 == 0 && x_coff % 8 == 0 && x_coff >= 0 && x_coff + C <= x_ctot,
               "maxpool2_nc8: bad channel slice of x (C %d, x_coff %d, x_ctot %d)", C, x_coff, x_ctot);
  B200_REQUIRE(y_ctot % 8 == 0 && y_coff % 8 == 0 && y_coff >= 0 && y_coff + C <= y_ctot,
               "maxpool2_nc8: bad channel slice of y (C %d, y_coff %d, y_ctot %d)", C, y_coff, y_ctot);
  B200_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0, "maxpool2_nc8: pointers must be 16-byte aligned");
  B200_REQUIRE(C / 8 <= 65535 && N <= 65535, "maxpool2_nc8: N or C too large for one launch");
  const long long So = (long long)(D / 2) * (H / 2) * (W / 2);
  if (So == 0) return B200_OK;
  dim3 grid(upsample_add_blocks(N, C, So), C / 8, N);
  maxpool2_nc8_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)x, x_ctot, x_coff, (__half*)y, y_ctot, y_coff, D, H, W);
  B200_LAUNCH_CHECK("maxpool2_nc8_kernel");
  return B200_OK;
}

extern "C" long long b200_upsample_add_nc8_workspace_bytes(int N, int C, int D, int H, int W, int scale) {
  if (N <= 0 || C <= 0 || C % 8 || D <= 0 || H <= 0 || W <= 0 || (scale != 1 && scale != 2)) return -1;
  const long long So = (long long)D * H * W * scale * scale * scale;
  return (long long)N * (C / 8) * upsample_add_blocks(N, C, So) * 16 * (long long)sizeof(float);
}

extern "C" int b200_upsample_add_nc8(const void* x, int x_ctot, int x_coff, int N, int C, int D, int H, int W, int scale,
                                     const void* skip, int skip_ctot, int skip_coff, void* y, int y_ctot, int y_coff, float* stats,
                                     void* workspace, void* stream) {
  B200_REQUIRE(x && skip && y, "upsample_add_nc8: null pointer");
  B200_REQUIRE(N > 0 && C > 0 && D > 0 && H > 0 && W > 0, "upsample_add_nc8: empty problem");
  B200_REQUIRE(scale == 1 || scale == 2, "upsample_add_nc8: scale must be 1 or 2 (got %d)", scale);
  B200_REQUIRE(C % 8 == 0 && x_ctot % 8 == 0 && x_coff % 8 == 0 && x_coff + C <= x_ctot, "upsample_add_nc8: bad channel slice of x");
  B200_REQUIRE(skip_ctot % 8 == 0 && skip_coff % 8 == 0 && skip_coff + C <= skip_ctot, "upsample_add_nc8: bad channel slice of skip");
  B200_REQUIRE(y_ctot % 8 == 0 && y_coff % 8 == 0 && y_coff + C <= y_ctot, "upsample_add_nc8: bad channel slice of y");
  B200_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(skip) | reinterpret_cast<uintptr_t>(y)) & 15) == 0,
               "upsample_add_nc8: pointers must be 16-byte aligned");
  B200_REQUIRE(!stats || workspace, "upsample_add_nc8: statistics need the workspace of b200_upsample_add_nc8_workspace_bytes()");
  B200_REQUIRE(C / 8 <= 65535 && N <= 65535, "upsample_add_nc8: N or C too large for one launch");
  UpAddP p;
  p.x = (const __half*)x; p.skip = (const __half*)skip; p.y = (__half*)y;
  p.x_ctot = x_ctot; p.x_coff = x_coff; p.s_ctot = skip_ctot; p.s_coff = skip_coff; p.y_ctot = y_ctot; p.y_coff = y_coff;
  p.C = C; p.D = D; p.H = H; p.W = W; p.Do = D * scale; p.Ho = H * scale; p.Wo = W * scale;
  p.part = stats ? (float*)workspace : nullptr;
  const long long So = (long long)p.Do * p.Ho * p.Wo;
  const int bx = upsample_add_blocks(N, C, So);
  dim3 grid(bx, C / 8, N);
  cudaStream_t st = (cudaStream_t)stream;
  if (scale == 2) upsample_add_nc8_kernel<2><<<grid, 256, 0, st>>>(p);
  else upsample_add_nc8_kernel<1><<<grid, 256, 0, st>>>(p);
  B200_LAUNCH_CHECK("upsample_add_nc8_kernel");
  if (stats) return launch_stats_finish((const float*)workspace, (long long)N * (C / 8), bx, 8, C / 8, C, stats, st);
  return B200_OK;
}
