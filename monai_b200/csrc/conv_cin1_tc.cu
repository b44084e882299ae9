// Single-input-channel convolutions on Hopper wgmma tensor cores (SURVEY.md §8 rows a8, a12, a14).
//
// Replaces, for a ONE-channel fp16/fp32 input volume,
//   * the 3x3x3 / stride 1 / pad 1 stem of UnetrBasicBlock.conv1 (monai/networks/blocks/dynunet_block.py:57-74), and
//   * PatchEmbed.proj, kernel 2 / stride 2 (monai/networks/blocks/patchembedding.py:141-219),
// which the CUDA-core kernel (swin.cu: conv_cin1_nc8_kernel) ran at 0.19 of HBM bandwidth: with Cout = 48 the 27-tap
// contraction is 1296 FMA per voxel, FMA-bound.  Here the contraction is an implicit GEMM with K = 27 -> 32 (8 -> 16):
//   M = 128 output voxels (a 16 x 8 patch of one D-plane, BD planes per tile), N = Cout, K = taps (zero padded),
// so the kernel is bound by the fp16 NC8 store of its output (2 * Cout bytes per voxel) instead.
//
// Warp roles (384 threads, one persistent CTA per SM):
//   warps 0-3  producers: stage the raw halo patch of a tile in shared memory (plain loads, zero outside the volume
//              = the convolution's zero padding), then build the im2col A operand -- thread r owns GEMM row r and
//              writes its K-vector as 16-byte pieces straight into the wgmma K-major / no-swizzle core-matrix image
//              ([k-chunk of 8][row][8 taps], LBO = 2048 B, SBO = 128 B); fence.proxy.async + mbarrier hand-over;
//   warps 4-11 two consumer warpgroups (rows 0-63 / 64-127 of the tile): BD x K/16 wgmma per tile with the accumulators in
//              registers, then the epilogue of conv_epi.cuh (bias, deterministic InstanceNorm sums, NC8 store).
// The weights [Cout][taps] fp32 are packed into the B image in shared memory once per CTA.
#include "common.cuh"
#include "tc90.cuh"
#include "conv_epi.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

template <int KS, int STRIDE, int NT, int BD>
struct Cin1Cfg {
  static constexpr int kTaps = KS * KS * KS;
  static constexpr int kKP = (kTaps + 15) / 16 * 16;             // padded K
  static constexpr int kHD = (BD - 1) * STRIDE + KS;             // halo extent of a tile
  static constexpr int kHHh = (kTH - 1) * STRIDE + KS;
  static constexpr int kHWw = (kTW - 1) * STRIDE + KS;
  static constexpr int kHaloElems = kHD * kHHh * kHWw;
  static constexpr int kHaloBytes = (kHaloElems * 2 + 127) / 128 * 128;
  static constexpr int kAPlane = (kKP / 8) * 2048;               // one plane's A tile: kKP/8 chunks of 128 rows x 16 B
  static constexpr int kAStage = BD * kAPlane;
  static constexpr int kStages = 2;
  static constexpr int kBBytes = NT * kKP * 2;
  static constexpr int kThreads = 384;                           // producer warpgroup + two consumer warpgroups
  static constexpr int kSmemBytes = kStages * (kAStage + kHaloBytes) + kBBytes + 256 + 4 * 2 * NT * 4 +
                                    2 * 2 * tc::kStageFloats * 4 + 128;
  static_assert(BD * NT <= 256, "accumulators exceed the register budget of a consumer thread");
  static_assert(NT % 16 == 0 && NT >= 16 && NT <= 256, "invalid wgmma N");
  static_assert(kSmemBytes <= 227 * 1024, "shared memory budget");
};

struct Cin1TcParams {
  const void* x;          // [N][1][D][H][W] raw volume
  const float* w;         // [Cout][taps]
  int D, H, W;            // INPUT spatial size
  int pad;
  ConvEpiP e;
};

__device__ __forceinline__ __half to_half(float v) { return __float2half_rn(v); }
__device__ __forceinline__ __half to_half(__half v) { return v; }

template <typename T, int KS, int STRIDE, int NT, int BD>
__global__ void __launch_bounds__(Cin1Cfg<KS, STRIDE, NT, BD>::kThreads, 1) conv_cin1_tc_kernel(Cin1TcParams p) {
  using Cfg = Cin1Cfg<KS, STRIDE, NT, BD>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = tc::align_smem128(smem_raw);   // keeps the shared address space (LDS/STS, not generic LD/ST)
  uint8_t* smem_a = smem;                                        // [kStages][BD][kKP/8][128][16 B]
  uint8_t* smem_h = smem_a + Cfg::kStages * Cfg::kAStage;        // [kStages] halo patches (fp16)
  uint8_t* smem_b = smem_h + Cfg::kStages * Cfg::kHaloBytes;     // packed weights
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + Cfg::kBBytes);
  uint64_t* a_full = bars;               // [2], 128 producer arrivals
  uint64_t* a_empty = bars + 2;          // [2], one arrival per consumer warpgroup
  float* s_stats = reinterpret_cast<float*>(bars + 32);          // [4][2*NT]
  float* s_stage = s_stats + 4 * 2 * NT;                         // [2 warpgroups][2][kStageFloats]

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { tc::mbar_init(&a_full[i], 128); tc::mbar_init(&a_empty[i], 2); }
    tc::fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 4 * 2 * NT; i += blockDim.x) s_stats[i] = 0.f;
  // B image [k16][khalf][NT/8][8 cout][8 k] (same as gemm_tc): element (cout, k) with k = (kd*KS + kh)*KS + kw
  {
    __half* sb = reinterpret_cast<__half*>(smem_b);
    const int co0 = 0;   // a single N tile (Cout == NT)
    for (int i = threadIdx.x; i < NT * Cfg::kKP; i += blockDim.x) {
      int r = i;
      const int kk = r % 8; r /= 8;
      const int row = r % 8; r /= 8;
      const int g = r % (NT / 8); r /= (NT / 8);
      const int khalf = r % 2; r /= 2;
      const int k16 = r;
      const int cout = co0 + g * 8 + row, k = k16 * 16 + khalf * 8 + kk;
      sb[i] = __float2half_rn(k < Cfg::kTaps ? p.w[cout * Cfg::kTaps + k] : 0.f);
    }
  }
  tc::fence_proxy_async();     // the generic-proxy writes of the weight image must be visible to the wgmma operand reads
  __syncthreads();

  if (warp < 4) {
    // ===================== producers: halo patch -> im2col A image =====================
    const int r = threadIdx.x;                     // GEMM row: h = r >> 3, w = r & 7 inside the 16 x 8 patch
    const int rh = (r >> 3) * STRIDE, rw = (r & 7) * STRIDE;
    const T* xg = reinterpret_cast<const T*>(p.x);
    // The raw halo patch of a tile is fetched into REGISTERS one tile ahead (all loads of a thread issued back to back, then
    // left in flight while the im2col of the current tile runs): a load -> convert -> store loop per element had the
    // producers waiting on one global-memory latency per element (9 in a row per tile) -- slower than the output store.
    constexpr int kHV = (Cfg::kHaloElems + 127) / 128;
    T hv[kHV];   // RAW values: converting here would make the warp wait for its loads inside fetch()
    auto fetch = [&](long long t) {
      const ConvTile c = conv_tile<BD>(p.e, t);
      const int z0 = c.d0 * STRIDE - p.pad, y0 = c.h0 * STRIDE - p.pad, x0 = c.w0 * STRIDE - p.pad;
      const T* xn = xg + (long long)c.n * p.D * p.H * p.W;
#pragma unroll
      for (int j = 0; j < kHV; ++j) {
        const int i = r + j * 128;
        const int hx = i % Cfg::kHWw, hy = (i / Cfg::kHWw) % Cfg::kHHh, hz = i / (Cfg::kHWw * Cfg::kHHh);
        const int iz = z0 + hz, iy = y0 + hy, ix = x0 + hx;
        const bool in = i < Cfg::kHaloElems && iz >= 0 && iz < p.D && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
        hv[j] = in ? __ldg(xn + ((long long)iz * p.H + iy) * p.W + ix) : T(0.f);
      }
    };
    if ((long long)blockIdx.x < p.e.total_tiles) fetch(blockIdx.x);
    int it = 0;
    for (long long t = blockIdx.x; t < p.e.total_tiles; t += gridDim.x, ++it) {
      const int st = it & 1;
      const uint32_t ph = (uint32_t)((it >> 1) & 1);
      tc::mbar_wait(&a_empty[st], ph ^ 1);         // the MMAs that read this stage's A image have completed
      __half* halo = reinterpret_cast<__half*>(smem_h + st * Cfg::kHaloBytes);
#pragma unroll
      for (int j = 0; j < kHV; ++j)
        if (r + j * 128 < Cfg::kHaloElems) halo[r + j * 128] = to_half(hv[j]);
      // all 128 producers have written the patch (and, transitively, finished reading the OTHER patch: a thread reaches
      // this barrier of tile i+1 only after its im2col of tile i)
      asm volatile("bar.sync 2, 128;" ::: "memory");
      if (t + gridDim.x < p.e.total_tiles) fetch(t + gridDim.x);   // next tile's patch: in flight during the im2col below
      uint8_t* a_st = smem_a + st * Cfg::kAStage;
#pragma unroll
      for (int pl = 0; pl < BD; ++pl) {
        __align__(16) __half kv[Cfg::kKP];
#pragma unroll
        for (int k = 0; k < Cfg::kKP; ++k) {
          if (k < Cfg::kTaps) {
            const int kd = k / (KS * KS), kh = (k / KS) % KS, kw = k % KS;
            kv[k] = halo[((pl * STRIDE + kd) * Cfg::kHHh + rh + kh) * Cfg::kHWw + rw + kw];
          } else {
            kv[k] = __float2half_rn(0.f);
          }
        }
#pragma unroll
        for (int ch = 0; ch < Cfg::kKP / 8; ++ch)
          *reinterpret_cast<uint4*>(a_st + pl * Cfg::kAPlane + ch * 2048 + r * 16) = *reinterpret_cast<const uint4*>(kv + ch * 8);
      }
      tc::fence_proxy_async();
      tc::mbar_arrive(&a_full[st]);
    }
  } else {
    // ===================== consumers: BD x K/16 wgmma per tile, then the epilogue of their 64 rows =====================
    const int g = (warp >> 2) - 1, wid = warp & 3;
    float* stage = s_stage + g * 2 * tc::kStageFloats;
    float* ws = s_stats + (2 * g + (wid & 1)) * (2 * NT);
    const uint32_t b_base = tc::smem_u32(smem_b);
    long long group = -1;
    int sl = 0, it = 0;
    for (long long t = blockIdx.x; t < p.e.total_tiles; t += gridDim.x, ++it) {
      const int st = it & 1;
      const uint32_t ph = (uint32_t)((it >> 1) & 1);
      const ConvTile c = conv_tile<BD>(p.e, t);
      float acc[BD * NT / 2];
      tc::mbar_wait(&a_full[st], ph);
      const uint32_t a_base = tc::smem_u32(smem_a + st * Cfg::kAStage) + g * 1024;
      tc::wg_fence();
      tc::static_for<0, BD>([&](auto plc) {
        constexpr int pl = decltype(plc)::value;
#pragma unroll
        for (int ks = 0; ks < Cfg::kKP / 16; ++ks) {
          const uint64_t adesc = tc::make_desc_kmajor_noswz(a_base + pl * Cfg::kAPlane + ks * 4096, 2048, 128);
          const uint64_t bdesc = tc::make_desc_kmajor_noswz(b_base + ks * NT * 32, NT * 16, 128);
          tc::wg_mma_ss<NT>(acc + pl * NT / 2, adesc, bdesc, ks != 0 ? 1u : 0u, 128);
        }
      });
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_fence_acc<BD * NT / 2>(acc);
      if (wid == 0 && lane == 0) tc::mbar_arrive(&a_empty[st]);
      conv_stats_turn(p.e, ws, NT, t, group, g, wid, lane);
      conv_epilogue<NT, BD>(p.e, c, acc, stage, ws, g, wid, lane, sl);
    }
    conv_stats_final(p.e, ws, NT, group, g, wid, lane);
  }
}

struct Cin1Call { const void* x; int dtype; const float* w; const float* bias; void* y; float* stats; void* ws; cudaStream_t st; long long ws_bytes; int query; };

template <int KS, int STRIDE, int NT, int BD>
static int launch_cin1_tc(int N, int D, int H, int W, int pad, int out_ctot, int out_coff, Cin1Call& c) {
  using Cfg = Cin1Cfg<KS, STRIDE, NT, BD>;
  Cin1TcParams p;
  p.x = c.x; p.w = c.w; p.D = D; p.H = H; p.W = W; p.pad = pad;
  ConvEpiP& e = p.e;
  e.D = (D + 2 * pad - KS) / STRIDE + 1; e.H = (H + 2 * pad - KS) / STRIDE + 1; e.W = (W + 2 * pad - KS) / STRIDE + 1;
  e.Cout = NT; e.out_ctot = out_ctot; e.out_coff = out_coff;
  e.tiles_w = ceil_div(e.W, kTW); e.tiles_h = ceil_div(e.H, kTH); e.tiles_d = ceil_div(e.D, BD); e.n_tiles = 1;
  e.total_tiles = (long long)e.tiles_w * e.tiles_h * e.tiles_d * N;
  const long long sp_tiles = (long long)e.tiles_w * e.tiles_h * e.tiles_d;
  const int R = stats_rows(sp_tiles, e.total_tiles);
  c.ws_bytes = stats_partial_bytes(N, R, NT, 4);
  if (c.query) return B200_OK;
  e.y = (__half*)c.y; e.bias = c.bias;
  e.sp.buf = c.stats ? (float*)c.ws : nullptr; e.sp.R = R; e.sp.tiles_per_group = sp_tiles; e.sp.rows_per_cta = 4;
  dim3 grid((unsigned)std::min<long long>(e.total_tiles, num_sms()));
  if (c.dtype == B200_DT_F16) {
    auto kern = conv_cin1_tc_kernel<__half, KS, STRIDE, NT, BD>;
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    kern<<<grid, Cfg::kThreads, Cfg::kSmemBytes, c.st>>>(p);
  } else {
    auto kern = conv_cin1_tc_kernel<float, KS, STRIDE, NT, BD>;
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    kern<<<grid, Cfg::kThreads, Cfg::kSmemBytes, c.st>>>(p);
  }
  B200_LAUNCH_CHECK("conv_cin1_tc_kernel");
  if (c.stats) return launch_stats_finish((const float*)c.ws, N, R * 4, NT, 1, NT, c.stats, c.st);
  return B200_OK;
}

template <int KS, int STRIDE>
static int dispatch_cin1_tc(int N, int D, int H, int W, int Cout, int pad, int out_ctot, int out_coff, Cin1Call& c) {
  switch (Cout) {
    case 16: return launch_cin1_tc<KS, STRIDE, 16, 4>(N, D, H, W, pad, out_ctot, out_coff, c);
    case 32: return launch_cin1_tc<KS, STRIDE, 32, 4>(N, D, H, W, pad, out_ctot, out_coff, c);
    case 48: return launch_cin1_tc<KS, STRIDE, 48, 4>(N, D, H, W, pad, out_ctot, out_coff, c);
    case 64: return launch_cin1_tc<KS, STRIDE, 64, 4>(N, D, H, W, pad, out_ctot, out_coff, c);
    case 96: return launch_cin1_tc<KS, STRIDE, 96, 2>(N, D, H, W, pad, out_ctot, out_coff, c);
    case 128: return launch_cin1_tc<KS, STRIDE, 128, 2>(N, D, H, W, pad, out_ctot, out_coff, c);
    default: return set_err(B200_ERR_UNSUPPORTED, "conv_cin1_tc: Cout must be 16, 32, 48, 64, 96 or 128 (got %d)", Cout);
  }
}

static int cin1_tc_dispatch(int N, int D, int H, int W, int Cout, int k, int stride, int pad, int out_ctot, int out_coff, Cin1Call& c) {
  B200_REQUIRE(N > 0 && D > 0 && H > 0 && W > 0, "conv_cin1_tc: empty problem");
  B200_REQUIRE(out_ctot % 8 == 0 && out_coff % 8 == 0 && out_coff + Cout <= out_ctot, "conv_cin1_tc: bad output channel slice");
  if (k == 3 && stride == 1 && pad == 1) return dispatch_cin1_tc<3, 1>(N, D, H, W, Cout, pad, out_ctot, out_coff, c);
  if (k == 2 && stride == 2 && pad == 0) {
    B200_REQUIRE(D >= 2 && H >= 2 && W >= 2, "conv_cin1_tc: input smaller than the kernel");
    return dispatch_cin1_tc<2, 2>(N, D, H, W, Cout, pad, out_ctot, out_coff, c);
  }
  return set_err(B200_ERR_UNSUPPORTED, "conv_cin1_tc: (kernel, stride, pad) must be (3,1,1) or (2,2,0), got (%d,%d,%d)", k, stride, pad);
}

}  // namespace b200

using namespace b200;

extern "C" long long b200_conv_cin1_tc_workspace_bytes(int N, int D, int H, int W, int Cout, int k, int stride, int pad) {
  Cin1Call c{nullptr, B200_DT_F16, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 1};
  if (cin1_tc_dispatch(N, D, H, W, Cout, k, stride, pad, Cout, 0, c)) return -1;
  return c.ws_bytes;
}

extern "C" int b200_conv_cin1_tc(const void* x, int dtype, int N, int D, int H, int W, const float* weight, const float* bias,
                                 int Cout, int k, int stride, int pad, void* y, int out_ctot, int out_coff, float* stats,
                                 void* workspace, void* stream) {
  B200_REQUIRE(x && y && weight, "conv_cin1_tc: null pointer");
  B200_REQUIRE(dtype == B200_DT_F16 || dtype == B200_DT_F32, "conv_cin1_tc: bad dtype");
  B200_REQUIRE(!stats || workspace, "conv_cin1_tc: statistics need the workspace of b200_conv_cin1_tc_workspace_bytes()");
  Cin1Call c{x, dtype, weight, bias, y, stats, workspace, (cudaStream_t)stream, 0, 0};
  return cin1_tc_dispatch(N, D, H, W, Cout, k, stride, pad, out_ctot, out_coff, c);
}
