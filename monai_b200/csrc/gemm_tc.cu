// Y = epilogue( X * W^T ) on Hopper wgmma tensor cores for channel-blocked (NC8) activations (SURVEY.md §8 rows a8, a12, a13).
//
// One kernel serves every GEMM-shaped layer of SwinUNETR outside the 3x3x3 convolutions:
//   * nn.Linear of WindowAttention.qkv / proj, MLPBlock.linear1 / linear2, PatchMerging.reduction
//     (monai/networks/nets/swin_unetr.py:509-532, 596-648, 749-773; monai/networks/blocks/mlp.py:75-80),
//   * 1x1x1 Conv3d (UnetResBlock.conv3, dynunet_block.py:75-87),
//   * ConvTranspose3d(kernel 2, stride 2) of UnetrUpBlock (unetr_block.py:56-64): a GEMM with N = 8*Cout followed by a
//     scatter of each (tap, cout) group to the 2x-upsampled voxel.
//
// Operands: X is NC8 [Nb][K/8][S][8] fp16 (rows = S tokens/voxels); a 128-row A tile of one 8-channel chunk is 2 KB
// contiguous in HBM and lands in shared memory as the wgmma K-major / no-swizzle core-matrix column
// (LBO = 128*16 B between K chunks, SBO = 128 B between 8-row groups).  W is pre-packed into the B image
// [nt][k16][khalf][NT/8][8][8] and streamed with 1-D bulk copies.  fp32 accumulators live in the registers of two
// consumer warpgroups.  Epilogue (variant chosen at compile time): + bias, GELU(erf), + residual,
// InstanceNorm partial sums, and a row map (identity / index table / 2x upsample scatter) before the fp16 NC8 store.
#include "common.cuh"
#include "tc90.cuh"
#include "stats.cuh"
#include "gelu.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

constexpr int kGemmStages = 4;
constexpr int kGemmK16PerStage = 4;                 // 64 K elements per pipeline stage
constexpr int kGemmAStage = kGemmK16PerStage * 2 * 128 * 16;  // 16 KB

// Width of the packed weight tiles (b200_gemm_tc_pack_weight): the widest multiple of 16 up to 256 that divides N.  Other
// kernels read these images too (the fused MLP, the folded residual of conv3x3x3_tc), so the packing does not depend on the
// tile the GEMM kernel runs.
__host__ __device__ inline int gemm_tc_nt(int N) {
  for (int nt = 256; nt >= 16; nt -= 16)
    if (N % nt == 0) return nt;
  return 16;
}
// N tile of the GEMM kernel: the widest compiled width that divides the packing width P (the accumulator of a 64-row half
// tile is NT / 2 registers per thread, so 128 is the widest that leaves room for the epilogue)
__host__ __device__ inline int gemm_tile_n(int P) {
  constexpr int kWidths[6] = {128, 96, 64, 48, 32, 16};
  for (int nt : kWidths)
    if (P % nt == 0) return nt;
  return 16;
}

struct GemmTcParams {
  b200_gemm_tc_desc d;
  const __half* x; const __half* w; const float* bias; __half* y; const __half* res; const int32_t* row_map;
  StatsPartials sp;   // deterministic InstanceNorm partial sums (stats.cuh)
  int P;              // width of the packed weight tiles (gemm_tc_nt(N)); the kernel's N tile divides it
};

__global__ void gemm_tc_pack_weight_kernel(const float* __restrict__ w, __half* __restrict__ out, int N, int K, int NT,
                                           long long w_stride_n, long long w_stride_k) {
  // out index: [nt][k16][khalf][g][row][kk]
  const long long total = (long long)N * K;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int kk = (int)(r % 8); r /= 8;
    const int row = (int)(r % 8); r /= 8;
    const int g = (int)(r % (NT / 8)); r /= (NT / 8);
    const int khalf = (int)(r % 2); r /= 2;
    const int k16 = (int)(r % (K / 16)); r /= (K / 16);
    const int nt = (int)r;
    const int n = nt * NT + g * 8 + row, k = k16 * 16 + khalf * 8 + kk;
    out[i] = __float2half_rn(w[n * w_stride_n + k * w_stride_k]);
  }
}

// Persistent, warp-specialised: each CTA loops over (batch, row tile, N tile) work items.  Warp 0 streams the operands
// through a shared-memory ring that runs across tile boundaries; two consumer warpgroups (warps 4-7: rows 0-63, warps
// 8-11: rows 64-127 of the 128-row tile) run the wgmma chain with the fp32 accumulators in registers and then the
// epilogue of their rows.  The epilogue variant (row mapping, activation, residual, statistics) is a template parameter:
// the per-step instruction stream is what bounds these HBM-shaped GEMMs, so nothing is decided at run time inside the
// column loop.
constexpr int kGemmThreads = 384;

// tile -> (N tile, row tile, batch item).  Without statistics the N tiles of a row tile run back to back (the A tile is
// re-read from L2); with statistics the row tiles of one (batch item, N tile) group are contiguous, which is what the
// deterministic partial sums of stats.cuh need.
template <bool STATS>
__device__ __forceinline__ void gemm_tile(long long tile, int n_tiles, int row_tiles, int& nt, int& rt, int& n) {
  if (STATS) {
    rt = (int)(tile % row_tiles);
    nt = (int)((tile / row_tiles) % n_tiles);
  } else {
    nt = (int)(tile % n_tiles);
    rt = (int)((tile / n_tiles) % row_tiles);
  }
  n = (int)(tile / ((long long)n_tiles * row_tiles));
}

template <int NT>
__host__ __device__ constexpr int gemm_smem_bytes() {
  return kGemmStages * (kGemmAStage + kGemmK16PerStage * NT * 32) + 128 /*barriers*/ + 4 * 2 * NT * 4 /*stats rows*/ +
         2 * 2 * tc::kStageFloats * 4 /*slice buffers*/ + 128 /*align slack*/;
}

template <int NT, int MODE, int ACT, bool RES, bool STATS>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_tc_kernel(GemmTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = tc::align_smem128(smem_raw);   // keeps the shared address space (LDS/STS, not generic LD/ST)
  constexpr int b_stage = kGemmK16PerStage * NT * 32;
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kGemmStages * kGemmAStage;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + kGemmStages * b_stage);
  uint64_t* full = bars;
  uint64_t* empty = bars + kGemmStages;
  float* s_stats = reinterpret_cast<float*>(bars + 16);  // [4][2*NT] (one row per 32-row quarter of the tile)
  float* s_stage = s_stats + 4 * 2 * NT;                 // [2 warpgroups][2][kStageFloats]

  const b200_gemm_tc_desc& d = p.d;
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform for ptxas
  const int num_k16 = d.K / 16;
  const int num_stages = (num_k16 + kGemmK16PerStage - 1) / kGemmK16PerStage;
  const int n_tiles = d.N / NT, row_tiles = (d.S + 127) / 128;
  const long long total_tiles = (long long)d.Nb * row_tiles * n_tiles;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kGemmStages; ++i) { tc::mbar_init(&full[i], 1); tc::mbar_init(&empty[i], 2); }
    tc::fence_barrier_init();
  }
  if (STATS)
    for (int i = threadIdx.x; i < 4 * 2 * NT; i += blockDim.x) s_stats[i] = 0.f;
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      int s = 0; uint32_t ph = 0;
      for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int nt, rt, n;
        gemm_tile<STATS>(tile, n_tiles, row_tiles, nt, rt, n);
        // the NT columns of this tile inside the packed image of width P: per K16 step two runs (k halves) of NT rows x 16 B
        const int col = nt * NT, ptile = col / p.P, pcol = col - ptile * p.P;
        const __half* wbase = p.w + (long long)ptile * num_k16 * (p.P * 16) + pcol * 8;
        for (int st = 0; st < num_stages; ++st) {
          const int steps = min(kGemmK16PerStage, num_k16 - st * kGemmK16PerStage);
          tc::mbar_wait(&empty[s], ph ^ 1);
          // A: one contiguous 1-D bulk copy per 8-channel chunk (128 rows x 16 B = 2 KB in NC8); the last row tile is
          // clamped to the valid rows so nothing is read past the chunk (stale smem rows are masked by the epilogue)
          const int rows = min(128, d.S - rt * 128);
          tc::mbar_arrive_expect_tx(&full[s], steps * 2 * rows * 16 + steps * NT * 32);
          const __half* abase = p.x + (((long long)n * (d.in_ctot / 8) + d.in_coff / 8 + st * kGemmK16PerStage * 2) * d.S + rt * 128) * 8;
          for (int c = 0; c < steps * 2; ++c)
            tc::bulk_load(smem_a + s * kGemmAStage + c * 2048, abase + (long long)c * d.S * 8, rows * 16, &full[s]);
          const __half* wst = wbase + (long long)st * kGemmK16PerStage * (p.P * 16);
          if (p.P == NT) {
            tc::bulk_load(smem_b + s * b_stage, wst, steps * NT * 32, &full[s]);
          } else {
            for (int k = 0; k < steps; ++k)
              for (int kh = 0; kh < 2; ++kh)
                tc::bulk_load(smem_b + s * b_stage + (k * 2 + kh) * NT * 16, wst + (long long)k * (p.P * 16) + kh * (p.P * 8), NT * 16, &full[s]);
          }
          if (++s == kGemmStages) { s = 0; ph ^= 1; }
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    const int g = (warp >> 2) - 1;          // consumer warpgroup: rows 64 g .. 64 g + 63 of the tile
    const int wid = warp & 3;
    const int q = 2 * g + (wid & 1);        // 32-row quarter of the tile this warp writes
    const int half = wid >> 1;              // which 8 columns of each 16-column slice this warp writes
    const int cout = MODE == 2 ? d.N / 8 : d.N;  // channels of the destination tensor written by this GEMM
    const long long cs = (long long)d.S_out * 8;   // halves between consecutive 8-channel chunks of the destination
    const float* __restrict__ bias = p.bias;
    const bool has_bias = bias != nullptr;
    const int W2 = 2 * d.W, HW4 = 4 * d.H * d.W;
    float* ws = s_stats + q * (2 * NT);     // running column sums of this quarter; the two warps of a quarter own disjoint columns
    float* stage = s_stage + g * 2 * tc::kStageFloats;
    long long group = -1;
    int s = 0; uint32_t ph = 0;
    int sl = 0;                             // slice counter: alternates the two slice buffers
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int nt, rt, n;
      gemm_tile<STATS>(tile, n_tiles, row_tiles, nt, rt, n);
      if (STATS) {
        const long long gg = tile / row_tiles;   // (batch item, N tile): tiles of a group are contiguous (row tile fastest)
        if (gg != group) {
          if (group >= 0) {
            tc::wg_bar(8 + g);
            if (half == 0) stats_flush(p.sp, ws, 2 * NT, group, q, lane, 0, NT);
          }
          group = gg;
        }
      }
      float acc[NT / 2];
      for (int st = 0; st < num_stages; ++st) {
        const int steps = min(kGemmK16PerStage, num_k16 - st * kGemmK16PerStage);
        tc::mbar_wait(&full[s], ph);
        const uint32_t a_base = tc::smem_u32(smem_a + s * kGemmAStage) + g * 1024, b_base = tc::smem_u32(smem_b + s * b_stage);
        tc::wg_fence();
        for (int k = 0; k < steps; ++k) {
          const uint64_t adesc = tc::make_desc_kmajor_noswz(a_base + k * 2 * 2048, 2048, 128);
          const uint64_t bdesc = tc::make_desc_kmajor_noswz(b_base + k * NT * 32, NT * 16, 128);
          tc::wg_mma_ss<NT>(acc, adesc, bdesc, (st | k) != 0 ? 1u : 0u, 128);
        }
        tc::wg_commit();
        tc::wg_wait<0>();
        tc::wg_fence_acc<NT / 2>(acc);
        if (wid == 0 && lane == 0) tc::mbar_arrive(&empty[s]);
        if (++s == kGemmStages) { s = 0; ph ^= 1; }
      }

      const int row = rt * 128 + q * 32 + lane;
      const bool row_ok = row < d.S;
      long long drow = row;
      if (MODE == 1) drow = row_ok ? (long long)__ldg(p.row_map + row) : -1;  // the map is shared by all batch items
      const bool dst_ok = row_ok && drow >= 0;
      const int co0 = nt * NT;
      if (MODE == 2) {
        const int vx = row % d.W, vy = (row / d.W) % d.H, vz = row / (d.W * d.H);
        drow = ((long long)(2 * vz) * (2 * d.H) + 2 * vy) * W2 + 2 * vx;
      }
      __half* ytile = p.y + ((long long)n * (d.out_ctot / 8) + (MODE == 2 ? 0 : (d.out_coff + co0) / 8)) * cs + drow * 8;
      const __half* rtile = RES ? p.res + ((long long)n * (d.res_ctot / 8) + (d.res_coff + co0) / 8) * cs + drow * 8 : nullptr;
#pragma unroll
      for (int c16 = 0; c16 < NT / 16; ++c16, ++sl) {
        float* buf = stage + (sl & 1) * tc::kStageFloats;
        tc::wg_stage16<0>(acc + c16 * 8, buf, wid, lane);
        tc::wg_bar(8 + g);
        float gv[8];
        tc::wg_read8(buf, wid, lane, gv);
        const int g8 = c16 * 2 + half;           // 8-column group inside this N tile
        __half* yp;
        int bidx;
        if (MODE == 2) {
          const int col = co0 + g8 * 8;          // GEMM columns are ordered [tap][cout]
          const int tap = col / cout, cc = col - tap * cout;
          const int tapoff = (tap >> 2) * HW4 + ((tap >> 1) & 1) * W2 + (tap & 1);
          yp = ytile + (long long)((d.out_coff + cc) >> 3) * cs + (long long)tapoff * 8;
          bidx = cc;
        } else {
          yp = ytile + (long long)g8 * cs;
          bidx = co0 + g8 * 8;
        }
        if (has_bias) {
          const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + bidx)), b1 = __ldg(reinterpret_cast<const float4*>(bias + bidx + 4));
          gv[0] += b0.x; gv[1] += b0.y; gv[2] += b0.z; gv[3] += b0.w;
          gv[4] += b1.x; gv[5] += b1.y; gv[6] += b1.z; gv[7] += b1.w;
        }
        if (ACT == 4) {
#pragma unroll
          for (int j = 0; j < 8; ++j) gv[j] = gelu_erf(gv[j]);
        }
        if (RES) {
          uint4 r = make_uint4(0, 0, 0, 0);
          if (dst_ok) r = *reinterpret_cast<const uint4*>(rtile + (long long)g8 * cs);
          const __half2* rh = reinterpret_cast<const __half2*>(&r);
#pragma unroll
          for (int j = 0; j < 4; ++j) { const float2 r2 = __half22float2(rh[j]); gv[2 * j] += r2.x; gv[2 * j + 1] += r2.y; }
        }
        if (dst_ok) {
          uint4 hv;
          __half2* hp = reinterpret_cast<__half2*>(&hv);
#pragma unroll
          for (int j = 0; j < 4; ++j) hp[j] = __floats2half2_rn(gv[2 * j], gv[2 * j + 1]);
          *reinterpret_cast<uint4*>(yp) = hv;
        }
        if (STATS) {
          float a8[8], b8[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) { a8[j] = dst_ok ? gv[j] : 0.f; b8[j] = a8[j] * a8[j]; }
          float csum, cq;
          transpose_reduce8(a8, b8, lane, csum, cq);
          if ((lane & 3) == 0) {
            const int col = g8 * 8 + transpose_reduce8_col(lane);
            ws[2 * col] += csum;
            ws[2 * col + 1] += cq;
          }
        }
      }
    }
    if (STATS && group >= 0) {
      tc::wg_bar(8 + g);
      if (half == 0) stats_flush(p.sp, ws, 2 * NT, group, q, lane, 0, NT);
    }
  }
}

using GemmKernelFn = void (*)(GemmTcParams);

template <int NT, int MODE, int ACT>
static GemmKernelFn gemm_pick2(bool res, bool stats) {
  if (res) return stats ? gemm_tc_kernel<NT, MODE, ACT, true, true> : gemm_tc_kernel<NT, MODE, ACT, true, false>;
  return stats ? gemm_tc_kernel<NT, MODE, ACT, false, true> : gemm_tc_kernel<NT, MODE, ACT, false, false>;
}

template <int NT>
static GemmKernelFn gemm_pick(int mode, int act, bool res, bool stats) {
  if (mode == 0) return act == 4 ? gemm_pick2<NT, 0, 4>(res, stats) : gemm_pick2<NT, 0, 0>(res, stats);
  if (mode == 1) return act == 4 ? gemm_pick2<NT, 1, 4>(res, stats) : gemm_pick2<NT, 1, 0>(res, stats);
  if (res) return nullptr;  // the upsample scatter has no residual form
  if (act == 4) return stats ? gemm_tc_kernel<NT, 2, 4, false, true> : gemm_tc_kernel<NT, 2, 4, false, false>;
  return stats ? gemm_tc_kernel<NT, 2, 0, false, true> : gemm_tc_kernel<NT, 2, 0, false, false>;
}

}  // namespace b200

using namespace b200;

extern "C" long long b200_gemm_tc_weight_bytes(int N, int K) {
  if (N <= 0 || K <= 0 || N % 16 || K % 16) return -1;
  return (long long)N * K * 2;
}

extern "C" int b200_gemm_tc_pack_weight(const float* w, int N, int K, long long stride_n, long long stride_k, void* packed,
                                        void* stream) {
  B200_REQUIRE(w && packed, "gemm_tc_pack_weight: null pointer");
  B200_REQUIRE(N > 0 && K > 0 && N % 16 == 0 && K % 16 == 0, "gemm_tc: N and K must be multiples of 16 (got %d, %d)", N, K);
  const long long total = (long long)N * K;
  const int blocks = (int)std::min<long long>((total + 255) / 256, 4096);
  gemm_tc_pack_weight_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, (__half*)packed, N, K, gemm_tc_nt(N), stride_n, stride_k);
  B200_LAUNCH_CHECK("gemm_tc_pack_weight_kernel");
  return B200_OK;
}

static int gemm_tc_check(const b200_gemm_tc_desc& d, const void* res, const int32_t* row_map) {
  B200_REQUIRE(d.Nb > 0 && d.S > 0 && d.S_out > 0, "gemm_tc: empty problem");
  B200_REQUIRE(d.K > 0 && d.K % 16 == 0 && d.N > 0 && d.N % 16 == 0, "gemm_tc: N and K must be multiples of 16 (got %d, %d)", d.N, d.K);
  B200_REQUIRE(d.in_ctot % 8 == 0 && d.in_coff % 8 == 0 && d.in_coff + d.K <= d.in_ctot, "gemm_tc: bad input channel slice");
  B200_REQUIRE(d.mode >= 0 && d.mode <= 2, "gemm_tc: mode must be 0 (rows), 1 (row map) or 2 (2x upsample scatter)");
  B200_REQUIRE(d.mode != 1 || row_map, "gemm_tc: mode 1 needs a row map");
  const int cout = d.mode == 2 ? d.N / 8 : d.N;
  B200_REQUIRE(d.mode != 2 || (d.N % 8 == 0 && cout % 8 == 0 && (long long)d.D * d.H * d.W == d.S && d.S_out == 8LL * d.S),
               "gemm_tc: upsample scatter needs N = 8*Cout, S = D*H*W and S_out = 8*S");
  B200_REQUIRE(d.out_ctot % 8 == 0 && d.out_coff % 8 == 0 && d.out_coff + cout <= d.out_ctot, "gemm_tc: bad output channel slice");
  B200_REQUIRE(!res || (d.res_ctot % 8 == 0 && d.res_coff % 8 == 0 && d.res_coff + cout <= d.res_ctot), "gemm_tc: bad residual channel slice");
  B200_REQUIRE(d.act == 0 || d.act == 4, "gemm_tc: activation must be 0 (none) or 4 (gelu)");
  return B200_OK;
}

extern "C" long long b200_gemm_tc_workspace_bytes(const b200_gemm_tc_desc* desc) {
  if (!desc || desc->N <= 0 || desc->N % 16 || desc->S <= 0 || desc->Nb <= 0) return -1;
  const int NT = gemm_tile_n(gemm_tc_nt(desc->N));   // the kernel's N tile: one statistics group per (batch item, N tile)
  const long long row_tiles = ceil_div(desc->S, 128), groups = (long long)desc->Nb * (desc->N / NT);
  return stats_partial_bytes(groups, stats_rows(row_tiles, row_tiles * groups), NT);
}

extern "C" int b200_gemm_tc(const b200_gemm_tc_desc* desc, const void* x, const void* packed_w, const float* bias,
                            const void* res, const int32_t* row_map, void* y, float* stats, void* workspace, void* stream) {
  B200_REQUIRE(desc && x && packed_w && y, "gemm_tc: null pointer");
  B200_REQUIRE(!stats || workspace, "gemm_tc: statistics need the workspace of b200_gemm_tc_workspace_bytes()");
  const b200_gemm_tc_desc& d = *desc;
  int rc = gemm_tc_check(d, res, row_map);
  if (rc) return rc;
  const int P = gemm_tc_nt(d.N), NT = gemm_tile_n(P);
  GemmTcParams p;
  p.d = d; p.x = (const __half*)x; p.w = (const __half*)packed_w; p.bias = bias; p.y = (__half*)y; p.res = (const __half*)res;
  p.row_map = row_map; p.P = P;
  int smem = 0;
  GemmKernelFn fn = nullptr;
  const bool has_res = res != nullptr, has_stats = stats != nullptr;
  switch (NT) {
    case 128: fn = gemm_pick<128>(d.mode, d.act, has_res, has_stats); smem = gemm_smem_bytes<128>(); break;
    case 96: fn = gemm_pick<96>(d.mode, d.act, has_res, has_stats); smem = gemm_smem_bytes<96>(); break;
    case 64: fn = gemm_pick<64>(d.mode, d.act, has_res, has_stats); smem = gemm_smem_bytes<64>(); break;
    case 48: fn = gemm_pick<48>(d.mode, d.act, has_res, has_stats); smem = gemm_smem_bytes<48>(); break;
    case 32: fn = gemm_pick<32>(d.mode, d.act, has_res, has_stats); smem = gemm_smem_bytes<32>(); break;
    default: fn = gemm_pick<16>(d.mode, d.act, has_res, has_stats); smem = gemm_smem_bytes<16>(); break;
  }
  B200_REQUIRE(fn != nullptr, "gemm_tc: the 2x upsample scatter (mode 2) does not take a residual");
  B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const long long row_tiles = ceil_div(d.S, 128), groups = (long long)d.Nb * (d.N / NT);
  const long long total_tiles = row_tiles * groups;
  p.sp.buf = stats ? (float*)workspace : nullptr;
  p.sp.R = stats_rows(row_tiles, total_tiles);
  p.sp.tiles_per_group = row_tiles;
  p.sp.rows_per_cta = 4;
  dim3 grid((unsigned)std::min<long long>(total_tiles, num_sms()));
  fn<<<grid, kGemmThreads, smem, (cudaStream_t)stream>>>(p);
  B200_LAUNCH_CHECK("gemm_tc_kernel");
  if (stats) return launch_stats_finish((const float*)workspace, groups, p.sp.R * 4, NT, d.N / NT, d.N, stats, (cudaStream_t)stream);
  return B200_OK;
}
