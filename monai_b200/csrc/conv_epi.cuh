// Shared output stage of the wgmma convolution kernels (conv_tc.cu: 3x3x3 stride 1; conv_cin1_tc.cu: the
// single-input-channel stems): tile geometry and the registers -> fp16 NC8 epilogue with bias and the
// deterministic InstanceNorm partial sums of stats.cuh.
//
// GEMM rows of a tile = one 16 (H) x 8 (W) patch of an output D-plane; a tile holds BD consecutive planes whose fp32
// accumulators are adjacent column blocks of NT columns in the registers of the two consumer warpgroups.
#pragma once
#include "common.cuh"
#include "stats.cuh"
#include "tc90.cuh"

namespace b200 {

constexpr int kTH = 16, kTW = 8;                 // output patch per D-plane: 16 (H) x 8 (W) = 128 GEMM rows

struct ConvEpiP {
  __half* y;                 // NC8 destination
  const float* bias;         // [Cout] or null
  StatsPartials sp;          // deterministic statistics (buf == null: none)
  int D, H, W;               // OUTPUT spatial size
  int Cout, out_ctot, out_coff;
  int tiles_w, tiles_h, tiles_d, n_tiles;
  long long total_tiles;     // tiles_w * tiles_h * tiles_d * n_tiles * N
};

struct ConvTile { int w0, h0, d0, nt, n; };

template <int BD>
__device__ __forceinline__ ConvTile conv_tile(const ConvEpiP& p, long long t) {
  // spatial tiles fastest, then the N tile, then the batch item: CTAs that run concurrently stream the same weights
  ConvTile c;
  c.w0 = (int)(t % p.tiles_w) * kTW; t /= p.tiles_w;
  c.h0 = (int)(t % p.tiles_h) * kTH; t /= p.tiles_h;
  c.d0 = (int)(t % p.tiles_d) * BD; t /= p.tiles_d;
  c.nt = (int)(t % p.n_tiles);
  c.n = (int)(t / p.n_tiles);
  return c;
}

// Epilogue of one tile, run by the consumer warpgroup `g` (rows 64 g .. 64 g + 63 of the tile) from its wgmma accumulators:
// `acc` holds the BD planes of the tile as consecutive blocks of NT columns (m64nN fragment layout, NT / 2 registers per
// plane).  16-column slices pass through the warpgroup's two slice buffers `stage` (tc::wg_stage16); afterwards warp `wid`
// owns row 32 (wid & 1) + lane of its half tile and the 8-column chunk 2 c16 + (wid >> 1) of every slice: + bias, fp16 NC8
// store, and the running InstanceNorm sums of the chunk in the quarter's shared-memory row `ws` (the two warps of a quarter
// own disjoint columns of the row).  `sl` counts slices across calls so the two buffers strictly alternate.
template <int NT, int BD>
__device__ __forceinline__ void conv_epilogue(const ConvEpiP& p, const ConvTile& c, const float* acc, float* stage, float* ws,
                                              int g, int wid, int lane, int& sl) {
  const int q = 2 * g + (wid & 1), half = wid >> 1;
  const int row = q * 32 + lane;
  const long long S = (long long)p.D * p.H * p.W;
  const int h = c.h0 + (row >> 3), w = c.w0 + (row & 7);
  const bool hw_ok = h < p.H && w < p.W;
  const int co0 = c.nt * NT;
  __half* ybase = p.y + (((long long)c.n * (p.out_ctot / 8) + (p.out_coff + co0) / 8) * S) * 8;
#pragma unroll
  for (int c16 = 0; c16 < NT / 16; ++c16) {
    const int cc = 2 * c16 + half;
    float bsum[8], bsq[8], bias8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { bsum[j] = 0.f; bsq[j] = 0.f; bias8[j] = p.bias ? p.bias[co0 + cc * 8 + j] : 0.f; }
#pragma unroll
    for (int sub = 0; sub < BD; ++sub, ++sl) {
      float* buf = stage + (sl & 1) * tc::kStageFloats;
      tc::wg_stage16<0>(acc + (sub * NT + c16 * 16) / 2, buf, wid, lane);
      tc::wg_bar(8 + g);
      float f[8];
      tc::wg_read8(buf, wid, lane, f);
      const int dz = c.d0 + sub;
      const bool ok = hw_ok && dz < p.D;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        f[j] += bias8[j];
        if (ok) { bsum[j] += f[j]; bsq[j] = fmaf(f[j], f[j], bsq[j]); }
      }
      if (ok) {
        uint4 hv;
        __half2* hp = reinterpret_cast<__half2*>(&hv);
#pragma unroll
        for (int j = 0; j < 4; ++j) hp[j] = __floats2half2_rn(f[2 * j], f[2 * j + 1]);
        *reinterpret_cast<uint4*>(ybase + ((long long)cc * S + ((long long)dz * p.H + h) * p.W + w) * 8) = hv;
      }
    }
    if (p.sp.buf) {
      float a1, b1;
      transpose_reduce8(bsum, bsq, lane, a1, b1);
      if ((lane & 3) == 0) {   // eight lanes, eight different columns of the quarter's row: no atomics
        const int col = cc * 8 + transpose_reduce8_col(lane);
        ws[2 * col] += a1;
        ws[2 * col + 1] += b1;
      }
    }
  }
}

// Statistics bookkeeping before the epilogue of tile t: when the (batch item, N tile) group changes, the quarter's row of
// running sums is written to the partial buffer (slot = quarter; rows_per_cta = 4) by the first warp of the quarter, after
// the warpgroup barrier has made the other warp's sums visible.
__device__ __forceinline__ void conv_stats_turn(const ConvEpiP& p, float* ws, int NT, long long t, long long& group, int g, int wid,
                                                int lane) {
  const long long g_t = t / ((long long)p.tiles_w * p.tiles_h * p.tiles_d);
  if (g_t == group) return;
  if (group >= 0 && p.sp.buf) {
    tc::wg_bar(8 + g);
    if ((wid >> 1) == 0) stats_flush(p.sp, ws, 2 * NT, group, 2 * g + (wid & 1), lane, 0, NT);
  }
  group = g_t;
}
__device__ __forceinline__ void conv_stats_final(const ConvEpiP& p, float* ws, int NT, long long group, int g, int wid, int lane) {
  if (group < 0 || !p.sp.buf) return;
  tc::wg_bar(8 + g);
  if ((wid >> 1) == 0) stats_flush(p.sp, ws, 2 * NT, group, 2 * g + (wid & 1), lane, 0, NT);
}

}  // namespace b200
