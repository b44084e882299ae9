// Deterministic InstanceNorm statistics for the tensor-core epilogues (SURVEY.md §8 row a9).
//
// nn.InstanceNorm3d needs per-(sample, channel) sum and sum of squares over the whole volume.  The convolution / GEMM
// epilogues already hold every output value in registers, so they produce the sums -- but never through floating-point
// atomics (their order changes from run to run).  Instead:
//   * every epilogue warp keeps RUNNING sums of its 32 rows in a warp-private shared-memory row [2*NT]
//     ({sum, sumsq} interleaved per column); tiles are walked in a fixed order, so the running sums are reproducible;
//   * when the (batch item, N tile) GROUP of the tile changes, the warp writes its row to the partial buffer
//         partials[group][c][q][2*NT],   c = rank of this CTA among the CTAs that own tiles of the group,  q = warp & 3
//     (tiles of a group are contiguous in the persistent tile order t = group * tiles_per_group + i and CTA b owns the
//     tiles t = b (mod gridDim.x), so  c = (b - group * tiles_per_group) mod gridDim.x  and exactly
//     R = min(tiles_per_group, gridDim.x) CTAs take part: every row the finishing pass reads has been written);
//   * stats_finish_kernel adds the R*4 rows of a group in a fixed order in double precision and stores the float
//     {sum, sumsq} pairs the normalisation kernels read.
// Result: bit-identical statistics run to run, no zero-initialisation, no barrier between the epilogue warps.
#pragma once
#include "common.cuh"

namespace b200 {

struct StatsPartials {
  float* buf;                 // [groups][R][rows_per_cta][2*NT]; null = no statistics
  int R;                      // min(tiles_per_group, gridDim.x)
  long long tiles_per_group;
  int rows_per_cta;           // partial rows one CTA writes per group: 4 (one per 32-row quarter of the tile)
};

// flush the warp-private running sums of columns [col_lo, col_hi) (in {sum,sumsq} pairs) and clear them; `slot` = this
// warp's row among the CTA's rows_per_cta rows
__device__ __forceinline__ void stats_flush(const StatsPartials& sp, float* ws, int nt2, long long group, int slot, int lane,
                                            int pair_lo, int pair_hi) {
  __syncwarp();
  const long long G = gridDim.x;
  const int c = (int)((((long long)blockIdx.x - (group * sp.tiles_per_group) % G) + G) % G);
  float* dst = sp.buf + (((group * sp.R + c) * sp.rows_per_cta + slot) * (long long)nt2);
  for (int i = 2 * pair_lo + lane; i < 2 * pair_hi; i += 32) { dst[i] = ws[i]; ws[i] = 0.f; }
  __syncwarp();
}

// host side: rows per group and bytes of the partial buffer
inline int stats_rows(long long tiles_per_group, long long total_tiles) {
  const long long grid = std::min<long long>(total_tiles, num_sms());
  return (int)std::min<long long>(tiles_per_group, grid);
}
inline long long stats_partial_bytes(long long groups, int R, int NT, int rows_per_cta = 4) { return groups * R * (long long)rows_per_cta * 2 * NT * (long long)sizeof(float); }

// stats[(n*Cout + nt*NT + col)*2 + {0,1}] = sum over the `rows` (= R * rows_per_cta) partial rows of group (n, nt), fixed order, fp64.
int launch_stats_finish(const float* partials, long long groups, int rows, int NT, int n_tiles, int Cout, float* stats, cudaStream_t st);

// InstanceNorm of channel c as one multiply-add, y = x * scale + shift, from its {sum, sumsq} over S voxels (invS = 1 / S).
// Every NC8 consumer of the statistics (norm_act_nc8_kernel, the operand table of conv3x3x3_tc, head_conv_norm_nc8_kernel)
// calls this, so a fused and an unfused normalisation produce the same fp16 values.  gamma / beta (float32 [C], either may be
// NULL) are the affine parameters: (gamma * rstd, beta - mean * rstd * gamma), as b200_norm_act computes them; with both NULL
// the pair is (rstd, -mean * rstd).
__device__ __forceinline__ float2 instnorm_scale_shift(float sum, float sumsq, float invS, float eps, const float* gamma,
                                                       const float* beta, int c) {
  const float mean = sum * invS, var = fmaxf(sumsq * invS - mean * mean, 0.f), rstd = 1.f / sqrtf(var + eps);
  if (!gamma && !beta) return make_float2(rstd, -mean * rstd);
  const float g = gamma ? __ldg(gamma + c) : 1.f, b = beta ? __ldg(beta + c) : 0.f;
  // explicit roundings: the shift is the same float wherever the helper is inlined (no site-dependent FMA contraction)
  return make_float2(__fmul_rn(rstd, g), __fsub_rn(b, __fmul_rn(__fmul_rn(mean, rstd), g)));
}

}  // namespace b200
