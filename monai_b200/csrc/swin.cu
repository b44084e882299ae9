// SwinUNETR token-side kernels on NC8 activations (SURVEY.md §8 rows a12, a13): LayerNorm + window gather,
// PatchMerging gather + LayerNorm, windowed attention, the single-input-channel stems and the 1x1x1 output head.
// Reference: monai/networks/nets/swin_unetr.py (WindowAttention 426-532, SwinTransformerBlock 535-698,
// PatchMerging 701-773, compute_mask 779-816, proj_out 1040-1053), monai/networks/blocks/patchembedding.py:141-219,
// monai/networks/blocks/dynunet_block.py:247-267.
#include "common.cuh"
#include "stats.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

__device__ __forceinline__ void ld8(const __half* p, float (&f)[8]) {
  __align__(16) __half v[8];
  *reinterpret_cast<uint4*>(v) = *reinterpret_cast<const uint4*>(p);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = __half2float(v[j]);
}
__device__ __forceinline__ void st8(__half* p, const float (&f)[8]) {
  __align__(16) __half v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = __float2half_rn(f[j]);
  *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(v);
}

// ---------------------------------------------------------------------------------------------------- LayerNorm
__device__ __forceinline__ void cvt8(const uint4& r, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
  for (int j = 0; j < 4; ++j) { const float2 t = __half22float2(h[j]); f[2 * j] = t.x; f[2 * j + 1] = t.y; }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 r;
  __half2* h = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(f[2 * j], f[2 * j + 1]);
  return r;
}
// y = (x - mean) * rstd * gamma + beta for one 8-channel vector; gamma / beta fetched as two float4 each
__device__ __forceinline__ uint4 ln_apply8(const uint4& raw, float mean, float rstd, const float* __restrict__ gamma,
                                           const float* __restrict__ beta, int ch) {
  float f[8];
  cvt8(raw, f);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = (f[j] - mean) * rstd;
  if (gamma) {
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + ch)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + ch + 4));
    f[0] *= g0.x; f[1] *= g0.y; f[2] *= g0.z; f[3] *= g0.w; f[4] *= g1.x; f[5] *= g1.y; f[6] *= g1.z; f[7] *= g1.w;
  }
  if (beta) {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + ch)), b1 = __ldg(reinterpret_cast<const float4*>(beta + ch + 4));
    f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w; f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
  }
  return pack8(f);
}

// One thread per token.  KC8 > 0: the token's C = 8*KC8 channels stay in registers as raw 16-byte vectors (one global
// read, one write; mean then centred variance, exactly the two-pass formula).  KC8 == 0: generic C, the centred second
// pass and the output pass re-read the token (L1 hits).
template <int KC8>
__global__ void __launch_bounds__(256) layernorm_nc8_kernel(const __half* __restrict__ x, __half* __restrict__ y, int C,
                                                            long long S_in, const int* __restrict__ src, long long S_out,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            float eps) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= S_out) return;
  const int n = blockIdx.y, C8 = KC8 > 0 ? KC8 : C / 8;
  const long long s = src ? (long long)__ldg(src + r) : r;
  __half* yo = y + ((long long)n * C8 * S_out + r) * 8;
  if (s < 0) {  // padded token: exact zeros (F.pad after norm1, swin_unetr.py:603-606)
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (int c = 0; c < C8; ++c) *reinterpret_cast<uint4*>(yo + (long long)c * S_out * 8) = z;
    return;
  }
  const __half* xi = x + ((long long)n * C8 * S_in + s) * 8;
  const float invC = 1.f / (float)(8 * C8);
  if (KC8 > 0) {
    uint4 raw[KC8 > 0 ? KC8 : 1];
#pragma unroll
    for (int c = 0; c < KC8; ++c) raw[c] = __ldg(reinterpret_cast<const uint4*>(xi + (long long)c * S_in * 8));
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < KC8; ++c) {
      float f[8]; cvt8(raw[c], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += f[j];
    }
    const float mean = sum * invC;
    float var = 0.f;
#pragma unroll
    for (int c = 0; c < KC8; ++c) {
      float f[8]; cvt8(raw[c], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = f[j] - mean; var = fmaf(d, d, var); }
    }
    const float rstd = 1.f / sqrtf(var * invC + eps);
#pragma unroll
    for (int c = 0; c < KC8; ++c) *reinterpret_cast<uint4*>(yo + (long long)c * S_out * 8) = ln_apply8(raw[c], mean, rstd, gamma, beta, c * 8);
  } else {
    float sum = 0.f;
    for (int c = 0; c < C8; ++c) {
      float f[8]; cvt8(__ldg(reinterpret_cast<const uint4*>(xi + (long long)c * S_in * 8)), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += f[j];
    }
    const float mean = sum * invC;
    float var = 0.f;
    for (int c = 0; c < C8; ++c) {
      float f[8]; cvt8(__ldg(reinterpret_cast<const uint4*>(xi + (long long)c * S_in * 8)), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = f[j] - mean; var = fmaf(d, d, var); }
    }
    const float rstd = 1.f / sqrtf(var * invC + eps);
    for (int c = 0; c < C8; ++c)
      *reinterpret_cast<uint4*>(yo + (long long)c * S_out * 8) =
          ln_apply8(__ldg(reinterpret_cast<const uint4*>(xi + (long long)c * S_in * 8)), mean, rstd, gamma, beta, c * 8);
  }
}

// ------------------------------------------------------------------------------------------ PatchMerging gather + LN
__constant__ int kMergeV1[8][3] = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {1, 1, 0}, {1, 0, 1}, {0, 1, 1}, {1, 1, 1}};
__constant__ int kMergeV2[8][3] = {{0, 0, 0}, {0, 0, 1}, {0, 1, 0}, {0, 1, 1}, {1, 0, 0}, {1, 0, 1}, {1, 1, 0}, {1, 1, 1}};

// Eight lanes per merged token (lane & 7 = neighbour q): every lane keeps its neighbour's C = 8*KC8 channels in registers
// as raw 16-byte vectors, the statistics are reduced over the 8 lanes with three shuffles, and each lane writes its own
// channel block (q*C .. q*C+C) of the output token.  One global read, one write; a warp's loads cover 4 (d,h) rows x 8
// consecutive voxels = four full 128-byte lines per instruction.
template <int KC8>
__global__ void __launch_bounds__(256, 2) patch_merge_ln8_nc8_kernel(const __half* __restrict__ x, __half* __restrict__ y, int C, int D,
                                                                     int H, int W, const float* __restrict__ gamma,
                                                                     const float* __restrict__ beta, float eps, int v2) {
  const int D2 = (D + 1) / 2, H2 = (H + 1) / 2, W2 = (W + 1) / 2;
  const long long S2 = (long long)D2 * H2 * W2, S = (long long)D * H * W;
  const int C8 = KC8 > 0 ? KC8 : C / 8;
  const int q = threadIdx.x & 7;
  const long long r_raw = (long long)blockIdx.x * 32 + (threadIdx.x >> 3);
  const bool tok_ok = r_raw < S2;
  const long long r = tok_ok ? r_raw : S2 - 1;   // lanes of an out-of-range token still take part in the shuffles
  const int n = blockIdx.y;
  const int w2 = (int)(r % W2), h2 = (int)((r / W2) % H2), d2 = (int)(r / ((long long)W2 * H2));
  const int* o = v2 ? kMergeV2[q] : kMergeV1[q];
  const int d = 2 * d2 + o[0], h = 2 * h2 + o[1], w = 2 * w2 + o[2];
  const bool ok = d < D && h < H && w < W;      // odd sizes: the reference pads with zeros, which enter the statistics
  const __half* xi = x + ((long long)n * C8 * S + (ok ? (((long long)d * H + h) * W + w) : 0)) * 8;
  const uint4 zero = make_uint4(0, 0, 0, 0);
  const float invC = 1.f / (float)(8 * 8 * C8);
  __half* yo = y + ((long long)n * (8 * C8) * S2 + r) * 8;
  if (KC8 > 0) {
    uint4 raw[KC8 > 0 ? KC8 : 1];
#pragma unroll
    for (int c = 0; c < KC8; ++c) raw[c] = ok ? __ldg(reinterpret_cast<const uint4*>(xi + (long long)c * S * 8)) : zero;
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < KC8; ++c) {
      float f[8]; cvt8(raw[c], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += f[j];
    }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1); sum += __shfl_xor_sync(0xffffffffu, sum, 2); sum += __shfl_xor_sync(0xffffffffu, sum, 4);
    const float mean = sum * invC;
    float var = 0.f;
#pragma unroll
    for (int c = 0; c < KC8; ++c) {
      float f[8]; cvt8(raw[c], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float dd = f[j] - mean; var = fmaf(dd, dd, var); }
    }
    var += __shfl_xor_sync(0xffffffffu, var, 1); var += __shfl_xor_sync(0xffffffffu, var, 2); var += __shfl_xor_sync(0xffffffffu, var, 4);
    const float rstd = 1.f / sqrtf(var * invC + eps);
    if (!tok_ok) return;
#pragma unroll
    for (int c = 0; c < KC8; ++c)
      *reinterpret_cast<uint4*>(yo + (long long)(q * KC8 + c) * S2 * 8) = ln_apply8(raw[c], mean, rstd, gamma, beta, (q * KC8 + c) * 8);
  } else {
    // wide channels (deep stages, few tokens): the lane re-reads its neighbour (L1 / L2 hits), loads unrolled by four
    float sum = 0.f;
#pragma unroll 4
    for (int c = 0; c < C8; ++c) {
      float f[8]; cvt8(ok ? __ldg(reinterpret_cast<const uint4*>(xi + (long long)c * S * 8)) : zero, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += f[j];
    }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1); sum += __shfl_xor_sync(0xffffffffu, sum, 2); sum += __shfl_xor_sync(0xffffffffu, sum, 4);
    const float mean = sum * invC;
    float var = 0.f;
#pragma unroll 4
    for (int c = 0; c < C8; ++c) {
      float f[8]; cvt8(ok ? __ldg(reinterpret_cast<const uint4*>(xi + (long long)c * S * 8)) : zero, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float dd = f[j] - mean; var = fmaf(dd, dd, var); }
    }
    var += __shfl_xor_sync(0xffffffffu, var, 1); var += __shfl_xor_sync(0xffffffffu, var, 2); var += __shfl_xor_sync(0xffffffffu, var, 4);
    const float rstd = 1.f / sqrtf(var * invC + eps);
    if (!tok_ok) return;
#pragma unroll 4
    for (int c = 0; c < C8; ++c) {
      const uint4 raw = ok ? __ldg(reinterpret_cast<const uint4*>(xi + (long long)c * S * 8)) : zero;
      *reinterpret_cast<uint4*>(yo + (long long)(q * C8 + c) * S2 * 8) = ln_apply8(raw, mean, rstd, gamma, beta, (q * C8 + c) * 8);
    }
  }
}

// LayerNorm with eight lanes per token for wide channels (C8 % 8 == 0, C8 / 8 <= 12: C = 64 .. 768): lane j keeps chunks
// j, j+8, ... in registers.  The deep stages have few tokens, so one thread per token would leave most of the chip idle
// behind a serial chain of 3 * C/8 loads.
template <int PER>
__global__ void __launch_bounds__(256) layernorm8_nc8_kernel(const __half* __restrict__ x, __half* __restrict__ y, long long S_in,
                                                             const int* __restrict__ src, long long S_out,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta, float eps) {
  constexpr int C8 = PER * 8;
  const int j8 = threadIdx.x & 7;
  const long long r_raw = (long long)blockIdx.x * 32 + (threadIdx.x >> 3);
  const bool tok_ok = r_raw < S_out;
  const long long r = tok_ok ? r_raw : S_out - 1;
  const int n = blockIdx.y;
  const long long s = src ? (long long)__ldg(src + r) : r;
  __half* yo = y + ((long long)n * C8 * S_out + r) * 8;
  const uint4 zero = make_uint4(0, 0, 0, 0);
  uint4 raw[PER];
  const __half* xi = x + ((long long)n * C8 * S_in + (s < 0 ? 0 : s)) * 8;
#pragma unroll
  for (int i = 0; i < PER; ++i) raw[i] = s < 0 ? zero : __ldg(reinterpret_cast<const uint4*>(xi + (long long)(i * 8 + j8) * S_in * 8));
  const float invC = 1.f / (float)(8 * C8);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    float f[8]; cvt8(raw[i], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) sum += f[j];
  }
  sum += __shfl_xor_sync(0xffffffffu, sum, 1); sum += __shfl_xor_sync(0xffffffffu, sum, 2); sum += __shfl_xor_sync(0xffffffffu, sum, 4);
  const float mean = sum * invC;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    float f[8]; cvt8(raw[i], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float dd = f[j] - mean; var = fmaf(dd, dd, var); }
  }
  var += __shfl_xor_sync(0xffffffffu, var, 1); var += __shfl_xor_sync(0xffffffffu, var, 2); var += __shfl_xor_sync(0xffffffffu, var, 4);
  const float rstd = 1.f / sqrtf(var * invC + eps);
  if (!tok_ok) return;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int c = i * 8 + j8;
    // padded token (s < 0): exact zeros, as F.pad after norm1 (swin_unetr.py:603-606)
    *reinterpret_cast<uint4*>(yo + (long long)c * S_out * 8) = s < 0 ? zero : ln_apply8(raw[i], mean, rstd, gamma, beta, c * 8);
  }
}

// ---------------------------------------------------------------------------------------------- window attention
// Flash-style attention for one (window, head, batch item) per block: K and V^T of the head are staged in shared
// memory once; each warp owns 16 query rows at a time and walks the keys 16 at a time:
//   S = Q K^T (2 x mma.m16n8k16, K = head_dim = 16 is a single MMA step), + relative-position bias + shift mask,
//   online softmax in the accumulator registers, O += P V (2 x mma.m16n8k16, P re-used from the S fragments).
// The relative-position bias is looked up in the (2w-1)^3-entry table held in shared memory:
//   index(i, j) = lin(i) - lin(j) + const,  lin(t) = d*(2w1-1)(2w2-1) + h*(2w2-1) + w  with the token's coordinates in
// the MODULE window (the reference slices relative_position_index[:n, :n], swin_unetr.py:514-516, so clamped windows
// keep base-`window_size` coordinates).  With head_dim 16 the kernel is bound by exp/softmax issue, not by the MMAs.  It
// serves the windows the wgmma kernel (attn_tc.cu) has no schedule for (more than 352 tokens or more than 8 shift-mask
// patterns).
constexpr int kAttKStride = 24;   // halfs per K row in smem (48 B: conflict-free b-fragment loads)

__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// One 32-key step of the online softmax for 16 query rows per warp.  All scores are kept in log2 units (the bias table
// is pre-multiplied by log2(e) when it is staged, scale2 = scale*log2(e)) so every exponential is a bare ex2.approx.
// MASK: shifted windows (region ids differ -> -100 as in compute_mask, swin_unetr.py:457-487).  TAIL: keys >= n exist.
// bare MUFU.EX2 (exp2f() adds a denormal-range test and two scalings per call; the arguments here are <= 0 or -inf)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct AttRow {
  int lin0, lin1, reg0, reg1;
  float m0, m1, l0, l1;
  float o[2][4];
};

template <bool MASK, bool TAIL>
__device__ __forceinline__ void att_step32(const uint32_t (&qa)[4], AttRow& r, int j0, int n, float scale2, const __half* __restrict__ sK,
                                           const __half* __restrict__ sVt, int vstride, const float* __restrict__ sTab,
                                           const unsigned short* __restrict__ sLin, const unsigned char* __restrict__ sReg, int g, int t4) {
  constexpr float kMaskAdd = -100.0f * 1.4426950408889634f;
  float sc[4][4];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
    const __half* kp = sK + (j0 + nt * 8 + g) * kAttKStride + 2 * t4;
    mma_16816(sc[nt], qa, *reinterpret_cast<const uint32_t*>(kp), *reinterpret_cast<const uint32_t*>(kp + 8));
  }
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int j = j0 + nt * 8 + 2 * t4;                       // this thread's two keys j, j+1 of the tile
    const uint32_t lj2 = *reinterpret_cast<const uint32_t*>(sLin + j);
    // sLin holds BYTE offsets (4 * lin) and r.lin0/1 the byte offset of the row's table origin: one subtract per lookup
    const int lja = (int)(lj2 & 0xffffu), ljb = (int)(lj2 >> 16);
    const char* tb = reinterpret_cast<const char*>(sTab);
    float v00 = fmaf(sc[nt][0], scale2, *reinterpret_cast<const float*>(tb + (r.lin0 - lja)));
    float v01 = fmaf(sc[nt][1], scale2, *reinterpret_cast<const float*>(tb + (r.lin0 - ljb)));
    float v10 = fmaf(sc[nt][2], scale2, *reinterpret_cast<const float*>(tb + (r.lin1 - lja)));
    float v11 = fmaf(sc[nt][3], scale2, *reinterpret_cast<const float*>(tb + (r.lin1 - ljb)));
    if (MASK) {
      const unsigned short rj2 = *reinterpret_cast<const unsigned short*>(sReg + j);
      const int rja = rj2 & 0xff, rjb = rj2 >> 8;
      if (rja != r.reg0) v00 += kMaskAdd;
      if (rjb != r.reg0) v01 += kMaskAdd;
      if (rja != r.reg1) v10 += kMaskAdd;
      if (rjb != r.reg1) v11 += kMaskAdd;
    }
    if (TAIL) {
      if (j >= n) { v00 = -INFINITY; v10 = -INFINITY; }
      if (j + 1 >= n) { v01 = -INFINITY; v11 = -INFINITY; }
    }
    sc[nt][0] = v00; sc[nt][1] = v01; sc[nt][2] = v10; sc[nt][3] = v11;
    mx0 = fmaxf(mx0, fmaxf(v00, v01)); mx1 = fmaxf(mx1, fmaxf(v10, v11));
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  const float mn0 = fmaxf(r.m0, mx0), mn1 = fmaxf(r.m1, mx1);
  const float c0 = ex2_approx(r.m0 - mn0), c1 = ex2_approx(r.m1 - mn1);
  r.m0 = mn0; r.m1 = mn1;
  float ps0 = 0.f, ps1 = 0.f;
  uint32_t pa[2][4];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const float p00 = ex2_approx(sc[nt][0] - mn0), p01 = ex2_approx(sc[nt][1] - mn0);
    const float p10 = ex2_approx(sc[nt][2] - mn1), p11 = ex2_approx(sc[nt][3] - mn1);
    ps0 += p00 + p01; ps1 += p10 + p11;
    pa[nt >> 1][(nt & 1) * 2] = pack_h2(p00, p01);       // a0 / a2: row r0
    pa[nt >> 1][(nt & 1) * 2 + 1] = pack_h2(p10, p11);   // a1 / a3: row r1
  }
  r.l0 = fmaf(r.l0, c0, ps0); r.l1 = fmaf(r.l1, c1, ps1);
#pragma unroll
  for (int dt = 0; dt < 2; ++dt) {
    r.o[dt][0] *= c0; r.o[dt][1] *= c0; r.o[dt][2] *= c1; r.o[dt][3] *= c1;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const __half* vp = sVt + (dt * 8 + g) * vstride + j0 + ks * 16 + 2 * t4;
      mma_16816(r.o[dt], pa[ks], *reinterpret_cast<const uint32_t*>(vp), *reinterpret_cast<const uint32_t*>(vp + 8));
    }
  }
}

template <bool MASK>
__global__ void __launch_bounds__(256) window_attention_nc8_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int C,
                                                                   int heads, int nW, int n, float scale,
                                                                   const float* __restrict__ table, int tab_len, int ws0, int ws1,
                                                                   int ws2, const int* __restrict__ region) {
  extern __shared__ __align__(16) uint8_t s_att[];
  const int npad = (n + 31) / 32 * 32;
  const int vstride = npad + 8;                       // halfs per V^T row (conflict-free b-fragment loads)
  __half* sK = reinterpret_cast<__half*>(s_att);      // [npad][kAttKStride]
  __half* sVt = sK + (size_t)npad * kAttKStride;      // [16][vstride]
  float* sTab = reinterpret_cast<float*>(sVt + 16 * vstride);  // [tab_len], times log2(e)
  unsigned short* sLin = reinterpret_cast<unsigned short*>(sTab + tab_len);      // [npad]
  unsigned char* sReg = reinterpret_cast<unsigned char*>(sLin + npad);  // [npad]
  const int w = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int C8 = C / 8;
  const long long T = (long long)nW * n;
  const __half* base = qkv + (long long)b * (3 * C8) * T * 8;
  const long long row0 = (long long)w * n;
  const int s1 = 2 * ws2 - 1, s0 = (2 * ws1 - 1) * s1;
  constexpr float kLog2e = 1.4426950408889634f;

  for (int i = threadIdx.x; i < npad * 2; i += blockDim.x) {
    const int t = i >> 1, hf = i & 1;
    uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
    if (t < n) {
      kv = *reinterpret_cast<const uint4*>(base + ((long long)(C8 + 2 * h + hf) * T + row0 + t) * 8);
      vv = *reinterpret_cast<const uint4*>(base + ((long long)(2 * C8 + 2 * h + hf) * T + row0 + t) * 8);
    }
    *reinterpret_cast<uint4*>(sK + t * kAttKStride + hf * 8) = kv;
    const __half* vh = reinterpret_cast<const __half*>(&vv);
#pragma unroll
    for (int j = 0; j < 8; ++j) sVt[(hf * 8 + j) * vstride + t] = vh[j];
  }
  for (int i = threadIdx.x; i < tab_len; i += blockDim.x) sTab[i] = table[(long long)i * heads + h] * kLog2e;
  for (int i = threadIdx.x; i < npad; i += blockDim.x) {
    const int td = i / (ws1 * ws2), th = (i / ws2) % ws1, tw = i % ws2;
    // padded keys (i >= n) are masked by the TAIL step; their index only has to stay inside the table
    sLin[i] = (unsigned short)(i < n ? 4 * (td * s0 + th * s1 + tw) : 0);   // byte offset into the fp32 table
    sReg[i] = (MASK && i < n) ? (unsigned char)region[(long long)w * n + i] : 0;
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  const int nwarps = blockDim.x >> 5;
  const int lin_c = (ws0 - 1) * s0 + (ws1 - 1) * s1 + (ws2 - 1);
  const float scale2 = scale * kLog2e;
  const int n_full = n / 32 * 32;
  __half* ob = out + (long long)b * C8 * T * 8;
  for (int rt = warp; rt * 16 < n; rt += nwarps) {
    const int r0 = rt * 16 + g, r1 = r0 + 8;
    // Q fragments (row-major A operand): a0 (r0, d 2t..), a1 (r1, d 2t..), a2 (r0, d 2t+8..), a3 (r1, d 2t+8..)
    uint32_t qa[4] = {0, 0, 0, 0};
    if (r0 < n) {
      qa[0] = *reinterpret_cast<const uint32_t*>(base + ((long long)(2 * h) * T + row0 + r0) * 8 + 2 * t4);
      qa[2] = *reinterpret_cast<const uint32_t*>(base + ((long long)(2 * h + 1) * T + row0 + r0) * 8 + 2 * t4);
    }
    if (r1 < n) {
      qa[1] = *reinterpret_cast<const uint32_t*>(base + ((long long)(2 * h) * T + row0 + r1) * 8 + 2 * t4);
      qa[3] = *reinterpret_cast<const uint32_t*>(base + ((long long)(2 * h + 1) * T + row0 + r1) * 8 + 2 * t4);
    }
    AttRow r;
    r.lin0 = sLin[min(r0, npad - 1)] + 4 * lin_c; r.lin1 = sLin[min(r1, npad - 1)] + 4 * lin_c;
    r.reg0 = sReg[min(r0, npad - 1)]; r.reg1 = sReg[min(r1, npad - 1)];
    r.m0 = r.m1 = -INFINITY; r.l0 = r.l1 = 0.f;
#pragma unroll
    for (int dt = 0; dt < 2; ++dt) r.o[dt][0] = r.o[dt][1] = r.o[dt][2] = r.o[dt][3] = 0.f;
    for (int j0 = 0; j0 < n_full; j0 += 32) att_step32<MASK, false>(qa, r, j0, n, scale2, sK, sVt, vstride, sTab, sLin, sReg, g, t4);
    if (n_full < n) att_step32<MASK, true>(qa, r, n_full, n, scale2, sK, sVt, vstride, sTab, sLin, sReg, g, t4);
    float l0 = r.l0, l1 = r.l1;
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
    for (int dt = 0; dt < 2; ++dt) {
      if (r0 < n) *reinterpret_cast<uint32_t*>(ob + ((long long)(2 * h + dt) * T + row0 + r0) * 8 + 2 * t4) = pack_h2(r.o[dt][0] * i0, r.o[dt][1] * i0);
      if (r1 < n) *reinterpret_cast<uint32_t*>(ob + ((long long)(2 * h + dt) * T + row0 + r1) * 8 + 2 * t4) = pack_h2(r.o[dt][2] * i1, r.o[dt][3] * i1);
    }
  }
}

// -------------------------------------------------------------------------------------- single-input-channel convs
// Each thread computes kVox consecutive output voxels along W for all Cout channels, 8 channels at a time: the k*k*
// (k + (kVox-1)*stride) input values live in registers, every weight vector is read from shared memory once (LDS.128)
// and reused for the kVox voxels, so the inner loop is FMA-bound (32 FMA per 2 LDS.128).
constexpr int kVox = 4;

template <typename T, int KS, int STRIDE>
__global__ void __launch_bounds__(128) conv_cin1_nc8_kernel(const T* __restrict__ x, __half* __restrict__ y, const float* __restrict__ wgt,
                                                            const float* __restrict__ bias, int D, int H, int W, int Do, int Ho, int Wo,
                                                            int Cout, int pad, int out_ctot, int out_coff, float* __restrict__ stats) {
  extern __shared__ __align__(16) float s_w[];  // [taps][Cout], then one warp-private statistics row [2*Cout] per warp
  constexpr int taps = KS * KS * KS;
  constexpr int XW = KS + (kVox - 1) * STRIDE;
  float* s_st = s_w + taps * Cout;
  // the weights are staged once per block and the block then walks voxel groups with a grid stride (a block that handled
  // a single group spent longer fetching its 27 x Cout weights from L2 than computing)
  for (int i = threadIdx.x; i < taps * Cout; i += blockDim.x) {
    const int t = i % taps, co = i / taps;      // read the [Cout][taps] tensor linearly
    s_w[t * Cout + co] = wgt[i];
  }
  for (int i = threadIdx.x; i < 4 * 2 * Cout; i += blockDim.x) s_st[i] = 0.f;
  __syncthreads();
  const int n = blockIdx.y;
  float* ws = s_st + (threadIdx.x >> 5) * (2 * Cout);
  const int Wq = (Wo + kVox - 1) / kVox;
  const long long So = (long long)Do * Ho * Wo;
  const long long total = (long long)Do * Ho * Wq;
  const long long span = (long long)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  const T* xn = x + (long long)n * D * H * W;
  for (long long r0 = (long long)blockIdx.x * blockDim.x; r0 < total; r0 += span) {   // block-uniform trip count (warp reductions inside)
    const long long r = r0 + threadIdx.x;
    const bool ok = r < total;
    const int ox0 = ok ? (int)(r % Wq) * kVox : 0, oy = ok ? (int)((r / Wq) % Ho) : 0, oz = ok ? (int)(r / ((long long)Wq * Ho)) : 0;
    float xv[KS][KS][XW];
    if (ok) {
#pragma unroll
      for (int kz = 0; kz < KS; ++kz)
#pragma unroll
        for (int ky = 0; ky < KS; ++ky) {
          const int iz = oz * STRIDE - pad + kz, iy = oy * STRIDE - pad + ky;
          const bool rok = iz >= 0 && iz < D && iy >= 0 && iy < H;
#pragma unroll
          for (int q = 0; q < XW; ++q) {
            const int ix = ox0 * STRIDE - pad + q;
            xv[kz][ky][q] = (rok && ix >= 0 && ix < W) ? io<T>::ld(xn + ((long long)iz * H + iy) * W + ix) : 0.f;
          }
        }
    }
    const long long vbase = ((long long)oz * Ho + oy) * Wo + ox0;
    __half* yo = y + (((long long)n * (out_ctot / 8) + out_coff / 8) * So + vbase) * 8;
    for (int c0 = 0; c0 < Cout; c0 += 8) {
      float acc[kVox][8];
#pragma unroll
      for (int v = 0; v < kVox; ++v)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[v][j] = bias ? bias[c0 + j] : 0.f;
      if (ok) {
#pragma unroll
        for (int kz = 0; kz < KS; ++kz)
#pragma unroll
          for (int ky = 0; ky < KS; ++ky)
#pragma unroll
            for (int kx = 0; kx < KS; ++kx) {
              const int t = (kz * KS + ky) * KS + kx;
              const float4 w0 = *reinterpret_cast<const float4*>(s_w + t * Cout + c0);
              const float4 w1 = *reinterpret_cast<const float4*>(s_w + t * Cout + c0 + 4);
#pragma unroll
              for (int v = 0; v < kVox; ++v) {
                const float xt = xv[kz][ky][v * STRIDE + kx];
                acc[v][0] = fmaf(xt, w0.x, acc[v][0]); acc[v][1] = fmaf(xt, w0.y, acc[v][1]);
                acc[v][2] = fmaf(xt, w0.z, acc[v][2]); acc[v][3] = fmaf(xt, w0.w, acc[v][3]);
                acc[v][4] = fmaf(xt, w1.x, acc[v][4]); acc[v][5] = fmaf(xt, w1.y, acc[v][5]);
                acc[v][6] = fmaf(xt, w1.z, acc[v][6]); acc[v][7] = fmaf(xt, w1.w, acc[v][7]);
              }
            }
#pragma unroll
        for (int v = 0; v < kVox; ++v)
          if (ox0 + v < Wo) st8(yo + ((long long)(c0 / 8) * So + v) * 8, acc[v]);
      }
      if (stats) {
        float a8[8], q8[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float a = 0.f, q2 = 0.f;
#pragma unroll
          for (int v = 0; v < kVox; ++v)
            if (ok && ox0 + v < Wo) { a += acc[v][j]; q2 = fmaf(acc[v][j], acc[v][j], q2); }
          a8[j] = a; q8[j] = q2;
        }
        float cs, cq;
        transpose_reduce8(a8, q8, lane, cs, cq);
        if ((lane & 3) == 0) {   // warp-private row, eight distinct columns: no atomics (deterministic, stats.cuh)
          const int col = c0 + transpose_reduce8_col(lane);
          ws[2 * col] += cs;
          ws[2 * col + 1] += cq;
        }
      }
    }
  }
  if (stats) {   // partial rows [n][block][warp][2*Cout]; every block writes its four rows (zeros if it had no work)
    __syncwarp();
    float* dst = stats + (((long long)n * gridDim.x + blockIdx.x) * 4 + (threadIdx.x >> 5)) * (2 * Cout);
    for (int i = lane; i < 2 * Cout; i += 32) dst[i] = ws[i];
  }
}

template <typename TO>
__global__ void __launch_bounds__(256) head_conv_nc8_kernel(const __half* __restrict__ x, TO* __restrict__ y, const float* __restrict__ wgt,
                                                            const float* __restrict__ bias, int C, long long S, int Cout) {
  extern __shared__ float s_hw[];  // [Cout][C]
  for (int i = threadIdx.x; i < Cout * C; i += blockDim.x) s_hw[i] = wgt[i];
  __syncthreads();
  const int n = blockIdx.y;
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= S) return;
  float acc[16];
#pragma unroll
  for (int o = 0; o < 16; ++o) acc[o] = (o < Cout && bias) ? bias[o] : 0.f;
  const __half* xi = x + ((long long)n * (C / 8) * S + r) * 8;
  for (int c = 0; c < C / 8; ++c) {
    float f[8]; ld8(xi + (long long)c * S * 8, f);
#pragma unroll
    for (int o = 0; o < 16; ++o)
      if (o < Cout) {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[o] = fmaf(f[j], s_hw[o * C + c * 8 + j], acc[o]);
      }
  }
#pragma unroll
  for (int o = 0; o < 16; ++o)
    if (o < Cout) io<TO>::st(y + ((long long)n * Cout + o) * S + r, acc[o]);
}

// Output head fused with the tail of the last residual or basic block (UnetResBlock / UnetBasicBlock.forward,
// dynunet_block.py:97-111 / 165-177, followed by UnetOutBlock): y = W * lrelu(instnorm(x) + instnorm?(res)) + b, x's norm
// optionally affine.  The normalised activation never goes to HBM.
struct HeadNormP {
  const __half* x; const __half* res; const float* stats; const float* res_stats; const float* wgt; const float* bias; void* y;
  int C, Cout, res_ctot, res_coff;
  long long S;
  float eps, slope;
  const float* gamma; const float* beta;   // affine parameters of x's InstanceNorm, float32 [C] (NULL = non-affine)
};

// CO = compile-time bound on the output channels (registers and FMAs are spent on CO, not on the ABI maximum of 16)
template <typename TO, int CO>
__global__ void __launch_bounds__(256) head_conv_norm_nc8_kernel(HeadNormP p) {
  extern __shared__ float s_hn[];  // [Cout][C] weights, then scale, shift, res scale, res shift [C] each
  float* s_sc = s_hn + p.Cout * p.C;
  float* s_sh = s_sc + p.C;
  float* s_rsc = s_sh + p.C;
  float* s_rsh = s_rsc + p.C;
  const int n = blockIdx.y;
  for (int i = threadIdx.x; i < p.Cout * p.C; i += blockDim.x) s_hn[i] = p.wgt[i];
  const float invS = 1.f / (float)p.S;
  for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
    // the helper of norm_act_nc8_kernel: same (scale, shift) bits
    const float2 k = instnorm_scale_shift(p.stats[2 * (n * p.C + c)], p.stats[2 * (n * p.C + c) + 1], invS, p.eps, p.gamma, p.beta, c);
    s_sc[c] = k.x; s_sh[c] = k.y;
    float rsc = 1.f, rsh = 0.f;
    if (p.res_stats) {
      const float2 r = instnorm_scale_shift(p.res_stats[2 * (n * p.C + c)], p.res_stats[2 * (n * p.C + c) + 1], invS, p.eps, nullptr, nullptr, c);
      rsc = r.x; rsh = r.y;
    }
    s_rsc[c] = rsc; s_rsh[c] = rsh;
  }
  __syncthreads();
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.S) return;
  float acc[CO];
#pragma unroll
  for (int o = 0; o < CO; ++o) acc[o] = (o < p.Cout && p.bias) ? p.bias[o] : 0.f;
  const __half* xi = p.x + ((long long)n * (p.C / 8) * p.S + r) * 8;
  const __half* ri = p.res ? p.res + (((long long)n * (p.res_ctot / 8) + p.res_coff / 8) * p.S + r) * 8 : nullptr;
  auto lds8 = [](const float* s, float (&v)[8]) {   // two 16-byte broadcast reads
    const float4 a = *reinterpret_cast<const float4*>(s), b = *reinterpret_cast<const float4*>(s + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  };
  for (int c = 0; c < p.C / 8; ++c) {
    float f[8], k0[8], k1[8];
    cvt8(__ldg(reinterpret_cast<const uint4*>(xi + (long long)c * p.S * 8)), f);
    lds8(s_sc + c * 8, k0); lds8(s_sh + c * 8, k1);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = fmaf(f[j], k0[j], k1[j]);
    if (ri) {
      float g[8];
      cvt8(__ldg(reinterpret_cast<const uint4*>(ri + (long long)c * p.S * 8)), g);
      lds8(s_rsc + c * 8, k0); lds8(s_rsh + c * 8, k1);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] += fmaf(g[j], k0[j], k1[j]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = f[j] >= 0.f ? f[j] : f[j] * p.slope;
#pragma unroll
    for (int o = 0; o < CO; ++o)
      if (o < p.Cout) {
        lds8(s_hn + o * p.C + c * 8, k0);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[o] = fmaf(f[j], k0[j], acc[o]);
      }
  }
#pragma unroll
  for (int o = 0; o < CO; ++o)
    if (o < p.Cout) io<TO>::st((TO*)p.y + ((long long)n * p.Cout + o) * p.S + r, acc[o]);
}

}  // namespace b200

using namespace b200;

// the body of b200_head_conv_norm_nc8 and b200_head_conv_norm_affine_nc8
static int head_conv_norm_nc8_launch(const void* x, int N, int C, long long S, const float* stats, float eps, const void* res,
                                     int res_ctot, int res_coff, const float* res_stats, float slope, const float* weight,
                                     const float* bias, int Cout, void* y, int out_dtype, const float* gamma, const float* beta,
                                     void* stream) {
  B200_REQUIRE(x && y && weight && stats, "head_conv_norm_nc8: null pointer");
  B200_REQUIRE(C % 8 == 0 && Cout >= 1 && Cout <= 16, "head_conv_norm_nc8: C must be a multiple of 8 and Cout <= 16 (got %d, %d)", C, Cout);
  B200_REQUIRE(!res || (res_ctot % 8 == 0 && res_coff % 8 == 0 && res_coff + C <= res_ctot), "head_conv_norm_nc8: bad residual channel slice");
  B200_REQUIRE(res || !res_stats, "head_conv_norm_nc8: residual statistics without a residual");
  B200_REQUIRE(out_dtype == B200_DT_F16 || out_dtype == B200_DT_F32, "head_conv_norm_nc8: bad dtype");
  HeadNormP p{(const __half*)x, (const __half*)res, stats, res_stats, weight, bias, y, C, Cout, res_ctot, res_coff, S, eps, slope, gamma, beta};
  dim3 grid(ceil_div(S, 256), N);
  const size_t smem = ((size_t)Cout * C + 4 * (size_t)C) * sizeof(float);
  B200_REQUIRE(smem <= 48 * 1024, "head_conv_norm_nc8: C too large (%d)", C);
  cudaStream_t st = (cudaStream_t)stream;
#define LHN(TO) do { if (Cout <= 2) head_conv_norm_nc8_kernel<TO, 2><<<grid, 256, smem, st>>>(p); \
                     else if (Cout <= 4) head_conv_norm_nc8_kernel<TO, 4><<<grid, 256, smem, st>>>(p); \
                     else head_conv_norm_nc8_kernel<TO, 16><<<grid, 256, smem, st>>>(p); } while (0)
  if (out_dtype == B200_DT_F16) LHN(__half);
  else if (out_dtype == B200_DT_F32) LHN(float);
  else return set_err(B200_ERR_INVALID, "head_conv_norm_nc8: bad dtype");
#undef LHN
  B200_LAUNCH_CHECK("head_conv_norm_nc8_kernel");
  return B200_OK;
}

extern "C" int b200_head_conv_norm_nc8(const void* x, int N, int C, long long S, const float* stats, float eps, const void* res,
                                       int res_ctot, int res_coff, const float* res_stats, float slope, const float* weight,
                                       const float* bias, int Cout, void* y, int out_dtype, void* stream) {
  return head_conv_norm_nc8_launch(x, N, C, S, stats, eps, res, res_ctot, res_coff, res_stats, slope, weight, bias, Cout, y, out_dtype,
                                   nullptr, nullptr, stream);
}

extern "C" int b200_head_conv_norm_affine_nc8(const void* x, int N, int C, long long S, const float* stats, float eps, const void* res,
                                              int res_ctot, int res_coff, const float* res_stats, float slope, const float* weight,
                                              const float* bias, int Cout, void* y, int out_dtype, const float* gamma,
                                              const float* beta, void* stream) {
  return head_conv_norm_nc8_launch(x, N, C, S, stats, eps, res, res_ctot, res_coff, res_stats, slope, weight, bias, Cout, y, out_dtype,
                                   gamma, beta, stream);
}

extern "C" int b200_layernorm_nc8(const void* x, int N, int C, long long S_in, const int32_t* src, long long S_out,
                                  const float* gamma, const float* beta, float eps, void* y, void* stream) {
  B200_REQUIRE(x && y, "layernorm_nc8: null pointer");
  B200_REQUIRE(N > 0 && C > 0 && C % 8 == 0 && S_in > 0 && S_out > 0, "layernorm_nc8: bad sizes");
  dim3 grid(ceil_div(S_out, 256), N);
  B200_REQUIRE((!gamma || reinterpret_cast<uintptr_t>(gamma) % 16 == 0) && (!beta || reinterpret_cast<uintptr_t>(beta) % 16 == 0),
               "layernorm_nc8: gamma / beta must be 16-byte aligned");
#define LLN(K) layernorm_nc8_kernel<K><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)x, (__half*)y, C, S_in, src, S_out, gamma, beta, eps)
#define LL8(P) layernorm8_nc8_kernel<P><<<dim3(ceil_div(S_out, 32), N), 256, 0, (cudaStream_t)stream>>>((const __half*)x, (__half*)y, S_in, src, S_out, gamma, beta, eps)
  if (C == 48) LLN(6);
  else if (C == 192) LL8(3);
  else if (C == 384) LL8(6);
  else if (C == 768) LL8(12);
  else LLN(0);
#undef LLN
#undef LL8
  B200_LAUNCH_CHECK("layernorm_nc8_kernel");
  return B200_OK;
}

extern "C" int b200_patch_merge_ln_nc8(const void* x, int N, int C, int D, int H, int W, const float* gamma,
                                       const float* beta, float eps, int v2, void* y, void* stream) {
  B200_REQUIRE(x && y, "patch_merge_ln_nc8: null pointer");
  B200_REQUIRE(N > 0 && C > 0 && C % 8 == 0 && D > 0 && H > 0 && W > 0, "patch_merge_ln_nc8: bad sizes");
  const long long S2 = (long long)((D + 1) / 2) * ((H + 1) / 2) * ((W + 1) / 2);
  B200_REQUIRE((!gamma || reinterpret_cast<uintptr_t>(gamma) % 16 == 0) && (!beta || reinterpret_cast<uintptr_t>(beta) % 16 == 0),
               "patch_merge_ln_nc8: gamma / beta must be 16-byte aligned");
  dim3 g8(ceil_div(S2, 32), N);
#define LPM(K) patch_merge_ln8_nc8_kernel<K><<<g8, 256, 0, (cudaStream_t)stream>>>((const __half*)x, (__half*)y, C, D, H, W, gamma, beta, eps, v2)
  if (C == 48) LPM(6); else if (C == 96) LPM(12); else LPM(0);
#undef LPM
  B200_LAUNCH_CHECK("patch_merge_ln_nc8_kernel");
  return B200_OK;
}

extern "C" int b200_window_attention_nc8(const void* qkv, int N, int C, int heads, int nW, int n, float scale,
                                         const float* table, int ws0, int ws1, int ws2, const int32_t* region, void* out,
                                         void* stream) {
  B200_REQUIRE(qkv && out && table, "window_attention_nc8: null pointer");
  B200_REQUIRE(N > 0 && heads > 0 && nW > 0 && n > 0, "window_attention_nc8: empty problem");
  B200_REQUIRE(C == heads * 16, "window_attention_nc8: head_dim must be 16 (C = %d, heads = %d)", C, heads);
  B200_REQUIRE(ws0 > 0 && ws1 > 0 && ws2 > 0 && n <= ws0 * ws1 * ws2, "window_attention_nc8: window of %d tokens exceeds the module window", n);
  B200_REQUIRE(heads <= 65535 && N <= 65535, "window_attention_nc8: grid too large");
  const int npad = (n + 31) / 32 * 32;
  const int tab_len = (2 * ws0 - 1) * (2 * ws1 - 1) * (2 * ws2 - 1);
  B200_REQUIRE(tab_len < 16384, "window_attention_nc8: relative position table too large");   // byte offsets are kept in 16 bits
  const size_t smem = (size_t)npad * kAttKStride * 2 + (size_t)16 * (npad + 8) * 2 + (size_t)tab_len * 4 + (size_t)npad * 2 + npad + 16;
  B200_REQUIRE(smem <= 200 * 1024, "window_attention_nc8: window of %d tokens does not fit in shared memory", n);
  auto kern = region ? window_attention_nc8_kernel<true> : window_attention_nc8_kernel<false>;
  B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  dim3 grid(nW, heads, N);
  const int threads = n >= 128 ? 256 : (n >= 64 ? 128 : 64);
  kern<<<grid, threads, smem, (cudaStream_t)stream>>>((const __half*)qkv, (__half*)out, C, heads, nW, n, scale, table, tab_len, ws0, ws1, ws2, region);
  B200_LAUNCH_CHECK("window_attention_nc8_kernel");
  return B200_OK;
}

static dim3 cin1_grid(int N, int Do, int Ho, int Wo) {
  const long long units = (long long)Do * Ho * ((Wo + kVox - 1) / kVox);
  // a few resident waves of blocks per batch item; each block strides over the voxel groups
  const long long per_item = std::max<long long>(1, (long long)num_sms() * 8 / std::max(1, N));
  return dim3((unsigned)std::min<long long>(ceil_div(units, 128), per_item), N);
}

template <typename T>
static int launch_cin1(const T* x, __half* y, const float* weight, const float* bias, int N, int D, int H, int W, int Do, int Ho, int Wo,
                       int Cout, int k, int stride, int pad, int out_ctot, int out_coff, float* partials, cudaStream_t st) {
  const dim3 grid = cin1_grid(N, Do, Ho, Wo);
  const size_t smem = ((size_t)k * k * k * Cout + 4 * 2 * Cout) * sizeof(float);
#define LCI(KS, SS) conv_cin1_nc8_kernel<T, KS, SS><<<grid, 128, smem, st>>>(x, y, weight, bias, D, H, W, Do, Ho, Wo, Cout, pad, out_ctot, out_coff, partials)
  if (k == 3 && stride == 1) LCI(3, 1);
  else if (k == 2 && stride == 2) LCI(2, 2);
  else if (k == 1 && stride == 1) LCI(1, 1);
  else if (k == 3 && stride == 2) LCI(3, 2);
  else return set_err(B200_ERR_UNSUPPORTED, "conv_cin1_nc8: (kernel, stride) must be (3,1), (2,2), (1,1) or (3,2), got (%d,%d)", k, stride);
#undef LCI
  B200_LAUNCH_CHECK("conv_cin1_nc8_kernel");
  return B200_OK;
}

extern "C" long long b200_conv_cin1_nc8_workspace_bytes(int N, int D, int H, int W, int Cout, int k, int stride, int pad) {
  if (N <= 0 || Cout <= 0 || k < 1 || stride < 1) return -1;
  const int Do = (D + 2 * pad - k) / stride + 1, Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  if (Do <= 0 || Ho <= 0 || Wo <= 0) return -1;
  return (long long)N * cin1_grid(N, Do, Ho, Wo).x * 4 * 2 * Cout * (long long)sizeof(float);
}

extern "C" int b200_conv_cin1_nc8(const void* x, int dtype, int N, int D, int H, int W, const float* weight, const float* bias,
                                  int Cout, int k, int stride, int pad, void* y, int out_ctot, int out_coff, float* stats,
                                  void* workspace, void* stream) {
  B200_REQUIRE(x && y && weight, "conv_cin1_nc8: null pointer");
  B200_REQUIRE(!stats || workspace, "conv_cin1_nc8: statistics need the workspace of b200_conv_cin1_nc8_workspace_bytes()");
  B200_REQUIRE(k >= 1 && k <= 3 && stride >= 1 && pad >= 0, "conv_cin1_nc8: kernel size must be 1..3");
  B200_REQUIRE(Cout > 0 && Cout % 8 == 0 && out_ctot % 8 == 0 && out_coff % 8 == 0 && out_coff + Cout <= out_ctot,
               "conv_cin1_nc8: channel counts must be multiples of 8");
  const int Do = (D + 2 * pad - k) / stride + 1, Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  B200_REQUIRE(Do > 0 && Ho > 0 && Wo > 0, "conv_cin1_nc8: empty output");
  B200_REQUIRE(((size_t)k * k * k * Cout + 4 * 2 * Cout) * sizeof(float) <= 48 * 1024, "conv_cin1_nc8: Cout too large");
  B200_REQUIRE(!stats || 2 * Cout <= 1024, "conv_cin1_nc8: Cout too large for the statistics pass");
  cudaStream_t st = (cudaStream_t)stream;
  float* part = stats ? (float*)workspace : nullptr;
  int rc;
  if (dtype == B200_DT_F16)
    rc = launch_cin1<__half>((const __half*)x, (__half*)y, weight, bias, N, D, H, W, Do, Ho, Wo, Cout, k, stride, pad, out_ctot, out_coff, part, st);
  else if (dtype == B200_DT_F32)
    rc = launch_cin1<float>((const float*)x, (__half*)y, weight, bias, N, D, H, W, Do, Ho, Wo, Cout, k, stride, pad, out_ctot, out_coff, part, st);
  else return set_err(B200_ERR_INVALID, "conv_cin1_nc8: bad dtype");
  if (rc || !stats) return rc;
  return launch_stats_finish(part, N, (int)cin1_grid(N, Do, Ho, Wo).x * 4, Cout, 1, Cout, stats, st);
}

extern "C" int b200_head_conv_nc8(const void* x, int N, int C, long long S, const float* weight, const float* bias, int Cout,
                                  void* y, int out_dtype, void* stream) {
  B200_REQUIRE(x && y && weight, "head_conv_nc8: null pointer");
  B200_REQUIRE(C % 8 == 0 && Cout >= 1 && Cout <= 16, "head_conv_nc8: C must be a multiple of 8 and Cout <= 16 (got %d, %d)", C, Cout);
  dim3 grid(ceil_div(S, 256), N);
  const size_t smem = (size_t)Cout * C * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  if (out_dtype == B200_DT_F16) head_conv_nc8_kernel<__half><<<grid, 256, smem, st>>>((const __half*)x, (__half*)y, weight, bias, C, S, Cout);
  else if (out_dtype == B200_DT_F32) head_conv_nc8_kernel<float><<<grid, 256, smem, st>>>((const __half*)x, (float*)y, weight, bias, C, S, Cout);
  else return set_err(B200_ERR_INVALID, "head_conv_nc8: bad dtype");
  B200_LAUNCH_CHECK("head_conv_nc8_kernel");
  return B200_OK;
}
