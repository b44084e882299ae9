// Affine-driven 3-D resampling and zero-padded separable filtering (SURVEY.md §8 rows a15, a16, a19).
//
// Resample: the reference materialises a dense coordinate grid (F.affine_grid or create_grid @ affine) and
// calls F.grid_sample (monai/networks/layers/spatial_transforms.py:584-591, monai/transforms/spatial/array.py:2102-2115).
// Coordinates are an affine function of the output index, so this kernel evaluates them on the fly in fp64
// (the reference's default coordinate dtype, spatial/array.py:355,1972) and never builds the grid.
// Sampling semantics follow ATen grid_sampler_3d (unnormalised coordinates are produced by the host):
//   padding zeros / border / reflection (reflection bounds depend on align_corners), nearest = round-half-even.
#include "common.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

struct ResampleP {
  const void* src; void* dst;
  int C, Di, Hi, Wi, Do, Ho, Wo;
  double m[12];
  int interp, pad, align;
};

__device__ __forceinline__ double reflect_coord(double in, double twice_low, double twice_high) {
  if (twice_low == twice_high) return 0.0;
  const double mn = twice_low / 2.0, span = (twice_high - twice_low) / 2.0;
  in = fabs(in - mn);
  const double extra = fmod(in, span);
  const int flips = (int)floor(in / span);
  return (flips & 1) ? span - extra + mn : extra + mn;
}

__device__ __forceinline__ double pad_coord(double x, int size, int pad, int align) {
  if (pad == 1) {
    x = fmin((double)(size - 1), fmax(x, 0.0));
  } else if (pad == 2) {
    x = align ? reflect_coord(x, 0.0, 2.0 * (size - 1)) : reflect_coord(x, -1.0, 2.0 * size - 1.0);
    x = fmin((double)(size - 1), fmax(x, 0.0));
  }
  return x;
}

constexpr int kRsVox = 4;   // consecutive output voxels along W per thread (independent gathers in flight, 16-byte stores)

// A block is 32 (w quads) x 8 (h rows) threads = a 128 x 8 output patch of one depth plane: one voxel per thread and one
// block per W row left the chip waiting on block turnover (204,800 tiny blocks for a 320^3 output, 3 % of HBM bandwidth).
// MODE 0: trilinear with zeros padding, 3: trilinear with border padding (both: fp64 base coordinate + fp32 increments),
// 1: trilinear with reflection padding (fp64 per voxel), 2: nearest.  Separate instantiations: the common paths carry no
// fp64 reflection code, and the border path needs no corner validity tests (a clamped coordinate has valid corners).
template <typename TI, typename TO, int MODE>
__global__ void __launch_bounds__(256) resample_affine_kernel(ResampleP p) {
  const int k0 = (blockIdx.x * 32 + threadIdx.x) * kRsVox;  // fastest output axis
  const int j = blockIdx.y * 8 + threadIdx.y, i = blockIdx.z;
  if (k0 >= p.Wo || j >= p.Ho) return;
  const long long in_cs = (long long)p.Di * p.Hi * p.Wi, out_cs = (long long)p.Do * p.Ho * p.Wo;
  const long long o0 = ((long long)i * p.Ho + j) * p.Wo + k0;
  const TI* src = (const TI*)p.src;
  TO* dst = (TO*)p.dst;
  // the (i, j) part of the affine map is shared by the thread's voxels; each voxel still evaluates the full fma chain
  // in the reference's order so the coordinates are bit-identical to the one-voxel formulation
  if (MODE == 2) {
#pragma unroll
    for (int v = 0; v < kRsVox; ++v) {
      const int k = k0 + v;
      if (k >= p.Wo) break;
      double a = fma(p.m[0], (double)i, fma(p.m[1], (double)j, fma(p.m[2], (double)k, p.m[3])));
      double b = fma(p.m[4], (double)i, fma(p.m[5], (double)j, fma(p.m[6], (double)k, p.m[7])));
      double c = fma(p.m[8], (double)i, fma(p.m[9], (double)j, fma(p.m[10], (double)k, p.m[11])));
      a = pad_coord(a, p.Di, p.pad, p.align); b = pad_coord(b, p.Hi, p.pad, p.align); c = pad_coord(c, p.Wi, p.pad, p.align);
      const int ia = (int)nearbyint(a), ib = (int)nearbyint(b), ic = (int)nearbyint(c);
      const bool ok = ia >= 0 && ia < p.Di && ib >= 0 && ib < p.Hi && ic >= 0 && ic < p.Wi;
      const long long off = ((long long)ia * p.Hi + ib) * p.Wi + ic;
      for (int ch = 0; ch < p.C; ++ch) io<TO>::st(dst + ch * out_cs + o0 + v, ok ? io<TI>::ld(src + ch * in_cs + off) : 0.f);
    }
    return;
  }
  float wgt[kRsVox][8];
  int off[kRsVox][8];   // element offsets inside one channel (the launcher requires Di*Hi*Wi < 2^31)
  // Trilinear, zeros / border padding: the coordinate of the thread's first voxel is evaluated in fp64 (the reference's
  // coordinate dtype) and split into integer + fraction; the next three voxels add v * m[.,k] to the fraction in fp32
  // (|error| < 1e-6 voxel).  Only 1/4 of the fp64 work per voxel remains -- the fp64 pipe, not HBM, bounded this kernel.
  constexpr bool split = MODE == 0 || MODE == 3;
  int IA = 0, IB = 0, IC = 0;
  float FA = 0.f, FB = 0.f, FC = 0.f;
  if (split) {
    const double a = fma(p.m[0], (double)i, fma(p.m[1], (double)j, fma(p.m[2], (double)k0, p.m[3])));
    const double b = fma(p.m[4], (double)i, fma(p.m[5], (double)j, fma(p.m[6], (double)k0, p.m[7])));
    const double c = fma(p.m[8], (double)i, fma(p.m[9], (double)j, fma(p.m[10], (double)k0, p.m[11])));
    // clamp far-away coordinates first so the integer conversion cannot overflow (anything beyond is fully outside / clamped anyway)
    const double lim = 1.0e9;
    const double ac = fmin(lim, fmax(-lim, a)), bc = fmin(lim, fmax(-lim, b)), cc = fmin(lim, fmax(-lim, c));
    const double fa = floor(ac), fb = floor(bc), fc = floor(cc);
    IA = (int)fa; IB = (int)fb; IC = (int)fc;
    FA = (float)(ac - fa); FB = (float)(bc - fb); FC = (float)(cc - fc);
  }
  const float sa = (float)p.m[2], sb = (float)p.m[6], sc = (float)p.m[10];
#pragma unroll
  for (int v = 0; v < kRsVox; ++v) {
    int a0, b0, c0;
    float ta, tb, tc;
    if (split) {
      const float av = fmaf((float)v, sa, FA), bv = fmaf((float)v, sb, FB), cv = fmaf((float)v, sc, FC);
      const float fa = floorf(av), fb = floorf(bv), fc = floorf(cv);
      a0 = IA + (int)fa; b0 = IB + (int)fb; c0 = IC + (int)fc;
      ta = av - fa; tb = bv - fb; tc = cv - fc;
      if (MODE == 3) {  // border: clamp the coordinate to [0, size-1]
        if (a0 < 0) { a0 = 0; ta = 0.f; } else if (a0 >= p.Di - 1) { a0 = p.Di - 1; ta = 0.f; }
        if (b0 < 0) { b0 = 0; tb = 0.f; } else if (b0 >= p.Hi - 1) { b0 = p.Hi - 1; tb = 0.f; }
        if (c0 < 0) { c0 = 0; tc = 0.f; } else if (c0 >= p.Wi - 1) { c0 = p.Wi - 1; tc = 0.f; }
      }
    } else {
      const int k = min(k0 + v, p.Wo - 1);
      double a = fma(p.m[0], (double)i, fma(p.m[1], (double)j, fma(p.m[2], (double)k, p.m[3])));
      double b = fma(p.m[4], (double)i, fma(p.m[5], (double)j, fma(p.m[6], (double)k, p.m[7])));
      double c = fma(p.m[8], (double)i, fma(p.m[9], (double)j, fma(p.m[10], (double)k, p.m[11])));
      a = pad_coord(a, p.Di, p.pad, p.align); b = pad_coord(b, p.Hi, p.pad, p.align); c = pad_coord(c, p.Wi, p.pad, p.align);
      const double fa = floor(a), fb = floor(b), fc = floor(c);
      a0 = (int)fa; b0 = (int)fb; c0 = (int)fc;
      ta = (float)(a - fa); tb = (float)(b - fb); tc = (float)(c - fc);
    }
    // per-axis weights with out-of-volume corners zeroed, and corner indices clamped into the volume so that every gather is
    // a valid address: eight offsets are then one base plus {0, dW} + {0, dH} + {0, dD}
    float wa[2] = {1.f - ta, ta}, wb[2] = {1.f - tb, tb}, wc[2] = {1.f - tc, tc};
    int a0c = a0, b0c = b0, c0c = c0, a1c, b1c, c1c;
    if (MODE == 3) {
      // the clamped coordinate lies in [0, size-1]: corner 0 is valid, corner 1 is at most `size` and then carries weight 0
      a1c = min(a0 + 1, p.Di - 1); b1c = min(b0 + 1, p.Hi - 1); c1c = min(c0 + 1, p.Wi - 1);
    } else {
      if (a0 < 0 || a0 >= p.Di) wa[0] = 0.f;
      if (a0 + 1 < 0 || a0 + 1 >= p.Di) wa[1] = 0.f;
      if (b0 < 0 || b0 >= p.Hi) wb[0] = 0.f;
      if (b0 + 1 < 0 || b0 + 1 >= p.Hi) wb[1] = 0.f;
      if (c0 < 0 || c0 >= p.Wi) wc[0] = 0.f;
      if (c0 + 1 < 0 || c0 + 1 >= p.Wi) wc[1] = 0.f;
      a0c = min(max(a0, 0), p.Di - 1); a1c = min(max(a0 + 1, 0), p.Di - 1);
      b0c = min(max(b0, 0), p.Hi - 1); b1c = min(max(b0 + 1, 0), p.Hi - 1);
      c0c = min(max(c0, 0), p.Wi - 1); c1c = min(max(c0 + 1, 0), p.Wi - 1);
    }
    const int base = (a0c * p.Hi + b0c) * p.Wi + c0c;
    const int dD = (a1c - a0c) * p.Hi * p.Wi, dH = (b1c - b0c) * p.Wi, dW = c1c - c0c;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int da = q >> 2, db = (q >> 1) & 1, dc = q & 1;
      wgt[v][q] = wa[da] * wb[db] * wc[dc];
      off[v][q] = base + (da ? dD : 0) + (db ? dH : 0) + (dc ? dW : 0);
    }
  }
  for (int ch = 0; ch < p.C; ++ch) {
    const TI* s = src + ch * in_cs;
    float r[kRsVox];
#pragma unroll
    for (int v = 0; v < kRsVox; ++v) {
      float acc = 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q) acc = fmaf(io<TI>::ld(s + off[v][q]), wgt[v][q], acc);
      r[v] = acc;
    }
#pragma unroll
    for (int v = 0; v < kRsVox; ++v)
      if (k0 + v < p.Wo) io<TO>::st(dst + ch * out_cs + o0 + v, r[v]);
  }
}

// out[i] = sum_t taps[t] * in[i + (t - r) * stride] along one axis, zero outside.
template <typename TI, typename TO>
__global__ void __launch_bounds__(256) filter1d_kernel(const TI* __restrict__ in, TO* __restrict__ out,
                                                       const float* __restrict__ taps, int n, long long total,
                                                       long long stride, int extent) {
  __shared__ float s_t[128];
  for (int t = threadIdx.x; t < n; t += blockDim.x) s_t[t] = taps[t];
  __syncthreads();
  const int r = (n - 1) / 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pos = (int)((i / stride) % extent);
    float acc = 0.f;
    for (int t = 0; t < n; ++t) {
      const int q = pos + t - r;
      if (q >= 0 && q < extent) acc = fmaf(s_t[t], io<TI>::ld(in + i + (long long)(t - r) * stride), acc);
    }
    io<TO>::st(out + i, acc);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Register sliding-window forms of the same 1-D filter (N taps known at compile time, W % 4 == 0, fp32 in / out):
// every input value is loaded once per pass (plus the halo at run boundaries) as part of a 16-byte vector.  The tap order
// and the fused multiply-adds are those of filter1d_kernel; a tap that falls outside the volume multiplies a zero, which
// leaves the accumulator unchanged, so the results are bit-identical.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kFiltRun = 16;   // consecutive outputs along the filter axis per thread

// Filter along D or H (stride >= W): a thread owns four consecutive W positions and a run of kFiltRun positions along the
// filter axis; `lines` = number of (other axis) lines, addressed through (line_stride, stride).
template <int N>
__global__ void __launch_bounds__(256) filter_slide_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                           const float* __restrict__ taps, int W4, int extent, long long stride,
                                                           int lines, long long line_stride, long long chan_stride, int runs) {
  constexpr int R = (N - 1) / 2;
  const int w4 = blockIdx.x * blockDim.x + threadIdx.x;
  if (w4 >= W4) return;
  const int run = blockIdx.y % runs, line = blockIdx.y / runs, ch = blockIdx.z;
  float tp[N];
#pragma unroll
  for (int t = 0; t < N; ++t) tp[t] = __ldg(taps + t);
  const long long base = (long long)ch * chan_stride + (long long)line * line_stride + (long long)w4 * 4;
  const int p0 = run * kFiltRun;
  float4 win[N];
#pragma unroll
  for (int t = 0; t < N - 1; ++t) {
    const int q = p0 - R + t;
    win[t] = (q >= 0 && q < extent) ? __ldg(reinterpret_cast<const float4*>(in + base + (long long)q * stride)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll
  for (int s = 0; s < kFiltRun; ++s) {
    const int pos = p0 + s;
    if (pos >= extent) break;
    const int q = pos + R;
    win[(N - 1 + s) % N] = (q < extent) ? __ldg(reinterpret_cast<const float4*>(in + base + (long long)q * stride)) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int t = 0; t < N; ++t) {
      const float4 v = win[(s + t) % N];
      acc.x = fmaf(tp[t], v.x, acc.x); acc.y = fmaf(tp[t], v.y, acc.y); acc.z = fmaf(tp[t], v.z, acc.z); acc.w = fmaf(tp[t], v.w, acc.w);
    }
    *reinterpret_cast<float4*>(out + base + (long long)pos * stride) = acc;
  }
}

// Filter along W (stride 1): a thread produces four consecutive outputs from the 4 + 2R inputs around them, fetched as
// aligned 16-byte vectors (R <= 4: three vectors).
template <int N>
__global__ void __launch_bounds__(256) filter_w4_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                        const float* __restrict__ taps, int W, long long rows) {
  constexpr int R = (N - 1) / 2;
  static_assert(R <= 4, "three aligned vectors cover the window");
  const int W4 = W / 4;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * W4) return;
  const int w4 = (int)(idx % W4);
  const long long row = idx / W4;
  const float* rp = in + row * W;
  float tp[N];
#pragma unroll
  for (int t = 0; t < N; ++t) tp[t] = __ldg(taps + t);
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 a = w4 > 0 ? __ldg(reinterpret_cast<const float4*>(rp) + w4 - 1) : z;
  const float4 b = __ldg(reinterpret_cast<const float4*>(rp) + w4);
  const float4 c = w4 + 1 < W4 ? __ldg(reinterpret_cast<const float4*>(rp) + w4 + 1) : z;
  const float v[12] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w};   // positions 4*w4 - 4 .. 4*w4 + 7
  float r[4];
#pragma unroll
  for (int o = 0; o < 4; ++o) {
    float acc = 0.f;
#pragma unroll
    for (int t = 0; t < N; ++t) acc = fmaf(tp[t], v[4 + o + t - R], acc);
    r[o] = acc;
  }
  *reinterpret_cast<float4*>(out + row * W + (long long)w4 * 4) = make_float4(r[0], r[1], r[2], r[3]);
}

template <int N>
static void launch_filter_fast(const float* src, float* tmp, float* tmp2, float* dst, const float* td, const float* th, const float* tw, int C,
                               int D, int H, int W, cudaStream_t st) {
  const int W4 = W / 4;
  const long long HW = (long long)H * W, vol = (long long)D * HW;
  dim3 block(W4 >= 64 ? 64 : 32);
  {  // along D: lines = H
    const int runs = ceil_div(D, kFiltRun);
    dim3 grid(ceil_div(W4, block.x), H * runs, C);
    filter_slide_kernel<N><<<grid, block, 0, st>>>(src, tmp, td, W4, D, HW, H, W, vol, runs);
  }
  {  // along H: lines = D
    const int runs = ceil_div(H, kFiltRun);
    dim3 grid(ceil_div(W4, block.x), D * runs, C);
    filter_slide_kernel<N><<<grid, block, 0, st>>>(tmp, tmp2, th, W4, H, W, D, HW, vol, runs);
  }
  const long long rows = (long long)C * D * H;
  filter_w4_kernel<N><<<(unsigned)((rows * W4 + 255) / 256), 256, 0, st>>>(tmp2, dst, tw, W, rows);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_resample_affine(const void* src, int src_dtype, int C, int Di, int Hi, int Wi, void* dst,
                                    int dst_dtype, int Do, int Ho, int Wo, const double* mat3x4, int interp, int pad,
                                    int align_corners, void* stream) {
  B200_REQUIRE(src && dst && mat3x4, "resample_affine: null pointer");
  B200_REQUIRE(C > 0 && Di > 0 && Hi > 0 && Wi > 0, "resample_affine: empty source");
  if ((long long)Do * Ho * Wo == 0) return B200_OK;
  B200_REQUIRE(interp == 0 || interp == 1, "resample_affine: interp must be 0 (nearest) or 1 (trilinear)");
  B200_REQUIRE(pad >= 0 && pad <= 2, "resample_affine: pad must be 0 (zeros), 1 (border) or 2 (reflection)");
  B200_REQUIRE(Do <= 65535 && ceil_div(Ho, 8) <= 65535, "resample_affine: output too large for the launch grid");
  B200_REQUIRE((long long)Di * Hi * Wi < (1LL << 31), "resample_affine: source channel larger than 2^31 elements");
  ResampleP p;
  p.src = src; p.dst = dst; p.C = C; p.Di = Di; p.Hi = Hi; p.Wi = Wi; p.Do = Do; p.Ho = Ho; p.Wo = Wo;
  for (int q = 0; q < 12; ++q) p.m[q] = mat3x4[q];
  p.interp = interp; p.pad = pad; p.align = align_corners;
  dim3 block(32, 8), grid(ceil_div(Wo, 32 * kRsVox), ceil_div(Ho, 8), Do);
  cudaStream_t st = (cudaStream_t)stream;
#define LR(TI, TO) do { if (interp == 0) resample_affine_kernel<TI, TO, 2><<<grid, block, 0, st>>>(p); \
                       else if (pad == 2) resample_affine_kernel<TI, TO, 1><<<grid, block, 0, st>>>(p); \
                       else if (pad == 1) resample_affine_kernel<TI, TO, 3><<<grid, block, 0, st>>>(p); \
                       else resample_affine_kernel<TI, TO, 0><<<grid, block, 0, st>>>(p); } while (0)
  if (src_dtype == B200_DT_F32 && dst_dtype == B200_DT_F32) LR(float, float);
  else if (src_dtype == B200_DT_F16 && dst_dtype == B200_DT_F32) LR(__half, float);
  else if (src_dtype == B200_DT_F32 && dst_dtype == B200_DT_F16) LR(float, __half);
  else if (src_dtype == B200_DT_F16 && dst_dtype == B200_DT_F16) LR(__half, __half);
  else return set_err(B200_ERR_INVALID, "resample_affine: bad dtype");
#undef LR
  B200_LAUNCH_CHECK("resample_affine_kernel");
  return B200_OK;
}

extern "C" int b200_separable_filter3d(const void* src, int dtype, int C, int D, int H, int W, const float* taps_d,
                                       int n_d, const float* taps_h, int n_h, const float* taps_w, int n_w, float* tmp,
                                       void* dst, void* stream) {
  B200_REQUIRE(src && dst && tmp, "separable_filter3d: null pointer");
  B200_REQUIRE(n_d <= 127 && n_h <= 127 && n_w <= 127, "separable_filter3d: more than 127 taps");
  B200_REQUIRE(n_d % 2 && n_h % 2 && n_w % 2, "separable_filter3d: tap counts must be odd");
  const long long total = (long long)C * D * H * W;
  if (total == 0) return B200_OK;
  const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 32);
  cudaStream_t st = (cudaStream_t)stream;
  // reference order (simplelayers.py:170-204): first spatial axis first, last spatial axis last.
  // src -(D)-> tmp[0:total] -(H)-> tmp[total:2*total] -(W)-> dst; intermediates stay fp32.
  const bool f16 = dtype == B200_DT_F16;
  B200_REQUIRE(f16 || dtype == B200_DT_F32, "separable_filter3d: bad dtype");
  B200_REQUIRE(taps_d && taps_h && taps_w, "separable_filter3d: all three axis kernels are required");
  float* tmp2 = tmp + total;
  // fast path: fp32 volume, the same odd tap count <= 9 on the three axes, W % 4 == 0, 16-byte aligned buffers
  if (!f16 && n_d == n_h && n_h == n_w && n_d <= 9 && W % 4 == 0 && (long long)H * ceil_div(D, kFiltRun) <= 65535 &&
      (long long)D * ceil_div(H, kFiltRun) <= 65535 && C <= 65535 &&
      ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(tmp)) & 15) == 0) {
    const float* s = (const float*)src;
    float* d = (float*)dst;
    switch (n_d) {
      case 1: launch_filter_fast<1>(s, tmp, tmp2, d, taps_d, taps_h, taps_w, C, D, H, W, st); break;
      case 3: launch_filter_fast<3>(s, tmp, tmp2, d, taps_d, taps_h, taps_w, C, D, H, W, st); break;
      case 5: launch_filter_fast<5>(s, tmp, tmp2, d, taps_d, taps_h, taps_w, C, D, H, W, st); break;
      case 7: launch_filter_fast<7>(s, tmp, tmp2, d, taps_d, taps_h, taps_w, C, D, H, W, st); break;
      default: launch_filter_fast<9>(s, tmp, tmp2, d, taps_d, taps_h, taps_w, C, D, H, W, st); break;
    }
    B200_LAUNCH_CHECK("filter_slide_kernel");
    return B200_OK;
  }
  if (f16) filter1d_kernel<__half, float><<<blocks, 256, 0, st>>>((const __half*)src, tmp, taps_d, n_d, total, (long long)H * W, D);
  else filter1d_kernel<float, float><<<blocks, 256, 0, st>>>((const float*)src, tmp, taps_d, n_d, total, (long long)H * W, D);
  B200_LAUNCH_CHECK("filter1d_kernel(d)");
  filter1d_kernel<float, float><<<blocks, 256, 0, st>>>(tmp, tmp2, taps_h, n_h, total, (long long)W, H);
  B200_LAUNCH_CHECK("filter1d_kernel(h)");
  if (f16) filter1d_kernel<float, __half><<<blocks, 256, 0, st>>>(tmp2, (__half*)dst, taps_w, n_w, total, 1, W);
  else filter1d_kernel<float, float><<<blocks, 256, 0, st>>>(tmp2, (float*)dst, taps_w, n_w, total, 1, W);
  B200_LAUNCH_CHECK("filter1d_kernel(w)");
  return B200_OK;
}
