/*
 * monai_b200 C ABI -- the drop-in boundary of the H100-native sliding-window / spatial-transform hot path.
 *
 * The reference (Project-MONAI/MONAI) has NO native boundary for this path: the seam is Python
 * (monai/inferers/utils.py, monai/networks/blocks/convolutions.py, monai/transforms/spatial/array.py), and
 * its only native module, monai._C (monai/csrc/ext.cpp:21-75), is a pybind11/ATen extension.  This header is
 * the plain-C equivalent a maintainer would bind with ctypes (see INTEGRATION.md): raw device pointers,
 * sizes and an opaque CUDA stream handle -- no torch types.  Every function
 *   - returns 0 on success, non-zero on failure (b200_last_error() gives the thread-local message),
 *   - launches asynchronously on `stream` (a cudaStream_t / CUstream cast to void*),
 *   - never allocates, frees or retains caller memory beyond the call (tensor maps are built per call).
 *
 * dtype codes: 0 = float32, 1 = float16.
 */
#ifndef MONAI_B200_H_
#define MONAI_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_ABI_VERSION 2

/* ---- library ---------------------------------------------------------------------------------------- */
int b200_abi_version(void);
const char* b200_last_error(void);
/* number of kernels launched by this library in this process (bench.py's gpu_launches evidence). */
long long b200_launch_count(void);

/* ---- sliding-window inference: gather + blend -------------------------------------------------------- */
/* replaces monai/inferers/utils.py:217-224 -- copy n_win windows (win_tab[n_win][4] = {batch, d0, h0, w0},
 * device int32) out of vol[B,C,D,H,W] into out[n_win,C,rd,rh,rw]; dtype conversion allowed.  starts_w_align: a common divisor of
 * every w0 in the table (0 / 1 = unknown): with 16-byte alignment all along W the copy runs on 16-byte vectors. */
int b200_sw_gather(const void* vol, int in_dtype, void* out, int out_dtype, const int32_t* win_tab, int n_win,
                   int C, int D, int H, int W, int rd, int rh, int rw, int starts_w_align, void* stream);

typedef struct b200_blend_desc {
  const void* preds;        /* resident window predictions, windows [win_begin, win_end) */
  int pred_dtype;
  long long pred_stride[5]; /* element strides of preds: window, channel, d, h, w */
  int win_begin, win_end;   /* flat window ids: batch-major, then meshgrid("ij") of the per-axis starts */
  int B, C, D, H, W;        /* blended (padded) volume */
  int rd, rh, rw;           /* roi */
  const int32_t* starts_d; int nd;  /* device: per-axis window starts (dense_patch_slices, data/utils.py:166-206) */
  const int32_t* starts_h; int nh;
  const int32_t* starts_w; int nw;
  const float* gd; const float* gh; const float* gw; /* device: 1-D importance factors (data/utils.py:1122-1127) */
  float clamp_min;          /* max(min(map), 1e-3) (data/utils.py:1132-1133) */
  const float* wmap;        /* optional device dense weight map [rd,rh,rw]; overrides gd/gh/gw when non-null */
  void* out;                /* mode 0/2: [B,C,D,H,W] in out_dtype; mode 1: fp32 accumulators (+=) */
  int out_dtype;
  const float* acc;         /* mode 2: fp32 accumulators */
  int box[4];               /* rows to visit: d in [box0,box1), h in [box2,box3); all-zero = whole volume */
  int starts_w_align;       /* host hint: a common divisor of every starts_w entry (2 -> 2 voxels/thread, 8 -> 8 voxels/thread; 1 or 0 = unknown) */
  int max_cover;            /* host hint: most windows covering one voxel along any single axis (0 = unknown; <= 3 enables the lean kernel) */
  const int32_t* slot_map;  /* mode 1, optional device array [B * n_windows]: flat window id -> slot of its prediction in `preds`
                               (-1 = not resident).  For callers that visit windows in another order than their ids (the buffered
                               mode of monai/inferers/utils.py:182-191, 239-253); win_begin / win_end are then ignored. */
  int n_slots;              /* resident predictions when slot_map is given */
  const double* resample;   /* optional HOST pointer to a 3x4 row-major matrix M: OUTPUT voxel index (d,h,w,1) -> coordinate in the
                               blended volume.  Non-null selects the FUSED blend + affine resample (modes 0 and 2): out is then
                               [B,C,out_D,out_H,out_W] = trilinear / nearest sample of the blended volume, which is never stored
                               (inferers/utils.py:286-298 composed with transforms/spatial/functional.py:68-184, e.g. the inverse of
                               Spacingd applied to the logits).  An identity M gives the bits of the plain blend. */
  int out_D, out_H, out_W;  /* output grid of the fused resample */
  int resample_interp;      /* 0 nearest (round half to even), 1 trilinear */
  int resample_pad;         /* 0 zeros, 1 border */
} b200_blend_desc;

/* replaces monai/inferers/utils.py:264-275, 286-288, 297-298, 351-360.
 * mode 0: all windows resident -> out = sum(w*pred)/sum(w);  mode 1: acc += sum over resident windows;
 * mode 2: out = acc / sum(w) (the count map is evaluated analytically, never stored). */
int b200_sw_blend(const b200_blend_desc* desc, int mode, void* stream);

/* ---- convolution / normalisation / activation (NCDHW, CUDA-core path) --------------------------------- */
typedef struct b200_conv_desc {
  int N, Cin, Cout;
  int Di, Hi, Wi;           /* input spatial */
  int Do, Ho, Wo;           /* output spatial */
  int kd, kh, kw;
  int sd, sh, sw;           /* stride */
  int pd, ph, pw;           /* padding */
  int transposed;           /* 0: Conv3d (weight [Cout,Cin,k]), 1: ConvTranspose3d (weight [Cin,Cout,k]) */
  int in_dtype, out_dtype;  /* weights and bias are always float32 */
  long long in_stride_n;    /* element stride between samples of x (lets x be a slice of a concat buffer) */
  long long out_stride_n;   /* element stride between samples of y */
} b200_conv_desc;

/* replaces nn.Conv3d / nn.ConvTranspose3d as used by monai/networks/blocks/convolutions.py:131-152.
 * fp32 accumulation on CUDA cores; exact-parity path for fp32 models and odd channel counts. */
int b200_conv3d_direct(const b200_conv_desc* desc, const void* x, const float* weight, const float* bias, void* y,
                       void* stream);

/* per-(n,c) sum and sum of squares over S = D*H*W elements of x[N,C,S] -> stats[N*C][2] (float32, overwritten;
 * deterministic: fixed summation order; with few large planes the work is split into chunks whose {sum, sumsq} pairs go through
 * `workspace` (b200_instnorm_stats_workspace_bytes, may be NULL: one block per plane then) and are added in chunk order).
 * x_stride_n = element stride between samples. */
long long b200_instnorm_stats_workspace_bytes(int N, int C, long long S);   /* 0: no scratch needed for this shape */
int b200_instnorm_stats(const void* x, int dtype, int N, int C, long long S, long long x_stride_n, float* stats,
                        void* workspace, void* stream);

/* y = act( (x - mean) * rstd * gamma + beta  [+ res] ) with mean/rstd from stats (biased variance, eps);
 * stats == NULL skips the normalisation.  replaces InstanceNorm3d + PReLU/LeakyReLU (ADN,
 * monai/networks/blocks/acti_norm.py:19-101) and the residual add of UnetResBlock (dynunet_block.py:97-111).
 * res_stats != NULL additionally instance-normalises the residual branch (norm3 of UnetResBlock).
 * act: 0 none, 1 leaky-relu(slope), 2 prelu (slope_ptr[c % n_slope]), 3 relu, 4 gelu(erf). */
int b200_norm_act(const void* x, int dtype, int N, int C, long long S, long long x_stride_n, const float* stats,
                  float eps, const float* gamma, const float* beta, const void* res, long long res_stride_n,
                  const float* res_stats, int act, float slope, const float* slope_ptr, int n_slope, void* y,
                  long long y_stride_n, void* stream);

/* MaxPool3d(kernel=2, stride=2) on [N,C,D,H,W] (basic_unet.py:61-89). */
int b200_maxpool3d_2(const void* x, int dtype, int NC, int D, int H, int W, void* y, void* stream);

/* replicate-pad / copy x[N,C,Di,Hi,Wi] into the channel slice of y (zero-copy concat helper, basic_unet.py:165-172):
 * y[n, c_off + c, d, h, w] = x[n, c, min(d,Di-1), ...]. */
int b200_copy_channels(const void* x, int dtype, int N, int C, int Di, int Hi, int Wi, void* y, int Ctot, int c_off,
                       int Do, int Ho, int Wo, void* stream);

/* ---- spatial transforms ----------------------------------------------------------------------------- */
/* out[c, i,j,k] = sample(src[c], M * (i,j,k,1)) for a 3x4 row-major double matrix M that maps OUTPUT voxel
 * indices to INPUT voxel indices (the composition the reference reaches through AffineTransform /
 * affine_grid + grid_sample: monai/networks/layers/spatial_transforms.py:502-592, spatial/array.py:2015-2117).
 * interp: 0 nearest, 1 trilinear.  pad: 0 zeros, 1 border, 2 reflection (align_corners flag selects the
 * reflection bounds and matches grid_sample's unnormalisation: coordinates are unnormalised by the caller). */
int b200_resample_affine(const void* src, int src_dtype, int C, int Di, int Hi, int Wi, void* dst, int dst_dtype,
                         int Do, int Ho, int Wo, const double* mat3x4, int interp, int pad, int align_corners,
                         void* stream);

/* Dense-grid spline resampling: replaces monai._C.grid_pull (monai/csrc/ext.cpp:66-74, csrc/resample/pushpull.h:58-110,
 * python wrapper monai/networks/layers/spatial_transforms.py:35-132) and the dense-grid form of Resample.__call__
 * (monai/transforms/spatial/array.py:2015-2117).  src [B,C,X,Y,Z] (f16/f32); grid holds three coordinate components per output
 * voxel, addressed as grid[b*stride_b + comp*stride_c + voxel*stride_v] (channel-last [B,Xo,Yo,Zo,3]: stride_c 1, stride_v 3;
 * channel-first [3|4,Xo,Yo,Zo]: stride_c Xo*Yo*Zo, stride_v 1), dtype 0 float32 or 2 float64; the VOXEL coordinate of axis a is
 * scale3[a] * value + shift3[a] (NULL = identity).  bound3 / order3 per axis: bound 0 replicate, 1 dct1, 2 dct2, 3 dst1, 4 dst2,
 * 5 dft, 7 zero (monai/csrc/resample/bounds_common.h); order 0..7 = centred cardinal B-spline weights without prefilter
 * (csrc/resample/interpolation_common.h).  extrapolate = 0 zeroes voxels whose coordinate leaves [-0.05, size-1+0.05).
 * nearest_half_even selects ATen's rounding for order 0 (grid_sample) instead of monai._C's std::round.  out [B,C,Xo,Yo,Zo]. */
int b200_grid_pull(const void* src, int src_dtype, int B, int C, int X, int Y, int Z, const void* grid, int grid_dtype,
                   long long grid_stride_b, long long grid_stride_c, long long grid_stride_v, int Xo, int Yo, int Zo,
                   const double* scale3, const double* shift3, const int* bound3, const int* order3, int extrapolate,
                   int nearest_half_even, void* out, int out_dtype, void* stream);

/* monai._C.grid_push / grid_count (monai/csrc/ext.cpp:66-74 -> csrc/resample/pushpull.h:112-216; python wrappers
 * monai/networks/layers/spatial_transforms.py:135-311): the adjoint of b200_grid_pull.  Every voxel of input [B,C,Xi,Yi,Zi] is
 * splatted with the same weights / bounds at the voxel coordinate grid[b, :, voxel] into out [B,C,X,Y,Z] (float32, zeroed by the
 * call).  input == NULL computes grid_count (C must be 1): the splat of ones.  Float atomics: equal to the reference to rounding. */
int b200_grid_push(const void* input, int in_dtype, int B, int C, int Xi, int Yi, int Zi, const void* grid, int grid_dtype,
                   long long grid_stride_b, long long grid_stride_c, long long grid_stride_v, int X, int Y, int Z,
                   const double* scale3, const double* shift3, const int* bound3, const int* order3, int extrapolate,
                   void* out, void* stream);

/* monai._C.grid_grad (csrc/resample/pushpull.h:218-270; python wrapper monai/networks/layers/spatial_transforms.py:314-408): spatial
 * gradients of the interpolated volume at the grid's coordinates, out [B,C,Xo,Yo,Zo,3] (last axis: d/dx0, d/dx1, d/dx2 in voxels).
 * Arguments as b200_grid_pull. */
int b200_grid_grad(const void* src, int src_dtype, int B, int C, int X, int Y, int Z, const void* grid, int grid_dtype,
                   long long grid_stride_b, long long grid_stride_c, long long grid_stride_v, int Xo, int Yo, int Zo,
                   const double* scale3, const double* shift3, const int* bound3, const int* order3, int extrapolate,
                   void* out, int out_dtype, void* stream);

/* zero-padded separable 3-D filter (GaussianFilter, monai/networks/layers/simplelayers.py:170-249, 542-595):
 * taps_* are float32 device arrays of odd length n_*; src/dst [C,D,H,W]; tmp is a float32 scratch buffer of
 * 2*C*D*H*W elements (the two intermediate passes stay fp32). */
int b200_separable_filter3d(const void* src, int dtype, int C, int D, int H, int W, const float* taps_d, int n_d,
                            const float* taps_h, int n_h, const float* taps_w, int n_w, float* tmp, void* dst,
                            void* stream);

/* ---- tensor-core path (wgmma / TMA), channel-blocked fp16 activations -------------------------- */
/* Activation layout "NC8": [N][C/8][D][H][W][8] float16 (C % 8 == 0).  */

/* NCDHW (f16/f32) <-> NC8 (f16) repack; c_off/Ctot address a channel slice of a concat buffer. */
int b200_pack_nc8(const void* x, int dtype, int N, int C, long long S, void* y, int Ctot, int c_off, void* stream);
int b200_unpack_nc8(const void* x, int Ctot, int c_off, int N, int C, long long S, void* y, int dtype, void* stream);

/* bytes needed for the packed weight image of b200_conv3x3x3_tc (depends on Cin, Cout only). */
long long b200_conv3x3x3_tc_weight_bytes(int Cin, int Cout);
/* pack Conv3d weight [Cout,Cin,3,3,3] float32 (device) into the wgmma B-operand image (device, fp16). */
int b200_conv3x3x3_tc_pack_weight(const float* w, int Cin, int Cout, void* packed, void* stream);

typedef struct b200_conv_tc_desc {
  int N, Cin, Cout, D, H, W;
  int in_ctot, in_coff;     /* x is channels [in_coff, in_coff+Cin) of an NC8 buffer with in_ctot channels */
  int out_ctot, out_coff;   /* y likewise */
  /* Fused InstanceNorm + activation of the INPUT (round 2; all zero = off): x is the raw output of the previous
   * convolution and in_stats its per-(n, channel of the slice) {sum, sumsq} (float32 device, [N][Cin][2], as written by the
   * `stats` output of these entry points).  The kernel feeds act((x - mean) * rstd) to the tensor core -- exactly the fp16
   * values b200_norm_act_nc8 would have stored (dynunet_block.py:97-103: conv1 -> norm1 -> lrelu -> conv2). */
  const float* in_stats;
  float in_eps;
  int in_act;               /* 0 none, 1 leaky-relu (in_slope), 3 relu */
  float in_slope;
  /* Folded 1x1x1 residual convolution (round 2; res_w == NULL = off; exclusive with in_stats; Cout <= 128): UnetResBlock.conv3
   * (dynunet_block.py:75-87, 104-108) reads the same input as conv1, so res_y = conv1x1x1(x, W3) is produced by the same launch
   * (one extra MMA per output plane and K slice on the centre view of the staged halo tile).  res_w = b200_gemm_tc_pack_weight image
   * of W3 [Cout, Cin]; res_y = NC8 destination (channel slice res_coff of res_ctot); res_stats (optional) = its {sum, sumsq}
   * per (n, cout), deterministic; the workspace of b200_conv3x3x3_tc_workspace_bytes(desc) covers both outputs. */
  const void* res_w;
  void* res_y;
  int res_ctot, res_coff;
  float* res_stats;
} b200_conv_tc_desc;

/* 3x3x3, stride 1, zero padding 1 implicit-GEMM convolution on wgmma tensor cores: halo tile staged once
 * into shared memory by TMA, 27 taps issued as shifted wgmma shared-memory descriptors, fp32 accumulators in
 * registers.  stats (optional, overwritten) receives per-(n,cout) {sum, sumsq} of the fp32 results so InstanceNorm needs no
 * extra pass.  The sums are DETERMINISTIC (bit-identical run to run): the epilogue warps write partial rows into
 * `workspace` (device scratch of b200_conv3x3x3_tc_workspace_bytes(desc) bytes, required when stats != NULL; no
 * initialisation needed) and a finishing pass adds them in a fixed order -- no floating-point atomics anywhere.
 * replaces the Conv3d inside UnetResBlock (monai/networks/blocks/dynunet_block.py:25-111) for SwinUNETR / DynUNet blocks. */
long long b200_conv3x3x3_tc_workspace_bytes(const b200_conv_tc_desc* desc);
int b200_conv3x3x3_tc(const b200_conv_tc_desc* desc, const void* x, const void* packed_w, const float* bias,
                      void* y, float* stats, void* workspace, void* stream);
/* The same with an AFFINE operand normalisation (InstanceNorm3d(affine=True), dynunet_block.py:114-177): desc->in_stats is
 * required and the kernel feeds act((x - mean) * rstd * in_gamma + in_beta), the fp16 values b200_norm_act_affine_nc8 would
 * have stored.  in_gamma / in_beta: float32 device [Cin] (either may be NULL: 1 / 0).  Workspace as for b200_conv3x3x3_tc. */
int b200_conv3x3x3_tc_affine(const b200_conv_tc_desc* desc, const float* in_gamma, const float* in_beta, const void* x,
                             const void* packed_w, const float* bias, void* y, float* stats, void* workspace, void* stream);

typedef struct b200_conv_gather_desc {
  int N, Cin, Cout;         /* Cin % 16 == 0; Cout arbitrary for NCDHW output, % 8 == 0 for NC8 output */
  int Di, Hi, Wi, Do, Ho, Wo;
  int k, stride, pad;       /* cubic kernel k <= 3, stride 1 or 2, zero padding */
  int transposed;           /* 0: Conv3d weight [Cout,Cin,k,k,k]; 1: ConvTranspose3d weight [Cin,Cout,k,k,k] */
  int in_ctot, in_coff;     /* x = channels [in_coff, in_coff+Cin) of an NC8 buffer */
  int out_ctot, out_coff;   /* NC8 destination slice (out_layout 0) */
  int out_layout;           /* 0: NC8 fp16; 1: NCDHW (out_dtype) with exactly Cout channels */
  int out_dtype;
} b200_conv_gather_desc;

/* General Conv3d / ConvTranspose3d (k <= 3, stride <= 2) as an implicit GEMM on wgmma with a cp.async im2col
 * producer -- the stride-2 and transposed 3x3x3 layers of UNet (monai/networks/nets/unet.py:150-182).  Weights are
 * packed per (N tile, parity class, live tap, 16-channel slice); stats as in b200_conv3x3x3_tc. */
long long b200_conv_gather_tc_weight_bytes(const b200_conv_gather_desc* desc);
int b200_conv_gather_tc_pack_weight(const b200_conv_gather_desc* desc, const float* w, void* packed, void* stream);
long long b200_conv_gather_tc_workspace_bytes(const b200_conv_gather_desc* desc);   /* statistics scratch, as for b200_conv3x3x3_tc */
int b200_conv_gather_tc(const b200_conv_gather_desc* desc, const void* x, const void* packed_w, const float* bias, void* y,
                        float* stats, void* workspace, void* stream);

/* Thin head: ConvTranspose3d(k3, s2, p1, output_padding 1) from NC8 features to <= 4 NCDHW logit channels
 * (top layer of UNet, monai/networks/nets/unet.py); weight float32 [Cin][Cout][3][3][3]. */
int b200_convt3s2_head_nc8(const void* x, int N, int Cin, int Di, int Hi, int Wi, int in_ctot, int in_coff,
                           const float* weight, const float* bias, int Cout, void* y, int out_dtype, void* stream);

typedef struct b200_gemm_tc_desc {
  int Nb;                   /* batch items (each with its own S rows) */
  int S;                    /* GEMM rows per batch item (tokens / voxels of x) */
  int K, N;                 /* reduction size (input channels) and GEMM columns */
  int in_ctot, in_coff;     /* x = channels [in_coff, in_coff+K) of an NC8 buffer with in_ctot channels */
  int out_ctot, out_coff;   /* destination channel slice */
  int res_ctot, res_coff;   /* residual (added before the store), indexed like the destination */
  long long S_out;          /* rows per batch item of the destination (== S unless mode 1/2) */
  int mode;                 /* 0: row r -> r; 1: row r -> row_map[r] (-1 = drop; shared by batch items); 2: ConvTranspose k2 s2 scatter */
  int act;                  /* 0 none, 4 GELU(erf) */
  int D, H, W;              /* mode 2: source grid (S == D*H*W); destination grid is (2D,2H,2W) */
} b200_gemm_tc_desc;

long long b200_gemm_tc_weight_bytes(int N, int K);
/* pack W[n,k] = w[n*stride_n + k*stride_k] (float32 device) into the wgmma B-operand image (fp16 device). */
int b200_gemm_tc_pack_weight(const float* w, int N, int K, long long stride_n, long long stride_k, void* packed,
                             void* stream);
/* y = [res +] act(x * W^T + bias) on wgmma: nn.Linear (swin_unetr.py:509-532, blocks/mlp.py:75-80, PatchMerging
 * 749-773), 1x1x1 Conv3d (dynunet_block.py:75-87) and ConvTranspose3d k2 s2 (unetr_block.py:56-64, mode 2 with
 * GEMM columns ordered [tap = kd*4+kh*2+kw][cout]).  stats (optional, overwritten) receives per-(batch, column)
 * {sum, sumsq} of the stored values for InstanceNorm, deterministically, through `workspace`
 * (b200_gemm_tc_workspace_bytes(desc) bytes; see b200_conv3x3x3_tc). */
long long b200_gemm_tc_workspace_bytes(const b200_gemm_tc_desc* desc);
int b200_gemm_tc(const b200_gemm_tc_desc* desc, const void* x, const void* packed_w, const float* bias, const void* res,
                 const int32_t* row_map, void* y, float* stats, void* workspace, void* stream);

/* Fused transformer MLP of a Swin block, one launch (swin_unetr.py:675-698: x + mlp(norm2(x)); blocks/mlp.py:75-80):
 *   y = x + W2 * gelu(W1 * LayerNorm(x) + b1) + b2,   x, y NC8 fp16 [Nb][C/8][S][8] (y may not alias x).
 * packed_w1 / packed_w2 are b200_gemm_tc_pack_weight() images of linear1.weight [hidden, C] and linear2.weight [C, hidden].
 * The hidden activations stay in shared memory.  Implemented for C = 48, hidden = 192 (anything else: B200_ERR_INVALID_ARGUMENT,
 * callers use layernorm_nc8 + two gemm_tc). */
int b200_mlp_fused_tc(const void* x, int x_ctot, int Nb, int S, int C, int hidden, const void* packed_w1, const float* b1,
                      const void* packed_w2, const float* b2, const float* gamma, const float* beta, float eps, void* y,
                      int y_ctot, void* stream);

/* Channels-first transformer pieces of the ViT encoder (UNETR; generic fp32-faithful forms, tokens [N, C, S]):
 * LayerNorm over the channel axis of every token (nn.LayerNorm(C): transformerblock.py:94-99, vit.py:128), gamma / beta may be NULL. */
int b200_layernorm_cf(const void* x, int dtype, int N, int C, long long S, const float* gamma, const float* beta, float eps,
                      void* y, void* stream);
/* Non-overlapping patches as channels: x [N, C, D, H, W] -> y [N, C*pd*ph*pw, (D/pd)*(H/ph)*(W/pw)] (channel = (c, a, b, e) row-major,
 * token = patch grid row-major), so that the patch projection of PatchEmbeddingBlock (patchembedding.py:104-108) is a Linear. */
int b200_patchify(const void* x, int dtype, int N, int C, int D, int H, int W, int pd, int ph, int pw, void* y, void* stream);
/* Multi-head self-attention softmax(q k^T * scale [+ bias] [+ mask]) v on channels-first tokens.
 * win == 0: global attention (SABlock.forward, selfattention.py:170-217).  win > 0: the token axis holds S / win windows of `win` tokens
 * and a query attends to its own window (WindowAttention.forward, swin_unetr.py:509-532); bias (optional) = float32 device
 * [heads][win][win] relative-position bias; region (optional) = int32 device [S / win][win] labels of compute_mask (swin_unetr.py:
 * 779-816): pairs with different labels get -100.
 * qkv [N, 3*heads*dim_head, S]: channels ordered (q|k|v, head, dim) as produced by the combined projection; out [N, heads*dim_head, S]
 * with channels (head, dim).  dim_head in {8, 16, 24, 32, 48, 64}. */
int b200_mhsa_cf(const void* qkv, int dtype, int N, int heads, int dim_head, long long S, float scale, int win, const float* bias,
                 const int32_t* region, void* out, void* stream);
/* y[n, c, r] = src[r] >= 0 ? x[n, c, src[r]] : 0 on channels-first tokens: window partition / reverse with cyclic shift and zero
 * padding through an index table (swin_unetr.py:596-648). */
int b200_gather_cf(const void* x, int dtype, int N, int C, long long S_in, const int32_t* src, long long S_out, void* y, void* stream);

/* LayerNorm over channels of NC8 tokens with an optional row gather (window partition + cyclic shift + zero pad of
 * swin_unetr.py:596-625): y[n, :, r] = LN(x[n, :, src[r]]) (src[r] < 0 -> zeros; src == NULL -> identity).
 * gamma/beta NULL = no affine (SwinTransformer.proj_out, swin_unetr.py:1040-1053).  src is shared by all batch items. */
int b200_layernorm_nc8(const void* x, int N, int C, long long S_in, const int32_t* src, long long S_out,
                       const float* gamma, const float* beta, float eps, void* y, void* stream);

/* PatchMerging gather + LayerNorm (swin_unetr.py:749-773): x NC8 [N][C/8][D][H][W][8] -> y NC8 [N][8C/8][D/2*H/2*W/2][8],
 * channel blocks in the reference order x0..x7 = (0,0,0),(1,0,0),(0,1,0),(0,0,1),(1,1,0),(1,0,1),(0,1,1),(1,1,1)
 * (v2 = 0) or itertools.product order (v2 = 1); odd sizes are zero padded. */
int b200_patch_merge_ln_nc8(const void* x, int N, int C, int D, int H, int W, const float* gamma, const float* beta,
                            float eps, int v2, void* y, void* stream);

/* Windowed multi-head self-attention (WindowAttention.forward, swin_unetr.py:509-532) on NC8 tokens in window order:
 * qkv NC8 [N][3C/8][nW*n][8] (channels = [q | k | v], head h = channels [16h, 16h+16) of each third; head_dim 16),
 * table float32 [(2ws0-1)(2ws1-1)(2ws2-1)][heads] = relative_position_bias_table of the MODULE window (ws0,ws1,ws2)
 * (tokens keep base-window coordinates when the window is clamped, as relative_position_index[:n,:n] does),
 * region int32 [nW][n] or NULL (shift mask: -100 where regions differ, swin_unetr.py:779-816),
 * out NC8 [N][C/8][nW*n][8]. */
int b200_window_attention_nc8(const void* qkv, int N, int C, int heads, int nW, int n, float scale, const float* table,
                              int ws0, int ws1, int ws2, const int32_t* region, void* out, void* stream);

/* The same attention on wgmma tensor cores (n <= 352 tokens per window, head_dim 16): S = q k^T is accumulated by wgmma
 * onto the relative-position bias + shift mask (pre-packed in the accumulator's register order, resident in shared
 * memory), online softmax in registers, P V runs on wgmma with the probabilities as register operands and V read in place
 * (MN-major operand).  The packed bias is opaque to callers: size it with b200_window_attention_tc_bias_bytes.
 * Differences to b200_window_attention_nc8:
 *   - q must be PRE-SCALED by scale * log2(e) (fold it into the q rows of the qkv projection): scores are in log2 units;
 *   - the bias table and the shift mask are pre-packed per (mask type, head, 192-row tile) with
 *     b200_window_attention_tc_pack_bias: region_types int32 [ntypes][n] holds ONE representative row of `region` per
 *     distinct mask pattern (NULL with ntypes = 1: no mask); ntypes <= 8;
 *   - sched int32 device array: count[8] (windows of each type), start[8] (offset of the type's window list),
 *     win[nW] (window ids grouped by type). */
long long b200_window_attention_tc_bias_bytes(int heads, int n, int ntypes);
int b200_window_attention_tc_pack_bias(const float* table, int heads, int n, int ws0, int ws1, int ws2,
                                       const int32_t* region_types, int ntypes, void* packed, void* stream);
int b200_window_attention_tc(const void* qkv, int N, int C, int heads, int nW, int n, const void* packed_bias,
                             const int32_t* sched, int ntypes, void* out, void* stream);

/* Global multi-head self-attention of the ViT encoder (SABlock.forward, selfattention.py:170-217; no bias, no mask) on
 * wgmma tensor cores, head_dim 64, any S >= 1:
 *   qkv NC8 fp16 [N][3C/8][S][8], channel = (which * heads + h) * 64 + d  (which = q | k | v),
 *   out NC8 fp16 [N][C/8][S][8],  channel = h * 64 + d.
 * q must be PRE-SCALED by dim_head^-0.5 * log2(e) (fold it into the q rows of the qkv projection): the softmax runs in
 * log2 units.  Deterministic.  C != 64 * heads: B200_ERR_UNSUPPORTED. */
int b200_mhsa_tc(const void* qkv, int N, int C, int heads, long long S, void* out, void* stream);

/* Convolution with ONE input channel straight from an NCDHW volume to NC8 (patch embedding k2 s2, the 3x3x3 stem of
 * UnetrBasicBlock and its 1x1x1 residual conv): weight float32 [Cout][1][k][k][k]; stats optional {sum,sumsq}. */
long long b200_conv_cin1_nc8_workspace_bytes(int N, int D, int H, int W, int Cout, int k, int stride, int pad);
int b200_conv_cin1_nc8(const void* x, int dtype, int N, int D, int H, int W, const float* weight, const float* bias,
                       int Cout, int k, int stride, int pad, void* y, int out_ctot, int out_coff, float* stats,
                       void* workspace, void* stream);

/* The same on wgmma tensor cores for (k, stride, pad) = (3, 1, 1) and (2, 2, 0), Cout in {16, 32, 48, 64, 96, 128}: an
 * implicit GEMM with K = taps padded to 32 / 16 whose im2col operand is built in shared memory from a staged halo patch
 * of the raw volume; bound by the fp16 store of its output instead of by CUDA-core FMAs.  Same arguments. */
long long b200_conv_cin1_tc_workspace_bytes(int N, int D, int H, int W, int Cout, int k, int stride, int pad);
int b200_conv_cin1_tc(const void* x, int dtype, int N, int D, int H, int W, const float* weight, const float* bias,
                      int Cout, int k, int stride, int pad, void* y, int out_ctot, int out_coff, float* stats,
                      void* workspace, void* stream);

/* Channel-wise post-processing of channel-first logits x[C][S] (the transforms that follow the inferer in a segmentation bundle):
 * op 0 softmax over C, 1 sigmoid  (Activations, monai/transforms/post/array.py:63-128);
 * op 2 argmax over C -> y[1][S] (index as float) or, with onehot > 0, y[onehot][S]; op 3 `x >= param`; op 4 round-half-even;
 * op 5 one-hot of a single-channel index map -> y[onehot][S]  (AsDiscrete, post/array.py:131-251).  dtypes: 0 f32, 1 f16. */
int b200_channel_post(const void* x, int in_dtype, int C, long long S, int op, float param, int onehot, void* y, int out_dtype,
                      void* stream);

/* AvgMerger of PatchInferer (monai/inferers/merger.py:103-205).  accumulate: values[NC][md][mh][mw] (fp32) += patch[NC][pd][ph][pw]
 * at spatial location (ld, lh, lw) and counts += 1 there (counts: uint8 (count_bytes 1) or int32 (4)); finalize: values /= counts. */
int b200_patch_accumulate(const void* patch, int dtype, long long NC, int pd, int ph, int pw, float* values, void* counts, int count_bytes,
                          int md, int mh, int mw, int ld, int lh, int lw, void* stream);
int b200_patch_finalize(float* values, const void* counts, int count_bytes, long long total, void* stream);

/* dst[i] += src[i], float32 (16-byte aligned): folds the partial numerators a peer rank sends into the local accumulators of the
 * depth-sharded sliding-window job (no reference counterpart: the reference does not shard a volume over GPUs). */
int b200_add_f32(float* dst, const float* src, long long n, void* stream);

/* 1x1x1 output head (UnetOutBlock, dynunet_block.py:247-267): NC8 fp16 [N][C/8][S][8] -> NCDHW [N][Cout][S]. */
int b200_head_conv_nc8(const void* x, int N, int C, long long S, const float* weight, const float* bias, int Cout,
                       void* y, int out_dtype, void* stream);

/* Output head fused with the tail of the last residual block: y = W * lrelu(instnorm(x) + instnorm?(res)) + b
 * (UnetResBlock.forward norm2 + residual + lrelu, dynunet_block.py:97-111, then UnetOutBlock :247-267).  x is a whole NC8
 * tensor of C channels with its (sum, sum of squares) statistics [N*C*2]; res is a channel slice of an NC8 buffer, normalised
 * with res_stats when given (the block's conv3 branch) or added as is. */
int b200_head_conv_norm_nc8(const void* x, int N, int C, long long S, const float* stats, float eps, const void* res,
                            int res_ctot, int res_coff, const float* res_stats, float slope, const float* weight,
                            const float* bias, int Cout, void* y, int out_dtype, void* stream);
/* The same with an affine InstanceNorm of x (DynUNet's last up block, dynunet_block.py:165-177): gamma / beta float32 device [C]
 * (either may be NULL: 1 / 0). */
int b200_head_conv_norm_affine_nc8(const void* x, int N, int C, long long S, const float* stats, float eps, const void* res,
                                   int res_ctot, int res_coff, const float* res_stats, float slope, const float* weight,
                                   const float* bias, int Cout, void* y, int out_dtype, const float* gamma, const float* beta,
                                   void* stream);

/* NC8 variant of b200_norm_act: y = act(instnorm(x) [+ instnorm?(res)]); act: 0 none, 1 leaky-relu(slope), 3 relu.
 * x / res / y are channel slices [coff, coff+C) of NC8 buffers with ctot channels. */
int b200_norm_act_nc8(const void* x, int x_ctot, int x_coff, int N, int C, long long S, const float* stats, float eps,
                      const void* res, int res_ctot, int res_coff, const float* res_stats, int act, float slope,
                      void* y, int y_ctot, int y_coff, void* stream);
/* The same with affine InstanceNorms: y = act(instnorm(x) * gamma + beta [+ instnorm(res) * res_gamma + res_beta]) (UnetResBlock
 * norm2 and norm3 with affine=True, dynunet_block.py:97-111).  Each parameter is float32 device [C] or NULL (1 / 0); gamma / beta
 * need stats, res_gamma / res_beta need res_stats.  With all four NULL the output is bit-identical to b200_norm_act_nc8. */
int b200_norm_act_affine_nc8(const void* x, int x_ctot, int x_coff, int N, int C, long long S, const float* stats, float eps,
                             const void* res, int res_ctot, int res_coff, const float* res_stats, int act, float slope,
                             void* y, int y_ctot, int y_coff, const float* gamma, const float* beta, const float* res_gamma,
                             const float* res_beta, void* stream);

/* Same, for a residual block whose input has ONE channel (SwinUNETR encoder1): the residual branch
 * instnorm(conv1x1x1(u)) of UnetResBlock (dynunet_block.py:75-111) is evaluated analytically from the statistics of the
 * raw input u [N][S] (fp16): conv3 gives w_c * u, so its instance norm is (w_c u - w_c mu) / sqrt(w_c^2 sigma^2 + eps).
 * raw_stats = {sum, sum of squares} of u per batch item [N*2]; raw_weight = the C conv3 weights (the conv has no bias).
 * The 1x1x1 convolution and its output tensor are never materialised. */
int b200_norm_act_cin1res_nc8(const void* x, int x_ctot, int x_coff, int N, int C, long long S, const float* stats, float eps,
                              const void* raw, const float* raw_stats, const float* raw_weight, int act, float slope, void* y,
                              int y_ctot, int y_coff, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MONAI_B200_H_ */
