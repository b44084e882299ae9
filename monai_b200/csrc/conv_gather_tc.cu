// General 3-D convolution / transposed convolution (kernel <= 3, stride <= 2, per axis) as an implicit GEMM on Hopper wgmma
// tensor cores with a software im2col producer (SURVEY.md §8 row a8: the stride-2 Conv3d and ConvTranspose3d(k3, s2) layers
// of UNet, monai/networks/nets/unet.py:150-182 via monai/networks/blocks/convolutions.py:131-152; the anisotropic strided and
// transposed convolutions of DynUNet).
//
// GEMM view: rows = 128 output voxels of ONE parity class (forward conv: a single class; transposed conv with
// stride (sd, sh, sw): sd*sh*sw classes, so that every row of a tile uses the same set of live taps -- no work is spent on taps that
// cannot reach an output voxel), columns = NT output channels, K = (live taps) x Cin walked in units of 16 channels.
// Producer warps (128 threads, one GEMM row each) gather the 16-channel vectors of the tap's input voxel with
// cp.async (16-byte pieces of the NC8 layout, zero-filled outside the volume = zero padding) straight into the wgmma
// K-major / no-swizzle core-matrix image; a proxy fence + mbarrier hands each stage to the two consumer warpgroups
// (rows 0-63 / 64-127 of the tile, accumulators in registers).  Weights are pre-packed per (N tile, class, tap,
// 16-channel slice) and arrive by bulk copies.  The kernel is persistent; the consumers' epilogue adds bias, reduces
// InstanceNorm partial sums and stores either NC8 fp16 (optionally into a channel slice of a concat buffer) or NCDHW (the Cout = 2 segmentation head).
#include "common.cuh"
#include "tc90.cuh"
#include "stats.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

constexpr int kCgStages = 4;
constexpr int kCgUnits = 4;                       // K16 units per pipeline stage
constexpr int kCgAStage = kCgUnits * 2 * 2048;    // 16 KB

struct CgTap { unsigned char id; signed char dz, dy, dx; };

struct CgParams {
  b200_conv_gather_desc d;
  const __half* x; const __half* w; const float* bias; void* y;
  StatsPartials sp;           // deterministic InstanceNorm partial sums (stats.cuh)
  int NT, cout_pad;
  int ncls, mul[3];           // classes; input coordinate = coarse * mul + tap offset (d, h, w)
  int Dc, Hc, Wc;             // coarse extent of one class
  int cls_ntaps[8], cls_unit_off[8];
  CgTap taps[8][27];
  int units_total;            // sum over classes of ntaps * Cin/16
};

// enumerate the live taps of every parity class (shared by the pack kernel and the conv kernel)
static void cg_build_taps(const b200_conv_gather_desc& d, CgParams& p) {
  const int* k = d.k; const int* s = d.stride; const int* pad = d.pad;
  p.ncls = d.transposed ? s[0] * s[1] * s[2] : 1;
  for (int a = 0; a < 3; ++a) p.mul[a] = d.transposed ? 1 : s[a];
  auto md = [](int v, int m) { return ((v % m) + m) % m; };
  auto fdiv = [md](int v, int m) { return (v - md(v, m)) / m; };
  int off = 0;
  for (int c = 0; c < p.ncls; ++c) {
    const int px = c % s[2], py = (c / s[2]) % s[1], pz = c / (s[2] * s[1]);
    int nt = 0;
    for (int kz = 0; kz < k[0]; ++kz)
      for (int ky = 0; ky < k[1]; ++ky)
        for (int kx = 0; kx < k[2]; ++kx) {
          CgTap t;
          t.id = (unsigned char)((kz * k[1] + ky) * k[2] + kx);
          if (d.transposed) {
            const int tz = pz + pad[0] - kz, ty = py + pad[1] - ky, tx = px + pad[2] - kx;
            if (md(tz, s[0]) || md(ty, s[1]) || md(tx, s[2])) continue;
            t.dz = (signed char)fdiv(tz, s[0]); t.dy = (signed char)fdiv(ty, s[1]); t.dx = (signed char)fdiv(tx, s[2]);
          } else {
            t.dz = (signed char)(kz - pad[0]); t.dy = (signed char)(ky - pad[1]); t.dx = (signed char)(kx - pad[2]);
          }
          p.taps[c][nt++] = t;
        }
    p.cls_ntaps[c] = nt;
    p.cls_unit_off[c] = off;
    off += nt * (d.Cin / 16);
  }
  p.units_total = off;
}

// packed layout: [nt][unit][khalf][NT/8][8][8], unit = cls_unit_off[cls] + tap_index_in_class * (Cin/16) + kc
__global__ void cg_pack_weight_kernel(const float* __restrict__ w, __half* __restrict__ out, CgParams p) {
  const b200_conv_gather_desc& d = p.d;
  const int NT = p.NT, kcs = d.Cin / 16, ktaps = d.k[0] * d.k[1] * d.k[2];
  const long long total = (long long)(p.cout_pad / NT) * p.units_total * NT * 16;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int kk = (int)(r % 8); r /= 8;
    const int row = (int)(r % 8); r /= 8;
    const int g = (int)(r % (NT / 8)); r /= (NT / 8);
    const int khalf = (int)(r % 2); r /= 2;
    const int unit = (int)(r % p.units_total); r /= p.units_total;
    const int nt = (int)r;
    int cls = 0;
    while (cls + 1 < p.ncls && unit >= p.cls_unit_off[cls + 1]) ++cls;
    const int u = unit - p.cls_unit_off[cls];
    const int ti = u / kcs, kc = u % kcs;
    const int tap = p.taps[cls][ti].id;
    const int cout = nt * NT + g * 8 + row, cin = kc * 16 + khalf * 8 + kk;
    float v = 0.f;
    if (cout < d.Cout)
      v = d.transposed ? w[((long long)cin * d.Cout + cout) * ktaps + tap] : w[((long long)cout * d.Cin + cin) * ktaps + tap];
    out[i] = __float2half_rn(v);
  }
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

template <int NT>
__global__ void __launch_bounds__(384, 1) conv_gather_tc_kernel(CgParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = tc::align_smem128(smem_raw);   // keeps the shared address space (LDS/STS, not generic LD/ST)
  constexpr int b_stage = kCgUnits * NT * 32;
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kCgStages * kCgAStage;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + kCgStages * b_stage);
  uint64_t* full = bars;                         // producers (128) + weight copy (1 + tx)
  uint64_t* empty = bars + kCgStages;            // one arrival per consumer warpgroup
  float* s_stats = reinterpret_cast<float*>(bars + 16);   // [4][2*NT]
  float* s_stage = s_stats + 4 * 2 * NT;                  // [2 warpgroups][2][kStageFloats]

  const b200_conv_gather_desc& d = p.d;
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int kcs = d.Cin / 16;
  const int n_tiles = p.cout_pad / NT;
  const long long coarse = (long long)p.Dc * p.Hc * p.Wc;
  const int row_tiles = (int)((coarse + 127) / 128);
  const long long total_tiles = (long long)d.N * p.ncls * row_tiles * n_tiles;
  const long long Si = (long long)d.Di * d.Hi * d.Wi, So = (long long)d.Do * d.Ho * d.Wo;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kCgStages; ++i) { tc::mbar_init(&full[i], 129); tc::mbar_init(&empty[i], 2); }
    tc::fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 4 * 2 * NT; i += blockDim.x) s_stats[i] = 0.f;
  __syncthreads();

  if (warp < 4) {
    // ===================== im2col producers: thread r gathers GEMM row r =====================
    const int r = threadIdx.x;
    int s = 0; uint32_t ph = 0;
    // up to kCgInflight cp.async groups (= stages) stay in flight per thread; a stage is handed to the MMA warp only
    // after its group completed (wait_group) and a proxy fence made the generic-proxy writes visible to wgmma
    constexpr int kCgInflight = 3;
    int pend_first = 0, pend_n = 0;   // pending stages are pend_first, pend_first+1, ... (mod kCgStages)
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      // tile order: row tile fastest, then parity class, then N tile, then batch item (consecutive tiles share their
      // weights; the tiles of one (batch item, N tile) group are contiguous for the deterministic statistics)
      const int rt = (int)(tile % row_tiles);
      long long t2 = tile / row_tiles;
      const int cls = (int)(t2 % p.ncls); t2 /= p.ncls;
      const int nt = (int)(t2 % n_tiles);
      const int n = (int)(t2 / n_tiles);
      const long long cv = (long long)rt * 128 + r;
      const bool row_ok = cv < coarse;
      const int cx = row_ok ? (int)(cv % p.Wc) : 0, cy = row_ok ? (int)((cv / p.Wc) % p.Hc) : 0, cz = row_ok ? (int)(cv / ((long long)p.Wc * p.Hc)) : 0;
      const int bz = cz * p.mul[0], by = cy * p.mul[1], bx = cx * p.mul[2];
      const int units = p.cls_ntaps[cls] * kcs;
      const __half* xn = p.x + ((long long)n * (d.in_ctot / 8) + d.in_coff / 8) * Si * 8;
      const __half* wbase = p.w + ((long long)nt * p.units_total + p.cls_unit_off[cls]) * (NT * 16);
      for (int u0 = 0; u0 < units; u0 += kCgUnits) {
        const int nu = min(kCgUnits, units - u0);
        tc::mbar_wait(&empty[s], ph ^ 1);
        const uint32_t a_dst = tc::smem_u32(smem_a + s * kCgAStage) + r * 16;
        for (int q = 0; q < nu; ++q) {
          const int u = u0 + q, ti = u / kcs, kc = u % kcs;
          const CgTap tp = p.taps[cls][ti];
          const int iz = bz + tp.dz, iy = by + tp.dy, ix = bx + tp.dx;
          const bool ok = row_ok && iz >= 0 && iz < d.Di && iy >= 0 && iy < d.Hi && ix >= 0 && ix < d.Wi;
          const __half* src = ok ? xn + ((long long)(kc * 2) * Si + ((long long)iz * d.Hi + iy) * d.Wi + ix) * 8 : p.x;
          cp_async16(a_dst + (q * 2) * 2048, src, ok ? 16 : 0);
          cp_async16(a_dst + (q * 2 + 1) * 2048, ok ? src + Si * 8 : p.x, ok ? 16 : 0);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        if (r == 0) {
          tc::mbar_arrive_expect_tx(&full[s], nu * NT * 32);
          tc::bulk_load(smem_b + s * b_stage, wbase + (long long)u0 * (NT * 16), nu * NT * 32, &full[s]);
        }
        if (pend_n == 0) pend_first = s;
        ++pend_n;
        if (pend_n == kCgInflight) {
          asm volatile("cp.async.wait_group 2;" ::: "memory");   // kCgInflight - 1 newest groups may still be pending
          tc::fence_proxy_async();
          tc::mbar_arrive(&full[pend_first]);
          pend_first = (pend_first + 1) % kCgStages;
          --pend_n;
        }
        if (++s == kCgStages) { s = 0; ph ^= 1; }
      }
    }
    if (pend_n > 0) {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      tc::fence_proxy_async();
      for (; pend_n > 0; --pend_n) { tc::mbar_arrive(&full[pend_first]); pend_first = (pend_first + 1) % kCgStages; }
    }
  } else {
    // ===================== consumers: warpgroup g runs rows 64 g .. 64 g + 63 (wgmma, then the epilogue) =====================
    const int g = (warp >> 2) - 1, wid = warp & 3;
    const int q = 2 * g + (wid & 1), half = wid >> 1;
    float* ws = s_stats + q * (2 * NT);
    float* stage = s_stage + g * 2 * tc::kStageFloats;
    long long group = -1;
    int s = 0; uint32_t ph = 0;
    int sl = 0;
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      if (p.sp.buf) {
        const long long gg = tile / ((long long)p.ncls * row_tiles);
        if (gg != group) {
          if (group >= 0) {
            tc::wg_bar(8 + g);
            if (half == 0) stats_flush(p.sp, ws, 2 * NT, group, q, lane, 0, NT);
          }
          group = gg;
        }
      }
      // tile order: row tile fastest, then parity class, then N tile, then batch item (consecutive tiles share their
      // weights; the tiles of one (batch item, N tile) group are contiguous for the deterministic statistics)
      const int rt = (int)(tile % row_tiles);
      long long t2 = tile / row_tiles;
      const int cls = (int)(t2 % p.ncls); t2 /= p.ncls;
      const int nt = (int)(t2 % n_tiles);
      const int n = (int)(t2 / n_tiles);
      const int units = p.cls_ntaps[cls] * kcs;
      float acc[NT / 2];
      for (int u0 = 0; u0 < units; u0 += kCgUnits) {
        const int nu = min(kCgUnits, units - u0);
        tc::mbar_wait(&full[s], ph);
        const uint32_t a_base = tc::smem_u32(smem_a + s * kCgAStage) + g * 1024, b_base = tc::smem_u32(smem_b + s * b_stage);
        tc::wg_fence();
        for (int qq = 0; qq < nu; ++qq) {
          const uint64_t adesc = tc::make_desc_kmajor_noswz(a_base + qq * 2 * 2048, 2048, 128);
          const uint64_t bdesc = tc::make_desc_kmajor_noswz(b_base + qq * NT * 32, NT * 16, 128);
          tc::wg_mma_ss<NT>(acc, adesc, bdesc, (u0 | qq) != 0 ? 1u : 0u, 128);
        }
        tc::wg_commit();
        tc::wg_wait<0>();
        tc::wg_fence_acc<NT / 2>(acc);
        if (wid == 0 && lane == 0) tc::mbar_arrive(&empty[s]);
        if (++s == kCgStages) { s = 0; ph ^= 1; }
      }
      // a parity class without live taps (a transposed conv with k < stride, e.g. the odd outputs of k1 s2) runs no MMA,
      // and only its first MMA would have cleared the accumulators: its outputs are the bias alone, as in torch
      if (units == 0) {
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
      }
      const long long cv = (long long)rt * 128 + q * 32 + lane;
      bool ok = cv < coarse;
      long long orow = 0;
      if (ok) {
        int ox = (int)(cv % p.Wc), oy = (int)((cv / p.Wc) % p.Hc), oz = (int)(cv / ((long long)p.Wc * p.Hc));
        if (d.transposed) {
          const int sd = d.stride[0], sh = d.stride[1], sw = d.stride[2];
          ox = ox * sw + cls % sw; oy = oy * sh + (cls / sw) % sh; oz = oz * sd + cls / (sw * sh);
        }
        ok = oz < d.Do && oy < d.Ho && ox < d.Wo;
        orow = ((long long)oz * d.Ho + oy) * d.Wo + ox;
      }
      const int co0 = nt * NT;
#pragma unroll
      for (int c16 = 0; c16 < NT / 16; ++c16, ++sl) {
        float* buf = stage + (sl & 1) * tc::kStageFloats;
        tc::wg_stage16<0>(acc + c16 * 8, buf, wid, lane);
        tc::wg_bar(8 + g);
        float f[8];
        tc::wg_read8(buf, wid, lane, f);
        const int cc = 2 * c16 + half;
        const int nc = co0 + cc * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += (p.bias && nc + j < d.Cout) ? p.bias[nc + j] : 0.f;
        if (ok) {
          if (d.out_layout == 0) {
            if (nc < d.Cout) {
              __align__(16) __half hv[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) hv[j] = __float2half_rn(f[j]);
              __half* yb = (__half*)p.y + ((long long)n * (d.out_ctot / 8) + (d.out_coff + nc) / 8) * So * 8;
              *reinterpret_cast<uint4*>(yb + orow * 8) = *reinterpret_cast<const uint4*>(hv);
            }
          } else {  // NCDHW (fp16 or fp32), only the real channels
#pragma unroll
            for (int j = 0; j < 8; ++j)
              if (nc + j < d.Cout) {
                const long long o = ((long long)n * d.Cout + nc + j) * So + orow;
                if (d.out_dtype == B200_DT_F16) ((__half*)p.y)[o] = __float2half_rn(f[j]);
                else ((float*)p.y)[o] = f[j];
              }
          }
        }
        if (p.sp.buf) {
          float a8[8], b8[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) { a8[j] = ok ? f[j] : 0.f; b8[j] = a8[j] * a8[j]; }
          float csum, cq;
          transpose_reduce8(a8, b8, lane, csum, cq);
          if ((lane & 3) == 0) {
            const int col = cc * 8 + transpose_reduce8_col(lane);
            ws[2 * col] += csum;
            ws[2 * col + 1] += cq;
          }
        }
      }
    }
    if (p.sp.buf && group >= 0) {
      tc::wg_bar(8 + g);
      if (half == 0) stats_flush(p.sp, ws, 2 * NT, group, q, lane, 0, NT);
    }
  }
}

// N tile: the widest compiled width that divides the padded Cout (NT / 2 accumulator registers per consumer thread)
static int cg_nt(int cout_pad) {
  constexpr int kWidths[6] = {128, 96, 64, 48, 32, 16};
  for (int nt : kWidths)
    if (cout_pad % nt == 0) return nt;
  return 16;
}

template <int NT>
static int cg_launch(const CgParams& p, long long total_tiles, cudaStream_t st) {
  const int smem = kCgStages * (kCgAStage + kCgUnits * NT * 32) + 128 + 4 * 2 * NT * 4 + 2 * 2 * tc::kStageFloats * 4 + 128;
  // per-device attribute: set on every call (cheap), so a second GPU in the same process works
  B200_CUDA(cudaFuncSetAttribute(conv_gather_tc_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  dim3 grid((unsigned)std::min<long long>(total_tiles, num_sms()));
  conv_gather_tc_kernel<NT><<<grid, 384, smem, st>>>(p);
  B200_LAUNCH_CHECK("conv_gather_tc_kernel");
  return B200_OK;
}

static int cg_setup(const b200_conv_gather_desc& d, CgParams& p) {
  B200_REQUIRE(d.N > 0 && d.Cin > 0 && d.Cin % 16 == 0 && d.Cout > 0, "conv_gather_tc: Cin must be a multiple of 16 (got %d)", d.Cin);
  for (int a = 0; a < 3; ++a)
    B200_REQUIRE(d.k[a] >= 1 && d.k[a] <= 3 && d.stride[a] >= 1 && d.stride[a] <= 2 && d.pad[a] >= 0 && d.pad[a] < 3,
                 "conv_gather_tc: kernel <= 3, stride <= 2, pad < 3 on every axis");
  B200_REQUIRE(d.in_ctot % 8 == 0 && d.in_coff % 8 == 0 && d.in_coff + d.Cin <= d.in_ctot, "conv_gather_tc: bad input channel slice");
  B200_REQUIRE(d.out_layout == 1 || (d.Cout % 8 == 0 && d.out_ctot % 8 == 0 && d.out_coff % 8 == 0 && d.out_coff + d.Cout <= d.out_ctot),
               "conv_gather_tc: NC8 output needs channel counts that are multiples of 8");
  p.d = d;
  p.cout_pad = (d.Cout + 15) / 16 * 16;
  p.NT = cg_nt(p.cout_pad);
  cg_build_taps(d, p);
  if (d.transposed) {
    p.Dc = ceil_div(d.Do, d.stride[0]); p.Hc = ceil_div(d.Ho, d.stride[1]); p.Wc = ceil_div(d.Wo, d.stride[2]);
  } else {
    p.Dc = d.Do; p.Hc = d.Ho; p.Wc = d.Wo;
  }
  return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" long long b200_conv_gather_tc_weight_bytes(const b200_conv_gather_desc* desc) {
  if (!desc) return -1;
  CgParams p;
  if (cg_setup(*desc, p)) return -1;
  return (long long)p.cout_pad * p.units_total * 16 * 2;
}

extern "C" int b200_conv_gather_tc_pack_weight(const b200_conv_gather_desc* desc, const float* w, void* packed, void* stream) {
  B200_REQUIRE(desc && w && packed, "conv_gather_tc_pack_weight: null pointer");
  CgParams p;
  int rc = cg_setup(*desc, p);
  if (rc) return rc;
  const long long total = (long long)p.cout_pad * p.units_total * 16;
  const int blocks = (int)std::min<long long>((total + 255) / 256, 4096);
  cg_pack_weight_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, (__half*)packed, p);
  B200_LAUNCH_CHECK("cg_pack_weight_kernel");
  return B200_OK;
}

extern "C" long long b200_conv_gather_tc_workspace_bytes(const b200_conv_gather_desc* desc) {
  if (!desc) return -1;
  CgParams p;
  if (cg_setup(*desc, p)) return -1;
  const long long coarse = (long long)p.Dc * p.Hc * p.Wc;
  const long long tpg = (long long)p.ncls * ((coarse + 127) / 128), groups = (long long)desc->N * (p.cout_pad / p.NT);
  return stats_partial_bytes(groups, stats_rows(tpg, tpg * groups), p.NT);
}

extern "C" int b200_conv_gather_tc(const b200_conv_gather_desc* desc, const void* x, const void* packed_w, const float* bias,
                                   void* y, float* stats, void* workspace, void* stream) {
  B200_REQUIRE(desc && x && packed_w && y, "conv_gather_tc: null pointer");
  B200_REQUIRE(!stats || workspace, "conv_gather_tc: statistics need the workspace of b200_conv_gather_tc_workspace_bytes()");
  CgParams p;
  int rc = cg_setup(*desc, p);
  if (rc) return rc;
  const b200_conv_gather_desc& d = *desc;
  // shape consistency with torch's conv arithmetic, per axis
  const int in_sp[3] = {d.Di, d.Hi, d.Wi}, out_sp[3] = {d.Do, d.Ho, d.Wo};
  for (int a = 0; a < 3; ++a) {
    if (!d.transposed) {
      B200_REQUIRE(out_sp[a] == (in_sp[a] + 2 * d.pad[a] - d.k[a]) / d.stride[a] + 1, "conv_gather_tc: output shape does not match conv arithmetic");
    } else {
      const int lo = (in_sp[a] - 1) * d.stride[a] - 2 * d.pad[a] + d.k[a];
      B200_REQUIRE(out_sp[a] >= lo && out_sp[a] < lo + d.stride[a], "conv_gather_tc: output shape does not match transposed-conv arithmetic");
    }
  }
  p.x = (const __half*)x; p.w = (const __half*)packed_w; p.bias = bias; p.y = y;
  const long long coarse = (long long)p.Dc * p.Hc * p.Wc;
  const long long tpg = (long long)p.ncls * ((coarse + 127) / 128), groups = (long long)d.N * (p.cout_pad / p.NT);
  const long long total_tiles = tpg * groups;
  p.sp.buf = stats ? (float*)workspace : nullptr;
  p.sp.R = stats_rows(tpg, total_tiles);
  p.sp.tiles_per_group = tpg;
  p.sp.rows_per_cta = 4;
  switch (p.NT) {
    case 128: rc = cg_launch<128>(p, total_tiles, (cudaStream_t)stream); break;
    case 96: rc = cg_launch<96>(p, total_tiles, (cudaStream_t)stream); break;
    case 64: rc = cg_launch<64>(p, total_tiles, (cudaStream_t)stream); break;
    case 48: rc = cg_launch<48>(p, total_tiles, (cudaStream_t)stream); break;
    case 32: rc = cg_launch<32>(p, total_tiles, (cudaStream_t)stream); break;
    default: rc = cg_launch<16>(p, total_tiles, (cudaStream_t)stream); break;
  }
  if (rc) return rc;
  if (stats) return launch_stats_finish((const float*)workspace, groups, p.sp.R * 4, p.NT, p.cout_pad / p.NT, d.Cout, stats, (cudaStream_t)stream);
  return B200_OK;
}
