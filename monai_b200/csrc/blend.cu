// Sliding-window gather + importance-weighted overlap blend (SURVEY.md §8 rows a3, a4, a5).
//
// Replaces monai/inferers/utils.py:217-224 (window gather), :264-275 (count map), :286-288 + :351-360
// (weighted scatter-add) and :297-298 (normalise) of the reference.  The blend is written in *gather form*:
// one thread owns one output voxel and walks the (Cartesian) window table in ascending window index, so
//   out[b,c,v] = ( sum_w imp(v - s_w) * pred_w[c, v - s_w] ) / ( sum_w imp(v - s_w) )
// is produced, for fp32 predictions, with the same fp32 operation order as the reference loop (mul, then sequential
// adds, then one IEEE divide); fp16 predictions use one fused multiply-add per term (blend_acc).  The count map is
// never materialised.  imp() is evaluated on the fly from the three 1-D
// vectors of compute_importance_map (monai/data/utils.py:1084-1134): ((g_d*g_h)*g_w) clamped from below.
#include "common.cuh"
#include "blend.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

// MODE 0: all windows resident -> write normalised result.  MODE 1: accumulate numerators (+=) for the
// resident window range.  MODE 2: divide accumulators by the analytic count (all windows).
//
// Each thread owns VEC (1 or 2) consecutive voxels along W.  It first lists the covering windows (at most kMaxCover,
// ascending window index = the reference's accumulation order) with their weights, then streams the predictions in
// groups of four independent loads so that ~16 requests per thread are in flight (the kernel is HBM-bound: every
// prediction is read exactly once, the output is written exactly once).

template <typename TP, int VEC> struct PredVec;
template <> struct PredVec<__half, 1> { static __device__ __forceinline__ void ld(const __half* p, float* v) { v[0] = __half2float(__ldg(p)); } };
template <> struct PredVec<float, 1> { static __device__ __forceinline__ void ld(const float* p, float* v) { v[0] = __ldg(p); } };
template <> struct PredVec<__half, 2> {
  static __device__ __forceinline__ void ld(const __half* p, float* v) {
    const __half2 h = __ldg(reinterpret_cast<const __half2*>(p));
    v[0] = __low2float(h); v[1] = __high2float(h);
  }
};
template <> struct PredVec<float, 2> {
  static __device__ __forceinline__ void ld(const float* p, float* v) {
    const float2 h = __ldg(reinterpret_cast<const float2*>(p));
    v[0] = h.x; v[1] = h.y;
  }
};

template <typename TP, typename TO, int MODE, int VEC>
__global__ void __launch_bounds__(128) sw_blend_kernel(BlendParams p) {
  __shared__ int s_w[kMaxStarts];
  __shared__ int s_did[32], s_hid[32];
  __shared__ int s_ndc, s_nhc;
  const int h = blockIdx.y + p.h0;
  const int d = blockIdx.z % (p.d1 - p.d0) + p.d0;
  const int b = blockIdx.z / (p.d1 - p.d0);
  for (int i = threadIdx.x; i < p.nw; i += blockDim.x) s_w[i] = p.starts_w[i];
  if (threadIdx.x == 0) {
    int n = 0;
    for (int i = 0; i < p.nd && n < 32; ++i) { int s = p.starts_d[i]; if (s <= d && d < s + p.rd) s_did[n++] = i; }
    s_ndc = n; n = 0;
    for (int i = 0; i < p.nh && n < 32; ++i) { int s = p.starts_h[i]; if (s <= h && h < s + p.rh) s_hid[n++] = i; }
    s_nhc = n;
  }
  __syncthreads();
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) * VEC;
  if (w >= p.W) return;
  const int num_win = p.nd * p.nh * p.nw;
  const long long vol = (long long)p.D * p.H * p.W;
  const long long voff = ((long long)d * p.H + h) * p.W + w;

  // covering windows along W form a contiguous index range [iw_lo, iw_lo + nwc) because the starts are sorted
  int iw_lo = 0, nwc = 0;
  for (int iw = 0; iw < p.nw; ++iw) {
    const int lw = w - s_w[iw];
    if (lw >= 0 && lw < p.rw) { if (nwc == 0) iw_lo = iw; ++nwc; }
  }
  const TP* preds = (const TP*)p.preds;
  float cnt[VEC];
  // channels are walked in pairs so that up to 8 independent loads are in flight per (d,h) window pair
  for (int c0 = 0; c0 < (MODE == 2 ? 1 : p.C); c0 += 2) {
    const bool two = (MODE != 2) && (c0 + 1 < p.C);
    float acc0[VEC], acc1[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
      cnt[v] = 0.f;
      acc0[v] = (MODE == 1) ? *((const float*)p.out + ((long long)b * p.C + c0) * vol + voff + v) : 0.f;
      acc1[v] = (MODE == 1 && two) ? *((const float*)p.out + ((long long)b * p.C + c0 + 1) * vol + voff + v) : 0.f;
    }
    for (int a = 0; a < s_ndc; ++a) {
      const int id = s_did[a];
      const int ld = d - p.starts_d[id];
      for (int e = 0; e < s_nhc; ++e) {
        const int ih = s_hid[e];
        const int lh = h - p.starts_h[ih];
        const float gdh = p.wmap ? 0.f : __fmul_rn(p.gd[ld], p.gh[lh]);
        const long long rowoff = (long long)ld * p.ps_d + (long long)lh * p.ps_h + (long long)c0 * p.ps_c;
        const int wbase = b * num_win + (id * p.nh + ih) * p.nw;
        for (int k0 = 0; k0 < nwc; k0 += 4) {
          float wt[4][VEC], v0[4][VEC], v1[4][VEC];
          bool res[4];
          int slotq[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int iw = iw_lo + k0 + q;
            const bool in = k0 + q < nwc;
            const int lw = in ? w - s_w[iw] : 0;
            const int widx = wbase + iw;
            // resident slot of this window: contiguous range [win_begin, win_end) or, with a slot map (buffered mode: the
            // windows are visited in another order than their ids), wherever the map says
            int slot = -1;
            if (in && MODE != 2) {
              if (p.slot_map) slot = __ldg(p.slot_map + widx);
              else if (widx >= p.win_begin && widx < p.win_end) slot = widx - p.win_begin;
            }
            slotq[q] = slot;
            res[q] = slot >= 0;
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
              float t = 0.f;
              if (in) t = p.wmap ? p.wmap[((long long)ld * p.rh + lh) * p.rw + lw + v] : fmaxf(__fmul_rn(gdh, p.gw[lw + v]), p.clamp_min);
              wt[q][v] = t; v0[q][v] = 0.f; v1[q][v] = 0.f;
            }
            if (res[q]) {
              const TP* pp = preds + (long long)slotq[q] * p.ps_n + rowoff + (long long)lw * p.ps_w;
              PredVec<TP, VEC>::ld(pp, v0[q]);
              if (two) PredVec<TP, VEC>::ld(pp + p.ps_c, v1[q]);
            }
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
              if (k0 + q < nwc) cnt[v] = __fadd_rn(cnt[v], wt[q][v]);
              if (res[q]) {
                acc0[v] = blend_acc<TP>(acc0[v], v0[q][v], wt[q][v]);
                if (two) acc1[v] = blend_acc<TP>(acc1[v], v1[q][v], wt[q][v]);
              }
            }
          }
        }
      }
    }
    if (MODE == 2) break;
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
      const long long o0 = ((long long)b * p.C + c0) * vol + voff + v;
      if (MODE == 0) {
        const float cf = BlendFin<TO>::prep(cnt[v]);
        io<TO>::st((TO*)p.out + o0, BlendFin<TO>::apply(acc0[v], cf));
        if (two) io<TO>::st((TO*)p.out + o0 + vol, BlendFin<TO>::apply(acc1[v], cf));
      } else {
        *((float*)p.out + o0) = acc0[v];
        if (two) *((float*)p.out + o0 + vol) = acc1[v];
      }
    }
  }
  if (MODE == 2) {
    for (int c = 0; c < p.C; ++c) {
      const long long o = ((long long)b * p.C + c) * vol + voff;
#pragma unroll
      for (int v = 0; v < VEC; ++v) io<TO>::st((TO*)p.out + o + v, BlendFin<TO>::apply(p.acc[o + v], BlendFin<TO>::prep(cnt[v])));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Eight voxels per thread (one 16-byte fp16 vector per prediction channel).  Usable when W, the roi and every window
// start along W are multiples of 8, so a thread's octet is covered by whole windows only.  A warp owns one (d, h) row
// segment: the covering ranges along D and H are warp-uniform, the loop over the covering W windows is per lane.
// Same fp32 operation order as the scalar kernel (ascending window index), hence bit-identical results.
// ---------------------------------------------------------------------------------------------------------------
template <typename TP> struct Pred8;
template <> struct Pred8<__half> {
  using Raw = uint4;
  static __device__ __forceinline__ Raw ld(const __half* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
  static __device__ __forceinline__ void cvt(const Raw& r, float (&v)[8]) {
    const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); v[2 * j] = f.x; v[2 * j + 1] = f.y; }
  }
};
template <> struct Pred8<float> {
  struct Raw { float4 a, b; };
  static __device__ __forceinline__ Raw ld(const float* p) {
    Raw r; r.a = __ldg(reinterpret_cast<const float4*>(p)); r.b = __ldg(reinterpret_cast<const float4*>(p) + 1); return r;
  }
  static __device__ __forceinline__ void cvt(const Raw& r, float (&v)[8]) {
    v[0] = r.a.x; v[1] = r.a.y; v[2] = r.a.z; v[3] = r.a.w; v[4] = r.b.x; v[5] = r.b.y; v[6] = r.b.z; v[7] = r.b.w;
  }
};
__device__ __forceinline__ void ld8f(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <typename TO> __device__ __forceinline__ void st8o(TO* p, const float (&v)[8]);
template <> __device__ __forceinline__ void st8o<float>(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
template <> __device__ __forceinline__ void st8o<__half>(__half* p, const float (&v)[8]) {
  uint4 r;
  __half2* h = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
  *reinterpret_cast<uint4*>(p) = r;
}

constexpr int kBlend8Rows = 8;   // warps (= h rows) per block
constexpr int kBlend8MaxRoiW = 512;
constexpr int kBlend8K = 3;      // W windows per (d, h) window pair handled by the pipelined path (overlap <= 2/3)

// (A variant without the load prefetch, 80 registers and three blocks per SM, measured 0.295 ms against 0.217 ms on C2.)
template <typename TP, typename TO, int MODE>
__global__ void __launch_bounds__(32 * kBlend8Rows, sizeof(TP) == 2 ? 2 : 1) sw_blend8_kernel(BlendParams p) {
  using Raw = typename Pred8<TP>::Raw;
  // A block covers 8 rows x 256 voxels of one depth plane; a WARP covers a compact 8 (h) x 32 (w) patch (lane = row*4 +
  // octet), because the number of covering windows changes only every few voxels along an axis: a compact patch rarely
  // straddles such a boundary, so the lanes of a warp agree on the loop trip counts (a 256-voxel row segment never does).
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
  const int w8 = (blockIdx.x * 32 + wrp * 4 + (lane & 3)) * 8;
  const int h = p.h0 + blockIdx.y * kBlend8Rows + (lane >> 2);
  const int nd_box = p.d1 - p.d0;
  const int d = blockIdx.z % nd_box + p.d0, b = blockIdx.z / nd_box;
  __shared__ __align__(16) float s_gw[kBlend8MaxRoiW];   // W-axis importance factors (pipelined path)
  __shared__ int s_cov[32 + kBlend8Rows + 1];            // covering window ranges (lo | count << 16): 32 octets, 8 rows, the plane
  if (p.gw && p.rw <= kBlend8MaxRoiW)
    for (int i = threadIdx.x; i < p.rw; i += blockDim.x) s_gw[i] = __ldg(p.gw + i);
  if (threadIdx.x < 32 + kBlend8Rows + 1) {
    // the window starts are sorted, so the windows covering a coordinate form a contiguous index range per axis
    const int t = threadIdx.x;
    const int* st = t < 32 ? p.starts_w : (t < 32 + kBlend8Rows ? p.starts_h : p.starts_d);
    const int ns = t < 32 ? p.nw : (t < 32 + kBlend8Rows ? p.nh : p.nd);
    const int r = t < 32 ? p.rw : (t < 32 + kBlend8Rows ? p.rh : p.rd);
    const int xq = t < 32 ? (blockIdx.x * 32 + t) * 8 : (t < 32 + kBlend8Rows ? p.h0 + blockIdx.y * kBlend8Rows + (t - 32) : d);
    int lo = 0, cn = 0;
    for (int i = 0; i < ns; ++i) { const int s = __ldg(st + i); if (s <= xq && xq < s + r) { if (!cn) lo = i; ++cn; } }
    s_cov[t] = lo | (cn << 16);
  }
  __syncthreads();
  if (h >= p.h1 || w8 >= p.W) return;
  const int cw = s_cov[wrp * 4 + (lane & 3)], ch = s_cov[32 + (lane >> 2)], cd = s_cov[32 + kBlend8Rows];
  const int id_lo = cd & 0xffff, ndc = cd >> 16, ih_lo = ch & 0xffff, nhc = ch >> 16, iw_lo = cw & 0xffff, nwc = cw >> 16;
  const int num_win = p.nd * p.nh * p.nw;
  const long long vol = (long long)p.D * p.H * p.W;
  const long long voff = ((long long)d * p.H + h) * p.W + w8;
  const TP* __restrict__ preds = (const TP*)p.preds;
  const bool dense = p.wmap != nullptr;
  // Pipelined path (the common geometry: at most 3 covering windows per axis, i.e. overlap <= 2/3): every per-axis
  // quantity (local coordinate, 1-D weight, address offset) lives in registers, a prediction address is
  // base + offA[a] + offE[e] + offK[k], and nothing but the predictions themselves is loaded inside the window loop.
  const bool piped = !dense && ndc <= kBlend8K && nhc <= kBlend8K && nwc <= kBlend8K && p.offsets_fit_i32 && p.rw <= kBlend8MaxRoiW;
  long long offA[kBlend8K];
  int offE[kBlend8K], offK[kBlend8K];
  float gda[kBlend8K], ghe[kBlend8K];
  int lwk[kBlend8K];
  if (piped) {
#pragma unroll
    for (int k = 0; k < kBlend8K; ++k) {
      const int ia = id_lo + (k < ndc ? k : 0), ie = ih_lo + (k < nhc ? k : 0), ik = iw_lo + (k < nwc ? k : 0);
      const int ld = d - __ldg(p.starts_d + ia), lh = h - __ldg(p.starts_h + ie), lw = w8 - __ldg(p.starts_w + ik);
      gda[k] = __ldg(p.gd + ld); ghe[k] = __ldg(p.gh + lh);
      lwk[k] = lw;
      offA[k] = (long long)ld * p.ps_d + (long long)ia * p.nh * p.nw * p.ps_n;
      offE[k] = (int)(lh * p.ps_h + (long long)ie * p.nw * p.ps_n);
      offK[k] = (int)(lw + (long long)ik * p.ps_n);
    }
  }
  float cnt[8];
  for (int c0 = 0; c0 < (MODE == 2 ? 1 : p.C); c0 += 2) {
    const bool two = (MODE != 2) && (c0 + 1 < p.C);
    float a0[8], a1[8];
#pragma unroll
    for (int v = 0; v < 8; ++v) { cnt[v] = 0.f; a0[v] = 0.f; a1[v] = 0.f; }
    if (MODE == 1) {
      ld8f((const float*)p.out + ((long long)b * p.C + c0) * vol + voff, a0);
      if (two) ld8f((const float*)p.out + ((long long)b * p.C + c0 + 1) * vol + voff, a1);
    }
    if (piped) {
      // The (d, h) window pairs are walked in ascending window order; the prediction vectors of pair q+1 are requested
      // before pair q is accumulated, so up to 12 16-byte loads per thread are in flight (every prediction is read
      // exactly once and nothing is reused, so memory-level parallelism is what the kernel lives on).
      const int P = ndc * nhc;
      const TP* pbase = preds + ((long long)b * num_win - p.win_begin) * p.ps_n + (long long)c0 * p.ps_c;
      const unsigned nres = (unsigned)(p.win_end - p.win_begin);
      const int wrel0 = b * num_win - p.win_begin + iw_lo;
      struct Pair { float gdh; int wrel; };
      auto issue = [&](int a, int e, Raw (&r0)[kBlend8K], Raw (&r1)[kBlend8K]) -> Pair {
        Pair pr;
        pr.gdh = __fmul_rn(a == 0 ? gda[0] : (a == 1 ? gda[1] : gda[2]), e == 0 ? ghe[0] : (e == 1 ? ghe[1] : ghe[2]));
        pr.wrel = wrel0 + ((id_lo + a) * p.nh + ih_lo + e) * p.nw;
        if (MODE != 2) {
          const TP* pp = pbase + (a == 0 ? offA[0] : (a == 1 ? offA[1] : offA[2])) + (e == 0 ? offE[0] : (e == 1 ? offE[1] : offE[2]));
#pragma unroll
          for (int k = 0; k < kBlend8K; ++k) {
            if (k < nwc && (unsigned)(pr.wrel + k) < nres) {
              r0[k] = Pred8<TP>::ld(pp + offK[k]);
              if (two) r1[k] = Pred8<TP>::ld(pp + offK[k] + p.ps_c);
            }
          }
        }
        return pr;
      };
      auto consume = [&](const Pair& pr, const Raw (&r0)[kBlend8K], const Raw (&r1)[kBlend8K]) {
#pragma unroll
        for (int k = 0; k < kBlend8K; ++k) {
          if (k < nwc) {
            float t[8];
            const float4 g0 = *reinterpret_cast<const float4*>(s_gw + lwk[k]), g1 = *reinterpret_cast<const float4*>(s_gw + lwk[k] + 4);
            t[0] = g0.x; t[1] = g0.y; t[2] = g0.z; t[3] = g0.w; t[4] = g1.x; t[5] = g1.y; t[6] = g1.z; t[7] = g1.w;
#pragma unroll
            for (int v = 0; v < 8; ++v) { t[v] = fmaxf(__fmul_rn(pr.gdh, t[v]), p.clamp_min); cnt[v] = __fadd_rn(cnt[v], t[v]); }
            if (MODE != 2 && (unsigned)(pr.wrel + k) < nres) {
              float xv[8];
              Pred8<TP>::cvt(r0[k], xv);
#pragma unroll
              for (int v = 0; v < 8; ++v) a0[v] = blend_acc<TP>(a0[v], xv[v], t[v]);
              if (two) {
                Pred8<TP>::cvt(r1[k], xv);
#pragma unroll
                for (int v = 0; v < 8; ++v) a1[v] = blend_acc<TP>(a1[v], xv[v], t[v]);
              }
            }
          }
        }
      };
      int ai = 0, ei = 0;   // (d, h) pair position of the load stream
      auto adv = [&](int& a, int& e) { if (++e == nhc) { e = 0; ++a; } };
      Raw A0[kBlend8K], A1[kBlend8K], B0[kBlend8K], B1[kBlend8K];
      Pair pa, pb;
      if (P > 0) { pa = issue(ai, ei, A0, A1); adv(ai, ei); }
      for (int q = 0; q < P; q += 2) {
        if (q + 1 < P) { pb = issue(ai, ei, B0, B1); adv(ai, ei); }
        consume(pa, A0, A1);
        if (q + 1 < P) {
          if (q + 2 < P) { pa = issue(ai, ei, A0, A1); adv(ai, ei); }
          consume(pb, B0, B1);
        }
      }
    } else {
      for (int a = 0; a < ndc; ++a) {
        const int id = id_lo + a;
        const int ld = d - __ldg(p.starts_d + id);
        for (int e = 0; e < nhc; ++e) {
          const int ih = ih_lo + e;
          const int lh = h - __ldg(p.starts_h + ih);
          const float gdh = dense ? 0.f : __fmul_rn(__ldg(p.gd + ld), __ldg(p.gh + lh));
          const long long rowoff = (long long)ld * p.ps_d + (long long)lh * p.ps_h + (long long)c0 * p.ps_c;
          const int wbase = b * num_win + (id * p.nh + ih) * p.nw;
          for (int k = 0; k < nwc; ++k) {
            const int iw = iw_lo + k;
            const int lw = w8 - __ldg(p.starts_w + iw);
            const int widx = wbase + iw;
            const bool res = (MODE != 2) && widx >= p.win_begin && widx < p.win_end;
            Raw r0, r1;
            if (res) {
              const TP* pp = preds + (long long)(widx - p.win_begin) * p.ps_n + rowoff + lw;
              r0 = Pred8<TP>::ld(pp);
              if (two) r1 = Pred8<TP>::ld(pp + p.ps_c);
            }
            float t[8];
            if (dense) {
              ld8f(p.wmap + ((long long)ld * p.rh + lh) * p.rw + lw, t);
            } else {
              ld8f(p.gw + lw, t);
#pragma unroll
              for (int v = 0; v < 8; ++v) t[v] = fmaxf(__fmul_rn(gdh, t[v]), p.clamp_min);
            }
#pragma unroll
            for (int v = 0; v < 8; ++v) cnt[v] = __fadd_rn(cnt[v], t[v]);
            if (res) {
              float xv[8];
              Pred8<TP>::cvt(r0, xv);
#pragma unroll
              for (int v = 0; v < 8; ++v) a0[v] = blend_acc<TP>(a0[v], xv[v], t[v]);
              if (two) {
                Pred8<TP>::cvt(r1, xv);
#pragma unroll
                for (int v = 0; v < 8; ++v) a1[v] = blend_acc<TP>(a1[v], xv[v], t[v]);
              }
            }
          }
        }
      }
    }
    if (MODE == 2) break;
    const long long o0 = ((long long)b * p.C + c0) * vol + voff;
    if (MODE == 0) {
#pragma unroll
      for (int v = 0; v < 8; ++v) { const float cf = BlendFin<TO>::prep(cnt[v]); a0[v] = BlendFin<TO>::apply(a0[v], cf); a1[v] = BlendFin<TO>::apply(a1[v], cf); }
      st8o<TO>((TO*)p.out + o0, a0);
      if (two) st8o<TO>((TO*)p.out + o0 + vol, a1);
    } else {
      st8o<float>((float*)p.out + o0, a0);
      if (two) st8o<float>((float*)p.out + o0 + vol, a1);
    }
  }
  if (MODE == 2) {
    for (int c = 0; c < p.C; ++c) {
      const long long o = ((long long)b * p.C + c) * vol + voff;
      float xv[8];
      ld8f(p.acc + o, xv);
#pragma unroll
      for (int v = 0; v < 8; ++v) xv[v] = BlendFin<TO>::apply(xv[v], BlendFin<TO>::prep(cnt[v]));
      st8o<TO>((TO*)p.out + o, xv);
    }
  }
}

template <typename TI, typename TO>
__global__ void __launch_bounds__(256) sw_gather_kernel(const TI* __restrict__ vol, TO* __restrict__ out,
                                                        const int* __restrict__ tab, int C, int D, int H, int W,
                                                        int rd, int rh, int rw) {
  // grid: x over w, y over (d*rh + h), z over (win*C + c)
  const int win = blockIdx.z / C, c = blockIdx.z % C;
  const int ld = blockIdx.y / rh, lh = blockIdx.y % rh;
  const int b = tab[win * 4 + 0], sd = tab[win * 4 + 1], sh = tab[win * 4 + 2], sw = tab[win * 4 + 3];
  const TI* src = vol + ((((long long)b * C + c) * D + sd + ld) * H + sh + lh) * W + sw;
  TO* dst = out + ((((long long)win * C + c) * rd + ld) * rh + lh) * (long long)rw;
  for (int lw = blockIdx.x * blockDim.x + threadIdx.x; lw < rw; lw += gridDim.x * blockDim.x)
    io<TO>::st(dst + lw, io<TI>::ld(src + lw));
}

// Same copy with 16-byte vectors (both element types equal, rw / W / every start along W multiples of the vector width):
// a thread moves one vector, a block walks (window, channel, d, h, vector) with a grid stride -- the one-row-per-block form
// above spends its time on block turnover (0.05 of HBM bandwidth on the 96^3 windows of C3).
template <typename T>
__global__ void __launch_bounds__(256) sw_gather_vec_kernel(const T* __restrict__ vol, T* __restrict__ out, const int* __restrict__ tab,
                                                            int n_win, int C, int D, int H, int W, int rd, int rh, int rw) {
  constexpr int V = 16 / sizeof(T);
  const int rwv = rw / V;
  const long long per_win = (long long)C * rd * rh * rwv;
  const long long total = per_win * n_win;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int win = (int)(i / per_win);
    long long r = i % per_win;
    const int wv = (int)(r % rwv); r /= rwv;
    const int lh = (int)(r % rh); r /= rh;
    const int ld = (int)(r % rd);
    const int c = (int)(r / rd);
    const int b = __ldg(tab + win * 4), sd = __ldg(tab + win * 4 + 1), sh = __ldg(tab + win * 4 + 2), sw = __ldg(tab + win * 4 + 3);
    const T* src = vol + ((((long long)b * C + c) * D + sd + ld) * H + sh + lh) * W + sw + wv * V;
    T* dst = out + ((((long long)win * C + c) * rd + ld) * rh + lh) * (long long)rw + wv * V;
    *reinterpret_cast<uint4*>(dst) = __ldg(reinterpret_cast<const uint4*>(src));
  }
}

// blend_fused.cu
int launch_blend8_lean(const BlendParams& p, int out_dtype, cudaStream_t st);
int launch_blend_resample(const BlendParams& p, const double* m, int oD, int oH, int oW, int interp, int pad, int mode, int pred_dtype,
                          int out_dtype, cudaStream_t st);

}  // namespace b200

using namespace b200;

template <int MODE, int VEC>
static int launch_blend_v(const BlendParams& p, int pred_dtype, int out_dtype, cudaStream_t st) {
  const int wq = (p.W + VEC - 1) / VEC;
  dim3 block(wq >= 128 ? 128 : (wq >= 64 ? 64 : 32));
  dim3 grid(ceil_div(wq, block.x), p.h1 - p.h0, (p.d1 - p.d0) * p.B);
  if (grid.y == 0 || grid.z == 0) return B200_OK;
  B200_REQUIRE(grid.z <= 65535 && grid.y <= 65535, "sw_blend: volume too large for the launch grid");
#define LB(TP, TO) sw_blend_kernel<TP, TO, MODE, VEC><<<grid, block, 0, st>>>(p)
  if (MODE == 1) {
    if (pred_dtype == B200_DT_F16) LB(__half, float); else LB(float, float);
  } else if (MODE == 2) {
    if (out_dtype == B200_DT_F16) LB(float, __half); else LB(float, float);
  } else {
    if (pred_dtype == B200_DT_F16 && out_dtype == B200_DT_F16) LB(__half, __half);
    else if (pred_dtype == B200_DT_F16) LB(__half, float);
    else if (out_dtype == B200_DT_F16) LB(float, __half);
    else LB(float, float);
  }
#undef LB
  B200_LAUNCH_CHECK("sw_blend_kernel");
  return B200_OK;
}

template <int MODE>
static int launch_blend8(const BlendParams& p, int pred_dtype, int out_dtype, cudaStream_t st) {
  dim3 block(32 * kBlend8Rows);
  dim3 grid(ceil_div(p.W / 8, 32), ceil_div(p.h1 - p.h0, kBlend8Rows), (p.d1 - p.d0) * p.B);
  if (grid.y == 0 || grid.z == 0) return B200_OK;
  B200_REQUIRE(grid.z <= 65535 && grid.y <= 65535, "sw_blend: volume too large for the launch grid");
#define LB(TP, TO) sw_blend8_kernel<TP, TO, MODE><<<grid, block, 0, st>>>(p)
  if (MODE == 1) {
    if (pred_dtype == B200_DT_F16) LB(__half, float); else LB(float, float);
  } else if (MODE == 2) {
    if (out_dtype == B200_DT_F16) LB(float, __half); else LB(float, float);
  } else {
    if (pred_dtype == B200_DT_F16 && out_dtype == B200_DT_F16) LB(__half, __half);
    else if (pred_dtype == B200_DT_F16) LB(__half, float);
    else if (out_dtype == B200_DT_F16) LB(float, __half);
    else LB(float, float);
  }
#undef LB
  B200_LAUNCH_CHECK("sw_blend8_kernel");
  return B200_OK;
}

template <int MODE>
static int launch_blend(const BlendParams& p, int pred_dtype, int out_dtype, bool vec2, bool vec8, cudaStream_t st) {
  if (vec8) return launch_blend8<MODE>(p, pred_dtype, out_dtype, st);
  return vec2 ? launch_blend_v<MODE, 2>(p, pred_dtype, out_dtype, st) : launch_blend_v<MODE, 1>(p, pred_dtype, out_dtype, st);
}

extern "C" int b200_sw_blend(const b200_blend_desc* dsc, int mode, void* stream) {
  B200_REQUIRE(dsc != nullptr, "sw_blend: null descriptor");
  B200_REQUIRE(mode >= 0 && mode <= 2, "sw_blend: mode must be 0 (final), 1 (accumulate) or 2 (finalize)");
  B200_REQUIRE(dsc->nw <= kMaxStarts, "sw_blend: more than %d window starts along the last axis", kMaxStarts);
  B200_REQUIRE(dsc->B > 0 && dsc->C > 0 && dsc->D > 0 && dsc->H > 0 && dsc->W > 0, "sw_blend: empty volume");
  B200_REQUIRE(dsc->rd <= dsc->D && dsc->rh <= dsc->H && dsc->rw <= dsc->W, "sw_blend: roi larger than the padded volume");
  B200_REQUIRE(dsc->pred_dtype == B200_DT_F32 || dsc->pred_dtype == B200_DT_F16, "sw_blend: bad pred dtype");
  B200_REQUIRE(dsc->out_dtype == B200_DT_F32 || dsc->out_dtype == B200_DT_F16, "sw_blend: bad out dtype");
  BlendParams p;
  p.preds = dsc->preds;
  p.ps_n = dsc->pred_stride[0]; p.ps_c = dsc->pred_stride[1]; p.ps_d = dsc->pred_stride[2];
  p.ps_h = dsc->pred_stride[3]; p.ps_w = dsc->pred_stride[4];
  p.win_begin = dsc->win_begin; p.win_end = dsc->win_end;
  p.B = dsc->B; p.C = dsc->C; p.D = dsc->D; p.H = dsc->H; p.W = dsc->W;
  p.rd = dsc->rd; p.rh = dsc->rh; p.rw = dsc->rw;
  p.starts_d = dsc->starts_d; p.nd = dsc->nd; p.starts_h = dsc->starts_h; p.nh = dsc->nh;
  p.starts_w = dsc->starts_w; p.nw = dsc->nw;
  p.gd = dsc->gd; p.gh = dsc->gh; p.gw = dsc->gw; p.clamp_min = dsc->clamp_min; p.wmap = dsc->wmap;
  p.out = dsc->out; p.acc = dsc->acc;
  p.d0 = dsc->box[0]; p.d1 = dsc->box[1]; p.h0 = dsc->box[2]; p.h1 = dsc->box[3];
  p.slot_map = dsc->slot_map; p.n_slots = dsc->n_slots;
  B200_REQUIRE(!p.slot_map || mode == 1, "sw_blend: a slot map goes with mode 1 (accumulate)");
  p.offsets_fit_i32 = mode == 2 || ((long long)(p.nh + 1) * p.nw * p.ps_n + (long long)p.rh * p.ps_h + p.rw < (1LL << 31));
  if (p.d1 <= 0) { p.d0 = 0; p.d1 = p.D; }
  if (p.h1 <= 0) { p.h0 = 0; p.h1 = p.H; }
  B200_REQUIRE(p.d0 >= 0 && p.d1 <= p.D && p.h0 >= 0 && p.h1 <= p.H, "sw_blend: box outside the volume");
  cudaStream_t st = (cudaStream_t)stream;
  if (dsc->resample)   // fused blend + affine resample: the blended volume is never materialised
    return launch_blend_resample(p, dsc->resample, dsc->out_D, dsc->out_H, dsc->out_W, dsc->resample_interp, dsc->resample_pad, mode,
                                 dsc->pred_dtype, dsc->out_dtype, st);
  // two voxels per thread when every window start, the roi and W are even and predictions are contiguous along W
  bool vec2 = (p.W % 2 == 0) && (p.rw % 2 == 0) && (mode == 2 || p.ps_w == 1) && dsc->starts_w_align >= 2 && dsc->starts_w_align % 2 == 0;
  if (vec2 && mode != 2) {
    const int esz = dsc->pred_dtype == B200_DT_F16 ? 2 : 4;
    vec2 = (reinterpret_cast<uintptr_t>(p.preds) % (2 * esz) == 0) && p.ps_n % 2 == 0 && p.ps_c % 2 == 0 && p.ps_d % 2 == 0 && p.ps_h % 2 == 0;
  }
  // eight voxels per thread: everything along W is a multiple of 8 and every vector access is 16-byte aligned
  bool vec8 = (p.W % 8 == 0) && (p.rw % 8 == 0) && (mode == 2 || p.ps_w == 1) && dsc->starts_w_align >= 8 && dsc->starts_w_align % 8 == 0 &&
              reinterpret_cast<uintptr_t>(p.out) % 16 == 0 && (mode != 2 || reinterpret_cast<uintptr_t>(p.acc) % 16 == 0) &&
              (p.wmap ? reinterpret_cast<uintptr_t>(p.wmap) % 16 == 0 : reinterpret_cast<uintptr_t>(p.gw) % 16 == 0);
  if (vec8 && mode != 2)
    vec8 = (reinterpret_cast<uintptr_t>(p.preds) % 16 == 0) && p.ps_n % 8 == 0 && p.ps_c % 8 == 0 && p.ps_d % 8 == 0 && p.ps_h % 8 == 0;
  if (p.slot_map) vec8 = false;   // only the general kernel looks windows up through a slot map
  // lean 8-voxel kernel: everything resident, fp16 predictions, separable weights, at most three covering windows per axis
  if (mode == 0 && vec8 && dsc->pred_dtype == B200_DT_F16 && !p.wmap && dsc->max_cover >= 1 && dsc->max_cover <= 3 && p.rw <= 512 &&
      p.win_begin == 0 && p.win_end == p.B * p.nd * p.nh * p.nw)
    return launch_blend8_lean(p, dsc->out_dtype, st);
  if (mode == 0) return launch_blend<0>(p, dsc->pred_dtype, dsc->out_dtype, vec2, vec8, st);
  if (mode == 1) return launch_blend<1>(p, dsc->pred_dtype, dsc->out_dtype, vec2, vec8, st);
  return launch_blend<2>(p, dsc->pred_dtype, dsc->out_dtype, vec2, vec8, st);
}

extern "C" int b200_sw_gather(const void* vol, int in_dtype, void* out, int out_dtype, const int32_t* win_tab,
                              int n_win, int C, int D, int H, int W, int rd, int rh, int rw, int starts_w_align, void* stream) {
  if (n_win == 0) return B200_OK;
  B200_REQUIRE(vol && out && win_tab, "sw_gather: null pointer");
  B200_REQUIRE(rd <= D && rh <= H && rw <= W, "sw_gather: roi larger than the volume");
  cudaStream_t st = (cudaStream_t)stream;
  // vector path: equal dtypes and everything along W aligned to 16 bytes; `starts_w_align` is the caller's promise about the
  // window starts along W (a common divisor of all of them; 0 / 1 = unknown), which cannot be seen from here
  const int esz = in_dtype == B200_DT_F16 ? 2 : 4, V = 16 / esz;
  if (in_dtype == out_dtype && starts_w_align >= V && starts_w_align % V == 0 && rw % V == 0 && W % V == 0 && reinterpret_cast<uintptr_t>(vol) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0) {
    const long long total = (long long)n_win * C * rd * rh * (rw / V);
    const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
    if (in_dtype == B200_DT_F16) sw_gather_vec_kernel<__half><<<blocks, 256, 0, st>>>((const __half*)vol, (__half*)out, win_tab, n_win, C, D, H, W, rd, rh, rw);
    else sw_gather_vec_kernel<float><<<blocks, 256, 0, st>>>((const float*)vol, (float*)out, win_tab, n_win, C, D, H, W, rd, rh, rw);
    B200_LAUNCH_CHECK("sw_gather_vec_kernel");
    return B200_OK;
  }
  B200_REQUIRE((long long)n_win * C <= 65535 && (long long)rd * rh <= 65535, "sw_gather: batch too large for one launch");
  dim3 block(rw >= 128 ? 128 : 64), grid(ceil_div(rw, block.x), rd * rh, n_win * C);
#define LG(TI, TO) sw_gather_kernel<TI, TO><<<grid, block, 0, st>>>((const TI*)vol, (TO*)out, win_tab, C, D, H, W, rd, rh, rw)
  if (in_dtype == B200_DT_F16 && out_dtype == B200_DT_F16) LG(__half, __half);
  else if (in_dtype == B200_DT_F16 && out_dtype == B200_DT_F32) LG(__half, float);
  else if (in_dtype == B200_DT_F32 && out_dtype == B200_DT_F16) LG(float, __half);
  else if (in_dtype == B200_DT_F32 && out_dtype == B200_DT_F32) LG(float, float);
  else return set_err(B200_ERR_INVALID, "sw_gather: bad dtype");
#undef LG
  B200_LAUNCH_CHECK("sw_gather_kernel");
  return B200_OK;
}
