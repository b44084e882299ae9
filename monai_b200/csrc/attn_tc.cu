// Windowed multi-head self-attention on Hopper wgmma tensor cores (SURVEY.md §8 row a13).
//
// Reference: WindowAttention.forward (monai/networks/nets/swin_unetr.py:509-532): per window of n <= 343 tokens and head
// (head_dim 16):  softmax(q k^T * scale + relative_position_bias[:n,:n] + shift_mask) v.
//
// With head_dim 16 the work is the n^2 exponentials (MUFU), not the MMAs, so the kernel is built to keep MUFU busy.
// One persistent CTA per SM works on tiles = (window, head, 192-query row tile); three consumer warpgroups take 64 query rows
// each and walk the keys in chunks of 64 (the last one may be 32; flash-attention style, online softmax):
//   S[64 x 64] = B' + Q K^T                     1 wgmma (SS form, K = 16 = the whole head, scale-d = 1)
// where B'[i][j] = log2(e) * (bias[i][j] + mask[i][j]) is loaded from shared memory straight into the accumulator
// registers: the packed image is stored in the accumulator's fragment order (16 fp16 per thread per 32 keys, two 16-byte
// vectors).  It depends on (mask type, head, row tile) only and stays RESIDENT in shared memory; tiles are scheduled
// (mask type, head, window group, row tile, window) so that a CTA reloads it once per group of kAtGroup windows while
// the K / V of those windows are still in L2 from the previous row tile.  Padded keys carry B' = -30000 (P = 0).  Scores
// are in log2 units: the caller folds scale * log2(e) into the q rows of the qkv projection.
//   softmax: running row maximum m (updated once per chunk) and row sum l in registers; P = 2^(S - m) rounded to fp16 --
//            the S accumulator fragment, packed to fp16 pairs, is the register A operand of the K = 16 steps of
//   O[64 x 16] += P V                           2-4 wgmma (RS form), V read in place as an MN-major B operand (NC8 rows
//            are 16-byte vectors of 8 dims); l sums the same fp16-rounded P values the MMA consumes;
//   epilogue: O / l -> fp16 NC8.
// Software pipeline per warpgroup: the S MMA of chunk c+1 is in flight while the exponentials of chunk c run, and the PV
// MMA of chunk c-1 retires only before O is rescaled (S and P are double-buffered in registers; P stays live until its
// MMA retires).  A warp whose 16 query rows are all padding (rows >= n) takes part in the MMAs but issues no
// exponential: its P is zero; a warpgroup whose 64 rows are all padding skips the tile.  Three consumer warpgroups (12
// warps issuing exponentials, against 8 with two) hide the latency of each warp's max / shuffle / wgmma-wait chain.
// Q, K, V tiles are 1-D bulk copies of NC8 rows (contiguous per 8-channel chunk); the producer runs up to two tiles ahead.
//
// Warp roles (512 threads): warp 0 = copy producer (warps 1-3 idle), warps 4-7 / 8-11 / 12-15 = the consumer warpgroups.
// Warpgroup 0 gives its registers to the consumers (setmaxnreg 56 / 152).
#include "common.cuh"
#include "tc90.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

constexpr int kAtNPadMax = 352;                       // keys per window, padded (n <= 343 -> 352)
constexpr int kAtWG = 3;                              // consumer warpgroups, 64 query rows each
constexpr int kAtRows = 64 * kAtWG;                   // query rows per tile
constexpr int kAtCT = 128 * kAtWG;                    // consumer threads
constexpr int kAtKChunk = kAtNPadMax * 16;            // bytes of one 8-dim chunk of K / V in shared memory
constexpr int kAtBiasBytes = kAtNPadMax * kAtCT;      // per 32 keys: every consumer thread x 16 fp16
constexpr int kAtQBytes = 2 * kAtRows * 16, kAtKBytes = 2 * kAtKChunk, kAtVBytes = 2 * kAtKChunk;   // one buffer of each (two of each are kept)
constexpr int kAtSmem = kAtBiasBytes + 2 * (kAtQBytes + kAtKBytes + kAtVBytes) + kAtWG * 2 * tc::kStageFloats * 4 + 256 + 128;
constexpr float kAtPadBias = -30000.f;
// windows per schedule group: the row tiles of a group run back to back on a CTA, so a window's K / V are read from HBM
// about once; 132 CTAs x 8 windows x 22 KB (K and V of one head at n = 343) = 23 MB stays well inside the 50 MB L2,
// and the 135 KB bias image is reloaded (from L2) once per 8 tiles
constexpr int kAtGroup = 8;

struct AttnTcParams {
  const __half* qkv; __half* out; const __half* bias; const int32_t* sched;
  int N, C8, heads, nW, n, n_pad, nrt, ntypes;
};

struct AttnTile { int ty, h, rt, b, w; };

// flattened tile index -> (mask type, head, row tile, batch item, window); order: type, head, group of kAtGroup (batch
// item, window) pairs, row tile, pair within the group
__device__ __forceinline__ AttnTile attn_decode(const AttnTcParams& p, long long f) {
  const int32_t* cnt = p.sched;
  const int32_t* start = p.sched + 8;
  const int32_t* win = p.sched + 16;
  AttnTile t;
  t.ty = 0;
  const long long hr_n = (long long)p.heads * p.nrt;
  for (;;) {
    const long long blk = (long long)cnt[t.ty] * p.N * hr_n;
    if (f < blk || t.ty + 1 >= p.ntypes) break;
    f -= blk; ++t.ty;
  }
  const int c = cnt[t.ty];
  const int per = c * p.N;                              // (batch item, window) pairs of this type
  const long long per_h = (long long)per * p.nrt;
  t.h = (int)(f / per_h);
  int r = (int)(f % per_h);
  const int full = per / kAtGroup * kAtGroup;           // pairs in whole groups; the last group may be smaller
  int l2;
  if (r < full * p.nrt) {
    const int grp = r / (kAtGroup * p.nrt);
    r %= kAtGroup * p.nrt;
    t.rt = r / kAtGroup;
    l2 = grp * kAtGroup + r % kAtGroup;
  } else {
    r -= full * p.nrt;
    const int rem = per - full;
    t.rt = r / rem;
    l2 = full + r % rem;
  }
  t.b = l2 / c;
  t.w = win[start[t.ty] + l2 % c];
  return t;
}

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 2^(a - m), 2^(b - m) as packed fp16; `sum` accumulates the two ROUNDED values (what the PV MMA multiplies)
__device__ __forceinline__ uint32_t exp2_pack(float a, float b, float m, float& sum) {
  const __half2 h = __floats2half2_rn(ex2(a - m), ex2(b - m));
  const float2 r = __half22float2(h);
  sum += r.x + r.y;
  return *reinterpret_cast<const uint32_t*>(&h);
}

// 8 fp16 of the packed bias -> 8 accumulator registers
__device__ __forceinline__ void bias_to_acc(const uint8_t* src, float* d) {
  const uint4 v = *reinterpret_cast<const uint4*>(src);
  const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = __half22float2(h[j]);
    d[2 * j] = f.x; d[2 * j + 1] = f.y;
  }
}

constexpr int kAtThreads = 128 * (kAtWG + 1);

template <int NPAD>
__global__ void __launch_bounds__(kAtThreads, 1) window_attention_tc_kernel(AttnTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = tc::align_smem128(smem_raw);   // keeps the shared address space (LDS/STS, not generic LD/ST)
  uint8_t* s_bias = smem;                             // [32-key block][2 halves][consumer thread][8 fp16]
  uint8_t* s_q = s_bias + kAtBiasBytes;               // [2 buffers][2 chunks][kAtRows rows][16 B]
  uint8_t* s_k = s_q + 2 * kAtQBytes;                 // [2 buffers][2 chunks][n_pad keys][16 B]
  uint8_t* s_v = s_k + 2 * kAtKBytes;                 // [2 buffers][2 chunks: V dims 0-7, 8-15][n_pad keys][16 B]
  float* s_stage = reinterpret_cast<float*>(s_v + 2 * kAtVBytes);   // [kAtWG warpgroups][2][kStageFloats]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stage + kAtWG * 2 * tc::kStageFloats);
  uint64_t* qk_full = bars + 0;     // [2]  Q / K (+ bias) of a tile have landed in buffer b
  uint64_t* qk_empty = bars + 2;    // [2]  the S MMAs (and bias loads) that read buffer b are done (one arrival per consumer warpgroup)
  uint64_t* v_full = bars + 4;      // [2]
  uint64_t* v_empty = bars + 6;     // [2]  the PV MMAs that read V buffer b are done

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  // NPAD (keys per window, padded to a multiple of 32) is a template parameter: the key loop is fully unrolled
  constexpr int n_pad = NPAD;
  constexpr int NB = NPAD / 32;          // 32-key blocks
  constexpr int NC = (NB + 1) / 2;       // 64-key chunks (the last one has 32 keys when NB is odd)
  const int n = p.n;
  const long long T = (long long)p.nW * n;
  const long long total = (long long)p.N * p.nW * p.heads * p.nrt;
  const long long lo = total * blockIdx.x / gridDim.x, hi = total * (blockIdx.x + 1) / gridDim.x;

  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&qk_full[i], 1); tc::mbar_init(&qk_empty[i], kAtWG); tc::mbar_init(&v_full[i], 1); tc::mbar_init(&v_empty[i], kAtWG);
    }
    tc::fence_barrier_init();
  }
  // zero Q / K / V (rows the bulk copies never write must be finite)
  {
    const uint4 z = make_uint4(0, 0, 0, 0);
    uint4* zq = reinterpret_cast<uint4*>(s_q);
    const int nz = (2 * kAtQBytes + 2 * kAtKBytes + 2 * kAtVBytes) / 16;
    for (int i = threadIdx.x; i < nz; i += blockDim.x) zq[i] = z;
  }
  tc::fence_proxy_async();
  __syncthreads();

  if (warp < 4) {
    // the copy producer needs few registers: warpgroup 0 hands them to the consumers, whose software pipeline keeps two S
    // and two P fragments live (with the launch's 128 per thread ptxas would serialise the wgmma)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 56;\n" ::: "memory");
    // ===================== copy producer: runs up to two tiles ahead of the MMAs =====================
    if (warp == 0 && lane == 0) {
      int last_combo = -1;
      int it = 0;
      for (long long f = lo; f < hi; ++f, ++it) {
        const AttnTile t = attn_decode(p, f);
        const int combo = (t.ty * p.heads + t.h) * p.nrt + t.rt;
        const int rows = min(kAtRows, n - t.rt * kAtRows);
        const int b = it & 1;
        const uint32_t use = (uint32_t)((it >> 1) & 1);
        tc::mbar_wait(&qk_empty[b], use ^ 1u);                  // the S MMAs that read this buffer two tiles ago are done
        uint32_t bias_bytes = 0u;
        if (combo != last_combo) {
          // the bias image is single-buffered: the consumers of the PREVIOUS tile (the other Q / K buffer) still read the old one
          if (it > 0) tc::mbar_wait(&qk_empty[b ^ 1], (uint32_t)(((it - 1) >> 1) & 1));
          bias_bytes = (uint32_t)(n_pad * kAtCT);
        }
        tc::mbar_arrive_expect_tx(&qk_full[b], bias_bytes + 2u * rows * 16u + 2u * n * 16u);
        if (bias_bytes) tc::bulk_load(s_bias, p.bias + (long long)combo * (n_pad * kAtCT / 2), bias_bytes, &qk_full[b]);
        last_combo = combo;
        const __half* base = p.qkv + (long long)t.b * (3 * p.C8) * T * 8;
        const long long row0 = (long long)t.w * n;
        for (int c = 0; c < 2; ++c) {
          tc::bulk_load(s_q + b * kAtQBytes + c * kAtRows * 16, base + ((long long)(2 * t.h + c) * T + row0 + t.rt * kAtRows) * 8, rows * 16, &qk_full[b]);
          tc::bulk_load(s_k + b * kAtKBytes + c * kAtKChunk, base + ((long long)(p.C8 + 2 * t.h + c) * T + row0) * 8, n * 16, &qk_full[b]);
        }
        tc::mbar_wait(&v_empty[b], use ^ 1u);                   // the PV MMAs that read this V buffer two tiles ago are done
        tc::mbar_arrive_expect_tx(&v_full[b], 2u * n * 16u);
        for (int c = 0; c < 2; ++c)
          tc::bulk_load(s_v + b * kAtVBytes + c * kAtKChunk, base + ((long long)(2 * p.C8 + 2 * t.h + c) * T + row0) * 8, n * 16, &v_full[b]);
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 152;\n" ::: "memory");
    // ===================== consumers: warpgroup g owns query rows 64 g .. 64 g + 63 of every tile =====================
    const int g = (warp >> 2) - 1, wid = warp & 3;
    const int ct = threadIdx.x - 128;   // consumer thread: its slot in the packed bias
    const uint32_t q_a = tc::smem_u32(s_q), k_a = tc::smem_u32(s_k), v_a = tc::smem_u32(s_v);
    float* stage = s_stage + g * 2 * tc::kStageFloats;
    int sl = 0;
    int it = 0;
    for (long long f = lo; f < hi; ++f, ++it) {
      const int b = it & 1;
      const uint32_t use = (uint32_t)((it >> 1) & 1);
      const AttnTile t = attn_decode(p, f);
      // all 16 rows of this warp are padding: no exponentials, P = 0 (the warp still takes part in the wgmma)
      const bool dead = t.rt * kAtRows + 64 * g + 16 * wid >= n;
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = 0.f;
      float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows 16 wid + lane/4 and + 8 of the warpgroup
      float s[2][32];          // S of chunks c (softmax) and c + 1 (MMA in flight)
      uint32_t pa[2][4][4];    // P of chunks c (being built) and c - 1 (PV MMA in flight)
      tc::mbar_wait(&qk_full[b], use);
      tc::mbar_wait(&v_full[b], use);
      if (t.rt * kAtRows + 64 * g >= n) {
        // all 64 rows of this warpgroup are padding (the last row tile of a small window): nothing to compute
        if (wid == 0 && lane == 0) { tc::mbar_arrive(&qk_empty[b]); tc::mbar_arrive(&v_empty[b]); }
        continue;
      }
      const uint64_t qd = tc::make_desc_kmajor_noswz(q_a + b * kAtQBytes + g * 1024, kAtRows * 16, 128);

      // S(c) = B' + Q K^T for the keys of chunk c, committed as one wgmma group
      auto issue_s = [&](auto cc) {
        constexpr int c = decltype(cc)::value;
        constexpr int nb = (2 * c + 1 < NB) ? 2 : 1;
        float* sc = s[c & 1];
#pragma unroll
        for (int k2 = 0; k2 < nb; ++k2)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) bias_to_acc(s_bias + ((2 * c + k2) * 2 + hh) * (kAtCT * 16) + ct * 16, sc + 16 * k2 + 8 * hh);
        tc::wg_fence();
        const uint64_t kd = tc::make_desc_kmajor_noswz(k_a + b * kAtKBytes + c * 64 * 16, kAtKChunk, 128);
        if constexpr (nb == 2) tc::Mma<64>::ss<0>(sc, qd, kd, 1u);
        else tc::Mma<32>::ss<0>(sc, qd, kd, 1u);
        tc::wg_commit();
      };

      issue_s(std::integral_constant<int, 0>{});
      tc::static_for<0, NC>([&](auto cc) {
        constexpr int c = decltype(cc)::value;
        constexpr int nb = (2 * c + 1 < NB) ? 2 : 1;
        constexpr int nv = 16 * nb;   // S registers of this chunk
        // pending groups here: S(c), PV(c-1); after the next issue also S(c+1)
        if constexpr (c + 1 < NC) {
          issue_s(std::integral_constant<int, c + 1>{});
          if constexpr (c == 0) tc::wg_wait<1>(); else tc::wg_wait<2>();
        } else {
          if constexpr (c == 0) tc::wg_wait<0>(); else tc::wg_wait<1>();
        }
        float* sc = s[c & 1];
        tc::wg_fence_acc<nv>(sc);
        // ---- online softmax over the chunk (the 4 lanes of a quad share a row) ----
        float a0 = 1.f, a1 = 1.f, ps0 = 0.f, ps1 = 0.f;
        if (!dead) {
          float x0 = sc[0], x1 = sc[2];
#pragma unroll
          for (int i = 0; i < nv / 4; ++i) {
            x0 = fmaxf(x0, fmaxf(sc[4 * i], sc[4 * i + 1]));
            x1 = fmaxf(x1, fmaxf(sc[4 * i + 2], sc[4 * i + 3]));
          }
          x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 1)); x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 2));
          x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 1)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 2));
          const float n0 = fmaxf(m0, x0), n1 = fmaxf(m1, x1);
          a0 = ex2(m0 - n0); a1 = ex2(m1 - n1);
          m0 = n0; m1 = n1;
#pragma unroll
          for (int kk = 0; kk < 2 * nb; ++kk) {
            pa[c & 1][kk][0] = exp2_pack(sc[8 * kk + 0], sc[8 * kk + 1], m0, ps0);
            pa[c & 1][kk][1] = exp2_pack(sc[8 * kk + 2], sc[8 * kk + 3], m1, ps1);
            pa[c & 1][kk][2] = exp2_pack(sc[8 * kk + 4], sc[8 * kk + 5], m0, ps0);
            pa[c & 1][kk][3] = exp2_pack(sc[8 * kk + 6], sc[8 * kk + 7], m1, ps1);
          }
        } else {
#pragma unroll
          for (int kk = 0; kk < 2 * nb; ++kk)
#pragma unroll
            for (int j = 0; j < 4; ++j) pa[c & 1][kk][j] = 0u;
        }
        // ---- retire PV(c-1), then rescale O and l ----
        if constexpr (c > 0) {
          if constexpr (c + 1 < NC) tc::wg_wait<1>(); else tc::wg_wait<0>();
          tc::wg_fence_acc<8>(o);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(pa[(c - 1) & 1][kk][j])::"memory");   // A registers stay live until the wait
        }
        l0 = l0 * a0 + ps0; l1 = l1 * a1 + ps1;
#pragma unroll
        for (int i = 0; i < 2; ++i) { o[4 * i] *= a0; o[4 * i + 1] *= a0; o[4 * i + 2] *= a1; o[4 * i + 3] *= a1; }
        // ---- O += P V (MN-major B: 8 keys x 16 B (8 dims) per core matrix, next 8 keys +128 B (LBO), next 8 dims +chunk (SBO)) ----
        tc::wg_fence();
#pragma unroll
        for (int kk = 0; kk < 2 * nb; ++kk) {
          const uint64_t vd = tc::make_desc_kmajor_noswz(v_a + b * kAtVBytes + (4 * c + kk) * 256, 128, kAtKChunk);
          tc::Mma<16>::rs<1>(o, pa[c & 1][kk], vd, 1u);
        }
        tc::wg_commit();
      });
      tc::wg_wait<0>();
      tc::wg_fence_acc<8>(o);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(pa[(NC - 1) & 1][kk][j])::"memory");
      if (wid == 0 && lane == 0) { tc::mbar_arrive(&qk_empty[b]); tc::mbar_arrive(&v_empty[b]); }
      // ---- epilogue: O / l -> fp16 NC8 (one row and 8 dims per thread after the slice exchange) ----
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      const float i0 = dead ? 0.f : 1.f / l0, i1 = dead ? 0.f : 1.f / l1;
#pragma unroll
      for (int i = 0; i < 2; ++i) { o[4 * i] *= i0; o[4 * i + 1] *= i0; o[4 * i + 2] *= i1; o[4 * i + 3] *= i1; }
      float* buf = stage + (sl & 1) * tc::kStageFloats;
      ++sl;
      tc::wg_stage16<0>(o, buf, wid, lane);
      tc::wg_bar(8 + g);
      float v[8];
      tc::wg_read8(buf, wid, lane, v);
      const int r = t.rt * kAtRows + 64 * g + 32 * (wid & 1) + lane;
      if (r < n) {
        const int dt = wid >> 1;
        __half* ob = p.out + (long long)t.b * p.C8 * T * 8 + ((long long)t.w * n + r) * 8;
        uint4 hv;
        __half2* hp = reinterpret_cast<__half2*>(&hv);
#pragma unroll
        for (int j = 0; j < 4; ++j) hp[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
        *reinterpret_cast<uint4*>(ob + (long long)(2 * t.h + dt) * T * 8) = hv;
      }
    }
  }
}

// B' images in the S accumulator's fragment order: [type][head][row tile][32-key block][2 halves][kAtCT consumer threads][8]
// fp16.  Consumer thread t = 128 g + 32 w + l (g < kAtWG) holds, for the 8-key column block i of a 32-key block, the values
// (4 i + e) of the m64n32 accumulator: row 64 g + 16 w + l/4 (+ 8 for e >= 2), key 8 i + 2 (l % 4) + (e & 1); half hh
// holds column blocks 2 hh and 2 hh + 1.
__global__ void attn_bias_pack_kernel(const float* __restrict__ table, const int32_t* __restrict__ region, __half* __restrict__ out,
                                      int heads, int n, int n_pad, int nrt, int ntypes, int ws0, int ws1, int ws2) {
  const long long total = (long long)ntypes * heads * nrt * n_pad * (kAtCT / 2);
  const int s1 = 2 * ws2 - 1, s0 = (2 * ws1 - 1) * s1;
  const int lin_c = (ws0 - 1) * s0 + (ws1 - 1) * s1 + (ws2 - 1);
  const int nb = n_pad / 32;
  constexpr float kLog2e = 1.4426950408889634f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int e8 = (int)(r % 8); r /= 8;
    const int ct = (int)(r % kAtCT); r /= kAtCT;
    const int hh = (int)(r % 2); r /= 2;
    const int kb = (int)(r % nb); r /= nb;
    const int rt = (int)(r % nrt); r /= nrt;
    const int h = (int)(r % heads); r /= heads;
    const int ty = (int)r;
    const int v16 = 8 * hh + e8, cb = v16 >> 2, e = v16 & 3, l = ct & 31;
    const int ig = rt * kAtRows + (ct >> 7) * 64 + ((ct >> 5) & 3) * 16 + (l >> 2) + (e >= 2 ? 8 : 0);
    const int j = kb * 32 + cb * 8 + 2 * (l & 3) + (e & 1);
    float v;
    if (j >= n) v = kAtPadBias;
    else if (ig >= n) v = 0.f;
    else {
      // tokens keep their coordinates in the MODULE window (relative_position_index[:n, :n], swin_unetr.py:514-516)
      const int li = (ig / (ws1 * ws2)) * s0 + ((ig / ws2) % ws1) * s1 + ig % ws2;
      const int lj = (j / (ws1 * ws2)) * s0 + ((j / ws2) % ws1) * s1 + j % ws2;
      v = table[(long long)(li - lj + lin_c) * heads + h] * kLog2e;
      if (region && region[(long long)ty * n + ig] != region[(long long)ty * n + j]) v += -100.f * kLog2e;   // compute_mask, swin_unetr.py:779-816
    }
    out[i] = __float2half_rn(v);
  }
}

}  // namespace b200

using namespace b200;

static bool attn_tc_shape_ok(int heads, int n, int ntypes) {
  return heads > 0 && n > 0 && n <= kAtNPadMax && ntypes >= 1 && ntypes <= 8;
}

extern "C" long long b200_window_attention_tc_bias_bytes(int heads, int n, int ntypes) {
  if (!attn_tc_shape_ok(heads, n, ntypes) || n > kAtNPadMax) return -1;
  const int n_pad = (n + 31) / 32 * 32, nrt = (n + kAtRows - 1) / kAtRows;
  return (long long)ntypes * heads * nrt * n_pad * kAtCT;
}

extern "C" int b200_window_attention_tc_pack_bias(const float* table, int heads, int n, int ws0, int ws1, int ws2,
                                                  const int32_t* region_types, int ntypes, void* packed, void* stream) {
  B200_REQUIRE(table && packed, "window_attention_tc_pack_bias: null pointer");
  B200_REQUIRE(attn_tc_shape_ok(heads, n, ntypes) && n <= kAtNPadMax, "window_attention_tc: unsupported shape (n = %d, types = %d)", n, ntypes);
  B200_REQUIRE(ws0 > 0 && ws1 > 0 && ws2 > 0 && n <= ws0 * ws1 * ws2, "window_attention_tc: window of %d tokens exceeds the module window", n);
  B200_REQUIRE(ntypes == 1 || region_types, "window_attention_tc_pack_bias: several mask types need their region rows");
  const int n_pad = (n + 31) / 32 * 32, nrt = (n + kAtRows - 1) / kAtRows;
  const long long total = (long long)ntypes * heads * nrt * n_pad * (kAtCT / 2);
  const int blocks = (int)std::min<long long>((total + 255) / 256, 8192);
  attn_bias_pack_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(table, region_types, (__half*)packed, heads, n, n_pad, nrt, ntypes, ws0, ws1, ws2);
  B200_LAUNCH_CHECK("attn_bias_pack_kernel");
  return B200_OK;
}

extern "C" int b200_window_attention_tc(const void* qkv, int N, int C, int heads, int nW, int n, const void* packed_bias,
                                        const int32_t* sched, int ntypes, void* out, void* stream) {
  B200_REQUIRE(qkv && out && packed_bias && sched, "window_attention_tc: null pointer");
  B200_REQUIRE(N > 0 && nW > 0, "window_attention_tc: empty problem");
  B200_REQUIRE(C == heads * 16, "window_attention_tc: head_dim must be 16 (C = %d, heads = %d)", C, heads);
  B200_REQUIRE(attn_tc_shape_ok(heads, n, ntypes) && n <= kAtNPadMax, "window_attention_tc: unsupported shape (n = %d, types = %d)", n, ntypes);
  AttnTcParams p;
  p.qkv = (const __half*)qkv; p.out = (__half*)out; p.bias = (const __half*)packed_bias; p.sched = sched;
  p.N = N; p.C8 = C / 8; p.heads = heads; p.nW = nW; p.n = n; p.n_pad = (n + 31) / 32 * 32; p.nrt = (n + kAtRows - 1) / kAtRows; p.ntypes = ntypes;
  const long long total = (long long)N * nW * heads * p.nrt;
  dim3 grid((unsigned)std::min<long long>(total, num_sms()));
  void (*kern)(AttnTcParams) = nullptr;
  switch (p.n_pad) {
#define B200_ATTN_CASE(NP) case NP: kern = window_attention_tc_kernel<NP>; break;
    B200_ATTN_CASE(32) B200_ATTN_CASE(64) B200_ATTN_CASE(96) B200_ATTN_CASE(128) B200_ATTN_CASE(160) B200_ATTN_CASE(192)
    B200_ATTN_CASE(224) B200_ATTN_CASE(256) B200_ATTN_CASE(288) B200_ATTN_CASE(320) B200_ATTN_CASE(352)
#undef B200_ATTN_CASE
  }
  B200_REQUIRE(kern != nullptr, "window_attention_tc: no kernel for %d padded keys", p.n_pad);
  // per-device attribute: set on every call (cheap), so a second GPU in the same process works
  B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kAtSmem));
  kern<<<grid, kAtThreads, kAtSmem, (cudaStream_t)stream>>>(p);
  B200_LAUNCH_CHECK("window_attention_tc_kernel");
  return B200_OK;
}
