// Windowed multi-head self-attention on Hopper wgmma tensor cores (SURVEY.md §8 row a13).
//
// Reference: WindowAttention.forward (monai/networks/nets/swin_unetr.py:509-532): per window of n <= 343 tokens and head
// (head_dim 16):  softmax(q k^T * scale + relative_position_bias[:n,:n] + shift_mask) v.
//
// One persistent CTA per SM works on tiles = (window, head, 128-query row tile); two consumer warpgroups take 64 query rows
// each and walk the keys in blocks of 32 (flash-attention style, online softmax):
//   S[64 x 32] = Q K^T                          1 wgmma (SS form, K = 16 = the whole head)
//              + I[64 x 64] * B'                4 wgmma (A = the identity rows of the warpgroup, resident in shared memory)
// where B'[i][j] = log2(e) * (bias[i][j] + mask[i][j]) is an fp16 B operand that stays RESIDENT in shared memory: it depends
// on (head, row tile, mask type) only, so tiles are scheduled (mask type, head, row tile)-major and a CTA reloads it a
// handful of times per launch.  Adding the bias with the tensor core (1.0 * fp16 value into the fp32 accumulator: exact)
// removes the per-element table lookup and mask test.  Padded keys carry B' = -30000 (P = 0).  Scores are in log2 units:
// the caller folds scale * log2(e) into the q rows of the qkv projection.
//   softmax: running row maximum m and row sum l in registers; P = 2^(S - m) rounded to fp16 -- the S accumulator fragment
//            of a 32-key block is, packed to fp16 pairs, the register A operand of two K = 16 steps of
//   O[64 x 16] += P V                           2 wgmma (RS form), V read in place as an MN-major B operand (NC8 rows are
//            16-byte vectors of 8 dims); l sums the same fp16-rounded P values the MMA consumes;
//   epilogue: O / l -> fp16 NC8.
// Q, K, V tiles are 1-D bulk copies of NC8 rows (contiguous per 8-channel chunk); the producer runs up to two tiles ahead.
//
// Warp roles (384 threads): warp 0 = copy producer, warps 4-7 / 8-11 = the two consumer warpgroups.
#include "common.cuh"
#include "tc90.cuh"
#include "../../include/monai_b200.h"

namespace b200 {

constexpr int kAtNPadMax = 352;                       // keys per window, padded (n <= 343 -> 352)
constexpr int kAtKChunk = kAtNPadMax * 16;            // bytes of one 8-dim chunk of K / V in shared memory
constexpr int kAtBiasBytes = 16 * kAtNPadMax * 16;    // 16 chunks of 8 query rows
constexpr int kAtIdBytes = 16 * 2048;                 // identity operand image: [k chunk of 8][128 rows][16 B]
constexpr int kAtQBytes = 2 * 2048, kAtKBytes = 2 * kAtKChunk, kAtVBytes = 2 * kAtKChunk;   // one buffer of each (two of each are kept)
constexpr int kAtSmem = kAtBiasBytes + kAtIdBytes + 2 * (kAtQBytes + kAtKBytes + kAtVBytes) + 2 * 2 * tc::kStageFloats * 4 + 256 + 128;
constexpr float kAtPadBias = -30000.f;

struct AttnTcParams {
  const __half* qkv; __half* out; const __half* bias; const int32_t* sched;
  int N, C8, heads, nW, n, n_pad, nrt, ntypes;
};

struct AttnTile { int ty, h, rt, b, w; };

// flattened tile index -> (mask type, head, row tile, batch item, window); order: type, (head, row tile), batch, window
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
  const long long per = (long long)c * p.N;
  const int hr = (int)(f / per);
  const int l2 = (int)(f % per);
  t.h = hr / p.nrt; t.rt = hr % p.nrt;
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

constexpr int kAtThreads = 384;

template <int NPAD>
__global__ void __launch_bounds__(kAtThreads, 1) window_attention_tc_kernel(AttnTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = tc::align_smem128(smem_raw);   // keeps the shared address space (LDS/STS, not generic LD/ST)
  uint8_t* s_bias = smem;
  uint8_t* s_id = s_bias + kAtBiasBytes;              // identity operand image
  uint8_t* s_q = s_id + kAtIdBytes;                   // [2 buffers][2 chunks][128 rows][16 B]
  uint8_t* s_k = s_q + 2 * kAtQBytes;                 // [2 buffers][2 chunks][n_pad keys][16 B]
  uint8_t* s_v = s_k + 2 * kAtKBytes;                 // [2 buffers][2 chunks: V dims 0-7, 8-15][n_pad keys][16 B]
  float* s_stage = reinterpret_cast<float*>(s_v + 2 * kAtVBytes);   // [2 warpgroups][2][kStageFloats]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stage + 2 * 2 * tc::kStageFloats);
  uint64_t* qk_full = bars + 0;     // [2]  Q / K (+ bias) of a tile have landed in buffer b
  uint64_t* qk_empty = bars + 2;    // [2]  the S MMAs that read buffer b are done (one arrival per consumer warpgroup)
  uint64_t* v_full = bars + 4;      // [2]
  uint64_t* v_empty = bars + 6;     // [2]  the PV MMAs that read V buffer b are done

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  // NPAD (keys per window, padded to a multiple of 32) is a template parameter: the key loop has a fixed trip count
  constexpr int n_pad = NPAD;
  const int n = p.n;
  const long long T = (long long)p.nW * n;
  const long long total = (long long)p.N * p.nW * p.heads * p.nrt;
  const long long lo = total * blockIdx.x / gridDim.x, hi = total * (blockIdx.x + 1) / gridDim.x;

  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&qk_full[i], 1); tc::mbar_init(&qk_empty[i], 2); tc::mbar_init(&v_full[i], 1); tc::mbar_init(&v_empty[i], 2);
    }
    tc::fence_barrier_init();
  }
  // zero the identity image and Q / K / V (rows the bulk copies never write must be finite)
  {
    const uint4 z = make_uint4(0, 0, 0, 0);
    uint4* zq = reinterpret_cast<uint4*>(s_id);
    const int nz = (kAtIdBytes + 2 * kAtQBytes + 2 * kAtKBytes + 2 * kAtVBytes) / 16;
    for (int i = threadIdx.x; i < nz; i += blockDim.x) zq[i] = z;
  }
  __syncthreads();
  {
    __half* id = reinterpret_cast<__half*>(s_id);   // [k chunk of 8][row][8]: element (row r, k = r) = 1
    for (int r = threadIdx.x; r < 128; r += blockDim.x) id[((r >> 3) * 128 + r) * 8 + (r & 7)] = __float2half_rn(1.f);
  }
  tc::fence_proxy_async();
  __syncthreads();

  if (warp == 0) {
    // ===================== copy producer: runs up to two tiles ahead of the MMAs =====================
    if (lane == 0) {
      int last_combo = -1;
      int it = 0;
      for (long long f = lo; f < hi; ++f, ++it) {
        const AttnTile t = attn_decode(p, f);
        const int combo = (t.ty * p.heads + t.h) * p.nrt + t.rt;
        const int rows = min(128, n - t.rt * 128);
        const int b = it & 1;
        const uint32_t use = (uint32_t)((it >> 1) & 1);
        tc::mbar_wait(&qk_empty[b], use ^ 1u);                  // the S MMAs that read this buffer two tiles ago are done
        uint32_t bias_bytes = 0u;
        if (combo != last_combo) {
          // the bias image is single-buffered: the S MMAs of the PREVIOUS tile (the other Q / K buffer) still read the old one
          if (it > 0) tc::mbar_wait(&qk_empty[b ^ 1], (uint32_t)(((it - 1) >> 1) & 1));
          bias_bytes = (uint32_t)(16 * n_pad * 16);
        }
        tc::mbar_arrive_expect_tx(&qk_full[b], bias_bytes + 2u * rows * 16u + 2u * n * 16u);
        if (bias_bytes) tc::bulk_load(s_bias, p.bias + (long long)combo * (16 * n_pad * 8), bias_bytes, &qk_full[b]);
        last_combo = combo;
        const __half* base = p.qkv + (long long)t.b * (3 * p.C8) * T * 8;
        const long long row0 = (long long)t.w * n;
        for (int c = 0; c < 2; ++c) {
          tc::bulk_load(s_q + b * kAtQBytes + c * 2048, base + ((long long)(2 * t.h + c) * T + row0 + t.rt * 128) * 8, rows * 16, &qk_full[b]);
          tc::bulk_load(s_k + b * kAtKBytes + c * kAtKChunk, base + ((long long)(p.C8 + 2 * t.h + c) * T + row0) * 8, n * 16, &qk_full[b]);
        }
        tc::mbar_wait(&v_empty[b], use ^ 1u);                   // the PV MMAs that read this V buffer two tiles ago are done
        tc::mbar_arrive_expect_tx(&v_full[b], 2u * n * 16u);
        for (int c = 0; c < 2; ++c)
          tc::bulk_load(s_v + b * kAtVBytes + c * kAtKChunk, base + ((long long)(2 * p.C8 + 2 * t.h + c) * T + row0) * 8, n * 16, &v_full[b]);
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    // ===================== consumers: warpgroup g owns query rows 64 g .. 64 g + 63 of every tile =====================
    const int g = (warp >> 2) - 1, wid = warp & 3;
    const uint32_t q_a = tc::smem_u32(s_q), k_a = tc::smem_u32(s_k), v_a = tc::smem_u32(s_v), b_a = tc::smem_u32(s_bias),
                   i_a = tc::smem_u32(s_id);
    float* stage = s_stage + g * 2 * tc::kStageFloats;
    int sl = 0;
    int it = 0;
    for (long long f = lo; f < hi; ++f, ++it) {
      const int b = it & 1;
      const uint32_t use = (uint32_t)((it >> 1) & 1);
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = 0.f;
      float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows 16 wid + lane/4 and + 8 of the warpgroup
      tc::mbar_wait(&qk_full[b], use);
      tc::mbar_wait(&v_full[b], use);
      const uint64_t qd = tc::make_desc_kmajor_noswz(q_a + b * kAtQBytes + g * 1024, 2048, 128);
#pragma unroll 1
      for (int kb = 0; kb < n_pad / 32; ++kb) {
        // ---- S = Q K^T + I B' for 32 keys ----
        float sc[16];
        tc::wg_fence();
        tc::Mma<32>::ss<0>(sc, qd, tc::make_desc_kmajor_noswz(k_a + b * kAtKBytes + kb * 32 * 16, kAtKChunk, 128), 0u);
#pragma unroll
        for (int s4 = 0; s4 < 4; ++s4) {
          const int ks = 4 * g + s4;   // the identity rows of this warpgroup are non-zero in K steps 4g .. 4g+3 only
          const uint64_t id_d = tc::make_desc_kmajor_noswz(i_a + ks * 4096 + g * 1024, 2048, 128);
          const uint64_t bd = tc::make_desc_kmajor_noswz(b_a + (2 * ks) * n_pad * 16 + kb * 32 * 16, n_pad * 16, 128);
          tc::Mma<32>::ss<0>(sc, id_d, bd, 1u);
        }
        tc::wg_commit();
        tc::wg_wait<0>();
        tc::wg_fence_acc<16>(sc);
        // ---- online softmax (the 4 lanes of a quad share a row) ----
        float x0 = sc[0], x1 = sc[2];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          x0 = fmaxf(x0, fmaxf(sc[4 * i], sc[4 * i + 1]));
          x1 = fmaxf(x1, fmaxf(sc[4 * i + 2], sc[4 * i + 3]));
        }
        x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 1)); x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 2));
        x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 1)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 2));
        const float n0 = fmaxf(m0, x0), n1 = fmaxf(m1, x1);
        const float a0 = ex2(m0 - n0), a1 = ex2(m1 - n1);
        m0 = n0; m1 = n1;
        l0 *= a0; l1 *= a1;
#pragma unroll
        for (int i = 0; i < 2; ++i) { o[4 * i] *= a0; o[4 * i + 1] *= a0; o[4 * i + 2] *= a1; o[4 * i + 3] *= a1; }
        uint32_t pa[2][4];
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
          pa[kk][0] = exp2_pack(sc[8 * kk + 0], sc[8 * kk + 1], m0, l0);
          pa[kk][1] = exp2_pack(sc[8 * kk + 2], sc[8 * kk + 3], m1, l1);
          pa[kk][2] = exp2_pack(sc[8 * kk + 4], sc[8 * kk + 5], m0, l0);
          pa[kk][3] = exp2_pack(sc[8 * kk + 6], sc[8 * kk + 7], m1, l1);
        }
        // ---- O += P V (MN-major B: 8 keys x 16 B (8 dims) per core matrix, next 8 keys +128 B (LBO), next 8 dims +chunk (SBO)) ----
        tc::wg_fence();
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
          const uint64_t vd = tc::make_desc_kmajor_noswz(v_a + b * kAtVBytes + (2 * kb + kk) * 256, 128, kAtKChunk);
          tc::Mma<16>::rs<1>(o, pa[kk], vd, 1u);
        }
        tc::wg_commit();
        tc::wg_wait<0>();
        tc::wg_fence_acc<8>(o);
#pragma unroll
        for (int kk = 0; kk < 2; ++kk)
#pragma unroll
          for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(pa[kk][j])::"memory");   // A registers stay live until the wait
      }
      if (wid == 0 && lane == 0) { tc::mbar_arrive(&qk_empty[b]); tc::mbar_arrive(&v_empty[b]); }
      // ---- epilogue: O / l -> fp16 NC8 (one row and 8 dims per thread after the slice exchange) ----
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
      for (int i = 0; i < 2; ++i) { o[4 * i] *= i0; o[4 * i + 1] *= i0; o[4 * i + 2] *= i1; o[4 * i + 3] *= i1; }
      float* buf = stage + (sl & 1) * tc::kStageFloats;
      ++sl;
      tc::wg_stage16<0>(o, buf, wid, lane);
      tc::wg_bar(8 + g);
      float v[8];
      tc::wg_read8(buf, wid, lane, v);
      const AttnTile t = attn_decode(p, f);
      const int r = t.rt * 128 + 64 * g + 32 * (wid & 1) + lane;
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

// B' operand images: [type][head][row tile][16 chunks of 8 query rows][n_pad keys][8] fp16 (see the header comment)
__global__ void attn_bias_pack_kernel(const float* __restrict__ table, const int32_t* __restrict__ region, __half* __restrict__ out,
                                      int heads, int n, int n_pad, int nrt, int ntypes, int ws0, int ws1, int ws2) {
  const long long total = (long long)ntypes * heads * nrt * 16 * n_pad * 8;
  const int s1 = 2 * ws2 - 1, s0 = (2 * ws1 - 1) * s1;
  const int lin_c = (ws0 - 1) * s0 + (ws1 - 1) * s1 + (ws2 - 1);
  constexpr float kLog2e = 1.4426950408889634f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int e = (int)(r % 8); r /= 8;
    const int j = (int)(r % n_pad); r /= n_pad;
    const int c = (int)(r % 16); r /= 16;
    const int rt = (int)(r % nrt); r /= nrt;
    const int h = (int)(r % heads); r /= heads;
    const int ty = (int)r;
    const int ig = rt * 128 + c * 8 + e;
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
  const int n_pad = (n + 31) / 32 * 32, nrt = (n + 127) / 128;
  return (long long)ntypes * heads * nrt * 16 * n_pad * 16;
}

extern "C" int b200_window_attention_tc_pack_bias(const float* table, int heads, int n, int ws0, int ws1, int ws2,
                                                  const int32_t* region_types, int ntypes, void* packed, void* stream) {
  B200_REQUIRE(table && packed, "window_attention_tc_pack_bias: null pointer");
  B200_REQUIRE(attn_tc_shape_ok(heads, n, ntypes) && n <= kAtNPadMax, "window_attention_tc: unsupported shape (n = %d, types = %d)", n, ntypes);
  B200_REQUIRE(ws0 > 0 && ws1 > 0 && ws2 > 0 && n <= ws0 * ws1 * ws2, "window_attention_tc: window of %d tokens exceeds the module window", n);
  B200_REQUIRE(ntypes == 1 || region_types, "window_attention_tc_pack_bias: several mask types need their region rows");
  const int n_pad = (n + 31) / 32 * 32, nrt = (n + 127) / 128;
  const long long total = (long long)ntypes * heads * nrt * 16 * n_pad * 8;
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
  p.N = N; p.C8 = C / 8; p.heads = heads; p.nW = nW; p.n = n; p.n_pad = (n + 31) / 32 * 32; p.nrt = (n + 127) / 128; p.ntypes = ntypes;
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
