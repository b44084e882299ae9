// 3x3x3 stride-1 implicit-GEMM convolution on Hopper wgmma tensor cores (SURVEY.md §8 rows a8, a14).
//
// Replaces the nn.Conv3d inside UnetResBlock / Convolution (monai/networks/blocks/dynunet_block.py:25-111,
// monai/networks/blocks/convolutions.py:131-152) for kernel 3, stride 1, zero padding 1.
//
// Data layout in HBM ("NC8"): activations are fp16 [N][C/8][D][H][W][8]: eight channels of one voxel are 16
// contiguous bytes and voxels run along W.  A shared-memory image of a (D,H,W) box of one 8-channel chunk is
// then exactly a column of wgmma "core matrices" (8 rows x 16 B) for the K-major / no-swizzle operand layout:
//   rows = 8 consecutive voxels along W, K = 8 channels.
//
// GEMM view: M = 128 output voxels (one 16(H) x 8(W) patch of one D-plane), N = NT output channels, K = 27*Cin.
// Per K-slice of 16 input channels the CTA stages ONE halo tile (BD+2) x 18 x 10 voxels with a single 5-D TMA
// box load (out-of-bounds => zero fill == the convolution's zero padding) and issues the taps as wgmma instructions
// whose A descriptors merely start at a shifted voxel of that tile (start += ((plane*18+kh)*10+kw)*16 B,
// SBO = 10*16 B between the 16 row groups, LBO = chunk stride).  Weights are pre-packed into the exact B-operand
// image and arrive by 1-D bulk copies (one (kh, kw) tap image per ring stage).  fp32 accumulators (BD planes x NT
// columns) live in the registers of two consumer warpgroups, 64 rows each; their epilogue adds bias, reduces InstanceNorm
// partial sums and stores fp16 NC8.  The kernel is persistent: one CTA per SM walks the tile list (see the kernel).
//
// Depth blocking: a tile holds BD output planes, so each staged halo tile (BD + 2 input planes) serves the 3 x BD
// (plane, kd) pairs of a (kh, kw) tap -- the halo is read from HBM once per BD planes instead of once per plane.
//
// Warp roles (384 threads): warp 0 = TMA producer, warps 4-11 = two consumer warpgroups (MMA + epilogue); with the
// fused input normalisation (NORM, see the kernel) warps 1-3 rewrite each staged halo tile in place.
#include "common.cuh"
#include "tc90.cuh"
#include "conv_epi.cuh"
#include "../../include/monai_b200.h"
#include <mutex>
#include <type_traits>
#include <cstdlib>

namespace b200 {

EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  });
  return fn;
}

// ----------------------------------------------------------------------------------------------------------
// NC8 pack / unpack
// ----------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) pack_nc8_kernel(const T* __restrict__ x, __half* __restrict__ y, int C, long long S,
                                                       int Ctot, int c_off) {
  const int chunk = blockIdx.y, n = blockIdx.z;
  const T* xs = x + ((long long)n * C + chunk * 8) * S;
  __half* yd = y + (((long long)n * (Ctot / 8) + c_off / 8 + chunk) * S) * 8;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (long long)gridDim.x * blockDim.x) {
    __align__(16) __half v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = __float2half_rn(io<T>::ld(xs + (long long)j * S + s));
    *reinterpret_cast<uint4*>(yd + s * 8) = *reinterpret_cast<const uint4*>(v);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) unpack_nc8_kernel(const __half* __restrict__ x, T* __restrict__ y, int C, long long S,
                                                         int Ctot, int c_off) {
  const int chunk = blockIdx.y, n = blockIdx.z;
  const __half* xs = x + (((long long)n * (Ctot / 8) + c_off / 8 + chunk) * S) * 8;
  T* yd = y + ((long long)n * C + chunk * 8) * S;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (long long)gridDim.x * blockDim.x) {
    __align__(16) __half v[8];
    *reinterpret_cast<uint4*>(v) = *reinterpret_cast<const uint4*>(xs + s * 8);
#pragma unroll
    for (int j = 0; j < 8; ++j) io<T>::st(yd + (long long)j * S + s, __half2float(v[j]));
  }
}

// ----------------------------------------------------------------------------------------------------------
// weight packing: Conv3d weight [Cout][Cin][27] fp32 -> [nt][kc][kh][kw][khalf][kd = 2,1,0][NT/8][8 cout][8 k] fp16
// (one K-major B image of 3*NT rows per (kh, kw): rows of kd = 2 first, so a kd range is a contiguous row range)
// ----------------------------------------------------------------------------------------------------------
__host__ __device__ inline int conv_tc_nt(int Cout) {
  if (Cout <= 128) return Cout;
  // very wide layers sit at the bottom of the networks (a few voxels per item): narrow N tiles there, so that enough CTAs
  // stream the weights in parallel (the layer is bound by weight bandwidth per SM, not by the tensor pipe)
  if (Cout >= 384 && Cout % 64 == 0) return 64;
  for (int nt = 128; nt >= 16; nt -= 16)
    if (Cout % nt == 0) return nt;
  return 16;
}

__global__ void conv_tc_pack_weight_kernel(const float* __restrict__ w, __half* __restrict__ out, int Cin, int Cout, int NT) {
  const long long total = (long long)Cout * Cin * 27;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int kk = (int)(r % 8); r /= 8;
    const int row = (int)(r % 8); r /= 8;
    const int g = (int)(r % (NT / 8)); r /= (NT / 8);
    const int kd = 2 - (int)(r % 3); r /= 3;
    const int khalf = (int)(r % 2); r /= 2;
    const int t9 = (int)(r % 9); r /= 9;    // kh*3 + kw
    const int kc = (int)(r % (Cin / 16)); r /= (Cin / 16);
    const int nt = (int)r;
    const int cout = nt * NT + g * 8 + row;
    const int cin = kc * 16 + khalf * 8 + kk;
    const int tap = kd * 9 + t9;
    out[i] = __float2half_rn(w[((long long)cout * Cin + cin) * 27 + tap]);
  }
}

// ----------------------------------------------------------------------------------------------------------
// the convolution kernel
// ----------------------------------------------------------------------------------------------------------
constexpr int kHH = kTH + 2, kHW = kTW + 2;      // halo patch (kTH x kTW output patch: conv_epi.cuh)

template <int NT, int BD, bool RES = false>
struct ConvTcCfg {
  static constexpr int kPlanes = BD + 2;
  static constexpr int kChunkBytes = kPlanes * kHH * kHW * 16;   // one 8-channel chunk of the halo tile
  static constexpr int kABytes = 2 * kChunkBytes;                // 16 input channels
  static constexpr int kBTapBytes = 3 * NT * 32;                 // one (kh, kw): the three kd taps stacked along N, 3*NT x 16 fp16
  // weight ring: one (kh, kw) tap image per stage, ~44 KB in flight so a bulk copy has > 1 us to land before its
  // MMAs are due
  static constexpr int kSB = (45056 / kBTapBytes) > 9 ? 9 : ((45056 / kBTapBytes) < 3 ? 3 : (45056 / kBTapBytes));
  static constexpr int kSA = 4;                                  // halo tiles in flight (one CTA per SM owns the whole shared memory)
  // RES: the 1x1x1 residual convolution of UnetResBlock is folded in (see the kernel): a second block of BD planes x NT columns
  static constexpr int kAccSet = (RES ? 2 : 1) * BD * NT;        // accumulator columns of a tile (kAccSet / 2 registers per thread)
  static constexpr int kRBytes = NT * 32;                        // RES: the 1x1x1 weights of one K slice (NT x 16 fp16), 2 stages
  static constexpr int kSR = 2;
  static constexpr int kThreads = 384;                           // producer warpgroup + two consumer warpgroups
  static constexpr int kStatRows = (RES ? 8 : 4);                // one row of running sums per 32-row quarter and output
  static constexpr int kSmemBytes = kSA * kABytes + kSB * kBTapBytes + (RES ? kSR * kRBytes : 0) + 384 /*barriers*/ +
                                    kStatRows * 2 * NT * 4 + 2 * 2 * tc::kStageFloats * 4 /*slice buffers*/ + 128 /*align slack*/;
  static_assert(kAccSet <= 256, "accumulators exceed the register budget of a consumer thread");
  static_assert(NT % 16 == 0 && NT >= 16 && NT <= 256, "invalid wgmma N");
  static_assert(kSmemBytes <= 227 * 1024, "shared memory budget");
};

struct ConvTcParams {
  b200_conv_tc_desc d;
  const __half* w;      // packed
  ConvEpiP e;           // output stage (conv_epi.cuh)
  const float* in_stats;   // NORM: {sum, sumsq} per (n, input channel) of the raw input (see b200_conv_tc_desc.in_stats)
  ConvEpiP r;             // RES: output stage of the folded 1x1x1 residual convolution
  const __half* res_w;     // RES: packed 1x1x1 weights (gemm_tc image: [nt][k16][khalf][NT/8][8][8])
};
// NORM: affine parameters of the operand's InstanceNorm, float32 [Cin] (NULL = 1 / 0); a kernel argument of its own, so that
// ConvTcParams (and the code generated around it) is what it was before the affine variant existed
struct ConvTcAffine { const float* gamma; const float* beta; };

// Persistent, warp-specialised (384 threads, one CTA per SM): warp 0 = TMA producer, warps 4-7 and 8-11 = two consumer
// warpgroups that run the wgmma chain of rows 0-63 / 64-127 of every tile with the fp32 accumulators in registers and then
// its epilogue.  Each CTA walks tiles blockIdx.x, blockIdx.x + gridDim.x, ...; the shared-memory rings run across tile
// boundaries, so the loads of tile i+1 are in flight during the epilogue of tile i.
//
// NORM: the input is the RAW output of the previous convolution and InstanceNorm + activation
// (monai/networks/blocks/dynunet_block.py:97-103: conv1 -> norm1 -> lrelu -> conv2) is applied on the operand load: warps 1-3
// rewrite every staged halo tile in place -- y = act(x * scale + shift) with the (optionally affine) per-channel pair of
// instnorm_scale_shift (stats.cuh), the exact expression and rounding of norm_act_nc8_kernel, so the MMAs consume
// bit-identical fp16 operands -- between the TMA completion (full_a) and the MMAs
// (ready_a).  Voxels outside the volume keep the TMA's zero fill: the convolution pads the NORMALISED tensor with zeros.
// This removes one read and one write of the activation tensor per residual block.
//
// RES: the 1x1x1 convolution of the residual branch (UnetResBlock.conv3, dynunet_block.py:75-87, 104-108) reads the SAME input as
// conv1, so it is folded into this kernel: per K slice one extra MMA per output plane multiplies the centre view of the staged
// halo tile (kh = kw = 1 of input plane o + 1) with the 1x1x1 weights into a second accumulator block, and the epilogue stores
// both tensors with their statistics.  This deletes a launch that re-reads the 2 x C input tensor.
template <int NT, int BD, bool NORM, bool RES>
__global__ void __launch_bounds__(ConvTcCfg<NT, BD, RES>::kThreads, 1) conv3x3x3_tc_kernel(const __grid_constant__ CUtensorMap tmap, ConvTcParams p,
                                                                                                  ConvTcAffine aff) {
  using Cfg = ConvTcCfg<NT, BD, RES>;
  static_assert(!(NORM && RES), "the residual fold is used by conv1, the operand normalisation by conv2");
  constexpr int kSA = Cfg::kSA, kSB = Cfg::kSB;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = tc::align_smem128(smem_raw);   // keeps the shared address space (LDS/STS, not generic LD/ST)
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kSA * Cfg::kABytes;
  uint8_t* smem_r = smem_b + kSB * Cfg::kBTapBytes;                   // RES: [kSR] 1x1x1 weight slices
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_r + (RES ? Cfg::kSR * Cfg::kRBytes : 0));
  uint64_t* full_a = bars;              // [kSA]
  uint64_t* empty_a = bars + kSA;       // [kSA]
  uint64_t* full_b = bars + 2 * kSA;    // [kSB]
  uint64_t* empty_b = full_b + kSB;     // [kSB]
  uint64_t* ready_a = empty_b + kSB;    // [kSA] NORM: 3 arrivals (one per transform warp)
  uint64_t* full_r = ready_a + kSA;     // [2] RES
  uint64_t* empty_r = full_r + 2;       // [2] RES
  static_assert(3 * kSA + 2 * kSB + 4 <= 48, "barrier block");
  float* s_stats = reinterpret_cast<float*>(bars + 48);  // [kStatRows][2*NT]
  float* s_stage = s_stats + Cfg::kStatRows * 2 * NT;    // [2 warpgroups][2][kStageFloats]
  float* s_norm = s_stage + 2 * 2 * tc::kStageFloats;    // NORM: [Cin][2] (scale, shift) of one batch item

  const b200_conv_tc_desc& d = p.d;
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int num_kc = d.Cin / 16;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kSA; ++i) { tc::mbar_init(&full_a[i], 1); tc::mbar_init(&empty_a[i], 2); tc::mbar_init(&ready_a[i], 3); }
    for (int i = 0; i < kSB; ++i) { tc::mbar_init(&full_b[i], 1); tc::mbar_init(&empty_b[i], 2); }
    for (int i = 0; i < 2; ++i) { tc::mbar_init(&full_r[i], 1); tc::mbar_init(&empty_r[i], 2); }
    tc::fence_barrier_init();
  }
  for (int i = threadIdx.x; i < Cfg::kStatRows * 2 * NT; i += blockDim.x) s_stats[i] = 0.f;
  __syncthreads();

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      tc::tma_prefetch_desc(&tmap);
      int sa = 0, sb = 0, sr = 0; uint32_t pa = 0, pb = 0, pr = 0;
      for (long long t = blockIdx.x; t < p.e.total_tiles; t += gridDim.x) {
        const ConvTile c = conv_tile<BD>(p.e, t);
        const __half* wbase = p.w + (long long)c.nt * num_kc * 9 * (Cfg::kBTapBytes / 2);
        for (int kc = 0; kc < num_kc; ++kc) {
          tc::mbar_wait(&empty_a[sa], pa ^ 1);
          tc::mbar_arrive_expect_tx(&full_a[sa], Cfg::kABytes);
          tc::tma_load_5d(smem_a + sa * Cfg::kABytes, &tmap, &full_a[sa], (c.w0 - 1) * 8, c.h0 - 1, c.d0 - 1,
                          (d.in_coff + kc * 16) / 8, c.n);
          if (++sa == kSA) { sa = 0; pa ^= 1; }
          if constexpr (RES) {
            tc::mbar_wait(&empty_r[sr], pr ^ 1);
            tc::mbar_arrive_expect_tx(&full_r[sr], Cfg::kRBytes);
            tc::bulk_load(smem_r + sr * Cfg::kRBytes, p.res_w + ((long long)c.nt * num_kc + kc) * (Cfg::kRBytes / 2), Cfg::kRBytes, &full_r[sr]);
            if (++sr == Cfg::kSR) { sr = 0; pr ^= 1; }
          }
          for (int t9 = 0; t9 < 9; ++t9) {
            tc::mbar_wait(&empty_b[sb], pb ^ 1);
            tc::mbar_arrive_expect_tx(&full_b[sb], Cfg::kBTapBytes);
            tc::bulk_load(smem_b + sb * Cfg::kBTapBytes, wbase + ((long long)kc * 9 + t9) * (Cfg::kBTapBytes / 2), Cfg::kBTapBytes,
                          &full_b[sb]);
            if (++sb == kSB) { sb = 0; pb ^= 1; }
          }
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    // ===================== consumers: wgmma + epilogue =====================
    const int g = (warp >> 2) - 1, wid = warp & 3;
    const bool leader = wid == 0 && lane == 0;
    const int q = 2 * g + (wid & 1);
    float* stage = s_stage + g * 2 * tc::kStageFloats;
    float* ws_m = s_stats + q * (2 * NT);
    float* ws_r = s_stats + (4 + q) * (2 * NT);
    int sa = 0, sb = 0, sr = 0; uint32_t pa = 0, pb = 0, pr = 0;
    int prev_sb = -1;
    int sl = 0;
    long long group_m = -1, group_r = -1;
    for (long long t = blockIdx.x; t < p.e.total_tiles; t += gridDim.x) {
      const ConvTile c = conv_tile<BD>(p.e, t);
      float acc[Cfg::kAccSet / 2];
      uint32_t a_base = 0;
      // One (kh, kw) tap of one K-slice: every input plane ip of the halo tile feeds output planes ip - kd.  One NT-wide MMA per
      // (ip, kd): in-flight wgmma instructions are ordered only between instructions of the same shape on the same
      // accumulator registers, so the kd taps of a plane are not fused into one wider MMA (that would write overlapping
      // register ranges at different offsets).  A plane accumulates kd = 0, 1, 2 in ip order; the accumulators start at zero.
      // The B stage of the previous tap is released as soon as its MMAs have completed (one wgmma group stays in flight).
      auto tap = [&](int kh, int kw) {
        tc::mbar_wait(&full_b[sb], pb);
        const uint32_t b_tap = tc::smem_u32(smem_b + sb * Cfg::kBTapBytes);
        tc::wg_fence();
        tc::static_for<0, BD + 2>([&](auto ipc) {
          constexpr int ip = decltype(ipc)::value;
          constexpr int kd_hi = ip < 2 ? ip : 2, kd_lo = ip - (BD - 1) > 0 ? ip - (BD - 1) : 0;
          const uint32_t a_addr = a_base + ((ip * kHH + kh) * kHW + kw) * 16;
          const uint64_t adesc = tc::make_desc_kmajor_noswz(a_addr, Cfg::kChunkBytes, kHW * 16);
          tc::static_for<0, 3>([&](auto kdc) {
            constexpr int kd = 2 - decltype(kdc)::value;
            if constexpr (kd <= kd_hi && kd >= kd_lo) {
              const uint64_t bdesc = tc::make_desc_kmajor_noswz(b_tap + (2 - kd) * NT * 16, 3 * NT * 16, 128);
              tc::wg_mma_ss<NT>(acc + (ip - kd) * NT / 2, adesc, bdesc, 1u, 128);
            }
          });
        });
        tc::wg_commit();
        tc::wg_wait<1>();
        if (prev_sb >= 0 && leader) tc::mbar_arrive(&empty_b[prev_sb]);
        prev_sb = sb;
        if (++sb == kSB) { sb = 0; pb ^= 1; }
      };
      // RES: D_res[plane o] += centre view of input plane o + 1 x W3 slice
      auto residual = [&]() {
        tc::mbar_wait(&full_r[sr], pr);
        const uint64_t bdesc = tc::make_desc_kmajor_noswz(tc::smem_u32(smem_r + sr * Cfg::kRBytes), NT * 16, 128);
        tc::wg_fence();
        tc::static_for<0, BD>([&](auto oc) {
          constexpr int o = decltype(oc)::value;
          const uint64_t adesc = tc::make_desc_kmajor_noswz(a_base + (((o + 1) * kHH + 1) * kHW + 1) * 16, Cfg::kChunkBytes, kHW * 16);
          tc::wg_mma_ss<NT>(acc + (BD * NT + o * NT) / 2, adesc, bdesc, 1u, 128);
        });
        tc::wg_commit();
      };
#pragma unroll
      for (int i = 0; i < Cfg::kAccSet / 2; ++i) acc[i] = 0.f;
      for (int kc = 0; kc < num_kc; ++kc) {
        tc::mbar_wait(NORM ? &ready_a[sa] : &full_a[sa], pa);
        a_base = tc::smem_u32(smem_a + sa * Cfg::kABytes) + g * 8 * kHW * 16;   // rows 64.. = patch rows h0 + 8 ..
#pragma unroll 1
        for (int t9 = 0; t9 < 9; ++t9) tap(t9 / 3, t9 % 3);
        if constexpr (RES) residual();
        tc::wg_wait<0>();
        tc::wg_fence_acc<Cfg::kAccSet / 2>(acc);
        if (leader) {
          tc::mbar_arrive(&empty_b[prev_sb]);
          tc::mbar_arrive(&empty_a[sa]);
          if constexpr (RES) tc::mbar_arrive(&empty_r[sr]);
        }
        prev_sb = -1;
        if constexpr (RES) { if (++sr == Cfg::kSR) { sr = 0; pr ^= 1; } }
        if (++sa == kSA) { sa = 0; pa ^= 1; }
      }
      conv_stats_turn(p.e, ws_m, NT, t, group_m, g, wid, lane);
      conv_epilogue<NT, BD>(p.e, c, acc, stage, ws_m, g, wid, lane, sl);
      if constexpr (RES) {
        conv_stats_turn(p.r, ws_r, NT, t, group_r, g, wid, lane);
        conv_epilogue<NT, BD>(p.r, c, acc + BD * NT / 2, stage, ws_r, g, wid, lane, sl);
      }
    }
    conv_stats_final(p.e, ws_m, NT, group_m, g, wid, lane);
    if constexpr (RES) conv_stats_final(p.r, ws_r, NT, group_r, g, wid, lane);
  } else if constexpr (NORM) {
    // ===================== operand transform (warps 1-3): InstanceNorm + activation in place =====================
    // Thread tt < kRowT * kHW owns voxel column px = tt % kHW of rows py = tt / kHW + kRowT * i of every plane of both chunk
    // images: the column bounds test is one per tile, the row test one per row, and a warp's 32 vectors are contiguous.
    // (scale, shift) of every input channel of the tile's batch item -- (rstd, -mean * rstd), or with the affine parameters
    // (gamma * rstd, beta - mean * rstd * gamma) -- sit in a shared table, rebuilt only when the item changes (named barrier 1
    // of the 96 transform threads; the consumer warpgroups use ids 8 and 9).
    constexpr int kRowT = 96 / kHW;                        // rows per pass
    static_assert(kHH % kRowT == 0, "the rows of a plane split evenly into passes");
    const int tt = threadIdx.x - 32;                       // 0..95
    const int px = tt % kHW, py0 = tt / kHW;
    const bool walker = tt < kRowT * kHW;
    const float invS = 1.f / ((float)d.D * (float)d.H * (float)d.W);
    const float slope = d.in_act == 1 ? d.in_slope : (d.in_act == 3 ? 0.f : 1.f), eps = d.in_eps;
    int sa = 0; uint32_t pa = 0;
    int table_n = -1;
    for (long long t = blockIdx.x; t < p.e.total_tiles; t += gridDim.x) {
      const ConvTile c = conv_tile<BD>(p.e, t);
      if (c.n != table_n) {
        tc::named_bar(1, 96);          // every transform thread is done with the previous item's table
        const float* st = p.in_stats + 2 * (long long)c.n * d.Cin;
        for (int ch = tt; ch < d.Cin; ch += 96)   // the helper of norm_act_nc8_kernel: same (scale, shift) bits
          reinterpret_cast<float2*>(s_norm)[ch] = instnorm_scale_shift(__ldg(st + 2 * ch), __ldg(st + 2 * ch + 1), invS, eps, aff.gamma, aff.beta, ch);
        tc::named_bar(1, 96);
        table_n = c.n;
      }
      const bool col_in = walker && (unsigned)(c.w0 - 1 + px) < (unsigned)d.W;
      for (int kc = 0; kc < num_kc; ++kc) {
        float sc[16], sh[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 v = reinterpret_cast<const float2*>(s_norm)[kc * 16 + j];
          sc[j] = v.x; sh[j] = v.y;
        }
        tc::mbar_wait(&full_a[sa], pa);
        uint8_t* img = smem_a + sa * Cfg::kABytes + (py0 * kHW + px) * 16;
        if (col_in) {
#pragma unroll 2
          for (int pz = 0; pz < Cfg::kPlanes; ++pz) {
            if ((unsigned)(c.d0 - 1 + pz) >= (unsigned)d.D) continue;
#pragma unroll
            for (int i = 0; i < kHH / kRowT; ++i) {
              if ((unsigned)(c.h0 - 1 + py0 + kRowT * i) >= (unsigned)d.H) continue;
#pragma unroll
              for (int chunk = 0; chunk < 2; ++chunk) {
                uint4* ptr = reinterpret_cast<uint4*>(img + chunk * Cfg::kChunkBytes + ((pz * kHH + kRowT * i) * kHW) * 16);
                uint4 raw = *ptr;
                __half2* h2 = reinterpret_cast<__half2*>(&raw);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const float2 f = __half22float2(h2[j]);
                  const float a = fmaf(f.x, sc[8 * chunk + 2 * j], sh[8 * chunk + 2 * j]);
                  const float b = fmaf(f.y, sc[8 * chunk + 2 * j + 1], sh[8 * chunk + 2 * j + 1]);
                  // one branch-free form for none / leaky-relu / relu: max(a, a * s) with s = 1 / slope / 0 (0 <= slope <= 1)
                  // returns exactly what `a >= 0 ? a : a * slope` returns
                  h2[j] = __floats2half2_rn(fmaxf(a, a * slope), fmaxf(b, b * slope));
                }
                *ptr = raw;
              }
            }
          }
        }
        tc::fence_proxy_async();       // generic-proxy stores -> visible to the wgmma operand reads
        __syncwarp();                  // one arrival per warp
        if (lane == 0) tc::mbar_arrive(&ready_a[sa]);
        if (++sa == kSA) { sa = 0; pa ^= 1; }
      }
    }
  }
}

// NC8 normalise + activation (same math as norm_act_kernel, 8 channels per 16-byte vector)
struct NormActNc8P {
  const __half* x; __half* y; const __half* res;
  int C, x_ctot, x_coff, y_ctot, y_coff, r_ctot, r_coff;
  long long S;
  const float* stats; const float* res_stats; float eps;
  int act; float slope;
  // single-channel residual branch evaluated analytically (see b200_norm_act_cin1res_nc8)
  const __half* raw; const float* raw_stats; const float* raw_w;
};
// affine parameters of the two InstanceNorms, float32 [C] (NULL = 1 / 0).  A kernel argument of its own: the non-affine
// instantiation then compiles to the code (and the 48 registers) it had before the affine variant existed.
struct NormAffineP { const float* gamma; const float* beta; const float* res_gamma; const float* res_beta; };

// AFFINE: apply the affine parameters `a` (a separate instantiation, so the non-affine launches keep their registers)
template <bool AFFINE>
__global__ void __launch_bounds__(256) norm_act_nc8_kernel(NormActNc8P p, NormAffineP a) {
  const int chunk = blockIdx.y, n = blockIdx.z;
  float sc[8], sh[8], rsc[8], rsh[8];
  const float invS = 1.f / (float)p.S;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = chunk * 8 + j;
    sc[j] = 1.f; sh[j] = 0.f; rsc[j] = 1.f; rsh[j] = 0.f;
    if (p.stats) {
      const float2 k = instnorm_scale_shift(p.stats[2 * (n * p.C + c)], p.stats[2 * (n * p.C + c) + 1], invS, p.eps,
                                            AFFINE ? a.gamma : nullptr, AFFINE ? a.beta : nullptr, c);
      sc[j] = k.x; sh[j] = k.y;
    }
    if (p.res_stats) {
      const float2 k = instnorm_scale_shift(p.res_stats[2 * (n * p.C + c)], p.res_stats[2 * (n * p.C + c) + 1], invS, p.eps,
                                            AFFINE ? a.res_gamma : nullptr, AFFINE ? a.res_beta : nullptr, c);
      rsc[j] = k.x; rsh[j] = k.y;
    }
    if (p.raw) {
      // residual = instnorm(w * u) of a 1-channel input u: mean = w mu, var = w^2 sigma^2  =>  alpha u + beta
      const float s = p.raw_stats[2 * n], q = p.raw_stats[2 * n + 1];
      const float mu = s * invS, var = fmaxf(q * invS - mu * mu, 0.f), w = p.raw_w[c];
      rsc[j] = w / sqrtf(w * w * var + p.eps); rsh[j] = -rsc[j] * mu;
    }
  }
  const __half* u = p.raw ? p.raw + (long long)n * p.S : nullptr;
  const __half* x = p.x + (((long long)n * (p.x_ctot / 8) + p.x_coff / 8 + chunk) * p.S) * 8;
  __half* y = p.y + (((long long)n * (p.y_ctot / 8) + p.y_coff / 8 + chunk) * p.S) * 8;
  const __half* r = p.res ? p.res + (((long long)n * (p.r_ctot / 8) + p.r_coff / 8 + chunk) * p.S) * 8 : nullptr;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < p.S; s += (long long)gridDim.x * blockDim.x) {
    __align__(16) __half v[8], rv[8];
    *reinterpret_cast<uint4*>(v) = *reinterpret_cast<const uint4*>(x + s * 8);
    if (r) *reinterpret_cast<uint4*>(rv) = *reinterpret_cast<const uint4*>(r + s * 8);
    const float uv = u ? __half2float(__ldg(u + s)) : 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float f = fmaf(__half2float(v[j]), sc[j], sh[j]);
      if (r) f += fmaf(__half2float(rv[j]), rsc[j], rsh[j]);
      if (u) f += fmaf(uv, rsc[j], rsh[j]);
      if (p.act == 1) f = f >= 0.f ? f : f * p.slope;
      else if (p.act == 3) f = fmaxf(f, 0.f);
      v[j] = __float2half_rn(f);
    }
    *reinterpret_cast<uint4*>(y + s * 8) = *reinterpret_cast<const uint4*>(v);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_pack_nc8(const void* x, int dtype, int N, int C, long long S, void* y, int Ctot, int c_off, void* stream) {
  B200_REQUIRE(x && y, "pack_nc8: null pointer");
  B200_REQUIRE(C % 8 == 0 && Ctot % 8 == 0 && c_off % 8 == 0 && c_off + C <= Ctot, "pack_nc8: channel counts must be multiples of 8");
  if ((long long)N * C * S == 0) return B200_OK;
  dim3 grid((unsigned)std::min<long long>((S + 255) / 256, 1024), C / 8, N);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == B200_DT_F16) pack_nc8_kernel<__half><<<grid, 256, 0, st>>>((const __half*)x, (__half*)y, C, S, Ctot, c_off);
  else if (dtype == B200_DT_F32) pack_nc8_kernel<float><<<grid, 256, 0, st>>>((const float*)x, (__half*)y, C, S, Ctot, c_off);
  else return set_err(B200_ERR_INVALID, "pack_nc8: bad dtype");
  B200_LAUNCH_CHECK("pack_nc8_kernel");
  return B200_OK;
}

extern "C" int b200_unpack_nc8(const void* x, int Ctot, int c_off, int N, int C, long long S, void* y, int dtype, void* stream) {
  B200_REQUIRE(x && y, "unpack_nc8: null pointer");
  B200_REQUIRE(C % 8 == 0 && Ctot % 8 == 0 && c_off % 8 == 0 && c_off + C <= Ctot, "unpack_nc8: channel counts must be multiples of 8");
  if ((long long)N * C * S == 0) return B200_OK;
  dim3 grid((unsigned)std::min<long long>((S + 255) / 256, 1024), C / 8, N);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == B200_DT_F16) unpack_nc8_kernel<__half><<<grid, 256, 0, st>>>((const __half*)x, (__half*)y, C, S, Ctot, c_off);
  else if (dtype == B200_DT_F32) unpack_nc8_kernel<float><<<grid, 256, 0, st>>>((const __half*)x, (float*)y, C, S, Ctot, c_off);
  else return set_err(B200_ERR_INVALID, "unpack_nc8: bad dtype");
  B200_LAUNCH_CHECK("unpack_nc8_kernel");
  return B200_OK;
}

extern "C" long long b200_conv3x3x3_tc_weight_bytes(int Cin, int Cout) {
  if (Cin <= 0 || Cout <= 0 || Cin % 16 || Cout % 16) return -1;
  return (long long)Cin * Cout * 27 * 2;
}

extern "C" int b200_conv3x3x3_tc_pack_weight(const float* w, int Cin, int Cout, void* packed, void* stream) {
  B200_REQUIRE(w && packed, "conv3x3x3_tc_pack_weight: null pointer");
  B200_REQUIRE(Cin > 0 && Cout > 0 && Cin % 16 == 0 && Cout % 16 == 0, "conv3x3x3_tc: Cin and Cout must be multiples of 16 (got %d, %d)", Cin, Cout);
  const long long total = (long long)Cin * Cout * 27;
  const int blocks = (int)std::min<long long>((total + 255) / 256, 4096);
  conv_tc_pack_weight_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, (__half*)packed, Cin, Cout, conv_tc_nt(Cout));
  B200_LAUNCH_CHECK("conv_tc_pack_weight_kernel");
  return B200_OK;
}

template <int NT, int BD>
struct ConvTcGeom {
  static void fill(const b200_conv_tc_desc& d, ConvEpiP& e) {
    e.D = d.D; e.H = d.H; e.W = d.W; e.Cout = d.Cout; e.out_ctot = d.out_ctot; e.out_coff = d.out_coff;
    e.tiles_w = ceil_div(d.W, kTW); e.tiles_h = ceil_div(d.H, kTH); e.tiles_d = ceil_div(d.D, BD); e.n_tiles = d.Cout / NT;
    e.total_tiles = (long long)e.tiles_w * e.tiles_h * e.tiles_d * e.n_tiles * d.N;
  }
};

// what a launch needs beyond the operands: mode 0 = run, mode 1 = only report the statistics workspace size
struct ConvTcCall {
  const void* x; const void* w; const float* bias; void* y; float* stats; void* ws; cudaStream_t st; long long ws_bytes; int query;
  const float* in_gamma; const float* in_beta;   // NORM: affine parameters of the operand normalisation (NULL = non-affine)
};

template <int NT, int BD, bool NORM, bool RES = false>
static int launch_conv_tc(const b200_conv_tc_desc& d, ConvTcCall& c) {
  using Cfg = ConvTcCfg<NT, BD, RES>;
  ConvTcParams p;
  p.d = d; p.w = (const __half*)c.w; p.in_stats = (const float*)d.in_stats;
  ConvTcGeom<NT, BD>::fill(d, p.e);
  const long long sp_tiles = (long long)p.e.tiles_w * p.e.tiles_h * p.e.tiles_d, groups = (long long)d.N * p.e.n_tiles;
  const int R = stats_rows(sp_tiles, p.e.total_tiles);
  constexpr int kRows = 4;                                          // partial rows a CTA writes per group (one per quarter)
  const long long one = stats_partial_bytes(groups, R, NT, kRows);
  c.ws_bytes = RES ? 2 * one : one;     // RES: main partials, then the residual's
  if (c.query) return B200_OK;
  EncodeTiledFn enc = get_encode_tiled();
  B200_REQUIRE(enc != nullptr, "conv3x3x3_tc: cuTensorMapEncodeTiled entry point unavailable");
  CUtensorMap tmap;
  const cuuint64_t S = (cuuint64_t)d.D * d.H * d.W;
  cuuint64_t gdim[5] = {(cuuint64_t)d.W * 8, (cuuint64_t)d.H, (cuuint64_t)d.D, (cuuint64_t)(d.in_ctot / 8), (cuuint64_t)d.N};
  cuuint64_t gstr[4] = {(cuuint64_t)d.W * 16, (cuuint64_t)d.H * d.W * 16, S * 16, S * 16 * (cuuint64_t)(d.in_ctot / 8)};
  cuuint32_t box[5] = {(cuuint32_t)kHW * 8, (cuuint32_t)kHH, (cuuint32_t)(BD + 2), 2, 1};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(c.x), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_REQUIRE(r == CUDA_SUCCESS, "conv3x3x3_tc: cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  p.e.y = (__half*)c.y; p.e.bias = c.bias;
  p.e.sp.buf = c.stats ? (float*)c.ws : nullptr; p.e.sp.R = R; p.e.sp.tiles_per_group = sp_tiles; p.e.sp.rows_per_cta = kRows;
  p.r = p.e; p.res_w = nullptr;
  if (RES) {
    p.r.y = (__half*)d.res_y; p.r.bias = nullptr; p.r.out_ctot = d.res_ctot; p.r.out_coff = d.res_coff;
    p.r.sp.buf = d.res_stats ? (float*)((char*)c.ws + one) : nullptr;
    p.res_w = (const __half*)d.res_w;
  }
  dim3 grid((unsigned)std::min<long long>(p.e.total_tiles, num_sms()));
  auto kern = conv3x3x3_tc_kernel<NT, BD, NORM, RES>;
  const int smem = Cfg::kSmemBytes + (NORM ? d.Cin * 8 : 0);   // NORM: the per-channel scale / shift table
  B200_REQUIRE(smem <= 227 * 1024, "conv3x3x3_tc: Cin %d is too wide for the operand normalisation table", d.Cin);
  // per-device attribute: set on every call (cheap), so a second GPU in the same process works
  B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kern<<<grid, Cfg::kThreads, smem, c.st>>>(tmap, p, ConvTcAffine{c.in_gamma, c.in_beta});
  B200_LAUNCH_CHECK("conv3x3x3_tc_kernel");
  if (c.stats) {
    const int rc = launch_stats_finish((const float*)c.ws, groups, R * kRows, NT, p.e.n_tiles, d.Cout, c.stats, c.st);
    if (rc) return rc;
  }
  if (RES && d.res_stats) return launch_stats_finish((const float*)((const char*)c.ws + one), groups, R * kRows, NT, p.e.n_tiles, d.Cout, d.res_stats, c.st);
  return B200_OK;
}

template <int NT, int BD>
static int launch_variant(const b200_conv_tc_desc& d, ConvTcCall& c) {
  if (d.in_stats) return launch_conv_tc<NT, BD, true>(d, c);
  if constexpr (NT <= 128 && 2 * BD * NT <= 256) {
    if (d.res_w) return launch_conv_tc<NT, BD, false, true>(d, c);
  }
  return launch_conv_tc<NT, BD, false>(d, c);
}

template <int NT>
static int dispatch_bd(const b200_conv_tc_desc& d, ConvTcCall& c) {
  // deeper CTA tiles amortise the halo and fuse more kd taps per MMA; the depth is bounded by the accumulators a consumer
  // thread can hold (BD * NT, twice that with the folded residual, <= 256 columns = 128 registers)
  const int res = d.res_w ? 2 : 1;
  if constexpr (NT * 4 <= 256) {
    if ((d.D % 4 == 0 || d.D >= 16) && 4 * NT * res <= 256) return launch_variant<NT, 4>(d, c);
  }
  if constexpr (NT * 2 <= 256) {
    if (d.D >= 2 && 2 * NT * res <= 256) return launch_variant<NT, 2>(d, c);
  }
  return launch_variant<NT, 1>(d, c);
}

static int conv_tc_dispatch(const b200_conv_tc_desc& d, ConvTcCall& c) {
  B200_REQUIRE(d.N > 0 && d.D > 0 && d.H > 0 && d.W > 0, "conv3x3x3_tc: empty problem");
  B200_REQUIRE(d.Cin > 0 && d.Cin % 16 == 0 && d.Cout > 0 && d.Cout % 16 == 0,
               "conv3x3x3_tc: Cin and Cout must be multiples of 16 (got %d, %d)", d.Cin, d.Cout);
  B200_REQUIRE(d.in_ctot % 8 == 0 && d.in_coff % 8 == 0 && d.in_coff + d.Cin <= d.in_ctot, "conv3x3x3_tc: bad input channel slice");
  B200_REQUIRE(d.out_ctot % 8 == 0 && d.out_coff % 8 == 0 && d.out_coff + d.Cout <= d.out_ctot, "conv3x3x3_tc: bad output channel slice");
  B200_REQUIRE(!d.in_stats || d.in_act == 0 || d.in_act == 1 || d.in_act == 3, "conv3x3x3_tc: in_act must be none, leaky-relu or relu");
  B200_REQUIRE(!d.in_stats || d.in_act != 1 || (d.in_slope >= 0.f && d.in_slope <= 1.f), "conv3x3x3_tc: in_slope must lie in [0, 1] (got %g)", (double)d.in_slope);
  if (d.res_w) {
    B200_REQUIRE(!d.in_stats, "conv3x3x3_tc: the folded residual convolution and the operand normalisation are exclusive");
    B200_REQUIRE(d.res_y && d.Cout <= 128, "conv3x3x3_tc: the folded residual convolution needs res_y and Cout <= 128 (got %d)", d.Cout);
    B200_REQUIRE(d.res_ctot % 8 == 0 && d.res_coff % 8 == 0 && d.res_coff + d.Cout <= d.res_ctot, "conv3x3x3_tc: bad residual output channel slice");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(d.res_w) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.res_y) & 15) == 0, "conv3x3x3_tc: residual pointers must be 16-byte aligned");
  }
  switch (conv_tc_nt(d.Cout)) {
    case 16: return dispatch_bd<16>(d, c);
    case 32: return dispatch_bd<32>(d, c);
    case 48: return dispatch_bd<48>(d, c);
    case 64: return dispatch_bd<64>(d, c);
    case 80: return dispatch_bd<80>(d, c);
    case 96: return dispatch_bd<96>(d, c);
    case 112: return dispatch_bd<112>(d, c);
    case 128: return dispatch_bd<128>(d, c);
    default: return set_err(B200_ERR_UNSUPPORTED, "conv3x3x3_tc: unsupported Cout %d", d.Cout);
  }
}

extern "C" long long b200_conv3x3x3_tc_workspace_bytes(const b200_conv_tc_desc* desc) {
  if (!desc) return -1;
  ConvTcCall c{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 1, nullptr, nullptr};
  if (conv_tc_dispatch(*desc, c)) return -1;
  return c.ws_bytes;
}

static int conv3x3x3_tc_run(const b200_conv_tc_desc* desc, const float* in_gamma, const float* in_beta, const void* x, const void* packed_w,
                            const float* bias, void* y, float* stats, void* workspace, void* stream) {
  B200_REQUIRE(desc && x && packed_w && y, "conv3x3x3_tc: null pointer");
  B200_REQUIRE(!(stats || (desc && desc->res_stats)) || workspace, "conv3x3x3_tc: statistics need the workspace of b200_conv3x3x3_tc_workspace_bytes()");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0 &&
               (reinterpret_cast<uintptr_t>(packed_w) & 15) == 0, "conv3x3x3_tc: pointers must be 16-byte aligned");
  B200_REQUIRE(desc->in_stats || !(in_gamma || in_beta), "conv3x3x3_tc: affine parameters of the operand normalisation without in_stats");
  ConvTcCall c{x, packed_w, bias, y, stats, workspace, (cudaStream_t)stream, 0, 0, in_gamma, in_beta};
  return conv_tc_dispatch(*desc, c);
}

extern "C" int b200_conv3x3x3_tc(const b200_conv_tc_desc* desc, const void* x, const void* packed_w, const float* bias,
                                 void* y, float* stats, void* workspace, void* stream) {
  return conv3x3x3_tc_run(desc, nullptr, nullptr, x, packed_w, bias, y, stats, workspace, stream);
}

extern "C" int b200_conv3x3x3_tc_affine(const b200_conv_tc_desc* desc, const float* in_gamma, const float* in_beta, const void* x,
                                        const void* packed_w, const float* bias, void* y, float* stats, void* workspace, void* stream) {
  return conv3x3x3_tc_run(desc, in_gamma, in_beta, x, packed_w, bias, y, stats, workspace, stream);
}

// y = act(instnorm(x) [+ instnorm?(res)]) with optional affine parameters per norm: the body of b200_norm_act_nc8 and
// b200_norm_act_affine_nc8
static int norm_act_nc8_launch(const void* x, int x_ctot, int x_coff, int N, int C, long long S, const float* stats, float eps,
                               const void* res, int res_ctot, int res_coff, const float* res_stats, int act, float slope, void* y,
                               int y_ctot, int y_coff, const float* gamma, const float* beta, const float* res_gamma,
                               const float* res_beta, void* stream) {
  B200_REQUIRE(x && y, "norm_act_nc8: null pointer");
  B200_REQUIRE(C % 8 == 0 && x_ctot % 8 == 0 && x_coff % 8 == 0 && y_ctot % 8 == 0 && y_coff % 8 == 0, "norm_act_nc8: channels must be multiples of 8");
  B200_REQUIRE(act == 0 || act == 1 || act == 3, "norm_act_nc8: activation must be none, leaky-relu or relu");
  B200_REQUIRE(stats || !(gamma || beta), "norm_act_nc8: affine parameters without statistics");
  B200_REQUIRE(res_stats || !(res_gamma || res_beta), "norm_act_nc8: residual affine parameters without residual statistics");
  if ((long long)N * C * S == 0) return B200_OK;
  NormActNc8P p;
  p.x = (const __half*)x; p.y = (__half*)y; p.res = (const __half*)res; p.C = C;
  p.x_ctot = x_ctot; p.x_coff = x_coff; p.y_ctot = y_ctot; p.y_coff = y_coff; p.r_ctot = res_ctot; p.r_coff = res_coff;
  p.S = S; p.stats = stats; p.res_stats = res_stats; p.eps = eps; p.act = act; p.slope = slope;
  p.raw = nullptr; p.raw_stats = nullptr; p.raw_w = nullptr;
  long long want = (long long)num_sms() * 16 / ((long long)N * (C / 8)) + 1;
  dim3 grid((unsigned)std::max<long long>(1, std::min<long long>(want, (S + 255) / 256)), C / 8, N);
  const NormAffineP a{gamma, beta, res_gamma, res_beta};
  if (gamma || beta || res_gamma || res_beta) norm_act_nc8_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(p, a);
  else norm_act_nc8_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(p, a);
  B200_LAUNCH_CHECK("norm_act_nc8_kernel");
  return B200_OK;
}

extern "C" int b200_norm_act_nc8(const void* x, int x_ctot, int x_coff, int N, int C, long long S, const float* stats,
                                 float eps, const void* res, int res_ctot, int res_coff, const float* res_stats, int act,
                                 float slope, void* y, int y_ctot, int y_coff, void* stream) {
  return norm_act_nc8_launch(x, x_ctot, x_coff, N, C, S, stats, eps, res, res_ctot, res_coff, res_stats, act, slope, y, y_ctot, y_coff,
                             nullptr, nullptr, nullptr, nullptr, stream);
}

extern "C" int b200_norm_act_affine_nc8(const void* x, int x_ctot, int x_coff, int N, int C, long long S, const float* stats,
                                        float eps, const void* res, int res_ctot, int res_coff, const float* res_stats, int act,
                                        float slope, void* y, int y_ctot, int y_coff, const float* gamma, const float* beta,
                                        const float* res_gamma, const float* res_beta, void* stream) {
  return norm_act_nc8_launch(x, x_ctot, x_coff, N, C, S, stats, eps, res, res_ctot, res_coff, res_stats, act, slope, y, y_ctot, y_coff,
                             gamma, beta, res_gamma, res_beta, stream);
}

extern "C" int b200_norm_act_cin1res_nc8(const void* x, int x_ctot, int x_coff, int N, int C, long long S, const float* stats,
                                         float eps, const void* raw, const float* raw_stats, const float* raw_weight, int act,
                                         float slope, void* y, int y_ctot, int y_coff, void* stream) {
  B200_REQUIRE(x && y && stats && raw && raw_stats && raw_weight, "norm_act_cin1res_nc8: null pointer");
  B200_REQUIRE(C % 8 == 0 && x_ctot % 8 == 0 && x_coff % 8 == 0 && y_ctot % 8 == 0 && y_coff % 8 == 0, "norm_act_cin1res_nc8: channels must be multiples of 8");
  B200_REQUIRE(act == 0 || act == 1 || act == 3, "norm_act_cin1res_nc8: activation must be none, leaky-relu or relu");
  if ((long long)N * C * S == 0) return B200_OK;
  NormActNc8P p;
  p.x = (const __half*)x; p.y = (__half*)y; p.res = nullptr; p.C = C;
  p.x_ctot = x_ctot; p.x_coff = x_coff; p.y_ctot = y_ctot; p.y_coff = y_coff; p.r_ctot = 0; p.r_coff = 0;
  p.S = S; p.stats = stats; p.res_stats = nullptr; p.eps = eps; p.act = act; p.slope = slope;
  p.raw = (const __half*)raw; p.raw_stats = raw_stats; p.raw_w = raw_weight;
  long long want = (long long)num_sms() * 16 / ((long long)N * (C / 8)) + 1;
  dim3 grid((unsigned)std::max<long long>(1, std::min<long long>(want, (S + 255) / 256)), C / 8, N);
  norm_act_nc8_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(p, NormAffineP{nullptr, nullptr, nullptr, nullptr});
  B200_LAUNCH_CHECK("norm_act_nc8_kernel");
  return B200_OK;
}
