// Shared helpers for the monai_b200 CUDA kernels (sm_90a only).
// Nothing here depends on torch; the C-ABI in include/monai_b200.h is plain pointers + sizes.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <algorithm>

#define B200_OK 0
#define B200_ERR_INVALID 1
#define B200_ERR_CUDA 2
#define B200_ERR_UNSUPPORTED 3

#define B200_DT_F32 0
#define B200_DT_F16 1

namespace b200 {

// thread-local last error message (returned by b200_last_error()).
char* err_buf();
int set_err(int code, const char* fmt, ...);

inline int cuda_check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) return set_err(B200_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return B200_OK;
}

#define B200_CUDA(expr)                                            \
  do {                                                             \
    int _rc = ::b200::cuda_check((expr), #expr);                   \
    if (_rc) return _rc;                                           \
  } while (0)

#define B200_LAUNCH_CHECK(name)                                    \
  do {                                                             \
    ::b200::note_launch();                                         \
    int _rc = ::b200::cuda_check(cudaGetLastError(), name);        \
    if (_rc) return _rc;                                           \
  } while (0)

#define B200_REQUIRE(cond, ...)                                    \
  do {                                                             \
    if (!(cond)) return ::b200::set_err(B200_ERR_INVALID, __VA_ARGS__); \
  } while (0)

int num_sms();
void note_launch();

template <typename T> struct io;
template <> struct io<float> {
  __device__ static __forceinline__ float ld(const float* p) { return __ldg(p); }
  __device__ static __forceinline__ void st(float* p, float v) { *p = v; }
  __device__ static __forceinline__ void st2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }  // 8-byte aligned
};
template <> struct io<__half> {
  __device__ static __forceinline__ float ld(const __half* p) { return __half2float(__ldg(p)); }
  __device__ static __forceinline__ void st(__half* p, float v) { *p = __float2half_rn(v); }
  __device__ static __forceinline__ void st2(__half* p, float a, float b) { *reinterpret_cast<__half2*>(p) = __floats2half2_rn(a, b); }  // 4-byte aligned
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Column sums of an 8-column x 32-lane tile held as 8 registers per lane (sum and sum of squares together): three
// exchange steps halve the number of columns a lane owns, two plain steps finish.  Afterwards the lanes with
// (lane & 3) == 0 hold the totals of column  ((lane>>4)&1)*4 + ((lane>>3)&1)*2 + ((lane>>2)&1).   (9 shuffles per array
// instead of 40 for eight butterfly reductions.)
__device__ __forceinline__ void transpose_reduce8(const float (&s)[8], const float (&q)[8], int lane, float& s_out, float& q_out) {
  float a4[4], b4[4];
  const bool hi16 = lane & 16;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float send = hi16 ? s[j] : s[j + 4], keep = hi16 ? s[j + 4] : s[j];
    a4[j] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    const float send2 = hi16 ? q[j] : q[j + 4], keep2 = hi16 ? q[j + 4] : q[j];
    b4[j] = keep2 + __shfl_xor_sync(0xffffffffu, send2, 16);
  }
  float a2[2], b2[2];
  const bool hi8 = lane & 8;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float send = hi8 ? a4[j] : a4[j + 2], keep = hi8 ? a4[j + 2] : a4[j];
    a2[j] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    const float send2 = hi8 ? b4[j] : b4[j + 2], keep2 = hi8 ? b4[j + 2] : b4[j];
    b2[j] = keep2 + __shfl_xor_sync(0xffffffffu, send2, 8);
  }
  const bool hi4 = lane & 4;
  float a1 = (hi4 ? a2[1] : a2[0]) + __shfl_xor_sync(0xffffffffu, hi4 ? a2[0] : a2[1], 4);
  float b1 = (hi4 ? b2[1] : b2[0]) + __shfl_xor_sync(0xffffffffu, hi4 ? b2[0] : b2[1], 4);
  a1 += __shfl_xor_sync(0xffffffffu, a1, 2); b1 += __shfl_xor_sync(0xffffffffu, b1, 2);
  a1 += __shfl_xor_sync(0xffffffffu, a1, 1); b1 += __shfl_xor_sync(0xffffffffu, b1, 1);
  s_out = a1; q_out = b1;
}
__device__ __forceinline__ int transpose_reduce8_col(int lane) { return ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1); }

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

}  // namespace b200
