// Antialiased bicubic resize taps (torch _upsample_bicubic2d_aa: separable Keys cubic a = -0.5, support widened by
// the down-scale factor, weights normalised) shared by the clip pre-processing (pre.cu) and the alpha resize
// (alpha.cu).  The tap tables (first tap, tap count, weights per output column / row) are built on the device so that
// a call needs no host arrays and no synchronisation.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace svr2 {
namespace {

constexpr int kMaxTaps = 32;

__device__ __forceinline__ float rn(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

__device__ __forceinline__ double cubic_aa(double x) {
  const double a = -0.5;
  x = fabs(x);
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0;
  if (x < 2.0) return (((x - 5.0) * x + 8.0) * x - 4.0) * a;
  return 0.0;
}

// table layout per axis: first[out], count[out], weights[out][K]
__global__ void aa_table_kernel(int in_size, int out_size, int K, int* __restrict__ first, int* __restrict__ count,
                                float* __restrict__ weights) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= out_size) return;
  const float scale = (float)in_size / (float)out_size;
  const float support = scale >= 1.0f ? 2.0f * scale : 2.0f;
  const float invscale = scale >= 1.0f ? 1.0f / scale : 1.0f;
  const float center = (float)((double)scale * ((double)i + 0.5));
  int lo = (int)(float)((double)center - (double)support + 0.5);
  if (lo < 0) lo = 0;
  int hi = (int)(float)((double)center + (double)support + 0.5);
  if (hi > in_size) hi = in_size;
  int n = hi - lo;
  if (n > K) n = K;
  const float lo_m_center = (float)((double)lo - (double)center);
  float tot = 0.f;
  float* w = weights + (long long)i * K;
  for (int j = 0; j < n; ++j) {
    const float arg = (float)(((double)j + (double)lo_m_center + 0.5) * (double)invscale);
    const float v = (float)cubic_aa((double)arg);
    w[j] = v;
    tot += v;
  }
  for (int j = 0; j < n; ++j)
    if (tot != 0.f) w[j] /= tot;
  for (int j = n; j < K; ++j) w[j] = 0.f;
  first[i] = lo;
  count[i] = n;
}

template <typename T>
__device__ __forceinline__ float load_bf16_rounded(const T* p);
template <>
__device__ __forceinline__ float load_bf16_rounded<float>(const float* p) { return rn(*p); }
template <>
__device__ __forceinline__ float load_bf16_rounded<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <>
__device__ __forceinline__ float load_bf16_rounded<__half>(const __half* p) { return rn(__half2float(*p)); }
// 8-bit frames as the reference CLI reads them (inference_cli.py:613, 336-339; generation_phases.py:380-387):
// fp32(u) / 255 correctly rounded, then fp16, then the bf16 compute dtype
template <>
__device__ __forceinline__ float load_bf16_rounded<uint8_t>(const uint8_t* p) {
  return rn(__half2float(__float2half_rn(__fdiv_rn((float)*p, 255.0f))));
}

inline size_t align256(size_t x) { return (x + 255) & ~size_t(255); }
inline int taps_for(int in_size, int out_size) {
  const float scale = (float)in_size / (float)out_size;
  const float support = scale >= 1.0f ? 2.0f * scale : 2.0f;
  return (int)ceilf(support) * 2 + 1;
}

}  // namespace
}  // namespace svr2
