// Antialiased bicubic resize taps (torch _upsample_bicubic2d_aa: separable Keys cubic a = -0.5, support widened by
// the down-scale factor, weights normalised) shared by the clip pre-processing (pre.cu) and the alpha resize
// (alpha.cu).  The tap tables (first tap, tap count, weights per output column / row) are built on the device so that
// a call needs no host arrays and no synchronisation.
//
// The tables are those of torch's CUDA kernel (ATen/native/cuda/UpSample.cuh, upsample_antialias::
// _compute_weights_span / _compute_weights / BicubicFilterFunctor), which is what the reference runs: it resizes the
// clip and the alpha on the GPU.  That kernel computes everything in fp32, and nvcc fuses its multiply-adds, also
// across statements; its sm_90 code evaluates, per output index i (ii = i + 0.5f, exact):
//   xmin  = max(int(fma(ii, scale, -support) + 0.5f), 0)        xmax = min(int(fma(ii, scale, support) + 0.5f), n_in)
//   xmin_m_center = fma(-ii, scale, float(xmin))                 invscale = 1 / scale (scale >= 1) or 1
//   arg_j = ((xmin_m_center + j) + 0.5f) * invscale              x = |arg_j|
//   w_j   = fma(x, x * fma(x, 1.5f, -2.5f), 1)  (x < 1)          fma(x, fma(x, x - 5, 8), -4) * -0.5  (1 <= x < 2)
//   total = w_0 + w_1 + ... left to right; w_j / total (IEEE division) when total != 0.
// The expressions below spell each of those roundings out (__fmaf_rn, __fadd_rn, __fmul_rn) so that contraction
// cannot change them.  torch's CPU kernel rounds differently (it computes the span and the argument without the
// fusions), so its weights differ from these in the last bits at non-dyadic ratios.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace svr2 {
namespace {

// At most 31 taps per output index: down-scale factors up to 7.5 (taps = 2 ceil(2 scale) + 1).
constexpr int kMaxTaps = 32;

__device__ __forceinline__ float rn(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// BicubicFilterFunctor (a = -0.5) as torch's sm_90 code evaluates it
__device__ __forceinline__ float cubic_aa(float x) {
  x = fabsf(x);
  if (x < 1.f) return __fmaf_rn(x, __fmul_rn(x, __fmaf_rn(x, 1.5f, -2.5f)), 1.f);
  if (x < 2.f) return __fmul_rn(__fmaf_rn(x, __fmaf_rn(x, __fadd_rn(x, -5.f), 8.f), -4.f), -0.5f);
  return 0.f;
}

// table layout per axis: first[out], count[out], weights[out][K]
__global__ void aa_table_kernel(int in_size, int out_size, int K, int* __restrict__ first, int* __restrict__ count,
                                float* __restrict__ weights) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= out_size) return;
  const float scale = __fdiv_rn((float)in_size, (float)out_size);
  const float support = scale >= 1.0f ? __fadd_rn(scale, scale) : 2.0f;
  const float invscale = scale >= 1.0f ? __fdiv_rn(1.0f, scale) : 1.0f;
  const float ii = __fadd_rn((float)i, 0.5f);
  int lo = (int)__fadd_rn(__fmaf_rn(ii, scale, -support), 0.5f);
  if (lo < 0) lo = 0;
  int hi = (int)__fadd_rn(__fmaf_rn(ii, scale, support), 0.5f);
  if (hi > in_size) hi = in_size;
  int n = hi - lo;
  if (n > K) n = K;
  const float lo_m_center = __fmaf_rn(-ii, scale, (float)lo);
  float tot = 0.f;
  float* w = weights + (long long)i * K;
  for (int j = 0; j < n; ++j) {
    const float v = cubic_aa(__fmul_rn(__fadd_rn(__fadd_rn(lo_m_center, (float)j), 0.5f), invscale));
    w[j] = v;
    tot = __fadd_rn(tot, v);
  }
  for (int j = 0; j < n; ++j)
    if (tot != 0.f) w[j] = __fdiv_rn(w[j], tot);
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
