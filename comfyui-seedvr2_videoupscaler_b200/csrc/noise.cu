// Input and latent noise (generation_phases.py:415-431, 679-704): the two per-value blends of the generation inputs
// `input_noise_scale` and `latent_noise_scale`.
//
//   input_noise_kernel   :416-429   out = tv * (1 - b) + (tv + 0.05 * n) * b on the transformed clip, out of place,
//                                   the draw n in any of the three memory orders the reference's clip can have
//   sr_condition_kernel  :680-697, infer.py:54-78
//                                   the DiT input rows [noise | cond | 1]; cond = A * latent + B * aug with
//                                   aug = noise * 0.1 + r * 0.05, or cond = latent without augmentation
//
// Every reference op is its own ATen kernel: its result is rounded (to bf16, or fp32 for the schedule's A * x0 and
// B * xT) before the next op reads it, so each step here is one __fmul_rn / __fadd_rn with no FMA contraction.
// Python scalars enter ATen's bf16 kernels as fp32 opmath values (0.05f, 0.1f, (float)(1 - b), (float)b).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "svr2_internal.h"

namespace svr2 {
namespace {

__device__ __forceinline__ float rbf(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

// bf16(bf16(x * c1) + bf16(bf16(x + bf16(n * 0.05)) * c2)) before the final rounding
__device__ __forceinline__ float input_blend(float x, float n, float c1, float c2) {
  const float kept = rbf(__fmul_rn(x, c1));              // transformed_video * (1 - blend_factor)
  const float scaled = rbf(__fmul_rn(n, 0.05f));         // noise * 0.05
  const float noisy = rbf(__fadd_rn(x, scaled));         // transformed_video + noise
  return __fadd_rn(kept, rbf(__fmul_rn(noisy, c2)));     // ... * blend_factor, then the sum
}

// x, out [3, T, plane] (c-major: the clip as the encoder reads it).  The noise is the raw draw in the memory order
// of the reference's randn_like on its transformed clip (see svr2.h): LAYOUT 0 [T, 3, plane], 1 [3, T, plane],
// 2 [T, plane, 3].  A thread takes one frame's pixels p .. p+7 (VEC: plane % 8 == 0, 16-byte aligned pointers) in
// all three channels, so every layout reads its noise in contiguous runs.
template <int LAYOUT, bool VEC>
__global__ void __launch_bounds__(256) input_noise_kernel(const __nv_bfloat16* __restrict__ x,
                                                          const __nv_bfloat16* __restrict__ n,
                                                          __nv_bfloat16* __restrict__ out, int T, int plane,
                                                          long long pixels, float c1, float c2) {
  constexpr int kVec = VEC ? 8 : 1;
  const long long stride = (long long)gridDim.x * blockDim.x * kVec;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * kVec; i < pixels; i += stride) {
    const long long t = i / plane;
    const long long p = i - t * plane;
    float nv[3][kVec];
    if constexpr (LAYOUT == 2) {
      const __nv_bfloat16* np = n + i * 3;
      if constexpr (VEC) {
        uint4 raw[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) raw[k] = reinterpret_cast<const uint4*>(np)[k];
        const __nv_bfloat16* v = reinterpret_cast<const __nv_bfloat16*>(raw);
#pragma unroll
        for (int k = 0; k < kVec; ++k)
#pragma unroll
          for (int c = 0; c < 3; ++c) nv[c][k] = __bfloat162float(v[k * 3 + c]);
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) nv[c][0] = __bfloat162float(np[c]);
      }
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const long long ni = (LAYOUT == 0 ? (t * 3 + c) : ((long long)c * T + t)) * plane + p;
        if constexpr (VEC) {
          const uint4 raw = *reinterpret_cast<const uint4*>(n + ni);
          const __nv_bfloat16* v = reinterpret_cast<const __nv_bfloat16*>(&raw);
#pragma unroll
          for (int k = 0; k < kVec; ++k) nv[c][k] = __bfloat162float(v[k]);
        } else {
          nv[c][0] = __bfloat162float(n[ni]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long xi = ((long long)c * T + t) * plane + p;
      if constexpr (VEC) {
        const uint4 xv = *reinterpret_cast<const uint4*>(x + xi);
        const __nv_bfloat162* xa = reinterpret_cast<const __nv_bfloat162*>(&xv);
        uint4 ov;
        __nv_bfloat162* oa = reinterpret_cast<__nv_bfloat162*>(&ov);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 xf = __bfloat1622float2(xa[k]);
          oa[k] = __floats2bfloat162_rn(input_blend(xf.x, nv[c][2 * k], c1, c2),
                                        input_blend(xf.y, nv[c][2 * k + 1], c1, c2));
        }
        *reinterpret_cast<uint4*>(out + xi) = ov;
      } else {
        out[xi] = __float2bfloat16_rn(input_blend(__bfloat162float(x[xi]), nv[c][0], c1, c2));
      }
    }
  }
}

constexpr int kCondRows = 128;   // latent rows per block

// out [L, 2c+1] = [noise | cond | 1] per row; noise, latent [L, c]; r [c, L] (channel-major, the memory order of the
// reference's randn_like on its channels-last latent view) or null.  A block stages its rows' r through shared memory
// so both the r reads and the row-major output stores are coalesced.
__global__ void __launch_bounds__(256) sr_condition_kernel(const __nv_bfloat16* __restrict__ noise,
                                                           const __nv_bfloat16* __restrict__ latent,
                                                           const __nv_bfloat16* __restrict__ r,
                                                           const float* __restrict__ coef_a,
                                                           const float* __restrict__ coef_b,
                                                           __nv_bfloat16* __restrict__ out, long long L, int c) {
  extern __shared__ __nv_bfloat16 sr[];                   // [c][kCondRows]
  const long long r0 = (long long)blockIdx.x * kCondRows;
  const int rows = (int)min((long long)kCondRows, L - r0);
  const int w = 2 * c + 1;
  float a = 0.f, b = 0.f;
  if (r) {
    a = *coef_a;
    b = *coef_b;
    for (int i = threadIdx.x; i < c * kCondRows; i += blockDim.x) {
      const int k = i / kCondRows, j = i - k * kCondRows;
      if (j < rows) sr[i] = r[(long long)k * L + r0 + j];
    }
    __syncthreads();
  }
  __nv_bfloat16* o = out + r0 * w;
  for (int i = threadIdx.x; i < rows * w; i += blockDim.x) {
    const int j = i / w, col = i - j * w;
    const long long row = r0 + j;
    __nv_bfloat16 v;
    if (col < c) {
      v = noise[row * c + col];
    } else if (col < 2 * c) {
      const int k = col - c;
      v = latent[row * c + k];
      if (r) {
        const float aug = rbf(__fadd_rn(rbf(__fmul_rn(__bfloat162float(noise[row * c + k]), 0.1f)),
                                        rbf(__fmul_rn(__bfloat162float(sr[k * kCondRows + j]), 0.05f))));
        v = __float2bfloat16_rn(__fadd_rn(__fmul_rn(a, __bfloat162float(v)), __fmul_rn(b, aug)));
      }
    } else {
      v = __float2bfloat16_rn(1.0f);
    }
    o[i] = v;
  }
}

inline int grid_for(long long n, int per_block = 256, int waves = 16) {
  long long g = (n + per_block - 1) / per_block;
  const long long cap = (long long)num_sms() * waves;
  if (g > cap) g = cap;
  return (int)(g < 1 ? 1 : g);
}

}  // namespace
}  // namespace svr2

using namespace svr2;

template <int LAYOUT>
static void launch_input_noise(bool vec, const void* x, const void* noise, void* out, int frames, int plane,
                               long long pixels, float c1, float c2, cudaStream_t s) {
  const __nv_bfloat16* xb = (const __nv_bfloat16*)x;
  const __nv_bfloat16* nb = (const __nv_bfloat16*)noise;
  if (vec)
    input_noise_kernel<LAYOUT, true><<<grid_for(pixels / 8), 256, 0, s>>>(xb, nb, (__nv_bfloat16*)out, frames, plane,
                                                                          pixels, c1, c2);
  else
    input_noise_kernel<LAYOUT, false><<<grid_for(pixels), 256, 0, s>>>(xb, nb, (__nv_bfloat16*)out, frames, plane,
                                                                       pixels, c1, c2);
}

extern "C" int svr2_input_noise_bf16(const void* x, const void* noise, int noise_layout, void* out, int frames,
                                     int64_t plane, float c1, float c2, void* stream) {
  if (frames <= 0 || plane <= 0) return set_error(SVR2_ERR_ARG, "svr2_input_noise_bf16: empty input");
  if (plane >= ((int64_t)1 << 31)) return set_error(SVR2_ERR_ARG, "svr2_input_noise_bf16: plane must be < 2^31");
  if (!x || !noise || !out) return set_error(SVR2_ERR_ARG, "svr2_input_noise_bf16: null tensor");
  if (noise_layout < 0 || noise_layout > 2)
    return set_error(SVR2_ERR_ARG, "svr2_input_noise_bf16: noise_layout must be 0, 1 or 2");
  const long long pixels = (long long)frames * plane;
  cudaStream_t s = (cudaStream_t)stream;
  const bool vec = plane % 8 == 0 && ((uintptr_t)x | (uintptr_t)noise | (uintptr_t)out) % 16 == 0;
  if (noise_layout == 0)
    launch_input_noise<0>(vec, x, noise, out, frames, (int)plane, pixels, c1, c2, s);
  else if (noise_layout == 1)
    launch_input_noise<1>(vec, x, noise, out, frames, (int)plane, pixels, c1, c2, s);
  else
    launch_input_noise<2>(vec, x, noise, out, frames, (int)plane, pixels, c1, c2, s);
  return check_launch("input_noise");
}

extern "C" int svr2_sr_condition_bf16(const void* noise, const void* latent, const void* latent_noise,
                                      const float* coef_a, const float* coef_b, void* out, int64_t rows, int channels,
                                      void* stream) {
  if (rows <= 0 || channels <= 0) return set_error(SVR2_ERR_ARG, "svr2_sr_condition_bf16: empty input");
  if (channels > 64) return set_error(SVR2_ERR_ARG, "svr2_sr_condition_bf16: channels must be <= 64");
  if (rows * (2 * channels + 1) >= ((int64_t)1 << 31))
    return set_error(SVR2_ERR_ARG, "svr2_sr_condition_bf16: rows * (2 * channels + 1) must be < 2^31");
  if (!noise || !latent || !out) return set_error(SVR2_ERR_ARG, "svr2_sr_condition_bf16: null tensor");
  if (latent_noise && (!coef_a || !coef_b))
    return set_error(SVR2_ERR_ARG, "svr2_sr_condition_bf16: latent_noise needs both coefficients");
  const int blocks = (int)((rows + kCondRows - 1) / kCondRows);
  const size_t smem = latent_noise ? (size_t)channels * kCondRows * sizeof(__nv_bfloat16) : 0;
  sr_condition_kernel<<<blocks, 256, smem, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)noise, (const __nv_bfloat16*)latent, (const __nv_bfloat16*)latent_noise, coef_a, coef_b,
      (__nv_bfloat16*)out, rows, channels);
  return check_launch("sr_condition");
}
