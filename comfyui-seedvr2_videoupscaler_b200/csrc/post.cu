// Post-decode colour correction and image formatting (SURVEY.md §8(f) rank 2): the step right after the VAE
// decode in the reference's phase 4 (generation_phases.py:1236-1345), as HBM-bound kernels.
//
//   wavelet_level_kernel   color_fix.py:122-184   one level of the a-trous (1,2,1)x(1,2,1)/16 pyramid, the
//                                                 high-frequency accumulation and the final recombination fused
//   adain_*                color_fix.py:72-119    per-(frame, channel) mean / unbiased std, normalise + restyle
//   rgb_to_lab / lab_to_rgb color_fix.py:368-474  sRGB <-> CIELAB (D65), fp32
//   histogram match        color_fix.py:477-521   exact rank mapping: radix sort (CUB) + scatter
//   sample_to_image        generation_phases.py:1322-1345   t c h w -> t h w c, clamp, [-1,1] -> [0,1]
//   sample_to_image_u8     + inference_cli.py:763           the same, then the CLI's * 255 -> uint8, in one pass
//
// Rounding points follow the reference's bf16 flow (every torch op on a bf16 tensor rounds once); the LAB
// part runs in fp32 as the reference does (ensure_float32_precision, color_fix.py:299-301).
#include <cub/device/device_radix_sort.cuh>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>

#include "svr2_internal.h"

namespace svr2 {
namespace {

__device__ __forceinline__ float bf2f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float rn(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }   // one rounding point

// Storage of the wavelet planes: bf16 rounds at every reference rounding point (the pipeline's compute dtype),
// fp32 is the same flow without intermediate rounding (wavelet_adaptive_color_correction casts its inputs to
// fp32 first, color_fix.py:808-812).
__device__ __forceinline__ float ld(__nv_bfloat16 v) { return bf2f(v); }
__device__ __forceinline__ float ld(float v) { return v; }
template <typename T> __device__ __forceinline__ float rnd(float x) { return rn(x); }
template <> __device__ __forceinline__ float rnd<float>(float x) { return x; }
template <typename T> __device__ __forceinline__ T cvt(float x) { return __float2bfloat16_rn(x); }
template <> __device__ __forceinline__ float cvt<float>(float x) { return x; }

// ---------------------------------------------------------------------------------------------------------
// One wavelet level on `planes` images of H x W (planar; img in TIn, the other planes in T):
//   low      = rnd( sum_{dy,dx} k[dy] k[dx] img[clamp(y + dy r)][clamp(x + dx r)] ),  k = (1,2,1)/4
//   high     = rnd( rnd(high + img) - low )        (content pass; `first` => high starts at 0)
//   out      = clamp( rnd(add_to + low), -1, 1 )   (last level of the style pass: content high + style low)
// bf16: the nine products are exact (bf16 x power of two) and the fp32 sum is order-independent up to the last
// fp32 bit, so `low` matches the reference's conv2d bit for bit in practice.  fp32: the taps are summed in the
// order of color_oracle.wavelet_blur (dy outer, dx inner, one rounded add each), so the sum is reproducible.
// Grid: (ceil(W / 256), H, planes); a thread owns two horizontally adjacent pixels.
template <typename TIn, typename T>
__global__ void __launch_bounds__(128) wavelet_level_kernel(const TIn* __restrict__ img, T* __restrict__ low,
                                                            T* __restrict__ high, const T* __restrict__ add_to,
                                                            T* __restrict__ out, int H, int W, int r, int first) {
  const int x0 = (blockIdx.x * 128 + threadIdx.x) * 2;
  if (x0 >= W) return;
  const int y = blockIdx.y;
  const long long plane = (long long)blockIdx.z * H * W;
  const TIn* p = img + plane;
  const int ym = max(y - r, 0), yp = min(y + r, H - 1);
  const int rows[3] = {ym, y, yp};
  float acc[2] = {0.f, 0.f};
#pragma unroll
  for (int px = 0; px < 2; ++px) {
    const int x = min(x0 + px, W - 1);
    const int xm = max(x - r, 0), xp = min(x + r, W - 1);
    float s = 0.f;
    if constexpr (std::is_same<T, float>::value) {
      const int cols[3] = {xm, x, xp};
      const float k[3] = {0.25f, 0.5f, 0.25f};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const TIn* row = p + (long long)rows[i] * W;
#pragma unroll
        for (int j = 0; j < 3; ++j) s = __fadd_rn(s, __fmul_rn(ld(row[cols[j]]), k[i] * k[j]));
      }
    } else {
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const TIn* row = p + (long long)rows[i] * W;
        const float h = 0.25f * ld(row[xm]) + 0.5f * ld(row[x]) + 0.25f * ld(row[xp]);
        s += (i == 1 ? 0.5f : 0.25f) * h;
      }
    }
    acc[px] = s;
  }
  const long long o = plane + (long long)y * W + x0;
  const bool two = (x0 + 1 < W);
#pragma unroll
  for (int px = 0; px < 2; ++px) {
    if (px == 1 && !two) break;
    const float lo = rnd<T>(acc[px]);
    if (add_to) {
      const float v = rnd<T>(ld(add_to[o + px]) + lo);
      out[o + px] = cvt<T>(fminf(fmaxf(v, -1.f), 1.f));
    } else {
      low[o + px] = cvt<T>(lo);
    }
    if (high) {
      const float im = ld(p[(long long)y * W + x0 + px]);
      const float hprev = first ? 0.f : ld(high[o + px]);
      high[o + px] = cvt<T>(rnd<T>(hprev + im) - lo);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// AdaIN statistics: one block per plane of content and of style; stats[plane] = (mean, std) with the
// reference's bf16 rounding of mean, var, var + eps and sqrt (calc_mean_std, color_fix.py:72-91).
__global__ void __launch_bounds__(1024) adain_stats_kernel(const __nv_bfloat16* __restrict__ content,
                                                           const __nv_bfloat16* __restrict__ style, long long n,
                                                           int planes, float eps, float2* __restrict__ stats) {
  const int pl = blockIdx.x;
  const __nv_bfloat16* p = (pl < planes ? content + (long long)pl * n : style + (long long)(pl - planes) * n);
  double s = 0.0, ss = 0.0;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = (double)bf2f(p[i]);
    s += v;
    ss += v * v;
  }
  __shared__ double sh[2][32];
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s; sh[1][threadIdx.x >> 5] = ss; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0.0, SS = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { S += sh[0][i]; SS += sh[1][i]; }   // fixed order
    const double mean = S / (double)n;
    const double var = n > 1 ? (SS - S * mean) / (double)(n - 1) : 0.0;
    const float var_eps = rn(rn((float)var) + eps);
    stats[pl] = make_float2(rn((float)mean), rn(sqrtf(var_eps)));
  }
}

__global__ void __launch_bounds__(256) adain_apply_kernel(const __nv_bfloat16* __restrict__ content,
                                                          __nv_bfloat16* __restrict__ out, long long n, int planes,
                                                          const float2* __restrict__ stats) {
  const int pl = blockIdx.y;
  const float2 c = stats[pl], s = stats[planes + pl];
  const __nv_bfloat16* p = content + (long long)pl * n;
  __nv_bfloat16* q = out + (long long)pl * n;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float nrm = rn(rn(bf2f(p[i]) - c.x) / c.y);
    q[i] = __float2bfloat16_rn(rn(nrm * s.y) + s.x);
  }
}

// ---------------------------------------------------------------------------------------------------------
// sRGB <-> CIELAB (D65), color_fix.py:299-321, 368-474.  epsilon^3 and kappa are the fp32 casts of the reference's
// double constants ((6/29)^3 = 216/24389, (29/3)^3 = 24389/27); cubing the fp32 quotients instead gives values one
// ulp higher (0.008856453, 903.2964), which shifts every dark pixel's L*, a*, b*.
constexpr float kLabEps3 = (float)(216.0 / 24389.0);
constexpr float kLabKappa = (float)(24389.0 / 27.0);
__device__ __forceinline__ float lab_f(float t) {
  return t > kLabEps3 ? powf(t, 1.0f / 3.0f) : (t * kLabKappa + 16.0f) / 116.0f;
}
__device__ __forceinline__ float lab_finv(float f) {
  return f > (6.0f / 29.0f) ? powf(f, 3.0f) : (f * 116.0f - 16.0f) / kLabKappa;
}

// rgb: [T,3,hw] bf16 in [-1,1]  ->  lab: [3][T*hw] fp32 (channel-major: each channel is one sortable array)
__global__ void __launch_bounds__(256) rgb_to_lab_kernel(const __nv_bfloat16* __restrict__ rgb,
                                                         float* __restrict__ lab, long long hw, long long total) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long t = i / hw, px = i - t * hw;
    const __nv_bfloat16* p = rgb + t * 3 * hw + px;
    float lin[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = (bf2f(p[c * hw]) + 1.0f) * 0.5f;
      v = fminf(fmaxf(v, 0.f), 1.f);
      lin[c] = v > 0.04045f ? powf((v + 0.055f) / 1.055f, 2.4f) : v / 12.92f;
    }
    const float X = (lin[0] * 0.4124564f + lin[1] * 0.3575761f + lin[2] * 0.1804375f) / 0.95047f;
    const float Y = lin[0] * 0.2126729f + lin[1] * 0.7151522f + lin[2] * 0.0721750f;
    const float Z = (lin[0] * 0.0193339f + lin[1] * 0.1191920f + lin[2] * 0.9503041f) / 1.08883f;
    const float fx = lab_f(X), fy = lab_f(Y), fz = lab_f(Z);
    lab[i] = fy * 116.0f - 16.0f;
    lab[total + i] = (fx - fy) * 500.0f;
    lab[2 * total + i] = (fy - fz) * 200.0f;
  }
}

// L = L_content * lw + L_matched * (1 - lw) (or L_content when L_matched is null), a, b: [T*hw] fp32
// -> rgb [T,3,hw] bf16 in [-1,1]
__global__ void __launch_bounds__(256) lab_to_rgb_kernel(const float* __restrict__ Lc, const float* __restrict__ Lm,
                                                         const float* __restrict__ a, const float* __restrict__ b,
                                                         float lw, float lw1, __nv_bfloat16* __restrict__ rgb,
                                                         long long hw, long long total) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const float L = Lm ? Lc[i] * lw + Lm[i] * lw1 : Lc[i];
    const float fy = (L + 16.0f) / 116.0f;
    const float fx = a[i] / 500.0f + fy;
    const float fz = fy - b[i] / 200.0f;
    const float X = lab_finv(fx) * 0.95047f, Y = lab_finv(fy), Z = lab_finv(fz) * 1.08883f;
    float lin[3];
    lin[0] = X * 3.2404542f + Y * -1.5371385f + Z * -0.4985314f;
    lin[1] = X * -0.9692660f + Y * 1.8760108f + Z * 0.0415560f;
    lin[2] = X * 0.0556434f + Y * -0.2040259f + Z * 1.0572252f;
    const long long t = i / hw, px = i - t * hw;
    __nv_bfloat16* q = rgb + t * 3 * hw + px;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = lin[c] > 0.0031308f ? powf(fmaxf(lin[c], 0.f), 1.0f / 2.4f) * 1.055f - 0.055f : lin[c] * 12.92f;
      v = fminf(fmaxf(v, 0.f), 1.f);
      q[c * hw] = __float2bfloat16_rn(v * 2.0f - 1.0f);
    }
  }
}

__global__ void __launch_bounds__(256) iota_kernel(uint32_t* __restrict__ idx, long long n) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
    idx[i] = (uint32_t)i;
}
// out[position of the r-th smallest source element] = r-th smallest reference value
__global__ void __launch_bounds__(256) rank_scatter_kernel(const uint32_t* __restrict__ order,
                                                           const float* __restrict__ ref_sorted,
                                                           float* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
    out[order[i]] = ref_sorted[i];
}

// [T,3,hw] -> [T,hw,3], clamp(-1,1) * 0.5 + 0.5 with the reference's bf16 rounding (mul exact, add rounds)
__global__ void __launch_bounds__(256) sample_to_image_kernel(const __nv_bfloat16* __restrict__ in,
                                                              __nv_bfloat16* __restrict__ out, long long hw,
                                                              long long total) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long t = i / hw, px = i - t * hw;
    const __nv_bfloat16* p = in + t * 3 * hw + px;
    __nv_bfloat16* q = out + i * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = fminf(fmaxf(bf2f(p[c * hw]), -1.f), 1.f);
      q[c] = __float2bfloat16_rn(rn(v * 0.5f) + 0.5f);
    }
  }
}

// The CLI's 8-bit frames (inference_cli.py:590, 763, 809: (frames.float() * 255.0).astype(uint8)) straight from the
// sample: the image value of sample_to_image_kernel, one fp32 product (no FMA), truncated.  Image values lie in [0, 1];
// an alpha outside it saturates (NaN -> 0), where numpy's cast is undefined.
__device__ __forceinline__ float image_value(float s) {
  const float v = fminf(fmaxf(s, -1.f), 1.f);
  return rn(rn(v * 0.5f) + 0.5f);
}
__device__ __forceinline__ uint32_t to_byte(float x) {
  return __float2uint_rz(fminf(fmaxf(__fmul_rn(x, 255.0f), 0.f), 255.f));
}

// [T,3,hw] bf16 (+ channel 3 of an RGBA bf16 image [T,hw,4] when C == 4) -> [T,hw,C] uint8, one pixel per thread
template <int C>
__global__ void __launch_bounds__(256) sample_to_image_u8_kernel(const __nv_bfloat16* __restrict__ in,
                                                                 const __nv_bfloat16* __restrict__ rgba,
                                                                 uint8_t* __restrict__ out, long long hw,
                                                                 long long total) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long t = i / hw, px = i - t * hw;
    const __nv_bfloat16* p = in + t * 3 * hw + px;
    uint8_t* q = out + i * C;
#pragma unroll
    for (int c = 0; c < 3; ++c) q[c] = (uint8_t)to_byte(image_value(bf2f(p[c * hw])));
    if (C == 4) q[3] = (uint8_t)to_byte(bf2f(rgba[i * 4 + 3]));
  }
}

// The same for hw % 4 == 0 and aligned buffers: four pixels per thread, 8-byte loads per channel plane, the 4*C output
// bytes stored as C 32-bit words
template <int C>
__global__ void __launch_bounds__(256) sample_to_image_u8_x4_kernel(const uint2* __restrict__ in,
                                                                    const __nv_bfloat16* __restrict__ rgba,
                                                                    uint32_t* __restrict__ out, long long hw4,
                                                                    long long total4) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total4; i += (long long)gridDim.x * 256) {
    const long long t = i / hw4, g = i - t * hw4;
    const uint2* p = in + t * 3 * hw4 + g;
    uint32_t b[4 * C];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const uint2 v = p[c * hw4];
      const uint32_t w[4] = {v.x << 16, v.x & 0xffff0000u, v.y << 16, v.y & 0xffff0000u};
#pragma unroll
      for (int k = 0; k < 4; ++k) b[k * C + c] = to_byte(image_value(__uint_as_float(w[k])));
    }
    if (C == 4) {
#pragma unroll
      for (int k = 0; k < 4; ++k) b[k * C + 3] = to_byte(bf2f(rgba[(i * 4 + k) * 4 + 3]));
    }
    uint32_t* q = out + i * C;
#pragma unroll
    for (int j = 0; j < C; ++j)
      q[j] = b[4 * j] | (b[4 * j + 1] << 8) | (b[4 * j + 2] << 16) | (b[4 * j + 3] << 24);
  }
}

// Temporal-overlap cross-fade (blend_overlapping_frames, generation_utils.py:284-312):
// out = rn(rn(prev * w_prev[f]) + rn(cur * w_cur[f])), frames of `frame_elems` bf16 values, 8 per thread
__global__ void __launch_bounds__(256) blend_overlap_kernel(const uint4* __restrict__ prev, const uint4* __restrict__ cur,
                                                            uint4* __restrict__ out, const float* __restrict__ w_prev,
                                                            const float* __restrict__ w_cur, long long vec_per_frame) {
  const int f = blockIdx.y;
  const float wp = w_prev[f], wc = w_cur[f];
  const long long base = (long long)f * vec_per_frame;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < vec_per_frame; i += (long long)gridDim.x * 256) {
    const uint4 a = prev[base + i], b = cur[base + i];
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float lo = rn(__uint_as_float(aw[e] << 16) * wp) + rn(__uint_as_float(bw[e] << 16) * wc);
      const float hi = rn(__uint_as_float(aw[e] & 0xffff0000u) * wp) + rn(__uint_as_float(bw[e] & 0xffff0000u) * wc);
      const __nv_bfloat162 pk = __floats2bfloat162_rn(lo, hi);
      o[e] = *reinterpret_cast<const uint32_t*>(&pk);
    }
    out[base + i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// fp32 frames (multi-GPU merge, inference_cli.py:1241-1270): prev * w_prev + cur * w_cur with torch's three
// separately rounded ops (no FMA contraction)
__global__ void __launch_bounds__(256) blend_overlap_f32_kernel(const float4* __restrict__ prev,
                                                                const float4* __restrict__ cur, float4* __restrict__ out,
                                                                const float* __restrict__ w_prev,
                                                                const float* __restrict__ w_cur, long long vec_per_frame) {
  const int f = blockIdx.y;
  const float wp = w_prev[f], wc = w_cur[f];
  const long long base = (long long)f * vec_per_frame;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < vec_per_frame; i += (long long)gridDim.x * 256) {
    const float4 a = prev[base + i], b = cur[base + i];
    out[base + i] = make_float4(__fadd_rn(__fmul_rn(a.x, wp), __fmul_rn(b.x, wc)), __fadd_rn(__fmul_rn(a.y, wp), __fmul_rn(b.y, wc)),
                                __fadd_rn(__fmul_rn(a.z, wp), __fmul_rn(b.z, wc)), __fadd_rn(__fmul_rn(a.w, wp), __fmul_rn(b.w, wc)));
  }
}

// The rank-seam cross-fade of a streamed multi-GPU run: fp32 open tail `prev` against a bf16 chunk head `cur`, the
// fp32 value of blend_overlap_f32_kernel on (prev, cur.float()) written to out_f (when not NULL) and its CLI byte
// (to_byte: * 255 without FMA, truncated, saturating, NaN -> 0) to out_b (when not NULL), in one pass.  Frames have
// any element count: with `vec`, the elements from the first multiple of 4 of the flat index on are moved 4 at a time
// (16-byte fp32, 8-byte bf16 and 4-byte u8 accesses, all aligned together), the few before and after one at a time.
template <bool F, bool B>
__device__ __forceinline__ void blend_u8_one(const float* prev, const __nv_bfloat16* cur, float* out_f, uint8_t* out_b,
                                             long long e, float wp, float wc) {
  const float v = __fadd_rn(__fmul_rn(prev[e], wp), __fmul_rn(bf2f(cur[e]), wc));
  if (F) out_f[e] = v;
  if (B) out_b[e] = (uint8_t)to_byte(v);
}

template <bool F, bool B>
__global__ void __launch_bounds__(256) blend_overlap_u8_kernel(const float* __restrict__ prev,
                                                               const __nv_bfloat16* __restrict__ cur,
                                                               float* __restrict__ out_f, uint8_t* __restrict__ out_b,
                                                               const float* __restrict__ w_prev,
                                                               const float* __restrict__ w_cur, long long frame_elems,
                                                               int vec) {
  const int f = blockIdx.y;
  const float wp = w_prev[f], wc = w_cur[f];
  const long long base = (long long)f * frame_elems;
  const long long lead = vec ? min((4 - base % 4) % 4, frame_elems) : frame_elems;   // elements before the body
  const long long nvec = (frame_elems - lead) / 4;
  const long long stride = (long long)gridDim.x * 256, t0 = (long long)blockIdx.x * 256 + threadIdx.x;
  for (long long i = t0; i < nvec; i += stride) {
    const long long e = base + lead + 4 * i;
    const float4 a = *reinterpret_cast<const float4*>(prev + e);
    const uint2 b = *reinterpret_cast<const uint2*>(cur + e);
    const float av[4] = {a.x, a.y, a.z, a.w};
    const float bv[4] = {__uint_as_float(b.x << 16), __uint_as_float(b.x & 0xffff0000u), __uint_as_float(b.y << 16),
                         __uint_as_float(b.y & 0xffff0000u)};
    float v[4];
    uint32_t word = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      v[k] = __fadd_rn(__fmul_rn(av[k], wp), __fmul_rn(bv[k], wc));
      word |= to_byte(v[k]) << (8 * k);
    }
    if (F) *reinterpret_cast<float4*>(out_f + e) = make_float4(v[0], v[1], v[2], v[3]);
    if (B) *reinterpret_cast<uint32_t*>(out_b + e) = word;
  }
  // the scalar elements: [0, lead) and [lead + 4 nvec, frame_elems) of the frame
  const long long rest = frame_elems - 4 * nvec;
  for (long long i = t0; i < rest; i += stride)
    blend_u8_one<F, B>(prev, cur, out_f, out_b, base + (i < lead ? i : 4 * nvec + i), wp, wc);
}

// Spatially tiled VAE (tiled_encode / tiled_decode, attn_video_vae.py:1302-1630): one tile accumulated into the running
// result with separable edge weights, in bf16 with torch's in-place op order — tile.mul_(wh).mul_(ww); result += tile;
// count.addcmul_(wh, ww) — i.e. every product / sum is rounded to bf16 where the reference rounds it.
__global__ void __launch_bounds__(256) tile_accumulate_kernel(const __nv_bfloat16* __restrict__ tile, long long tile_plane,
                                                              int tile_ld, int planes, int eh, int ew,
                                                              const __nv_bfloat16* __restrict__ wh,
                                                              const __nv_bfloat16* __restrict__ ww,
                                                              __nv_bfloat16* __restrict__ result,
                                                              __nv_bfloat16* __restrict__ count, int H, int W, int y0,
                                                              int x0) {
  const long long n = (long long)planes * eh * ew;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int x = (int)(i % ew), y = (int)((i / ew) % eh);
    const long long pl = i / ((long long)ew * eh);
    const float a = __bfloat162float(wh[y]), b = __bfloat162float(ww[x]);
    const float t = rn(rn(__bfloat162float(tile[pl * tile_plane + (long long)y * tile_ld + x]) * a) * b);
    const long long ro = (pl * H + (y0 + y)) * W + (x0 + x);
    result[ro] = __float2bfloat16_rn(__bfloat162float(result[ro]) + t);
    if (pl == 0) {
      const long long co = (long long)(y0 + y) * W + (x0 + x);
      count[co] = __float2bfloat16_rn(fmaf(a, b, __bfloat162float(count[co])));     // addcmul_: one rounding
    }
  }
}
// result.div_(count.clamp(min=1e-6))
__global__ void __launch_bounds__(256) tile_normalize_kernel(__nv_bfloat16* __restrict__ result,
                                                             const __nv_bfloat16* __restrict__ count, int planes,
                                                             long long hw) {
  const long long n = (long long)planes * hw;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float c = rn(fmaxf(__bfloat162float(count[i % hw]), 1e-6f));
    result[i] = __float2bfloat16_rn(__bfloat162float(result[i]) / c);
  }
}
// ramp(n) of vae.py's _tiled on the device: torch.linspace(0, 1, n, dtype=bf16) on CUDA (ATen's kernel in bf16
// arithmetic: step = bf16(1 / bf16(n - 1)); entry i < n / 2 is 0 + step * bf16(i), the rest 1 - step * bf16(n - 1 - i),
// every product and sum rounded), then * pi, cos, * 0.5, 0.5 - (each rounded), and 1 - r behind it
__device__ __forceinline__ float tile_ramp_value(int n, int i) {
  float t = 0.f;
  if (n > 1) {
    const float step = rn(1.0f / rn((float)(n - 1)));
    t = i < n / 2 ? rn(0.0f + rn(step * rn((float)i))) : rn(1.0f - rn(step * rn((float)(n - 1 - i))));
  }
  const float c = rn(cosf(rn(t * (float)M_PI)));
  return rn(0.5f - rn(0.5f * c));
}
__global__ void __launch_bounds__(256) tile_ramp_kernel(__nv_bfloat16* __restrict__ rh, int nh, __nv_bfloat16* __restrict__ rw,
                                                        int nw) {
  for (int i = blockIdx.x * 256 + threadIdx.x; i < nh + nw; i += gridDim.x * 256) {
    __nv_bfloat16* out = i < nh ? rh : rw;
    const int n = i < nh ? nh : nw, j = i < nh ? i : i - nh;
    const float r = tile_ramp_value(n, j);
    out[j] = __float2bfloat16_rn(r);
    out[n + j] = __float2bfloat16_rn(1.0f - r);
  }
}

inline int grid_for(long long n, int per_block = 256, int waves = 16) {
  long long b = (n + per_block - 1) / per_block;
  const long long cap = (long long)num_sms() * waves;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

inline size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

}  // namespace
}  // namespace svr2

using namespace svr2;

// argument checks shared by both storage types; returns the capped dilation, or -1 after set_error
static int wavelet_level_radius(const char* fn, const void* low, const void* add_to, const void* out, int planes,
                                int H, int W, int radius) {
  const char* why = nullptr;
  if (planes <= 0 || H <= 0 || W <= 0) why = "empty image";
  else if (planes > 65535 || H > 65535) why = "planes, H <= 65535";
  else if ((add_to != nullptr) != (out != nullptr)) why = "add_to and out go together";
  else if (!add_to && !low) why = "low is required";
  if (why) {
    char buf[160];
    snprintf(buf, sizeof buf, "%s: %s", fn, why);
    set_error(SVR2_ERR_ARG, buf);
    return -1;
  }
  int cap = (H < W ? H : W) / 8;                          // max_safe_radius, color_fix.py:136-140
  if (cap < 1) cap = 1;
  return radius > cap ? cap : radius;
}

extern "C" int svr2_wavelet_level_bf16(const void* img, void* low, void* high, const void* add_to, void* out,
                                       int planes, int H, int W, int radius, int first, void* stream) {
  const int r = wavelet_level_radius("svr2_wavelet_level_bf16", low, add_to, out, planes, H, W, radius);
  if (r < 0) return SVR2_ERR_ARG;
  dim3 grid((W + 255) / 256, H, planes);
  wavelet_level_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)img, (__nv_bfloat16*)low,
                                                               (__nv_bfloat16*)high, (const __nv_bfloat16*)add_to,
                                                               (__nv_bfloat16*)out, H, W, r, first);
  return check_launch("wavelet_level");
}

extern "C" int svr2_wavelet_level_f32(const void* img, int img_bf16, float* low, float* high, const float* add_to,
                                      float* out, int planes, int H, int W, int radius, int first, void* stream) {
  const int r = wavelet_level_radius("svr2_wavelet_level_f32", low, add_to, out, planes, H, W, radius);
  if (r < 0) return SVR2_ERR_ARG;
  dim3 grid((W + 255) / 256, H, planes);
  if (img_bf16)
    wavelet_level_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)img, low, high, add_to, out, H,
                                                                 W, r, first);
  else
    wavelet_level_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((const float*)img, low, high, add_to, out, H, W, r,
                                                                 first);
  return check_launch("wavelet_level_f32");
}

extern "C" int svr2_adain_bf16(const void* content, const void* style, void* out, int planes, int64_t hw,
                               float* stats_scratch, void* stream) {
  if (planes <= 0 || hw <= 0) return set_error(SVR2_ERR_ARG, "svr2_adain_bf16: empty input");
  if (planes > 65535) return set_error(SVR2_ERR_ARG, "svr2_adain_bf16: planes <= 65535");   // the apply grid's y
  if (!stats_scratch) return set_error(SVR2_ERR_ARG, "svr2_adain_bf16: stats scratch (planes * 4 floats) required");
  cudaStream_t s = (cudaStream_t)stream;
  adain_stats_kernel<<<2 * planes, 1024, 0, s>>>((const __nv_bfloat16*)content, (const __nv_bfloat16*)style, hw,
                                                 planes, 1e-5f, (float2*)stats_scratch);
  int rc = check_launch("adain_stats");
  if (rc) return rc;
  int bx = grid_for(hw, 256, 16) / planes;
  if (bx < 1) bx = 1;
  adain_apply_kernel<<<dim3(bx, planes), 256, 0, s>>>((const __nv_bfloat16*)content, (__nv_bfloat16*)out, hw, planes,
                                                      (const float2*)stats_scratch);
  return check_launch("adain_apply");
}

extern "C" int svr2_rgb_to_lab_f32(const void* rgb, float* lab, int frames, int64_t hw, void* stream) {
  if (frames <= 0 || hw <= 0) return set_error(SVR2_ERR_ARG, "svr2_rgb_to_lab_f32: empty input");
  const long long total = (long long)frames * hw;
  rgb_to_lab_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)rgb, lab, hw, total);
  return check_launch("rgb_to_lab");
}

extern "C" int svr2_lab_to_rgb_bf16(const float* L_content, const float* L_matched, const float* a, const float* b,
                                    float luminance_weight, void* rgb, int frames, int64_t hw, void* stream) {
  if (frames <= 0 || hw <= 0) return set_error(SVR2_ERR_ARG, "svr2_lab_to_rgb_bf16: empty input");
  const long long total = (long long)frames * hw;
  // mul(lw) and mul(1.0 - lw) with the python-double difference cast to fp32 (color_fix.py:337-339)
  const float lw = luminance_weight, lw1 = (float)(1.0 - (double)luminance_weight);
  lab_to_rgb_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(L_content, L_matched, a, b, lw, lw1,
                                                                       (__nv_bfloat16*)rgb, hw, total);
  return check_launch("lab_to_rgb");
}

// scratch layout: keys_out[n] f32 | idx_in[n] u32 | idx_out[n] u32 | ref_sorted[n] f32 | cub temp
static size_t hist_cub_temp(int64_t n) {
  size_t t1 = 0, t2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t1, (const float*)nullptr, (float*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, n);
  cub::DeviceRadixSort::SortKeys(nullptr, t2, (const float*)nullptr, (float*)nullptr, n);
  return t1 > t2 ? t1 : t2;
}

extern "C" int64_t svr2_histogram_match_scratch_bytes(int64_t n) {
  if (n <= 0) return 0;
  return (int64_t)(4 * align256((size_t)n * 4) + align256(hist_cub_temp(n)));
}

extern "C" int svr2_histogram_match_f32(const float* source, const float* reference, float* out, int64_t n,
                                        void* scratch, int64_t scratch_bytes, void* stream) {
  if (n <= 0) return set_error(SVR2_ERR_ARG, "svr2_histogram_match_f32: empty input");
  if (n >= (int64_t)1 << 32) return set_error(SVR2_ERR_ARG, "svr2_histogram_match_f32: n must be < 2^32");
  if (!scratch || scratch_bytes < svr2_histogram_match_scratch_bytes(n))
    return set_error(SVR2_ERR_ARG, "svr2_histogram_match_f32: scratch too small (svr2_histogram_match_scratch_bytes)");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t seg = align256((size_t)n * 4);
  uint8_t* base = (uint8_t*)scratch;
  float* keys_out = (float*)base;
  uint32_t* idx_in = (uint32_t*)(base + seg);
  uint32_t* idx_out = (uint32_t*)(base + 2 * seg);
  float* ref_sorted = (float*)(base + 3 * seg);
  void* temp = base + 4 * seg;
  size_t temp_bytes = hist_cub_temp(n);
  iota_kernel<<<grid_for(n), 256, 0, s>>>(idx_in, n);
  int rc = check_launch("iota");
  if (rc) return rc;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, source, keys_out, idx_in, idx_out, n, 0, 32, s);
  if (e != cudaSuccess) return set_error(SVR2_ERR_CUDA, cudaGetErrorString(e));
  e = cub::DeviceRadixSort::SortKeys(temp, temp_bytes, reference, ref_sorted, n, 0, 32, s);
  if (e != cudaSuccess) return set_error(SVR2_ERR_CUDA, cudaGetErrorString(e));
  rank_scatter_kernel<<<grid_for(n), 256, 0, s>>>(idx_out, ref_sorted, out, n);
  return check_launch("rank_scatter");
}

extern "C" int svr2_sample_to_image_bf16(const void* sample, void* image, int frames, int64_t hw, void* stream) {
  if (frames <= 0 || hw <= 0) return set_error(SVR2_ERR_ARG, "svr2_sample_to_image_bf16: empty input");
  const long long total = (long long)frames * hw;
  sample_to_image_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)sample,
                                                                            (__nv_bfloat16*)image, hw, total);
  return check_launch("sample_to_image");
}

extern "C" int svr2_sample_to_image_u8(const void* sample, const void* alpha_rgba, void* image, int frames, int64_t hw,
                                       void* stream) {
  if (frames <= 0 || hw <= 0) return set_error(SVR2_ERR_ARG, "svr2_sample_to_image_u8: empty input");
  if (!sample || !image) return set_error(SVR2_ERR_ARG, "svr2_sample_to_image_u8: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const long long total = (long long)frames * hw;
  const __nv_bfloat16* a = (const __nv_bfloat16*)alpha_rgba;
  const bool vec = hw % 4 == 0 && ((uintptr_t)sample % 8) == 0 && ((uintptr_t)image % (alpha_rgba ? 16 : 4)) == 0;
  if (vec) {
    const long long total4 = total / 4;
    if (alpha_rgba)
      sample_to_image_u8_x4_kernel<4><<<grid_for(total4), 256, 0, s>>>((const uint2*)sample, a, (uint32_t*)image,
                                                                        hw / 4, total4);
    else
      sample_to_image_u8_x4_kernel<3><<<grid_for(total4), 256, 0, s>>>((const uint2*)sample, a, (uint32_t*)image,
                                                                        hw / 4, total4);
  } else if (alpha_rgba) {
    sample_to_image_u8_kernel<4><<<grid_for(total), 256, 0, s>>>((const __nv_bfloat16*)sample, a, (uint8_t*)image, hw,
                                                                  total);
  } else {
    sample_to_image_u8_kernel<3><<<grid_for(total), 256, 0, s>>>((const __nv_bfloat16*)sample, a, (uint8_t*)image, hw,
                                                                  total);
  }
  return check_launch("sample_to_image_u8");
}

extern "C" int svr2_blend_overlap_bf16(const void* prev_tail, const void* cur_head, void* out, const float* w_prev,
                                       const float* w_cur, int overlap, int64_t frame_elems, void* stream) {
  if (overlap <= 0 || frame_elems <= 0) return set_error(SVR2_ERR_ARG, "svr2_blend_overlap_bf16: empty input");
  if (frame_elems % 8) return set_error(SVR2_ERR_ARG, "svr2_blend_overlap_bf16: frame_elems must be a multiple of 8");
  if (overlap > 65535) return set_error(SVR2_ERR_ARG, "svr2_blend_overlap_bf16: overlap <= 65535");
  const long long vec = frame_elems / 8;
  int bx = grid_for(vec, 256, 8) / overlap;
  if (bx < 1) bx = 1;
  blend_overlap_kernel<<<dim3(bx, overlap), 256, 0, (cudaStream_t)stream>>>((const uint4*)prev_tail, (const uint4*)cur_head,
                                                                             (uint4*)out, w_prev, w_cur, vec);
  return check_launch("blend_overlap");
}

extern "C" int svr2_blend_overlap_f32(const float* prev_tail, const float* cur_head, float* out, const float* w_prev,
                                      const float* w_cur, int overlap, int64_t frame_elems, void* stream) {
  if (overlap <= 0 || frame_elems <= 0) return set_error(SVR2_ERR_ARG, "svr2_blend_overlap_f32: empty input");
  if (frame_elems % 4) return set_error(SVR2_ERR_ARG, "svr2_blend_overlap_f32: frame_elems must be a multiple of 4");
  if (overlap > 65535) return set_error(SVR2_ERR_ARG, "svr2_blend_overlap_f32: overlap <= 65535");
  const long long vec = frame_elems / 4;
  int bx = grid_for(vec, 256, 8) / overlap;
  if (bx < 1) bx = 1;
  blend_overlap_f32_kernel<<<dim3(bx, overlap), 256, 0, (cudaStream_t)stream>>>((const float4*)prev_tail, (const float4*)cur_head,
                                                                                 (float4*)out, w_prev, w_cur, vec);
  return check_launch("blend_overlap_f32");
}

extern "C" int svr2_blend_overlap_u8(const float* prev_tail, const void* cur_head, float* out_f32, void* out_u8,
                                     const float* w_prev, const float* w_cur, int overlap, int64_t frame_elems,
                                     void* stream) {
  if (overlap <= 0 || frame_elems <= 0) return set_error(SVR2_ERR_ARG, "svr2_blend_overlap_u8: empty input");
  if (overlap > 65535) return set_error(SVR2_ERR_ARG, "svr2_blend_overlap_u8: overlap <= 65535");
  if (!prev_tail || !cur_head || !w_prev || !w_cur || (!out_f32 && !out_u8))
    return set_error(SVR2_ERR_ARG, "svr2_blend_overlap_u8: null input, or neither output given");
  const int vec = ((uintptr_t)prev_tail % 16) == 0 && ((uintptr_t)cur_head % 8) == 0 && ((uintptr_t)out_f32 % 16) == 0 &&
                  ((uintptr_t)out_u8 % 4) == 0;
  int bx = grid_for(vec ? frame_elems / 4 + 1 : frame_elems, 256, 8) / overlap;
  if (bx < 1) bx = 1;
  const dim3 grid(bx, overlap);
  cudaStream_t s = (cudaStream_t)stream;
  const __nv_bfloat16* cur = (const __nv_bfloat16*)cur_head;
  uint8_t* ob = (uint8_t*)out_u8;
  if (out_f32 && out_u8)
    blend_overlap_u8_kernel<true, true><<<grid, 256, 0, s>>>(prev_tail, cur, out_f32, ob, w_prev, w_cur, frame_elems, vec);
  else if (out_f32)
    blend_overlap_u8_kernel<true, false><<<grid, 256, 0, s>>>(prev_tail, cur, out_f32, ob, w_prev, w_cur, frame_elems, vec);
  else
    blend_overlap_u8_kernel<false, true><<<grid, 256, 0, s>>>(prev_tail, cur, out_f32, ob, w_prev, w_cur, frame_elems, vec);
  return check_launch("blend_overlap_u8");
}

extern "C" int svr2_tile_accumulate_bf16(const void* tile, int64_t tile_plane_stride, int tile_row_stride, int planes,
                                         int eff_h, int eff_w, const void* weight_h, const void* weight_w, void* result,
                                         void* count, int H, int W, int y0, int x0, void* stream) {
  if (planes <= 0 || eff_h <= 0 || eff_w <= 0) return SVR2_OK;
  if (y0 < 0 || x0 < 0 || y0 + eff_h > H || x0 + eff_w > W)
    return set_error(SVR2_ERR_ARG, "svr2_tile_accumulate_bf16: tile does not fit the result");
  const long long n = (long long)planes * eff_h * eff_w;
  tile_accumulate_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)tile, tile_plane_stride, tile_row_stride, planes, eff_h, eff_w,
      (const __nv_bfloat16*)weight_h, (const __nv_bfloat16*)weight_w, (__nv_bfloat16*)result, (__nv_bfloat16*)count, H, W,
      y0, x0);
  return check_launch("tile_accumulate");
}

extern "C" int svr2_tile_normalize_bf16(void* result, const void* count, int planes, int64_t hw, void* stream) {
  if (planes <= 0 || hw <= 0) return SVR2_OK;
  tile_normalize_kernel<<<grid_for((long long)planes * hw), 256, 0, (cudaStream_t)stream>>>(
      (__nv_bfloat16*)result, (const __nv_bfloat16*)count, planes, hw);
  return check_launch("tile_normalize");
}

int svr2::tile_ramp(void* ramp_h, int len_h, void* ramp_w, int len_w, void* stream) {
  if (len_h < 0 || len_w < 0 || (len_h > 0 && !ramp_h) || (len_w > 0 && !ramp_w))
    return set_error(SVR2_ERR_ARG, "svr2_tile_ramp_bf16: lengths >= 0, tables of positive length not NULL");
  const int n = len_h + len_w;
  if (n == 0) return SVR2_OK;
  tile_ramp_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)ramp_h, len_h, (__nv_bfloat16*)ramp_w,
                                                                     len_w);
  return check_launch("tile_ramp");
}
extern "C" int svr2_tile_ramp_bf16(void* ramp_h, int len_h, void* ramp_w, int len_w, void* stream) {
  return tile_ramp(ramp_h, len_h, ramp_w, len_w, stream);
}
