// Alpha channel of RGBA clips (edge_guided_alpha_upscale, src/core/alpha_upscaling.py:289-438): the input alpha is
// resized to the output size and refined by a guided filter whose guide is the decoded RGB; binary masks are then
// tightened around the RGB's Sobel edges.  Everything the reference does in fp32 torch passes, OpenCV on the host
// and three host round trips runs here as HBM-bound kernels; the branch decisions (binary mask or gradient alpha,
// whether the guide is normalised from [-1, 1]) are device flags in the scratch header, read by the later kernels, so
// the sequence makes no host synchronisation and captures into a CUDA graph.
//
//   alpha_init / alpha_stats / alpha_finalize   :319-334  binary-mask ratio of the alpha, global min of the guide
//   alpha_resize_kernel                         :342-348  antialiased bicubic resize of the alpha, clamp(0, 1)
//   sobel_sq_kernel                             :125-188  RGB -> uint8 -> gray -> 3x3 Sobel (reflect-101):
//                                                         gx^2 + gy^2 and the per-frame maximum
//   guided_a_kernel                             :234-273  box means of I, p, I*I, I*p -> coefficients a, b
//   guided_b_kernel                             :276-286, 370-426  box means of a, b -> q, the binary-mask
//                                                         refinement, clamp(0, 1)
//
// Rounding follows the reference's fp32 torch ops one by one (no FMA contraction where torch rounds the product);
// window sums run in the order of ATen's avg_pool2d (row-major over the window).  The Sobel edges are reproduced bit
// for bit: every step there is integer or correctly rounded.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "aa_resize.cuh"
#include "svr2_internal.h"

namespace svr2 {
namespace {

// Scratch header.  The first six words are part of the ABI (include/svr2.h).
struct AlphaHdr {
  int binary;          // binary_ratio > 0.95
  int normalise;       // guide.min() < 0: guide = (rgb + 1) / 2
  int normalise_twice; // the edge detector's own min() < 0 on the normalised guide: once more (x + 1) / 2
  int radius;          // guided-filter radius: 2 (binary) or 3
  float ratio;         // binary_ratio
  float rgb_min;       // min of the guide before normalisation
  int min_key;         // order-preserving integer key of the running min
  int pad;
  unsigned long long n_low, n_high;   // count(alpha < 0.1), count(alpha > 0.9)
};
constexpr int kTile = 32;          // output tile edge of the stencil kernels (256 threads, 4 rows each)
constexpr float kEps = 0.002f;     // guided-filter eps (alpha_upscaling.py:367, 422)

__device__ __forceinline__ int min_key(float f) { const int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__device__ __forceinline__ float key_min(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }
__device__ __forceinline__ float bf(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float half01(float x) { return __fdiv_rn(__fadd_rn(x, 1.f), 2.f); }   // (x + 1) / 2

__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i < 0 ? 0 : (i >= n ? n - 1 : i);
}

// Guide value of one channel and the grayscale guide I = guide.mean(dim=1) as torch's CUDA reduction computes it on the
// reference's GPU tensor: the channel sum in order, then MeanOps' multiply by its fp32 factor (guide_factor)
__device__ __forceinline__ float guide_gray(const __nv_bfloat16* px, long long plane, int norm, float factor) {
  float c[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float v = bf(px + k * plane);
    c[k] = norm ? half01(v) : v;
  }
  return __fmul_rn(__fadd_rn(__fadd_rn(c[0], c[1]), c[2]), factor);
}

// ATen's mean factor, float(outputs) / numel with numel converted to float: fl(1/3) unless 3 T H W rounds in fp32
inline float guide_factor(long long outputs) { return (float)outputs / (float)(3 * outputs); }

// cv2.cvtColor(RGB2GRAY) of the uint8 image made by detect_edges_batch (:148-159)
__device__ __forceinline__ int gray_u8(const __nv_bfloat16* px, long long plane, int norm, int twice) {
  int u[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float x = bf(px + k * plane);
    if (norm) x = half01(x);
    if (twice) x = half01(x);
    const float y = fminf(fmaxf(__fmul_rn(x, 255.f), 0.f), 255.f);
    u[k] = (int)y;
  }
  return (9798 * u[0] + 19235 * u[1] + 3735 * u[2] + (1 << 14)) >> 15;
}

// edges = uint8(sqrt(s) / sqrt(max s) * 255) / 255 in fp64 as numpy does (:166-174); a flat frame gives 0
__device__ __forceinline__ float edge_value(unsigned s, unsigned smax) {
  if (smax == 0) return 0.f;
  const double e = sqrt((double)s) / sqrt((double)smax) * 255.0;
  return __fdiv_rn((float)(int)e, 255.f);
}

__global__ void alpha_init_kernel(AlphaHdr* __restrict__ hdr, unsigned* __restrict__ frame_max, int frames) {
  if (threadIdx.x == 0) {
    hdr->min_key = 0x7fffffff;
    hdr->n_low = hdr->n_high = 0ull;
  }
  for (int t = threadIdx.x; t < frames; t += blockDim.x) frame_max[t] = 0u;
}

// One pass over the alpha (channel `chan` of `channels`, rounded to bf16 on load) and over the guide.
template <typename T>
__global__ void __launch_bounds__(256) alpha_stats_kernel(const T* __restrict__ alpha, int channels, long long n_alpha,
                                                          const __nv_bfloat16* __restrict__ rgb, long long n_rgb,
                                                          AlphaHdr* __restrict__ hdr) {
  unsigned long long lo = 0, hi = 0;
  float m = INFINITY;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long long i = i0; i < n_alpha; i += stride) {
    const float a = load_bf16_rounded<T>(alpha + i * channels + (channels - 1));
    lo += a < 0.1f;
    hi += a > 0.9f;
  }
  for (long long i = i0; i < n_rgb; i += stride) m = fminf(m, bf(rgb + i));
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    lo += __shfl_xor_sync(0xffffffffu, lo, o);
    hi += __shfl_xor_sync(0xffffffffu, hi, o);
    m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (lo) atomicAdd(&hdr->n_low, lo);
    if (hi) atomicAdd(&hdr->n_high, hi);
    atomicMin(&hdr->min_key, min_key(m));
  }
}

// The flags, in the reference's fp32 order: (near_zero.float() + near_one.float()) / numel > 0.95, the division by
// the Python int numel as torch's CUDA kernel does it: a multiply by fl(1 / fl(numel)) (div_true_kernel_cuda)
__global__ void alpha_finalize_kernel(AlphaHdr* __restrict__ hdr, long long n_alpha, int allow_twice) {
  const float m = key_min(hdr->min_key);
  const int norm = m < 0.f;
  hdr->rgb_min = m;
  hdr->normalise = norm;
  hdr->normalise_twice = allow_twice && norm && half01(m) < 0.f;
  const float ratio = n_alpha > 0 ? __fmul_rn(__fadd_rn(__ull2float_rn(hdr->n_low), __ull2float_rn(hdr->n_high)),
                                              __frcp_rn(__ll2float_rn(n_alpha)))
                                  : 0.f;
  hdr->ratio = ratio;
  hdr->binary = ratio > 0.95f;
  hdr->radius = hdr->binary ? 2 : 3;
}

// F.interpolate(alpha, (H, W), bicubic, antialias=True).clamp(0, 1) in fp32 (:342-348) as torch's CUDA kernel
// computes it on the reference's GPU tensor: its tap tables (aa_resize.cuh) and its accumulation (horizontal taps
// first, then rows, each a product and an fma chain), as in pre.cu's resize; one output channel, input read through
// the channel stride of the frames.
template <typename T>
__global__ void __launch_bounds__(256) alpha_resize_kernel(const T* __restrict__ in, int channels, int h, int w,
                                                           float* __restrict__ out, int H, int W, int K,
                                                           const int* __restrict__ xfirst, const int* __restrict__ xcount,
                                                           const float* __restrict__ xw, const int* __restrict__ yfirst,
                                                           const int* __restrict__ ycount, const float* __restrict__ yw) {
  const int ox = blockIdx.x * 64 + (threadIdx.x & 63);
  const int oy = blockIdx.y * 4 + (threadIdx.x >> 6);
  const int t = blockIdx.z;
  if (ox >= W || oy >= H) return;
  const int x0 = xfirst[ox], nx = xcount[ox], y0 = yfirst[oy], ny = ycount[oy];
  const float* wx = xw + (long long)ox * K;
  const float* wy = yw + (long long)oy * K;
  const T* base = in + (long long)t * h * w * channels + (channels - 1);
  float acc = 0.f;
  for (int j = 0; j < ny; ++j) {
    const T* row = base + ((long long)(y0 + j) * w + x0) * channels;
    float r = __fmul_rn(load_bf16_rounded<T>(row), wx[0]);
    for (int i = 1; i < nx; ++i) r = __fmaf_rn(load_bf16_rounded<T>(row + (long long)i * channels), wx[i], r);
    acc = (j == 0) ? __fmul_rn(r, wy[j]) : __fmaf_rn(r, wy[j], acc);
  }
  out[((long long)t * H + oy) * W + ox] = fminf(fmaxf(acc, 0.f), 1.f);
}

// gx^2 + gy^2 of cv2.Sobel(gray, CV_64F, 1, 0 / 0, 1, ksize=3, BORDER_REFLECT_101) (exact integers) and the per-frame
// maximum.  The edge value is a monotone function of it, so consumers derive the edges and their 3x3 max-pool from it.
__global__ void __launch_bounds__(256) sobel_sq_kernel(const __nv_bfloat16* __restrict__ rgb, int H, int W,
                                                       unsigned* __restrict__ sq, unsigned* __restrict__ frame_max,
                                                       const AlphaHdr* __restrict__ hdr) {
  constexpr int TW = kTile + 2;
  __shared__ int g[TW * TW];
  const int t = blockIdx.z, x0 = blockIdx.x * kTile, y0 = blockIdx.y * kTile;
  const long long plane = (long long)H * W;
  const __nv_bfloat16* img = rgb + (long long)t * 3 * plane;
  const int norm = hdr->normalise, twice = hdr->normalise_twice;
  for (int i = threadIdx.x; i < TW * TW; i += 256) {
    const int y = reflect101(y0 + i / TW - 1, H), x = reflect101(x0 + i % TW - 1, W);
    g[i] = gray_u8(img + (long long)y * W + x, plane, norm, twice);
  }
  __syncthreads();
  const int tx = threadIdx.x & 31;
  unsigned m = 0;
  for (int ty = threadIdx.x >> 5; ty < kTile; ty += 8) {
    const int y = y0 + ty, x = x0 + tx;
    if (y >= H || x >= W) continue;
    const int* c = g + (ty + 1) * TW + tx + 1;
    const int gx = (c[-TW + 1] - c[-TW - 1]) + 2 * (c[1] - c[-1]) + (c[TW + 1] - c[TW - 1]);
    const int gy = (c[TW - 1] - c[-TW - 1]) + 2 * (c[TW] - c[-TW]) + (c[TW + 1] - c[-TW + 1]);
    const unsigned s = (unsigned)(gx * gx + gy * gy);
    sq[(long long)t * plane + (long long)y * W + x] = s;
    m = max(m, s);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (tx == 0 && m) atomicMax(frame_max + t, m);
}

__global__ void __launch_bounds__(256) edges_kernel(const unsigned* __restrict__ sq, const unsigned* __restrict__ frame_max,
                                                    float* __restrict__ edges, long long plane, long long total) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256)
    edges[i] = edge_value(sq[i], frame_max[i / plane]);
}

// Loads a (kTile + 2R)^2 tile of `src` around the block's outputs, zeros outside the image (avg_pool2d's zero padding:
// adding 0 leaves every partial sum unchanged, so the window sums equal ATen's sums over the valid elements).
template <int R, typename F>
__device__ __forceinline__ void load_tile(float* __restrict__ dst, int x0, int y0, int H, int W, F&& at) {
  constexpr int TW = kTile + 2 * R;
  for (int i = threadIdx.x; i < TW * TW; i += 256) {
    const int y = y0 + i / TW - R, x = x0 + i % TW - R;
    dst[i] = (y >= 0 && y < H && x >= 0 && x < W) ? at(y, x) : 0.f;
  }
}

// Box mean of one window, summed row-major as ATen's avg_pool2d, divided by (2R+1)^2 (count_include_pad)
template <int R>
__device__ __forceinline__ float box_mean(const float* __restrict__ c) {
  constexpr int TW = kTile + 2 * R;
  float s = 0.f;
#pragma unroll
  for (int dy = 0; dy <= 2 * R; ++dy)
#pragma unroll
    for (int dx = 0; dx <= 2 * R; ++dx) s = __fadd_rn(s, c[dy * TW + dx]);
  return __fdiv_rn(s, (float)((2 * R + 1) * (2 * R + 1)));
}

template <int R>
__device__ __forceinline__ void guided_a(float* __restrict__ sI, float* __restrict__ sP,
                                         const __nv_bfloat16* __restrict__ img, const float* __restrict__ p,
                                         float* __restrict__ A, float* __restrict__ B, int H, int W, int norm,
                                         float factor) {
  constexpr int TW = kTile + 2 * R;
  constexpr float K = (float)((2 * R + 1) * (2 * R + 1));
  const int x0 = blockIdx.x * kTile, y0 = blockIdx.y * kTile;
  const long long plane = (long long)H * W;
  load_tile<R>(sI, x0, y0, H, W, [&](int y, int x) { return guide_gray(img + (long long)y * W + x, plane, norm, factor); });
  load_tile<R>(sP, x0, y0, H, W, [&](int y, int x) { return p[(long long)y * W + x]; });
  __syncthreads();
  const int tx = threadIdx.x & 31;
  for (int ty = threadIdx.x >> 5; ty < kTile; ty += 8) {
    const int y = y0 + ty, x = x0 + tx;
    if (y >= H || x >= W) continue;
    const float* ci = sI + ty * TW + tx;
    const float* cp = sP + ty * TW + tx;
    float si = 0.f, sp = 0.f, sii = 0.f, sip = 0.f;
#pragma unroll
    for (int dy = 0; dy <= 2 * R; ++dy)
#pragma unroll
      for (int dx = 0; dx <= 2 * R; ++dx) {
        const float i = ci[dy * TW + dx], v = cp[dy * TW + dx];
        si = __fadd_rn(si, i);
        sp = __fadd_rn(sp, v);
        sii = __fadd_rn(sii, __fmul_rn(i, i));
        sip = __fadd_rn(sip, __fmul_rn(i, v));
      }
    const float mi = __fdiv_rn(si, K), mp = __fdiv_rn(sp, K), cii = __fdiv_rn(sii, K), cip = __fdiv_rn(sip, K);
    const float var = __fsub_rn(cii, __fmul_rn(mi, mi));
    const float cov = __fsub_rn(cip, __fmul_rn(mi, mp));
    const float a = __fdiv_rn(cov, __fadd_rn(var, kEps));
    const long long o = (long long)y * W + x;
    A[o] = a;
    B[o] = __fsub_rn(mp, __fmul_rn(a, mi));
  }
}

// Pass A: one frame per blockIdx.z; the radius comes from the statistics (uniform per launch).
__global__ void __launch_bounds__(256) guided_a_kernel(const __nv_bfloat16* __restrict__ rgb, const float* __restrict__ p,
                                                       float* __restrict__ A, float* __restrict__ B, int H, int W,
                                                       float factor, const AlphaHdr* __restrict__ hdr) {
  __shared__ float sI[(kTile + 6) * (kTile + 6)], sP[(kTile + 6) * (kTile + 6)];
  const long long plane = (long long)H * W, t = blockIdx.z;
  const int norm = hdr->normalise;
  if (hdr->radius == 2)
    guided_a<2>(sI, sP, rgb + t * 3 * plane, p + t * plane, A + t * plane, B + t * plane, H, W, norm, factor);
  else
    guided_a<3>(sI, sP, rgb + t * 3 * plane, p + t * plane, A + t * plane, B + t * plane, H, W, norm, factor);
}

// Steps 3-8 of the binary-mask branch (:370-408) for one pixel: q is the guided-filter output, e the edge value and z
// the 3x3 max-pooled edge value.
__device__ __forceinline__ float binary_refine(float q, float e, float z) {
  const float binary = q > 0.5f ? 1.f : 0.f;
  const float sig = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-__fmul_rn(__fsub_rn(q, 0.5f), 12.f))));
  const float es = fminf(fmaxf(__fdiv_rn(e, 0.25f), 0.f), 1.f);
  const float in_edges = __fadd_rn(__fmul_rn(q, __fsub_rn(1.f, es)), __fmul_rn(sig, es));
  const float combined = z < 0.05f ? binary : in_edges;
  float f = z < 0.03f ? (combined > 0.5f ? 1.f : 0.f) : combined;
  if (f > 0.3f && f < 0.7f && !(e > 0.15f)) f = f > 0.5f ? 1.f : 0.f;
  return f;
}

template <int R, bool BIN>
__device__ __forceinline__ void guided_b(float* __restrict__ sA, float* __restrict__ sB, unsigned* __restrict__ sS,
                                         const __nv_bfloat16* __restrict__ img, const float* __restrict__ A,
                                         const float* __restrict__ B, const unsigned* __restrict__ sq, unsigned smax,
                                         int H, int W, int norm, float factor, int t, float* __restrict__ out_f32,
                                         __nv_bfloat16* __restrict__ out_rgba) {
  constexpr int TW = kTile + 2 * R, SW = kTile + 2;
  const int x0 = blockIdx.x * kTile, y0 = blockIdx.y * kTile;
  const long long plane = (long long)H * W;
  load_tile<R>(sA, x0, y0, H, W, [&](int y, int x) { return A[(long long)y * W + x]; });
  load_tile<R>(sB, x0, y0, H, W, [&](int y, int x) { return B[(long long)y * W + x]; });
  if (BIN) {   // max_pool2d pads with -inf; every s >= 0 and the centre is always inside, so 0 padding gives the same max
    for (int i = threadIdx.x; i < SW * SW; i += 256) {
      const int y = y0 + i / SW - 1, x = x0 + i % SW - 1;
      sS[i] = (y >= 0 && y < H && x >= 0 && x < W) ? sq[(long long)y * W + x] : 0u;
    }
  }
  __syncthreads();
  const int tx = threadIdx.x & 31;
  for (int ty = threadIdx.x >> 5; ty < kTile; ty += 8) {
    const int y = y0 + ty, x = x0 + tx;
    if (y >= H || x >= W) continue;
    const long long o = (long long)y * W + x;
    const float ma = box_mean<R>(sA + ty * TW + tx), mb = box_mean<R>(sB + ty * TW + tx);
    float v = __fadd_rn(__fmul_rn(ma, guide_gray(img + o, plane, norm, factor)), mb);
    if (BIN) {
      const unsigned* c = sS + (ty + 1) * SW + tx + 1;
      unsigned zmax = 0;
#pragma unroll
      for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) zmax = max(zmax, c[dy * SW + dx]);
      v = binary_refine(v, edge_value(c[0], smax), edge_value(zmax, smax));
    }
    v = fminf(fmaxf(v, 0.f), 1.f);
    if (out_rgba)
      out_rgba[((long long)t * plane + o) * 4 + 3] = __float2bfloat16_rn(v);
    else
      out_f32[(long long)t * plane + o] = v;
  }
}

__global__ void __launch_bounds__(256) guided_b_kernel(const __nv_bfloat16* __restrict__ rgb, const float* __restrict__ A,
                                                       const float* __restrict__ B, const unsigned* __restrict__ sq,
                                                       const unsigned* __restrict__ frame_max, int H, int W,
                                                       float factor, const AlphaHdr* __restrict__ hdr,
                                                       float* __restrict__ out_f32,
                                                       __nv_bfloat16* __restrict__ out_rgba) {
  __shared__ float sA[(kTile + 6) * (kTile + 6)], sB[(kTile + 6) * (kTile + 6)];
  __shared__ unsigned sS[(kTile + 2) * (kTile + 2)];
  const long long plane = (long long)H * W;
  const int t = blockIdx.z, norm = hdr->normalise;
  const __nv_bfloat16* img = rgb + (long long)t * 3 * plane;
  if (hdr->binary)
    guided_b<2, true>(sA, sB, sS, img, A + t * plane, B + t * plane, sq + t * plane, frame_max[t], H, W, norm, factor,
                      t, out_f32, out_rgba);
  else
    guided_b<3, false>(sA, sB, sS, img, A + t * plane, B + t * plane, sq + t * plane, 0u, H, W, norm, factor, t,
                       out_f32, out_rgba);
}

// [T,3,hw] -> channels 0..2 of [T,hw,4]: clamp(-1,1) * 0.5 + 0.5 with the rounding of sample_to_image (post.cu);
// channel 3 (the alpha) is left as it is.
__global__ void __launch_bounds__(256) sample_to_image_rgba_kernel(const __nv_bfloat16* __restrict__ in,
                                                                   __nv_bfloat16* __restrict__ out, long long hw,
                                                                   long long total) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long t = i / hw, px = i - t * hw;
    const __nv_bfloat16* p = in + t * 3 * hw + px;
    __nv_bfloat16* q = out + i * 4;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = fminf(fmaxf(bf(p + c * hw), -1.f), 1.f);
      q[c] = __float2bfloat16_rn(rn(v * 0.5f) + 0.5f);
    }
  }
}

inline int grid_for(long long n, int waves = 16) {
  long long b = (n + 255) / 256;
  const long long cap = (long long)num_sms() * waves;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

// scratch: header + per-frame Sobel maxima | gx^2+gy^2 plane | tap tables | p | a | b
struct Layout {
  size_t hdr, sq, tables, plane, total;
  int K, L;
};
inline Layout layout(int frames, int h, int w, int H, int W) {
  Layout l;
  const size_t n = (size_t)frames * H * W;
  l.hdr = align256(sizeof(AlphaHdr) + (size_t)frames * sizeof(unsigned));
  l.sq = align256(n * sizeof(unsigned));
  l.K = taps_for(h, H) > taps_for(w, W) ? taps_for(h, H) : taps_for(w, W);
  l.L = H > W ? H : W;
  l.tables = 2 * align256((size_t)l.L * 2 * sizeof(int)) + 2 * align256((size_t)l.L * l.K * sizeof(float));
  l.plane = align256(n * sizeof(float));
  l.total = l.hdr + l.sq + l.tables + 3 * l.plane;
  return l;
}

inline unsigned* frame_max_of(void* scratch) { return (unsigned*)((uint8_t*)scratch + sizeof(AlphaHdr)); }

int launch_stats(const void* alpha, int dtype, int channels, long long n_alpha, const void* rgb, long long n_rgb,
                 int frames, void* scratch, int allow_twice, cudaStream_t s) {
  AlphaHdr* hdr = (AlphaHdr*)scratch;
  alpha_init_kernel<<<1, 256, 0, s>>>(hdr, frame_max_of(scratch), frames);
  const int grid = grid_for(n_rgb > n_alpha ? n_rgb : n_alpha, 4);
#define SVR2_STATS(T) \
  alpha_stats_kernel<T><<<grid, 256, 0, s>>>((const T*)alpha, channels, n_alpha, (const __nv_bfloat16*)rgb, n_rgb, hdr)
  if (dtype == 0) SVR2_STATS(float);
  else if (dtype == 1) SVR2_STATS(__nv_bfloat16);
  else if (dtype == 2) SVR2_STATS(__half);
  else SVR2_STATS(uint8_t);
#undef SVR2_STATS
  alpha_finalize_kernel<<<1, 1, 0, s>>>(hdr, n_alpha, allow_twice);
  return check_launch("alpha_stats");
}

}  // namespace
}  // namespace svr2

using namespace svr2;

extern "C" int64_t svr2_alpha_upscale_scratch_bytes(int frames, int h, int w, int H, int W) {
  if (frames <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0) return 0;
  return (int64_t)layout(frames, h, w, H, W).total;
}

extern "C" int svr2_alpha_upscale(const void* alpha_src, int src_dtype, int src_channels, int frames, int h, int w,
                                  const void* rgb_up, int H, int W, void* out, int out_kind, void* scratch,
                                  int64_t scratch_bytes, void* stream) {
  if (frames <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0) return set_error(SVR2_ERR_ARG, "svr2_alpha_upscale: empty image");
  if (frames > 65535) return set_error(SVR2_ERR_ARG, "svr2_alpha_upscale: at most 65535 frames per call");
  if (src_dtype < 0 || src_dtype > 3)
    return set_error(SVR2_ERR_ARG, "svr2_alpha_upscale: src_dtype 0 fp32 | 1 bf16 | 2 fp16 | 3 uint8");
  if (src_channels != 1 && src_channels != 4)
    return set_error(SVR2_ERR_ARG, "svr2_alpha_upscale: src_channels must be 1 (alpha plane) or 4 (RGBA frames)");
  if (out_kind < 0 || out_kind > 2) return set_error(SVR2_ERR_ARG, "svr2_alpha_upscale: out_kind 0 | 1 | 2");
  if (!alpha_src || !rgb_up || !out) return set_error(SVR2_ERR_ARG, "svr2_alpha_upscale: null pointer");
  const Layout l = layout(frames, h, w, H, W);
  if (l.K > kMaxTaps) return set_error(SVR2_ERR_ARG, "svr2_alpha_upscale: down-scale factor above 7.5 (more than 31 taps)");
  if (!scratch || scratch_bytes < (int64_t)l.total)
    return set_error(SVR2_ERR_ARG, "svr2_alpha_upscale: scratch too small (svr2_alpha_upscale_scratch_bytes)");
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* base = (uint8_t*)scratch;
  AlphaHdr* hdr = (AlphaHdr*)base;
  unsigned* fmax = frame_max_of(scratch);
  unsigned* sq = (unsigned*)(base + l.hdr);
  uint8_t* tab = base + l.hdr + l.sq;
  const size_t seg_i = align256((size_t)l.L * 2 * sizeof(int)), seg_w = align256((size_t)l.L * l.K * sizeof(float));
  int* xfirst = (int*)tab;
  int* xcount = xfirst + l.L;
  int* yfirst = (int*)(tab + seg_i);
  int* ycount = yfirst + l.L;
  float* xw = (float*)(tab + 2 * seg_i);
  float* yw = (float*)(tab + 2 * seg_i + seg_w);
  float* p = (float*)(tab + l.tables);
  float* A = (float*)((uint8_t*)p + l.plane);
  float* B = (float*)((uint8_t*)A + l.plane);
  const long long plane = (long long)H * W;

  int rc = launch_stats(alpha_src, src_dtype, src_channels, (long long)frames * h * w, rgb_up, 3LL * frames * plane,
                        frames, scratch, 1, s);
  if (rc) return rc;
  aa_table_kernel<<<(W + 127) / 128, 128, 0, s>>>(w, W, l.K, xfirst, xcount, xw);
  aa_table_kernel<<<(H + 127) / 128, 128, 0, s>>>(h, H, l.K, yfirst, ycount, yw);
  float* resized = out_kind == 2 ? (float*)out : p;
  const dim3 rgrid((W + 63) / 64, (H + 3) / 4, frames);
#define SVR2_ARESIZE(T)                                                                                                \
  alpha_resize_kernel<T><<<rgrid, 256, 0, s>>>((const T*)alpha_src, src_channels, h, w, resized, H, W, l.K, xfirst, \
                                               xcount, xw, yfirst, ycount, yw)
  if (src_dtype == 0) SVR2_ARESIZE(float);
  else if (src_dtype == 1) SVR2_ARESIZE(__nv_bfloat16);
  else if (src_dtype == 2) SVR2_ARESIZE(__half);
  else SVR2_ARESIZE(uint8_t);
#undef SVR2_ARESIZE
  rc = check_launch("alpha_resize");
  if (rc || out_kind == 2) return rc;
  const dim3 tgrid((W + kTile - 1) / kTile, (H + kTile - 1) / kTile, frames);
  const __nv_bfloat16* rgb = (const __nv_bfloat16*)rgb_up;
  sobel_sq_kernel<<<tgrid, 256, 0, s>>>(rgb, H, W, sq, fmax, hdr);
  const float factor = guide_factor((long long)frames * plane);
  guided_a_kernel<<<tgrid, 256, 0, s>>>(rgb, p, A, B, H, W, factor, hdr);
  guided_b_kernel<<<tgrid, 256, 0, s>>>(rgb, A, B, sq, fmax, H, W, factor, hdr, out_kind == 0 ? (float*)out : nullptr,
                                        out_kind == 1 ? (__nv_bfloat16*)out : nullptr);
  return check_launch("alpha_guided_filter");
}

extern "C" int svr2_sobel_edges_f32(const void* rgb_up, int frames, int H, int W, float* edges, void* scratch,
                                    int64_t scratch_bytes, void* stream) {
  if (frames <= 0 || H <= 0 || W <= 0) return set_error(SVR2_ERR_ARG, "svr2_sobel_edges_f32: empty image");
  if (frames > 65535) return set_error(SVR2_ERR_ARG, "svr2_sobel_edges_f32: at most 65535 frames per call");
  if (!rgb_up || !edges) return set_error(SVR2_ERR_ARG, "svr2_sobel_edges_f32: null pointer");
  const Layout l = layout(frames, 1, 1, H, W);
  if (!scratch || scratch_bytes < (int64_t)(l.hdr + l.sq))
    return set_error(SVR2_ERR_ARG, "svr2_sobel_edges_f32: scratch too small (svr2_alpha_upscale_scratch_bytes)");
  cudaStream_t s = (cudaStream_t)stream;
  const long long plane = (long long)H * W;
  int rc = launch_stats(nullptr, 0, 1, 0, rgb_up, 3LL * frames * plane, frames, scratch, 0, s);
  if (rc) return rc;
  unsigned* sq = (unsigned*)((uint8_t*)scratch + l.hdr);
  const dim3 tgrid((W + kTile - 1) / kTile, (H + kTile - 1) / kTile, frames);
  sobel_sq_kernel<<<tgrid, 256, 0, s>>>((const __nv_bfloat16*)rgb_up, H, W, sq, frame_max_of(scratch),
                                        (const AlphaHdr*)scratch);
  const long long total = (long long)frames * plane;
  edges_kernel<<<grid_for(total), 256, 0, s>>>(sq, frame_max_of(scratch), edges, plane, total);
  return check_launch("sobel_edges");
}

extern "C" int svr2_sample_to_image_rgba_bf16(const void* sample, void* image, int frames, int64_t hw, void* stream) {
  if (frames <= 0 || hw <= 0) return set_error(SVR2_ERR_ARG, "svr2_sample_to_image_rgba_bf16: empty input");
  const long long total = (long long)frames * hw;
  sample_to_image_rgba_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)sample,
                                                                                 (__nv_bfloat16*)image, hw, total);
  return check_launch("sample_to_image_rgba");
}
