// HSV colour correction (src/utils/color_fix.py:524-872): hue-conditional saturation histogram matching
// (`hsv`) and its blend into an fp32 wavelet base where the output is over-saturated (`wavelet_adaptive`).
//
//   hsv_bin_kernel      color_fix.py:567-575, 614-649, 717-731   RGB -> HSV of content and style, 12 hue bins:
//                                                                 per-bin counts and one radix-sort entry per
//                                                                 (pixel, bin) it belongs to
//   2 x CUB radix sort  color_fix.py:744-747                      stable, on (bin << 30 | bits(saturation))
//   hsv_match_kernel    color_fix.py:733-737, 749-769             rank -> quantile index -> style saturation
//   hsv_compose_kernel  color_fix.py:593-607, 652-695, 817-851    HSV -> RGB, clamp, [-1,1]; optionally the
//                                                                 saturation maps, sigmoid weight and blend
//
// Everything is fp32 with torch's rounding points on the GPU (each op rounds; no FMA contraction).  No host
// synchronisation: the bin counts, qualify decisions and quantile indices stay on the device, so a clip with these
// modes captures into one CUDA graph.
#include <cub/device/device_radix_sort.cuh>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "svr2_internal.h"

namespace svr2 {
namespace {

constexpr int kBins = 12;                 // num_bins, color_fix.py:710
constexpr uint32_t kMinPixels = 100;      // min_pixels, color_fix.py:712
constexpr int kSegShift = 30;             // saturation in [0, 1]: its fp32 bits are < 2^30
constexpr int kSortBits = kSegShift + 4;  // segment 0..11, sentinel 15
constexpr uint64_t kSentinel = 15ull << kSegShift;
constexpr uint32_t kWrapFlag = 0x80000000u;   // value of the second (bin 0) entry of a wrap-around pixel

// Scratch header (the first 256 bytes of the scratch), written on the device by every call:
//   u32 content_count[12] | u32 style_count[12] | u32 qualify[12]
// counts are the sizes of the reference's boolean masks (a wrap-around pixel counts in bin 0 and bin 11);
// qualify[b] = content_count[b] > 100 && style_count[b] > 100.
struct HsvHeader {
  uint32_t content_count[kBins];
  uint32_t style_count[kBins];
  uint32_t qualify[kBins];
};
constexpr size_t kHeaderBytes = 256;
static_assert(sizeof(HsvHeader) <= kHeaderBytes, "header");

__device__ __forceinline__ float bf2f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to01(float x) {        // add(1.0).mul_(0.5).clamp_(0.0, 1.0)
  return fminf(fmaxf(__fmul_rn(__fadd_rn(x, 1.0f), 0.5f), 0.0f), 1.0f);
}
// where(maxc > 1e-10, range / clamp(maxc, min=1e-10), 0)   (color_fix.py:643, 866-870)
__device__ __forceinline__ float saturation(float maxc, float minc) {
  return maxc > 1e-10f ? __fdiv_rn(__fsub_rn(maxc, minc), fmaxf(maxc, 1e-10f)) : 0.0f;
}
__device__ __forceinline__ float saturation3(float r, float g, float b) {
  return saturation(fmaxf(fmaxf(r, g), b), fminf(fminf(r, g), b));
}

// _rgb_to_hsv_batch (color_fix.py:614-649) on [0,1] values.  The masked assignments run r, g, b, so on ties blue
// wins over green over red; `% 6.0` is torch.remainder (fmod, then + 6 for a negative result: a tiny negative
// (g-b)/range gives exactly 6, i.e. h == 1).  h.div_(6.0) by a python scalar runs on the GPU as a multiplication by
// the fp32 reciprocal.
__device__ __forceinline__ void rgb_to_hsv(float r, float g, float b, float& h, float& s, float& v) {
  const float maxc = fmaxf(fmaxf(r, g), b), minc = fminf(fminf(r, g), b);
  const float range = __fsub_rn(maxc, minc);
  float hh = 0.0f;
  if (range > 1e-10f) {
    if (maxc == b) {
      hh = __fadd_rn(__fdiv_rn(__fsub_rn(r, g), range), 4.0f);
    } else if (maxc == g) {
      hh = __fadd_rn(__fdiv_rn(__fsub_rn(b, r), range), 2.0f);
    } else {
      hh = fmodf(__fdiv_rn(__fsub_rn(g, b), range), 6.0f);
      if (hh != 0.0f && hh < 0.0f) hh = __fadd_rn(hh, 6.0f);
    }
  }
  h = __fmul_rn(hh, 1.0f / 6.0f);
  s = saturation(maxc, minc);
  v = maxc;
}

// _hsv_to_rgb_batch (color_fix.py:652-695), then clamp_(0, 1) and mul_(2).sub_(1) (:599-602)
__device__ __forceinline__ void hsv_to_rgb_pm1(float h, float s, float v, float out[3]) {
  const float h6 = __fmul_rn(h, 6.0f);
  const float fl = floorf(h6);
  const int i = ((int)fl) % 6;
  const float f = __fsub_rn(h6, fl);
  const float p = __fmul_rn(v, __fsub_rn(1.0f, s));
  const float q = __fmul_rn(v, __fsub_rn(1.0f, __fmul_rn(s, f)));
  const float t = __fmul_rn(v, __fsub_rn(1.0f, __fmul_rn(s, __fsub_rn(1.0f, f))));
  float r, g, b;
  switch (i) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
  out[0] = __fsub_rn(__fmul_rn(fminf(fmaxf(r, 0.0f), 1.0f), 2.0f), 1.0f);
  out[1] = __fsub_rn(__fmul_rn(fminf(fmaxf(g, 0.0f), 1.0f), 2.0f), 1.0f);
  out[2] = __fsub_rn(__fmul_rn(fminf(fmaxf(b, 0.0f), 1.0f), 2.0f), 1.0f);
}

// Hue bins of _hue_conditional_saturation_match (color_fix.py:717-727): bin b = [b/12, (b+1)/12) with the python-double
// edges rounded to fp32 as torch compares them; bin 0 also takes h >= 1 - 1/12 (the same fp32 value as bin 11's
// lower edge), so a pixel with 11/12 <= h < 1 lies in bin 11 and in bin 0, and h == 1 in bin 0 only.
// primary: the bin the pixel's first sort entry goes to; wrap: it has a second entry in bin 0.
__device__ __forceinline__ int hue_bin(float h, bool& wrap) {
  const double bw = 1.0 / kBins;
  wrap = h >= (float)(1.0 - bw) && h < (float)(kBins * bw);
  int bin = 0;                                               // h == 1 (only reachable through the wrap clause)
#pragma unroll
  for (int b = kBins - 1; b >= 1; --b)
    if (h >= (float)(b * bw) && h < (float)((b + 1) * bw)) bin = b;
  return bin;
}

// One pass over content and style: matched saturation initialised to the content saturation, sort entries at 2i
// (primary bin) and 2i+1 (bin 0 for a wrap-around pixel, else a sentinel), so that within every bin the entries
// are in pixel order and the stable sort breaks saturation ties by pixel index.  Bin counts into the header.
__global__ void __launch_bounds__(256) hsv_bin_kernel(const __nv_bfloat16* __restrict__ content,
                                                      const __nv_bfloat16* __restrict__ style, long long hw,
                                                      long long n, float* __restrict__ msat,
                                                      uint64_t* __restrict__ ckeys, uint32_t* __restrict__ cvals,
                                                      uint64_t* __restrict__ skeys, HsvHeader* __restrict__ hdr) {
  __shared__ uint32_t cnt[2][kBins];
  if (threadIdx.x < 2 * kBins) cnt[threadIdx.x / kBins][threadIdx.x % kBins] = 0;
  __syncthreads();
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const long long t = i / hw, px = i - t * hw;
    const long long base = t * 3 * hw + px;
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      const __nv_bfloat16* p = (side == 0 ? content : style) + base;
      float h, s, v;
      rgb_to_hsv(to01(bf2f(p[0])), to01(bf2f(p[hw])), to01(bf2f(p[2 * hw])), h, s, v);
      bool wrap;
      const int bin = hue_bin(h, wrap);
      const uint64_t bits = __float_as_uint(s);
      atomicAdd(&cnt[side][bin], 1u);
      if (wrap) atomicAdd(&cnt[side][0], 1u);
      const ulonglong2 k = make_ulonglong2(((uint64_t)bin << kSegShift) | bits, wrap ? bits : kSentinel);
      if (side == 0) {
        msat[i] = s;
        reinterpret_cast<ulonglong2*>(ckeys)[i] = k;
        reinterpret_cast<uint2*>(cvals)[i] = make_uint2((uint32_t)i, (uint32_t)i | kWrapFlag);
      } else {
        reinterpret_cast<ulonglong2*>(skeys)[i] = k;
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < 2 * kBins) {
    const uint32_t c = cnt[threadIdx.x / kBins][threadIdx.x % kBins];
    if (c) atomicAdd((threadIdx.x < kBins ? hdr->content_count : hdr->style_count) + threadIdx.x % kBins, c);
  }
}

// torch.linspace(0, 1, steps, device="cuda")[r] (ATen's CUDA kernel: step = 1 / float(steps - 1); the first half is
// step * r, the second half counts back from the end as 1 - step * k, which that kernel evaluates as one fused
// multiply-add), times float(n_ref - 1), .long(), clamp (color_fix.py:755-757)
__device__ __forceinline__ long long quantile_index(long long r, long long steps, long long n_ref) {
  const float step = __fdiv_rn(1.0f, (float)(steps - 1));
  const float q = r < steps / 2 ? __fmul_rn(step, (float)r) : __fmaf_rn(-step, (float)(steps - r - 1), 1.0f);
  const long long k = (long long)__fmul_rn(q, (float)(n_ref - 1));
  return k < 0 ? 0 : (k > n_ref - 1 ? n_ref - 1 : k);
}

// Over the sorted content entries: entry j of bin b has rank r = j - start(b) among the bin's content pixels; in a
// qualifying bin its pixel gets the style saturation of rank r (equal counts) or of the quantile index.  The
// reference's loop runs bin 0 before bin 11, so a wrap-around pixel keeps bin 11's match when bin 11 qualifies.
__global__ void __launch_bounds__(256) hsv_match_kernel(const uint64_t* __restrict__ ckeys,
                                                        const uint32_t* __restrict__ cvals,
                                                        const uint64_t* __restrict__ skeys, long long entries,
                                                        float* __restrict__ msat, HsvHeader* __restrict__ hdr) {
  __shared__ long long cstart[kBins], sstart[kBins], ccount[kBins], scount[kBins];
  __shared__ int qual[kBins];
  if (threadIdx.x == 0) {
    long long c = 0, s = 0;
    for (int b = 0; b < kBins; ++b) {
      cstart[b] = c, sstart[b] = s;
      ccount[b] = hdr->content_count[b], scount[b] = hdr->style_count[b];
      c += ccount[b], s += scount[b];
      qual[b] = ccount[b] > kMinPixels && scount[b] > kMinPixels;
      if (blockIdx.x == 0) hdr->qualify[b] = qual[b];
    }
  }
  __syncthreads();
  for (long long j = (long long)blockIdx.x * 256 + threadIdx.x; j < entries; j += (long long)gridDim.x * 256) {
    const uint64_t key = ckeys[j];
    const int bin = (int)(key >> kSegShift);
    if (bin >= kBins || !qual[bin]) continue;
    const uint32_t val = cvals[j];
    if ((val & kWrapFlag) && qual[kBins - 1]) continue;
    const long long r = j - cstart[bin], nc = ccount[bin], ns = scount[bin];
    const long long k = nc == ns ? r : quantile_index(r, nc, ns);
    msat[val & ~kWrapFlag] = __uint_as_float((uint32_t)(skeys[sstart[bin] + k] & ((1ull << kSegShift) - 1)));
  }
}

// HSV -> RGB with the matched saturation (h and v recomputed from the content, bit-identical to the first pass).
// wav == nullptr: out = bf16(rgb).  Otherwise wavelet_adaptive (color_fix.py:817-851): weight =
// clamp(sigmoid(5 * ((c_sat - s_sat) - 0.15)) * ((w_sat - s_sat) > 0.075), 0, 1), out = bf16(wav * (1 - weight) +
// rgb * weight), every op rounded separately.
__global__ void __launch_bounds__(256) hsv_compose_kernel(const __nv_bfloat16* __restrict__ content,
                                                          const __nv_bfloat16* __restrict__ style,
                                                          const float* __restrict__ wav, const float* __restrict__ msat,
                                                          __nv_bfloat16* __restrict__ out, long long hw, long long n) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const long long t = i / hw, px = i - t * hw;
    const long long base = t * 3 * hw + px;
    const float cr = to01(bf2f(content[base])), cg = to01(bf2f(content[base + hw])), cb = to01(bf2f(content[base + 2 * hw]));
    float h, c_sat, v;
    rgb_to_hsv(cr, cg, cb, h, c_sat, v);
    float rgb[3];
    hsv_to_rgb_pm1(h, msat[i], v, rgb);
    if (wav) {
      const float s_sat = saturation3(to01(bf2f(style[base])), to01(bf2f(style[base + hw])), to01(bf2f(style[base + 2 * hw])));
      const float w0 = wav[base], w1 = wav[base + hw], w2 = wav[base + 2 * hw];
      const float w_sat = saturation3(to01(w0), to01(w1), to01(w2));
      const float x = __fmul_rn(5.0f, __fsub_rn(__fsub_rn(c_sat, s_sat), 0.15f));
      float weight = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x)));
      weight = (__fsub_rn(w_sat, s_sat) > 0.075f) ? weight : 0.0f;
      weight = fminf(fmaxf(weight, 0.0f), 1.0f);
      const float keep = __fsub_rn(1.0f, weight);
      const float w[3] = {w0, w1, w2};
#pragma unroll
      for (int c = 0; c < 3; ++c) rgb[c] = __fadd_rn(__fmul_rn(w[c], keep), __fmul_rn(rgb[c], weight));
    }
    out[base] = __float2bfloat16_rn(rgb[0]);
    out[base + hw] = __float2bfloat16_rn(rgb[1]);
    out[base + 2 * hw] = __float2bfloat16_rn(rgb[2]);
  }
}

inline int grid_for(long long n, int per_block = 256, int waves = 16) {
  long long b = (n + per_block - 1) / per_block;
  const long long cap = (long long)num_sms() * waves;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

inline size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// scratch layout: header | msat f32[n] | keys u64[2n] x 3 | vals u32[2n] x 2 | CUB temp
struct HsvLayout {
  size_t msat, keys[3], vals[2], temp, temp_bytes, total;
};
HsvLayout hsv_layout(int64_t n) {
  HsvLayout L;
  const size_t e = 2 * (size_t)n;
  size_t t1 = 0, t2 = 0;
  cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
  cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, t1, k, v, (int64_t)e, 0, kSortBits);
  cub::DeviceRadixSort::SortKeys(nullptr, t2, k, (int64_t)e, 0, kSortBits);
  size_t o = kHeaderBytes;
  L.msat = o, o += align256((size_t)n * 4);
  for (auto& x : L.keys) x = o, o += align256(e * 8);
  for (auto& x : L.vals) x = o, o += align256(e * 4);
  L.temp = o, L.temp_bytes = t1 > t2 ? t1 : t2;
  L.total = o + align256(L.temp_bytes);
  return L;
}

}  // namespace
}  // namespace svr2

using namespace svr2;

extern "C" int64_t svr2_hsv_scratch_bytes(int64_t n) {
  if (n <= 0 || n >= ((int64_t)1 << 31)) return 0;
  return (int64_t)hsv_layout(n).total;
}

extern "C" int svr2_hsv_saturation_match_bf16(const void* content, const void* style, const float* wavelet, void* out,
                                              int frames, int64_t hw, void* scratch, int64_t scratch_bytes,
                                              void* stream) {
  if (frames <= 0 || hw <= 0) return set_error(SVR2_ERR_ARG, "svr2_hsv_saturation_match_bf16: empty input");
  const long long n = (long long)frames * hw;
  if (n >= ((long long)1 << 31)) return set_error(SVR2_ERR_ARG, "svr2_hsv_saturation_match_bf16: frames * hw must be < 2^31");
  if (!content || !style || !out) return set_error(SVR2_ERR_ARG, "svr2_hsv_saturation_match_bf16: null tensor");
  const HsvLayout L = hsv_layout(n);
  if (!scratch || scratch_bytes < (int64_t)L.total)
    return set_error(SVR2_ERR_ARG, "svr2_hsv_saturation_match_bf16: scratch too small (svr2_hsv_scratch_bytes)");
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* base = (uint8_t*)scratch;
  HsvHeader* hdr = (HsvHeader*)base;
  float* msat = (float*)(base + L.msat);
  uint64_t* keys[3] = {(uint64_t*)(base + L.keys[0]), (uint64_t*)(base + L.keys[1]), (uint64_t*)(base + L.keys[2])};
  uint32_t* vals[2] = {(uint32_t*)(base + L.vals[0]), (uint32_t*)(base + L.vals[1])};
  const long long entries = 2 * n;
  cudaError_t e = cudaMemsetAsync(hdr, 0, kHeaderBytes, s);
  if (e != cudaSuccess) return set_error(SVR2_ERR_CUDA, cudaGetErrorString(e));
  hsv_bin_kernel<<<grid_for(n), 256, 0, s>>>((const __nv_bfloat16*)content, (const __nv_bfloat16*)style, hw, n, msat,
                                             keys[0], vals[0], keys[2], hdr);
  int rc = check_launch("hsv_bin");
  if (rc) return rc;
  size_t temp_bytes = L.temp_bytes;
  cub::DoubleBuffer<uint64_t> ck(keys[0], keys[1]);
  cub::DoubleBuffer<uint32_t> cv(vals[0], vals[1]);
  e = cub::DeviceRadixSort::SortPairs(base + L.temp, temp_bytes, ck, cv, (int64_t)entries, 0, kSortBits, s);
  if (e != cudaSuccess) return set_error(SVR2_ERR_CUDA, cudaGetErrorString(e));
  // the style keys sort into the content keys' spare buffer (the selector is host state: no synchronisation)
  cub::DoubleBuffer<uint64_t> sk(keys[2], ck.Alternate());
  e = cub::DeviceRadixSort::SortKeys(base + L.temp, temp_bytes, sk, (int64_t)entries, 0, kSortBits, s);
  if (e != cudaSuccess) return set_error(SVR2_ERR_CUDA, cudaGetErrorString(e));
  hsv_match_kernel<<<grid_for(entries), 256, 0, s>>>(ck.Current(), cv.Current(), sk.Current(), entries, msat, hdr);
  rc = check_launch("hsv_match");
  if (rc) return rc;
  hsv_compose_kernel<<<grid_for(n), 256, 0, s>>>((const __nv_bfloat16*)content, (const __nv_bfloat16*)style, wavelet,
                                                 msat, (__nv_bfloat16*)out, hw, n);
  return check_launch("hsv_compose");
}
