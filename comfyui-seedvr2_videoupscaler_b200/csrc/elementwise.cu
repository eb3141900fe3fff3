// HBM-bound kernels of the hot path: everything that is not a contraction.
// All are one-read/one-write, 16-byte vectorised, fp32 math with bf16 rounding
// at the reference's rounding points (SURVEY.md §8 G3).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "ptx.cuh"
#include "svr2_internal.h"

namespace svr2 {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]),
                    pack_bf16x2(f[6], f[7]));
}

// ------------------------------------------------------------------ RMSNorm + AdaSingle "in"
// Persistent blocks (8 warps), one warp per row per iteration: all of a row's 16-byte vectors are loaded up front (kVec per
// lane in flight), fp32 statistics by warp shuffle, one write.  The fp32 scale / shift (/ weight) vectors are staged in
// shared memory ONCE per block: read per row from L1/L2 they were 8 bytes of cache traffic per 4 bytes of HBM traffic and
// capped the kernel at ~3.4 TB/s.  dim % 8 == 0, dim <= 32*8*kVec.
template <int kVec>
__global__ void __launch_bounds__(256) rmsnorm_ada_kernel(const __nv_bfloat16* __restrict__ x,
                                                          __nv_bfloat16* __restrict__ y, int rows, int dim, float eps,
                                                          const float* __restrict__ weight,
                                                          const float* __restrict__ scale,
                                                          const float* __restrict__ shift, int mode) {
  extern __shared__ float sm_vec[];               // [scale | shift | weight] x dim
  float* s_scale = sm_vec;
  float* s_shift = sm_vec + dim;
  float* s_weight = sm_vec + 2 * dim;
  for (int i = threadIdx.x; i < dim; i += 256) {
    s_scale[i] = scale[i];
    s_shift[i] = shift[i];
    if (weight) s_weight[i] = weight[i];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int nvec = dim / 8;
  const float inv_dim = 1.0f / (float)dim;
  for (long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); row < rows; row += (long long)gridDim.x * 8) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * dim);
    uint4* yr = reinterpret_cast<uint4*>(y + row * dim);
    uint4 raw[kVec];
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const int c = lane + i * 32;
      raw[i] = c < nvec ? __ldcs(xr + c) : make_uint4(0, 0, 0, 0);
    }
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      float v[8];
      unpack8(raw[i], v);
#pragma unroll
      for (int e = 0; e < 8; ++e) ss += v[e] * v[e];
    }
    ss = warp_sum(ss);
    const float rrms = 1.0f / sqrtf(ss * inv_dim + eps);
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        float v[8], o[8];
        unpack8(raw[i], v);
        const float4 s0 = *reinterpret_cast<const float4*>(s_scale + c * 8), s1 = *reinterpret_cast<const float4*>(s_scale + c * 8 + 4);
        const float4 h0 = *reinterpret_cast<const float4*>(s_shift + c * 8), h1 = *reinterpret_cast<const float4*>(s_shift + c * 8 + 4);
        const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
        const float sh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float r = v[e] * rrms;
          if (weight) r *= s_weight[c * 8 + e];
          if (mode == 0) {
            o[e] = r * sc[e] + sh[e];
          } else {
            r = bf16_round(r);
            r = bf16_round(r * sc[e]);
            o[e] = r + sh[e];
          }
        }
        yr[c] = pack8(o);
      }
    }
  }
}

// ------------------------------------------------------------------ q/k norm + RoPE + window gather
// one block per output row (window-ordered); warp w handles heads w, w+nwarps, ...; lane = 4 dims.
__global__ void __launch_bounds__(256) qk_norm_rope_window_kernel(
    const __nv_bfloat16* __restrict__ qkv_vid, const __nv_bfloat16* __restrict__ qkv_txt,
    const int32_t* __restrict__ row_src, const int32_t* __restrict__ row_rope, const float* __restrict__ cos_tab,
    const float* __restrict__ sin_tab, int nfreq, const float* __restrict__ wq_vid, const float* __restrict__ wk_vid,
    const float* __restrict__ wq_txt, const float* __restrict__ wk_txt, float eps, int heads,
    __nv_bfloat16* __restrict__ q, __nv_bfloat16* __restrict__ k, __nv_bfloat16* __restrict__ v,
    const int32_t* __restrict__ row_list) {
  const long long r = row_list ? (long long)row_list[blockIdx.x] : (long long)blockIdx.x;   // optional subset of the rows
  const int src = row_src[r];
  const bool is_txt = src < 0;
  const int inner = heads * 128;
  const __nv_bfloat16* base = is_txt ? qkv_txt + (long long)(-src - 1) * 3 * inner : qkv_vid + (long long)src * 3 * inner;
  const float* wq = is_txt ? wq_txt : wq_vid;
  const float* wk = is_txt ? wk_txt : wk_vid;
  const int ri[3] = {row_rope[r * 3 + 0], row_rope[r * 3 + 1], row_rope[r * 3 + 2]};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int d0 = lane * 4;
  const int rot = 6 * nfreq;  // rotated dims
  // per-lane cos/sin for the two pairs (d0,d0+1), (d0+2,d0+3)
  float cs[2], sn[2];
#pragma unroll
  for (int pi = 0; pi < 2; ++pi) {
    const int d = d0 + 2 * pi;
    cs[pi] = 1.f;
    sn[pi] = 0.f;
    if (d < rot) {
      const int axis = d / (2 * nfreq), j = (d % (2 * nfreq)) >> 1;
      const int tr = ri[axis];
      if (tr >= 0) {
        cs[pi] = cos_tab[tr * nfreq + j];
        sn[pi] = sin_tab[tr * nfreq + j];
      }
    }
  }
  const float4 wq4 = *reinterpret_cast<const float4*>(wq + d0);
  const float4 wk4 = *reinterpret_cast<const float4*>(wk + d0);
  // The kernel is latency-bound (one 256-byte row segment per warp and load): fetch q, k and v of up to three heads
  // per warp before touching any of them, so ~2.3 KB per warp are in flight instead of 256 B.
  constexpr int kHeadsPerPass = 3;
  for (int h0 = warp; h0 < heads; h0 += nwarps * kHeadsPerPass) {
    uint2 raw[kHeadsPerPass][3];
#pragma unroll
    for (int i = 0; i < kHeadsPerPass; ++i) {
      const int h = h0 + i * nwarps;
      if (h < heads) {
#pragma unroll
        for (int which = 0; which < 3; ++which)
          raw[i][which] = *reinterpret_cast<const uint2*>(base + which * inner + h * 128 + d0);
      }
    }
#pragma unroll
    for (int i = 0; i < kHeadsPerPass; ++i) {
      const int h = h0 + i * nwarps;
      if (h >= heads) break;
      const long long o_off = (r * heads + h) * 128 + d0;
#pragma unroll
      for (int which = 0; which < 2; ++which) {
        const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw[i][which]);
        float2 a = __bfloat1622float2(hh[0]), b = __bfloat1622float2(hh[1]);
        float ss = a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y;
        ss = warp_sum(ss);
        const float rr = 1.0f / sqrtf(ss * (1.0f / 128.0f) + eps);
        const float4 w4 = which == 0 ? wq4 : wk4;
        float x0 = a.x * rr * w4.x, x1 = a.y * rr * w4.y, x2 = b.x * rr * w4.z, x3 = b.y * rr * w4.w;
        // interleaved-pair rotation: (x0,x1) -> (x0 c - x1 s, x1 c + x0 s)
        const float y0 = x0 * cs[0] - x1 * sn[0], y1 = x1 * cs[0] + x0 * sn[0];
        const float y2 = x2 * cs[1] - x3 * sn[1], y3 = x3 * cs[1] + x2 * sn[1];
        uint2 outv = make_uint2(pack_bf16x2(y0, y1), pack_bf16x2(y2, y3));
        *reinterpret_cast<uint2*>((which == 0 ? q : k) + o_off) = outv;
      }
      *reinterpret_cast<uint2*>(v + o_off) = raw[i][2];
    }
  }
}

// ------------------------------------------------------------------ text mean over windows
__global__ void txt_window_mean_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out,
                                       int n_win, int l, int dim) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over l*dim/8 vectors
  const long long nvec = (long long)l * dim / 8;
  if (idx >= nvec) return;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int w = 0; w < n_win; ++w) {
    float f[8];
    unpack8(reinterpret_cast<const uint4*>(in + (long long)w * l * dim)[idx], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += f[e];
  }
  const float inv = 1.0f / (float)n_win;
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] *= inv;
  reinterpret_cast<uint4*>(out)[idx] = pack8(acc);
}

// ------------------------------------------------------------------ patchify / unpatchify (1,2,2)
__global__ void patchify_kernel(const __nv_bfloat16* __restrict__ vid, __nv_bfloat16* __restrict__ out, int T, int H,
                                int W, int C, int ld_out) {
  const int Hp = H / 2, Wp = W / 2;
  const long long l = blockIdx.x;  // token
  const int wp = l % Wp, hp = (l / Wp) % Hp, t = l / ((long long)Wp * Hp);
  for (int i = threadIdx.x; i < ld_out; i += blockDim.x) {
    float val = 0.f;
    if (i < 4 * C) {
      const int c = i % C, dw = (i / C) & 1, dh = i / (2 * C);
      val = __bfloat162float(vid[(((long long)t * H + 2 * hp + dh) * W + 2 * wp + dw) * C + c]);
    }
    out[l * ld_out + i] = __float2bfloat16_rn(val);
  }
}
__global__ void unpatchify_kernel(const __nv_bfloat16* __restrict__ in, int ld_in, __nv_bfloat16* __restrict__ out,
                                  int T, int H, int W, int C) {
  const int Hp = H / 2, Wp = W / 2;
  const long long l = blockIdx.x;
  const int wp = l % Wp, hp = (l / Wp) % Hp, t = l / ((long long)Wp * Hp);
  for (int i = threadIdx.x; i < 4 * C; i += blockDim.x) {
    const int c = i % C, dw = (i / C) & 1, dh = i / (2 * C);
    out[(((long long)t * H + 2 * hp + dh) * W + 2 * wp + dw) * C + c] = in[l * ld_in + i];
  }
}

// ------------------------------------------------------------------ GroupNorm(32) per frame
// Deterministic three-step reduction (no floating-point atomics, so results are bit-reproducible):
//   1. stats   : block = slab of pixels of one frame, thread = 8 fixed channels; per-block partial
//                (sum, sumsq) per group reduced in a fixed order -> partial[f][blk][32][2] (double).
//                The per-thread chains are fp64 too: var = E[x^2] - mean^2 cancels by (mean/std)^2, which an fp32
//                chain of thousands of adds does not survive on offset or near-flat frames (a black frame after
//                conv_in); bf16 squares are exact in fp32 (v * v below), so the sums are the only rounding.
//   2. finalize: one block per frame sums the partials in block order and emits per-channel
//                fp32 coefficients a = rstd*gamma, b = beta - mean*a
//   3. apply   : y = silu(bf16(a*x + b)) (+ halo duplication of frame 0)
__global__ void __launch_bounds__(256) groupnorm_stats_kernel(const __nv_bfloat16* __restrict__ x, int hw, int C,
                                                              int pix_per_block, double* __restrict__ partial) {
  __shared__ double sm[256][4];
  const int f = blockIdx.y;
  const int cvec = C / 8;               // vectors per pixel
  const int cpg = C / 32;               // channels per group (4, 8, 16)
  const long long p0 = (long long)blockIdx.x * pix_per_block;
  const long long p1 = min((long long)hw, p0 + pix_per_block);
  const __nv_bfloat16* xf = x + (long long)f * hw * C;
  const int cv = threadIdx.x % cvec, pl = threadIdx.x / cvec, pstride = 256 / cvec;
  double s0 = 0.0, q0 = 0.0, s1 = 0.0, q1 = 0.0;  // (s0,q0): channels 0-3 of the vector, (s1,q1): 4-7
  long long p = p0 + pl;
  for (; p + 3LL * pstride < p1; p += 4LL * pstride) {
    uint4 r[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) r[u] = *reinterpret_cast<const uint4*>(xf + (p + (long long)u * pstride) * C + cv * 8);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float v[8];
      unpack8(r[u], v);
#pragma unroll
      for (int e = 0; e < 4; ++e) { s0 += v[e]; q0 += v[e] * v[e]; s1 += v[4 + e]; q1 += v[4 + e] * v[4 + e]; }
    }
  }
  for (; p < p1; p += pstride) {
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(xf + p * C + cv * 8), v);
#pragma unroll
    for (int e = 0; e < 4; ++e) { s0 += v[e]; q0 += v[e] * v[e]; s1 += v[4 + e]; q1 += v[4 + e] * v[4 + e]; }
  }
  sm[threadIdx.x][0] = s0; sm[threadIdx.x][1] = q0; sm[threadIdx.x][2] = s1; sm[threadIdx.x][3] = q1;
  __syncthreads();
  if (threadIdx.x < 32) {
    const int g = threadIdx.x;
    double ds = 0.0, dq = 0.0;
    if (cpg == 4) {               // group g = half (g&1) of vector g>>1
      const int v = g >> 1, h = (g & 1) * 2;
      for (int l = 0; l < pstride; ++l) { ds += sm[l * cvec + v][h]; dq += sm[l * cvec + v][h + 1]; }
    } else {                      // group g = vectors [g*cpg/8, (g+1)*cpg/8)
      const int nv = cpg / 8;
      for (int l = 0; l < pstride; ++l)
        for (int v = g * nv; v < (g + 1) * nv; ++v) {
          ds += sm[l * cvec + v][0] + sm[l * cvec + v][2];
          dq += sm[l * cvec + v][1] + sm[l * cvec + v][3];
        }
    }
    double* dst = partial + (((long long)f * gridDim.x + blockIdx.x) * 32 + g) * 2;
    dst[0] = ds;
    dst[1] = dq;
  }
}

// grid = frames, block = 256: coef[f][c] = (a, b)
__global__ void __launch_bounds__(256) groupnorm_finalize_kernel(const double* __restrict__ partial, int nblk, int hw,
                                                                 int C, const __nv_bfloat16* __restrict__ gamma,
                                                                 const __nv_bfloat16* __restrict__ beta, float eps,
                                                                 float2* __restrict__ coef) {
  __shared__ float s_mean[32], s_rstd[32];
  const int f = blockIdx.x, cpg = C / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // warp w reduces groups w, w+8, ... : lanes stride over blocks, then a fixed-order shuffle tree
  for (int g = warp; g < 32; g += 8) {
    double ds = 0.0, dq = 0.0;
    for (int b = lane; b < nblk; b += 32) {
      const double* src = partial + (((long long)f * nblk + b) * 32 + g) * 2;
      ds += src[0];
      dq += src[1];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ds += __shfl_xor_sync(0xffffffffu, ds, o);
      dq += __shfl_xor_sync(0xffffffffu, dq, o);
    }
    if (lane == 0) {
      const double n = (double)hw * cpg;
      const double mean = ds / n, var = dq / n - mean * mean;
      s_mean[g] = (float)mean;
      s_rstd[g] = rsqrtf(fmaxf((float)var, 0.f) + eps);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += 256) {
    const int g = c / cpg;
    const float a = s_rstd[g] * __bfloat162float(gamma[c]);
    coef[(long long)f * C + c] = make_float2(a, __bfloat162float(beta[c]) - s_mean[g] * a);
  }
}

// fixed-order tree over a block of 256 threads; every thread gets the totals
__device__ __forceinline__ void block_sum2_256(double& ds, double& dq, double* sh_s, double* sh_q) {
  sh_s[threadIdx.x] = ds;
  sh_q[threadIdx.x] = dq;
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if (threadIdx.x < st) {
      sh_s[threadIdx.x] += sh_s[threadIdx.x + st];
      sh_q[threadIdx.x] += sh_q[threadIdx.x + st];
    }
    __syncthreads();
  }
  ds = sh_s[0];
  dq = sh_q[0];
  __syncthreads();
}

// finalize from conv-epilogue partials: part [frames][slots][C/8] (sum0, sq0, sum1, sq1) per channel octet
// (x/y: channels 0-3 of the octet, z/w: channels 4-7).  One block per (group, frame); every thread sums a
// fixed strided subset of the slots in double, then a fixed-order shared-memory tree -> deterministic.
// The partials are fp32 sums, so var = E[x^2] - mean^2 from them is off by ~1e-4 (mean/std)^2 of var.  A group with
// mean^2 > 16 var (a near-flat or strongly offset group) is summed again from x, shifted by that mean:
// sum (x - m~) and sum (x - m~)^2 do not cancel.  Only such groups pay the extra read of their channels.
__global__ void __launch_bounds__(256) groupnorm_finalize_fused_kernel(const float4* __restrict__ part, int slots,
                                                                       const __nv_bfloat16* __restrict__ x, int hw, int C,
                                                                       const __nv_bfloat16* __restrict__ gamma,
                                                                       const __nv_bfloat16* __restrict__ beta,
                                                                       float eps, float2* __restrict__ coef) {
  __shared__ double sh_s[256], sh_q[256];
  const int g = blockIdx.x, f = blockIdx.y, cpg = C / 32, noct = C / 8;
  double ds = 0.0, dq = 0.0;
  const float4* base = part + (long long)f * slots * noct;
  if (cpg == 4) {
    const int o = g >> 1, hi = g & 1;
    for (int sl = threadIdx.x; sl < slots; sl += 256) {
      const float4 v = base[(long long)sl * noct + o];
      ds += hi ? v.z : v.x;
      dq += hi ? v.w : v.y;
    }
  } else {
    const int no = cpg / 8;
    for (int sl = threadIdx.x; sl < slots; sl += 256) {
      for (int o = g * no; o < (g + 1) * no; ++o) {
        const float4 v = base[(long long)sl * noct + o];
        ds += (double)v.x + (double)v.z;
        dq += (double)v.y + (double)v.w;
      }
    }
  }
  block_sum2_256(ds, dq, sh_s, sh_q);
  const double n = (double)hw * cpg;
  double mean = ds / n, var = dq / n - mean * mean;
  if (16.0 * var < mean * mean) {                 // block-uniform
    const float shift = (float)mean;
    const int lg = cpg == 4 ? 0 : cpg == 8 ? 1 : 2;  // 4-channel chunks per pixel: 1 << lg
    const __nv_bfloat16* xg = x + (long long)f * hw * C + g * cpg;
    ds = 0.0;
    dq = 0.0;
    for (long long i = threadIdx.x; i < ((long long)hw << lg); i += 256) {
      const uint2 r = *reinterpret_cast<const uint2*>(xg + (i >> lg) * C + (i & ((1 << lg) - 1)) * 4);
      const float d0 = __uint_as_float(r.x << 16) - shift, d1 = __uint_as_float(r.x & 0xffff0000u) - shift;
      const float d2 = __uint_as_float(r.y << 16) - shift, d3 = __uint_as_float(r.y & 0xffff0000u) - shift;
      ds += (d0 + d1) + (d2 + d3);
      dq += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
    }
    block_sum2_256(ds, dq, sh_s, sh_q);
    const double dm = ds / n;
    mean = (double)shift + dm;
    var = dq / n - dm * dm;
  }
  const float rstd = rsqrtf(fmaxf((float)var, 0.f) + eps);
  if (threadIdx.x < cpg) {
    const int c = g * cpg + threadIdx.x;
    const float a = rstd * __bfloat162float(gamma[c]);
    coef[(long long)f * C + c] = make_float2(a, __bfloat162float(beta[c]) - (float)mean * a);
  }
}

// The bf16 rounding of the normalised value is one cvt.rn.bf16x2 per channel pair, six 16-byte loads are in flight per
// thread and at most 64 registers are used so that four blocks fit an SM — the kernel is latency-bound at the
// power-capped clock, not DRAM-bound.
template <bool SILU>
__global__ void __launch_bounds__(256, 4) groupnorm_apply_kernel(const __nv_bfloat16* __restrict__ x,
                                                                 __nv_bfloat16* __restrict__ y, int hw, int C,
                                                                 int out_t_pad, int out_dup_head,
                                                                 const float2* __restrict__ coef) {
  const int f = blockIdx.y;
  const int cvec = C / 8;
  const long long nvec = (long long)hw * cvec;
  const uint4* __restrict__ xf = reinterpret_cast<const uint4*>(x + (long long)f * hw * C);
  uint4* __restrict__ yf = reinterpret_cast<uint4*>(y + (long long)(f + out_t_pad) * hw * C);
  const long long halo = nvec;                       // vectors per frame
  const int cv = threadIdx.x % cvec;                 // every stride below is a multiple of 256: fixed channel octet
  float ca[8], cb[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float2 t = coef[(long long)f * C + cv * 8 + e];
    ca[e] = t.x;
    cb[e] = t.y;
  }
  const bool dup = out_dup_head && f == 0;
  auto apply = [&](const uint4& r) -> uint4 {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float t0 = fmaf(__uint_as_float(w[e] << 16), ca[2 * e], cb[2 * e]);
      const float t1 = fmaf(__uint_as_float(w[e] & 0xffff0000u), ca[2 * e + 1], cb[2 * e + 1]);
      uint32_t pk = pack_bf16x2(t0, t1);              // F.group_norm output is bf16
      if constexpr (SILU) pk = pack_bf16x2(silu_fast(__uint_as_float(pk << 16)), silu_fast(__uint_as_float(pk & 0xffff0000u)));
      o[e] = pk;
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
  };
  const long long stride = (long long)gridDim.x * 256;
  long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  for (; i + 5 * stride < nvec; i += 6 * stride) {
    uint4 r[6];
#pragma unroll
    for (int u = 0; u < 6; ++u) r[u] = __ldcs(xf + i + u * stride);        // streamed once
#pragma unroll
    for (int u = 0; u < 6; ++u) {
      const uint4 pk = apply(r[u]);
      yf[i + u * stride] = pk;
      if (dup) {
        yf[i + u * stride - halo] = pk;
        yf[i + u * stride - 2 * halo] = pk;
      }
    }
  }
  for (; i < nvec; i += stride) {
    const uint4 pk = apply(xf[i]);
    yf[i] = pk;
    if (dup) {
      yf[i - halo] = pk;
      yf[i - 2 * halo] = pk;
    }
  }
}

static void launch_gn_apply(const void* x, void* y, int frames, int hw, int C, int silu, int out_t_pad, int out_dup_head,
                            const float2* coef, cudaStream_t s) {
  const long long nvec = (long long)hw * C / 8;
  int bx = (int)((nvec + 256 * 12 - 1) / (256 * 12));
  if (bx < 1) bx = 1;
  if (silu)
    groupnorm_apply_kernel<true><<<dim3(bx, frames), 256, 0, s>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, hw, C,
                                                                  out_t_pad, out_dup_head, coef);
  else
    groupnorm_apply_kernel<false><<<dim3(bx, frames), 256, 0, s>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, hw, C,
                                                                   out_t_pad, out_dup_head, coef);
}

// ------------------------------------------------------------------ attention pass-1 combine
// partial [rows][slots] (max, sum exp2) -> lse2[row] = M + log2(sum_i l_i 2^(m_i - M))
__global__ void rowstat_combine_kernel(const float2* __restrict__ part, int slots, long long ld, float* __restrict__ lse,
                                       int rows) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float2* pr = part + row * ld;
  float mx = -INFINITY;
  for (int i = lane; i < slots; i += 32) mx = fmaxf(mx, pr[i].x);
  mx = warp_max(mx);
  float s = 0.f;
  for (int i = lane; i < slots; i += 32) {
    const float2 v = pr[i];
    if (v.x > -INFINITY) s += v.y * exp2f(v.x - mx);
  }
  s = warp_sum(s);
  if (lane == 0) lse[row] = mx + log2f(s);
}

// Single-pass variant (no duplicated Q K^T): a cheap GEMM over a SUBSET of the keys gives a reference exponent m^ per
// row (any value within ~100 powers of two of the true row maximum works: probabilities are written un-normalised as
// bf16(exp2(s - m^)) with full relative precision, their fp32 sum normalises the output afterwards).
// partial [rows][slots] (max, sum) over the sampled keys -> mhat[row] = max; optionally clears the fallback flag.
__global__ void rowstat_max_kernel(const float2* __restrict__ part, int slots, long long ld, float* __restrict__ mhat,
                                   int rows, int* __restrict__ flag_reset) {
  if (flag_reset && blockIdx.x == 0 && threadIdx.x == 0) *flag_reset = 0;
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float2* pr = part + row * ld;
  float mx = -INFINITY;
  for (int i = lane; i < slots; i += 32) mx = fmaxf(mx, pr[i].x);
  mx = warp_max(mx);
  if (lane == 0) mhat[row] = mx;
}
// partial [rows][slots] (unused, sum of exp2(score - mhat)) over ALL keys -> rowscale[row] = 1 / sum, and the safety check
// of the reference exponent: the row sum l must lie in (1e-30, 1e30).  l < 1e30 bounds every probability (no overflow in
// bf16, in the fp32 sums, or in the fp32 accumulators of P~ V); l > 1e-30 keeps the dominant probabilities above bf16's
// normal range.  A violated row raises *flag: the caller's conditional fallback launches then recompute the chunk with the
// exact two-pass kernels.
__global__ void pexp_stat_combine_kernel(const float2* __restrict__ part, int slots, long long ld,
                                         const float* __restrict__ mhat, float* __restrict__ rowscale, int rows,
                                         int* __restrict__ flag) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= rows) return;
  (void)mhat;
  const float2* pr = part + row * ld;
  float s = 0.f;
  for (int i = lane; i < slots; i += 32) s += pr[i].y;
  s = warp_sum(s);
  if (lane == 0) {
    const bool ok = (s > 1e-30f) && (s < 1e30f);
    rowscale[row] = ok ? 1.0f / s : 0.f;
    if (!ok) atomicOr(flag, 1);
  }
}

// ------------------------------------------------------------------ transpose bf16 [rows, cols] -> [cols, rows]
__global__ void transpose_kernel(const __nv_bfloat16* __restrict__ in, long long ld_in, __nv_bfloat16* __restrict__ out,
                                 long long ld_out, int rows, int cols) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < rows && c < cols) ? in[(long long)r * ld_in + c] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < rows && c < cols) out[(long long)c * ld_out + r] = tile[threadIdx.x][i];
  }
}

// ------------------------------------------------------------------ layout glue
template <typename TIn>
__device__ __forceinline__ float ld_as_float(const TIn* p, long long i);
template <> __device__ __forceinline__ float ld_as_float<float>(const float* p, long long i) { return p[i]; }
template <> __device__ __forceinline__ float ld_as_float<__nv_bfloat16>(const __nv_bfloat16* p, long long i) { return __bfloat162float(p[i]); }
template <> __device__ __forceinline__ float ld_as_float<__half>(const __half* p, long long i) { return __half2float(p[i]); }

// in: [C,T,H,W] window (channel / frame / row strides in elements) -> out: [out_t_pad + T, H, W, C_pad] (channels >= C
// zero), frame 0 duplicated into the halo
template <typename TIn>
__global__ void ncdhw_to_ndhwc_kernel(const TIn* __restrict__ in, int C, int T, int H, int W, long long chan_stride,
                                      long long frame_stride, int row_stride, __nv_bfloat16* __restrict__ out, int C_pad,
                                      int out_t_pad, float div) {
  const long long hw = (long long)H * W;
  const long long total = (long long)T * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / hw, pix = i % hw;
    const long long src = t * frame_stride + (pix / W) * row_stride + pix % W;
    for (int c = 0; c < C_pad; ++c) {
      const float v = c < C ? bf16_round(ld_as_float<TIn>(in, (long long)c * chan_stride + src)) / div : 0.f;
      const __nv_bfloat16 b = __float2bfloat16_rn(v);
      out[((t + out_t_pad) * hw + pix) * C_pad + c] = b;
      if (t == 0)
        for (int d = 0; d < out_t_pad; ++d) out[((long long)d * hw + pix) * C_pad + c] = b;
    }
  }
}
// in: [T,H,W,ld_in] -> out [C,T,H,W] (first C channels)
template <typename TOut>
__global__ void ndhwc_to_ncdhw_kernel(const __nv_bfloat16* __restrict__ in, int ld_in, int C, int T, int H, int W,
                                      TOut* __restrict__ out, long long chan_stride) {
  const long long hw = (long long)H * W, total = (long long)T * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / hw, pix = i % hw;
    for (int c = 0; c < C; ++c) {
      const float v = __bfloat162float(in[i * ld_in + c]);
      if constexpr (sizeof(TOut) == 4) out[(long long)c * chan_stride + t * hw + pix] = v;
      else out[(long long)c * chan_stride + t * hw + pix] = __float2bfloat16_rn(v);
    }
  }
}

// ------------------------------------------------------------------ spatially tiled VAE seams
// The final kernel of a tile accumulates straight into the clip-sized result instead of storing the tile: what
// svr2_tile_accumulate_bf16 (post.cu tile_accumulate_kernel) does with the stored tile, with the same rounding points —
// result = bf16(result + rn(rn(v * wh[y]) * ww[x])), count = bf16(fma(wh[y], ww[x], count)) once per pixel.  The edge
// weights come from the clip's ramp tables (svr2_tile_ramp_bf16: [r | 1 - r]) as vae.py's _tiled builds them: ones,
// the first ov = min(len, n - 1) entries r on a side with a neighbour before, the last ov entries 1 - r on a side with
// a neighbour after (which wins where both overlap).
struct SeamDev {
  __nv_bfloat16* result;          // at the tile's top-left corner, frame 0 of this call
  __nv_bfloat16* count;           // at the tile's corner (row stride rs); NULL: not updated
  long long cs, fs;
  int rs;
  const __nv_bfloat16 *ramp_h, *ramp_w;
  int len_h, len_w, edges;
};
__device__ __forceinline__ float seam_weight(const __nv_bfloat16* ramp, int len, bool lo, bool hi, int n, int i) {
  const int ov = len < n - 1 ? len : n - 1;
  float w = 1.f;
  if (ov > 0 && lo && i < ov) w = __bfloat162float(ramp[i]);
  if (ov > 0 && hi && i >= n - ov) w = __bfloat162float(ramp[len + i - (n - ov)]);
  return w;
}
// v[c]: the tile's bf16 values of pixel (t, y, x) of an H x W tile
__device__ __forceinline__ void seam_add(const SeamDev& s, int C, const float* v, long long t, int y, int x, int H, int W) {
  const float a = seam_weight(s.ramp_h, s.len_h, s.edges & SVR2_SEAM_TOP, s.edges & SVR2_SEAM_BOTTOM, H, y);
  const float b = seam_weight(s.ramp_w, s.len_w, s.edges & SVR2_SEAM_LEFT, s.edges & SVR2_SEAM_RIGHT, W, x);
  const long long o = t * s.fs + (long long)y * s.rs + x;
  for (int c = 0; c < C; ++c) {
    const float u = bf16_round(bf16_round(v[c] * a) * b);
    __nv_bfloat16* r = s.result + (long long)c * s.cs + o;
    *r = __float2bfloat16_rn(__bfloat162float(*r) + u);
  }
  if (s.count && t == 0) {
    __nv_bfloat16* k = s.count + (long long)y * s.rs + x;
    *k = __float2bfloat16_rn(fmaf(a, b, __bfloat162float(*k)));
  }
}
// ndhwc_to_ncdhw_kernel's seam variant (the encoder's 16 mean channels of conv_out)
__global__ void __launch_bounds__(256) ndhwc_to_ncdhw_seam_kernel(const __nv_bfloat16* __restrict__ in, int ld_in, int C,
                                                                  int T, int H, int W, SeamDev s) {
  const long long hw = (long long)H * W, total = (long long)T * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / hw, pix = i % hw;
    float v[16];
    for (int c = 0; c < C; ++c) v[c] = __bfloat162float(in[i * ld_in + c]);
    seam_add(s, C, v, t, (int)(pix / W), (int)(pix % W), H, W);
  }
}

// 3x3x3 im2col, zero spatial padding, causal halo = 2 real frames in front of x.
// x [2+T, H, W, 8] (3 real channels: one aligned 16-byte load per pixel) -> out [T*H*W, 128], column
// ((kt*3+kh)*3+kw)*3 + c, columns 81..127 zero.  One thread assembles one output row in registers
// (27 pixel loads, mostly L1 hits shared with the neighbouring rows) and writes its 256 bytes.
__global__ void __launch_bounds__(128) im2col3_c3_kernel(const uint4* __restrict__ x, int T, int H, int W,
                                                         uint4* __restrict__ out) {
  const long long total = (long long)T * H * W;
  const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= total) return;
  const int w = row % W, h = (row / W) % H;
  const long long t = row / ((long long)W * H);
  uint32_t v[44];                      // 88 bf16 slots: 81 values + zero tail
#pragma unroll
  for (int i = 0; i < 44; ++i) v[i] = 0;
#pragma unroll
  for (int tap = 0; tap < 27; ++tap) {
    const int kw = tap % 3, kh = (tap / 3) % 3, kt = tap / 9;
    const int hh = h + kh - 1, ww = w + kw - 1;
    uint32_t c01 = 0, c2 = 0;
    if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
      const uint4 px = x[((t + kt) * H + hh) * W + ww];
      c01 = px.x;
      c2 = px.y & 0xffffu;
    }
    // place 3 halfwords at halfword offset 3*tap
    const int o = 3 * tap;
    if ((o & 1) == 0) {               // aligned: [c0 c1] -> word o/2, c2 -> low half of word o/2+1
      v[o / 2] |= c01;
      v[o / 2 + 1] |= c2;
    } else {                          // c0 -> high half of word (o-1)/2, [c1 c2] -> next word
      v[o / 2] |= c01 << 16;
      v[o / 2 + 1] |= (c01 >> 16) | (c2 << 16);
    }
  }
  uint4* dst = out + row * 16;
#pragma unroll
  for (int j = 0; j < 11; ++j) dst[j] = make_uint4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
#pragma unroll
  for (int j = 11; j < 16; ++j) dst[j] = make_uint4(0, 0, 0, 0);
}

// generic fallback: one thread per 16-byte chunk
__global__ void __launch_bounds__(256) im2col3_kernel(const __nv_bfloat16* __restrict__ x, int T, int H, int W, int C,
                                                      int ld_in, __nv_bfloat16* __restrict__ out, int ld_out) {
  const int cpr = ld_out / 8;
  const long long total = (long long)T * H * W * cpr;
  const unsigned short* xs = reinterpret_cast<const unsigned short*>(x);
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / cpr;
    const int c8 = (int)(idx - row * cpr) * 8;
    const int w = row % W, h = (row / W) % H, t = row / ((long long)W * H);
    unsigned short v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int i = c8 + e;
      v[e] = 0;
      if (i < 27 * C) {
        const int tap = i / C, c = i - tap * C, kw = tap % 3, kh = (tap / 3) % 3, kt = tap / 9;
        const int hh = h + kh - 1, ww = w + kw - 1;
        if (hh >= 0 && hh < H && ww >= 0 && ww < W) v[e] = xs[(((long long)(t + kt) * H + hh) * W + ww) * ld_in + c];
      }
    }
    uint4 pk = make_uint4(v[0] | (uint32_t(v[1]) << 16), v[2] | (uint32_t(v[3]) << 16), v[4] | (uint32_t(v[5]) << 16),
                          v[6] | (uint32_t(v[7]) << 16));
    reinterpret_cast<uint4*>(out + row * ld_out)[c8 / 8] = pk;
  }
}

// ------------------------------------------------------------------ conv_out tap gather
// Decoder conv_out (128 -> 3, 3x3x3 causal) as (1) one GEMM z[tap*co_n + co][pixel] = W_tap[co,:] . x[pixel,:]
// over ALL input pixels incl. the 2 halo frames (x is read once instead of 27 times), fp32, and (2) this
// gather: out[co][t][h][w] = bias[co] + sum_taps z[tap, co][(t+kt), h+kh-1, w+kw-1] (zero outside the frame).
__device__ __forceinline__ void conv_tap_sum(const float* __restrict__ z, long long ldz, int co_n, int H, int W,
                                             long long t, int h, int w, float* acc) {
  const long long hw = (long long)H * W;
#pragma unroll
  for (int kt = 0; kt < 3; ++kt)
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hh = h + kh - 1;
      if (hh < 0 || hh >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int ww = w + kw - 1;
        if (ww < 0 || ww >= W) continue;
        const long long q = (t + kt) * hw + (long long)hh * W + ww;     // halo: input frame index = t + kt
        const int tap = (kt * 3 + kh) * 3 + kw;
        for (int c = 0; c < co_n; ++c) acc[c] += z[(long long)(tap * co_n + c) * ldz + q];
      }
    }
}
template <typename TOut>
__global__ void __launch_bounds__(256) conv_tap_gather_kernel(const float* __restrict__ z, long long ldz, int co_n,
                                                              const __nv_bfloat16* __restrict__ bias, int T, int H, int W,
                                                              TOut* __restrict__ out, long long chan_stride) {
  const long long hw = (long long)H * W, total = (long long)T * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int w = i % W, h = (i / W) % H;
    const long long t = i / hw;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    conv_tap_sum(z, ldz, co_n, H, W, t, h, w, acc);
    for (int c = 0; c < co_n; ++c) {
      const float v = bf16_round(acc[c] + __bfloat162float(bias[c]));
      if constexpr (sizeof(TOut) == 4) out[(long long)c * chan_stride + i] = v;
      else out[(long long)c * chan_stride + i] = __float2bfloat16_rn(v);
    }
  }
}
// conv_tap_gather_kernel's seam variant (the decoder's last kernel): v = bf16(bias + sum over the taps), accumulated
__global__ void __launch_bounds__(256) conv_tap_gather_seam_kernel(const float* __restrict__ z, long long ldz, int co_n,
                                                                   const __nv_bfloat16* __restrict__ bias, int T, int H,
                                                                   int W, SeamDev s) {
  const long long hw = (long long)H * W, total = (long long)T * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int w = i % W, h = (i / W) % H;
    const long long t = i / hw;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    conv_tap_sum(z, ldz, co_n, H, W, t, h, w, acc);
    for (int c = 0; c < co_n; ++c) acc[c] = bf16_round(acc[c] + __bfloat162float(bias[c]));
    seam_add(s, co_n, acc, t, h, w, H, W);
  }
}

}  // namespace svr2

using namespace svr2;

extern "C" int svr2_rmsnorm_ada_bf16(const void* x, void* y, int rows, int dim, float eps, const float* weight,
                                     const float* scale, const float* shift, int mode, void* stream) {
  if (dim % 8 || dim > 32 * 8 * 16) return set_error(SVR2_ERR_ARG, "svr2_rmsnorm_ada_bf16: dim % 8 != 0 or dim > 4096");
  if (rows <= 0) return SVR2_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const long long want = (rows + 7) / 8;
  const long long cap = (long long)num_sms() * 6;                 // persistent: a few blocks per SM, each loops over rows
  const unsigned grid = (unsigned)(want < cap ? want : cap);
  const size_t smem = (size_t)3 * dim * sizeof(float);             // <= 48 KB for dim <= 4096
  const __nv_bfloat16* xi = (const __nv_bfloat16*)x;
  __nv_bfloat16* yo = (__nv_bfloat16*)y;
  if (dim <= 1024) rmsnorm_ada_kernel<4><<<grid, 256, smem, s>>>(xi, yo, rows, dim, eps, weight, scale, shift, mode);
  else if (dim <= 2560) rmsnorm_ada_kernel<10><<<grid, 256, smem, s>>>(xi, yo, rows, dim, eps, weight, scale, shift, mode);
  else if (dim <= 3072) rmsnorm_ada_kernel<12><<<grid, 256, smem, s>>>(xi, yo, rows, dim, eps, weight, scale, shift, mode);
  else rmsnorm_ada_kernel<16><<<grid, 256, smem, s>>>(xi, yo, rows, dim, eps, weight, scale, shift, mode);
  return check_launch("rmsnorm_ada");
}

static int qk_norm_rope_launch(const void* qkv_vid, const void* qkv_txt, const int32_t* row_src, const int32_t* row_rope,
                               const float* cos_tab, const float* sin_tab, int nfreq, const float* wq_vid,
                               const float* wk_vid, const float* wq_txt, const float* wk_txt, float eps, int n_rows,
                               int heads, void* q, void* k, void* v, const int32_t* row_list, void* stream) {
  if (n_rows <= 0) return SVR2_OK;
  if (6 * nfreq > 128) return set_error(SVR2_ERR_ARG, "rope: 6*nfreq > head_dim");
  const int threads = heads >= 8 ? 256 : 32 * heads;   // 8 warps loop over the heads (one warp per head was slower: 54 vs 34 ms)
  qk_norm_rope_window_kernel<<<n_rows, threads, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)qkv_vid, (const __nv_bfloat16*)qkv_txt, row_src, row_rope, cos_tab, sin_tab, nfreq, wq_vid,
      wk_vid, wq_txt, wk_txt, eps, heads, (__nv_bfloat16*)q, (__nv_bfloat16*)k, (__nv_bfloat16*)v, row_list);
  return check_launch("qk_norm_rope_window");
}

extern "C" int svr2_qk_norm_rope_window_bf16(const void* qkv_vid, const void* qkv_txt, const int32_t* row_src,
                                             const int32_t* row_rope, const float* cos_tab, const float* sin_tab,
                                             int nfreq, const float* wq_vid, const float* wk_vid, const float* wq_txt,
                                             const float* wk_txt, float eps, int total, int heads, void* q, void* k,
                                             void* v, void* stream) {
  return qk_norm_rope_launch(qkv_vid, qkv_txt, row_src, row_rope, cos_tab, sin_tab, nfreq, wq_vid, wk_vid, wq_txt, wk_txt,
                             eps, total, heads, q, k, v, nullptr, stream);
}

// Same, for the subset of output rows listed in row_list (the text rows of every window when the video rows come out
// of svr2_linear_qkv_rope_bf16's epilogue).
extern "C" int svr2_qk_norm_rope_rows_bf16(const void* qkv_vid, const void* qkv_txt, const int32_t* row_src,
                                           const int32_t* row_rope, const float* cos_tab, const float* sin_tab, int nfreq,
                                           const float* wq_vid, const float* wk_vid, const float* wq_txt,
                                           const float* wk_txt, float eps, const int32_t* row_list, int n_rows, int heads,
                                           void* q, void* k, void* v, void* stream) {
  if (!row_list) return set_error(SVR2_ERR_ARG, "svr2_qk_norm_rope_rows_bf16: row_list must not be NULL");
  return qk_norm_rope_launch(qkv_vid, qkv_txt, row_src, row_rope, cos_tab, sin_tab, nfreq, wq_vid, wk_vid, wq_txt, wk_txt,
                             eps, n_rows, heads, q, k, v, row_list, stream);
}

extern "C" int svr2_txt_window_mean_bf16(const void* in, void* out, int n_win, int l, int dim, void* stream) {
  if (dim % 8) return set_error(SVR2_ERR_ARG, "txt_window_mean: dim % 8");
  const long long nvec = (long long)l * dim / 8;
  txt_window_mean_kernel<<<(unsigned)((nvec + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)in, (__nv_bfloat16*)out, n_win, l, dim);
  return check_launch("txt_window_mean");
}

extern "C" int svr2_patchify_bf16(const void* vid, void* out, int T, int H, int W, int C, int ld_out, void* stream) {
  if ((H | W) & 1) return set_error(SVR2_ERR_ARG, "patchify: H, W must be even");
  const long long L = (long long)T * (H / 2) * (W / 2);
  patchify_kernel<<<(unsigned)L, 64, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)vid, (__nv_bfloat16*)out, T, H, W, C, ld_out);
  return check_launch("patchify");
}
extern "C" int svr2_unpatchify_bf16(const void* in, int ld_in, void* out, int T, int H, int W, int C, void* stream) {
  const long long L = (long long)T * (H / 2) * (W / 2);
  unpatchify_kernel<<<(unsigned)L, 64, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)in, ld_in, (__nv_bfloat16*)out, T, H, W, C);
  return check_launch("unpatchify");
}

extern "C" int svr2_groupnorm_bf16(const void* x, void* y, int frames, int hw, int C, const void* gamma,
                                   const void* beta, float eps, int silu, int out_t_pad, int out_dup_head,
                                   double* scratch, int64_t scratch_bytes, void* stream) {
  if (C % 32 || (C / 32 != 4 && C / 32 != 8 && C / 32 != 16))
    return set_error(SVR2_ERR_ARG, "groupnorm: C must be 128, 256 or 512");
  if (out_dup_head && out_t_pad != 2)        // the apply kernel copies frame 0 into exactly two halo frames
    return set_error(SVR2_ERR_ARG, "groupnorm: out_dup_head needs out_t_pad == 2");
  cudaStream_t s = (cudaStream_t)stream;
  int blocks_x = (int)((hw + 4095) / 4096);
  if (blocks_x < 1) blocks_x = 1;
  const int ppb = (hw + blocks_x - 1) / blocks_x;
  const size_t partial_bytes = sizeof(double) * 64 * (size_t)blocks_x * frames;
  const size_t coef_bytes = sizeof(float2) * (size_t)frames * C;
  if ((size_t)scratch_bytes < partial_bytes + coef_bytes) {
    char msg[160];
    snprintf(msg, sizeof msg, "groupnorm: scratch too small (%lld < %zu bytes)", (long long)scratch_bytes,
             partial_bytes + coef_bytes);
    return set_error(SVR2_ERR_ARG, msg);
  }
  float2* coef = reinterpret_cast<float2*>(reinterpret_cast<char*>(scratch) + partial_bytes);
  groupnorm_stats_kernel<<<dim3(blocks_x, frames), 256, 0, s>>>((const __nv_bfloat16*)x, hw, C, ppb, scratch);
  int rc = check_launch("groupnorm_stats");
  if (rc) return rc;
  groupnorm_finalize_kernel<<<frames, 256, 0, s>>>(scratch, blocks_x, hw, C, (const __nv_bfloat16*)gamma,
                                                   (const __nv_bfloat16*)beta, eps, coef);
  rc = check_launch("groupnorm_finalize");
  if (rc) return rc;
  launch_gn_apply(x, y, frames, hw, C, silu, out_t_pad, out_dup_head, coef, s);
  return check_launch("groupnorm_apply");
}

// GroupNorm(+SiLU) whose statistics were produced by svr2_conv3d_stats_bf16: finalize + apply only
// (saves the separate statistics read pass).  coef_scratch: frames * C * 8 bytes.
extern "C" int svr2_groupnorm_from_stats_bf16(const void* x, void* y, int frames, int hw, int C, const void* gamma,
                                              const void* beta, float eps, int silu, int out_t_pad, int out_dup_head,
                                              const void* stat_partial, int stat_slots, void* coef_scratch,
                                              void* stream) {
  if (C % 32 || (C / 32 != 4 && C / 32 != 8 && C / 32 != 16))
    return set_error(SVR2_ERR_ARG, "groupnorm: C must be 128, 256 or 512");
  if (out_dup_head && out_t_pad != 2)        // the apply kernel copies frame 0 into exactly two halo frames
    return set_error(SVR2_ERR_ARG, "groupnorm: out_dup_head needs out_t_pad == 2");
  cudaStream_t s = (cudaStream_t)stream;
  float2* coef = (float2*)coef_scratch;
  groupnorm_finalize_fused_kernel<<<dim3(32, frames), 256, 0, s>>>((const float4*)stat_partial, stat_slots,
                                                                   (const __nv_bfloat16*)x, hw, C,
                                                         (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta, eps,
                                                         coef);
  int rc = check_launch("groupnorm_finalize_fused");
  if (rc) return rc;
  launch_gn_apply(x, y, frames, hw, C, silu, out_t_pad, out_dup_head, coef, s);
  return check_launch("groupnorm_apply");
}

/* bytes of scratch svr2_groupnorm_bf16 needs for (frames, hw, C) */
extern "C" int64_t svr2_groupnorm_scratch_bytes(int frames, int hw, int C) {
  long long blocks_x = (hw + 4095) / 4096;
  if (blocks_x < 1) blocks_x = 1;
  return (int64_t)(sizeof(double) * 64 * blocks_x * frames + sizeof(float2) * (long long)frames * C);
}

extern "C" int svr2_rowstat_combine(const void* partial, int slots, int64_t ld, float* lse, int rows, void* stream) {
  if (rows <= 0) return SVR2_OK;
  rowstat_combine_kernel<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>((const float2*)partial, slots, ld, lse, rows);
  return check_launch("rowstat_combine");
}

extern "C" int svr2_rowstat_max(const void* partial, int slots, int64_t ld, float* mhat, int rows, int* flag_reset,
                                void* stream) {
  if (rows <= 0) return SVR2_OK;
  rowstat_max_kernel<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>((const float2*)partial, slots, ld, mhat, rows,
                                                                        flag_reset);
  return check_launch("rowstat_max");
}

extern "C" int svr2_pexp_stat_combine(const void* partial, int slots, int64_t ld, const float* mhat, float* rowscale,
                                      int rows, int* flag, void* stream) {
  if (rows <= 0) return SVR2_OK;
  if (!flag) return set_error(SVR2_ERR_ARG, "svr2_pexp_stat_combine: flag must not be NULL");
  pexp_stat_combine_kernel<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>((const float2*)partial, slots, ld, mhat,
                                                                              rowscale, rows, flag);
  return check_launch("pexp_stat_combine");
}

extern "C" int svr2_transpose_bf16(const void* in, int64_t ld_in, void* out, int64_t ld_out, int rows, int cols,
                                   void* stream) {
  dim3 grid((cols + 31) / 32, (rows + 31) / 32), block(32, 8);
  transpose_kernel<<<grid, block, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)in, ld_in, (__nv_bfloat16*)out, ld_out, rows, cols);
  return check_launch("transpose");
}

// strides of the NCDHW side in elements: a rectangle of a clip's frames (a spatial tile) or all of them
int svr2::ncdhw_to_ndhwc_window(const void* in, int in_dtype, int C, int T, int H, int W, int64_t chan_stride,
                                int64_t frame_stride, int row_stride, void* out, int C_pad, int out_t_pad, float div,
                                void* stream) {
  const long long total = (long long)T * H * W;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  cudaStream_t s = (cudaStream_t)stream;
  const long long cs = chan_stride, fs = frame_stride;
  const int rs = row_stride;
  if (in_dtype == 0) ncdhw_to_ndhwc_kernel<float><<<blocks, 256, 0, s>>>((const float*)in, C, T, H, W, cs, fs, rs, (__nv_bfloat16*)out, C_pad, out_t_pad, div);
  else if (in_dtype == 1) ncdhw_to_ndhwc_kernel<__nv_bfloat16><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)in, C, T, H, W, cs, fs, rs, (__nv_bfloat16*)out, C_pad, out_t_pad, div);
  else if (in_dtype == 2) ncdhw_to_ndhwc_kernel<__half><<<blocks, 256, 0, s>>>((const __half*)in, C, T, H, W, cs, fs, rs, (__nv_bfloat16*)out, C_pad, out_t_pad, div);
  else return set_error(SVR2_ERR_ARG, "ncdhw_to_ndhwc: dtype must be 0 (f32), 1 (bf16) or 2 (f16)");
  return check_launch("ncdhw_to_ndhwc");
}
// channel stride of the NCDHW side in elements (T*H*W for a contiguous tensor; larger for a temporal slice of a clip)
int svr2::ncdhw_to_ndhwc_strided(const void* in, int in_dtype, int C, int T, int H, int W, int64_t chan_stride, void* out,
                                 int C_pad, int out_t_pad, float div, void* stream) {
  return ncdhw_to_ndhwc_window(in, in_dtype, C, T, H, W, chan_stride, (int64_t)H * W, W, out, C_pad, out_t_pad, div, stream);
}
extern "C" int svr2_ncdhw_to_ndhwc_bf16(const void* in, int in_dtype, int C, int T, int H, int W, void* out, int C_pad,
                                        int out_t_pad, float div, void* stream) {
  return ncdhw_to_ndhwc_strided(in, in_dtype, C, T, H, W, (int64_t)T * H * W, out, C_pad, out_t_pad, div, stream);
}
int svr2::ndhwc_to_ncdhw_strided(const void* in, int ld_in, int C, int T, int H, int W, void* out, int out_dtype,
                                 int64_t chan_stride, void* stream) {
  const long long total = (long long)T * H * W;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  cudaStream_t s = (cudaStream_t)stream;
  const long long cs = chan_stride;
  if (out_dtype == 0) ndhwc_to_ncdhw_kernel<float><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)in, ld_in, C, T, H, W, (float*)out, cs);
  else if (out_dtype == 1) ndhwc_to_ncdhw_kernel<__nv_bfloat16><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)in, ld_in, C, T, H, W, (__nv_bfloat16*)out, cs);
  else return set_error(SVR2_ERR_ARG, "ndhwc_to_ncdhw: dtype must be 0 (f32) or 1 (bf16)");
  return check_launch("ndhwc_to_ncdhw");
}
extern "C" int svr2_ndhwc_to_ncdhw(const void* in, int ld_in, int C, int T, int H, int W, void* out, int out_dtype,
                                   void* stream) {
  return ndhwc_to_ncdhw_strided(in, ld_in, C, T, H, W, out, out_dtype, (int64_t)T * H * W, stream);
}
extern "C" int svr2_im2col3_bf16(const void* x, int T, int H, int W, int C, int ld_in, void* out, int ld_out,
                                 void* stream) {
  if (ld_out % 8) return set_error(SVR2_ERR_ARG, "im2col3: ld_out % 8");
  if (C == 3 && ld_in == 8 && ld_out == 128) {
    const long long rows = (long long)T * H * W;
    im2col3_c3_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, (cudaStream_t)stream>>>((const uint4*)x, T, H, W, (uint4*)out);
    return check_launch("im2col3_c3");
  }
  const long long total = (long long)T * H * W * (ld_out / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 64) blocks = 132LL * 64;
  im2col3_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, T, H, W, C, ld_in, (__nv_bfloat16*)out, ld_out);
  return check_launch("im2col3");
}

// z: [27*co_n rows][ldz] fp32 (row = tap*co_n + co, column = input pixel incl. 2 halo frames); out: [co_n,T,H,W] with
// channel stride chan_stride elements
int svr2::conv_tap_gather_strided(const float* z, int64_t ldz, int co_n, const void* bias, int T, int H, int W, void* out,
                                  int out_dtype, int64_t chan_stride, void* stream) {
  if (co_n < 1 || co_n > 4) return set_error(SVR2_ERR_ARG, "conv_tap_gather: 1 <= co_n <= 4");
  const long long total = (long long)T * H * W;
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 32) blocks = 132LL * 32;
  cudaStream_t s = (cudaStream_t)stream;
  const long long cs = chan_stride;
  if (out_dtype == 0)
    conv_tap_gather_kernel<float><<<(unsigned)blocks, 256, 0, s>>>(z, ldz, co_n, (const __nv_bfloat16*)bias, T, H, W, (float*)out, cs);
  else if (out_dtype == 1)
    conv_tap_gather_kernel<__nv_bfloat16><<<(unsigned)blocks, 256, 0, s>>>(z, ldz, co_n, (const __nv_bfloat16*)bias, T, H, W, (__nv_bfloat16*)out, cs);
  else return set_error(SVR2_ERR_ARG, "conv_tap_gather: dtype must be 0 (f32) or 1 (bf16)");
  return check_launch("conv_tap_gather");
}
extern "C" int svr2_conv_tap_gather(const float* z, int64_t ldz, int co_n, const void* bias, int T, int H, int W,
                                    void* out, int out_dtype, void* stream) {
  return conv_tap_gather_strided(z, ldz, co_n, bias, T, H, W, out, out_dtype, (int64_t)T * H * W, stream);
}

static SeamDev seam_dev(const svr2::Seam& s) {
  return SeamDev{(__nv_bfloat16*)s.result, (__nv_bfloat16*)s.count, (long long)s.cs, (long long)s.fs, s.rs,
                 (const __nv_bfloat16*)s.ramp_h, (const __nv_bfloat16*)s.ramp_w, s.len_h, s.len_w, s.edges};
}
static int seam_check(const svr2::Seam& s, const char* what) {
  if (!s.result || (s.len_h > 0 && !s.ramp_h) || (s.len_w > 0 && !s.ramp_w) || s.len_h < 0 || s.len_w < 0) {
    char buf[160];
    snprintf(buf, sizeof buf, "%s: result NULL, or a ramp table of positive length NULL", what);
    return set_error(SVR2_ERR_ARG, buf);
  }
  return SVR2_OK;
}
int svr2::conv_tap_gather_seam(const float* z, int64_t ldz, int co_n, const void* bias, int T, int H, int W, const Seam& s,
                               void* stream) {
  if (co_n < 1 || co_n > 4) return set_error(SVR2_ERR_ARG, "conv_tap_gather_seam: 1 <= co_n <= 4");
  if (int rc = seam_check(s, "conv_tap_gather_seam")) return rc;
  const long long total = (long long)T * H * W;
  if (total <= 0) return SVR2_OK;
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 32) blocks = 132LL * 32;
  conv_tap_gather_seam_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(z, ldz, co_n, (const __nv_bfloat16*)bias,
                                                                                   T, H, W, seam_dev(s));
  return check_launch("conv_tap_gather_seam");
}
int svr2::ndhwc_to_ncdhw_seam(const void* in, int ld_in, int C, int T, int H, int W, const Seam& s, void* stream) {
  if (C < 1 || C > 16 || ld_in < C) return set_error(SVR2_ERR_ARG, "ndhwc_to_ncdhw_seam: 1 <= C <= 16, ld_in >= C");
  if (int rc = seam_check(s, "ndhwc_to_ncdhw_seam")) return rc;
  const long long total = (long long)T * H * W;
  if (total <= 0) return SVR2_OK;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  ndhwc_to_ncdhw_seam_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)in, ld_in, C, T, H, W,
                                                                       seam_dev(s));
  return check_launch("ndhwc_to_ncdhw_seam");
}
extern "C" int svr2_conv_tap_gather_seam_bf16(const float* z, int64_t ldz, int co_n, const void* bias, int T, int H, int W,
                                              void* result, int64_t chan_stride, int64_t frame_stride, int row_stride,
                                              void* count, const void* ramp_h, int len_h, const void* ramp_w, int len_w,
                                              int edges, void* stream) {
  const Seam s{result, chan_stride, frame_stride, row_stride, count, ramp_h, ramp_w, len_h, len_w, edges};
  return conv_tap_gather_seam(z, ldz, co_n, bias, T, H, W, s, stream);
}
extern "C" int svr2_ndhwc_to_ncdhw_seam_bf16(const void* in, int ld_in, int C, int T, int H, int W, void* result,
                                             int64_t chan_stride, int64_t frame_stride, int row_stride, void* count,
                                             const void* ramp_h, int len_h, const void* ramp_w, int len_w, int edges,
                                             void* stream) {
  const Seam s{result, chan_stride, frame_stride, row_stride, count, ramp_h, ramp_w, len_h, len_w, edges};
  return ndhwc_to_ncdhw_seam(in, ld_in, C, T, H, W, s, stream);
}
