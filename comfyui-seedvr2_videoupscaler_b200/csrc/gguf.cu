// GGUF block dequantization to fp16 (gguf_dequant.py:146-342): the eleven block formats the reference's
// `dequantize_functions` table handles, decoded once at load so the DiT loader receives dense fp16 tensors.
//
// Rounding: the reference runs every block function with dtype float16, so each torch op is one Half op — computed in
// fp32, rounded to fp16 before the next op reads it.  Here every product / sum / difference is one __fmul_rn /
// __fadd_rn / __fsub_rn followed by a rounding to fp16 (h() below, or the final store), never an FMA.  Scales are
// little-endian fp16.  The integer parts (nibbles, bits, signed offsets) are exact in fp16, as in the reference.
//
// Element order inside a block (E = element index within the block; "q[i]" = byte i of the named byte array):
//   Q8_0  (32 el, 34 B)   d | q[32] int8                     E -> q[E]
//   Q4_0  (32 el, 18 B)   d | q[16]                          E < 16: low nibble of q[E]; E >= 16: high nibble of q[E-16]
//   Q4_1  (32 el, 20 B)   d | m | q[16]                      nibbles as Q4_0
//   Q5_0  (32 el, 22 B)   d | qh u32 | q[16]                 nibble as Q4_0, 5th bit = bit E of qh
//   Q5_1  (32 el, 24 B)   d | m | qh u32 | q[16]             as Q5_0
//   Q2_K  (256 el, 84 B)  sc[16] | q[64] | d | dmin          E = 128g + 32s + l: (q[32g+l] >> 2s) & 3; sub-block E/16
//                                                            scales sc[j] & 15, mins sc[j] >> 4
//   Q3_K  (256 el, 110 B) hm[32] | q[64] | sc[12] | d        low 2 bits as Q2_K; high bit = bit (E/32) of hm[E%32],
//                                                            a clear bit subtracts 4; sub-block j = E/16 has the 6-bit
//                                                            scale (j < 8 ? sc[j] & 15 : sc[j-8] >> 4) | ((sc[8 + j%4]
//                                                            >> 2(j/4)) & 3) << 4, offset by -32
//   Q4_K  (256 el, 144 B) d | dmin | sc[12] | q[128]         sub-block j = E/32, l = E%32: (q[32(j/2)+l] >> 4(j%2)) & 15
//                                                            6-bit scale / min of j < 4: sc[j] & 63 / sc[j+4] & 63;
//                                                            j >= 4: (sc[j+4] & 15) | (sc[j-4] >> 6) << 4 /
//                                                                    (sc[j+4] >> 4) | (sc[j] >> 6) << 4
//   Q5_K  (256 el, 176 B) d | dmin | sc[12] | qh[32] | q[128] nibble and scales as Q4_K, 5th bit = bit j of qh[l]
//   Q6_K  (256 el, 210 B) ql[128] | qh[64] | sc[16] int8 | d E = 128h + r: low 4 bits (ql[64h + r%64] >> 4(r/64)) & 15,
//                                                            high 2 bits (qh[32h + r%32] >> 2(r/32)) & 3, minus 32;
//                                                            sub-block E/16 scales by sc[E/16]
//   BF16  (1 el, 2 B)                                        widened to fp32, then rounded to fp16 (out of range: inf)
//
// Shape: a CTA owns kElemsPerCta consecutive outputs, i.e. a whole number of blocks whose bytes are contiguous in the
// source.  It stages them into shared memory with coalesced 16-byte loads (4-byte ones when the source is only 4-byte
// aligned; blocks are mostly not 4-byte multiples, so per-thread loads from global would be unaligned), then each thread
// decodes 8 consecutive outputs — always inside one sub-block — and writes them as one 16-byte vector.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "svr2_internal.h"

namespace svr2 {
namespace {

enum GgmlType : int {
  kQ4_0 = 2, kQ4_1 = 3, kQ5_0 = 6, kQ5_1 = 7, kQ8_0 = 8, kQ2_K = 10, kQ3_K = 11, kQ4_K = 12, kQ5_K = 13, kQ6_K = 14,
  kBF16 = 30
};

// GGML's block geometry (elements, bytes) of the types this file decodes; false for any other type
constexpr bool geometry(int type, int* elems, int* bytes) {
  switch (type) {
    case kQ4_0: *elems = 32; *bytes = 18; return true;
    case kQ4_1: *elems = 32; *bytes = 20; return true;
    case kQ5_0: *elems = 32; *bytes = 22; return true;
    case kQ5_1: *elems = 32; *bytes = 24; return true;
    case kQ8_0: *elems = 32; *bytes = 34; return true;
    case kQ2_K: *elems = 256; *bytes = 84; return true;
    case kQ3_K: *elems = 256; *bytes = 110; return true;
    case kQ4_K: *elems = 256; *bytes = 144; return true;
    case kQ5_K: *elems = 256; *bytes = 176; return true;
    case kQ6_K: *elems = 256; *bytes = 210; return true;
    case kBF16: *elems = 1; *bytes = 2; return true;
    default: return false;
  }
}

constexpr int block_elems(int type) { int e = 0, b = 0; geometry(type, &e, &b); return e; }
constexpr int block_bytes(int type) { int e = 0, b = 0; geometry(type, &e, &b); return b; }

constexpr int kThreads = 256;
constexpr int kElemsPerCta = kThreads * 8;

__device__ __forceinline__ float h(float x) { return __half2float(__float2half_rn(x)); }
__device__ __forceinline__ float f16_at(const uint8_t* p) {
  return __half2float(__ushort_as_half((unsigned short)(p[0] | (p[1] << 8))));
}
__device__ __forceinline__ uint32_t u32_at(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// 6-bit scale and min of sub-block j (0..7) of a Q4_K / Q5_K block's 12 packed bytes
__device__ __forceinline__ void k_scale_min(const uint8_t* sc, int j, int* s, int* m) {
  if (j < 4) {
    *s = sc[j] & 63;
    *m = sc[j + 4] & 63;
  } else {
    *s = (sc[j + 4] & 15) | ((sc[j - 4] >> 6) << 4);
    *m = (sc[j + 4] >> 4) | ((sc[j] >> 6) << 4);
  }
}

// v[0..7] = elements e .. e+7 of the block at p before their final fp16 rounding (the caller's store rounds)
template <int TYPE>
__device__ __forceinline__ void decode8(const uint8_t* p, int e, float v[8]) {
  if constexpr (TYPE == kQ8_0) {
    const float d = f16_at(p);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = __fmul_rn(d, (float)(int8_t)p[2 + e + k]);
  } else if constexpr (TYPE == kQ4_0 || TYPE == kQ4_1 || TYPE == kQ5_0 || TYPE == kQ5_1) {
    constexpr bool has_min = TYPE == kQ4_1 || TYPE == kQ5_1;
    constexpr bool has_qh = TYPE == kQ5_0 || TYPE == kQ5_1;
    const float d = f16_at(p);
    const float m = has_min ? f16_at(p + 2) : 0.f;
    const uint8_t* qh = p + (has_min ? 4 : 2);
    const uint8_t* qs = qh + (has_qh ? 4 : 0);
    const uint32_t hbits = has_qh ? u32_at(qh) : 0u;
    const int shift = e < 16 ? 0 : 4;
    const int b0 = e & 15;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      int q = (qs[b0 + k] >> shift) & 15;
      if constexpr (has_qh) q |= (int)((hbits >> (e + k)) & 1u) << 4;
      if constexpr (has_min) {
        v[k] = __fadd_rn(h(__fmul_rn(d, (float)q)), m);
      } else {
        v[k] = __fmul_rn(d, (float)(q - (has_qh ? 16 : 8)));
      }
    }
  } else if constexpr (TYPE == kQ2_K) {
    const uint8_t* sc = p;
    const uint8_t* qs = p + 16;
    const float d = f16_at(p + 80), dmin = f16_at(p + 82);
    const int j = e >> 4, g = e >> 7, s = (e >> 5) & 3, l = e & 31;
    const float dl = h(__fmul_rn(d, (float)(sc[j] & 15)));
    const float ml = h(__fmul_rn(dmin, (float)(sc[j] >> 4)));
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int q = (qs[32 * g + l + k] >> (2 * s)) & 3;
      v[k] = __fsub_rn(h(__fmul_rn(dl, (float)q)), ml);
    }
  } else if constexpr (TYPE == kQ3_K) {
    const uint8_t* hm = p;
    const uint8_t* qs = p + 32;
    const uint8_t* sc = p + 96;
    const float d = f16_at(p + 108);
    const int j = e >> 4, g = e >> 7, s = (e >> 5) & 3, hb = e >> 5, l = e & 31;
    const int lo = j < 8 ? (sc[j] & 15) : (sc[j - 8] >> 4);
    const int hi = (sc[8 + (j & 3)] >> (2 * (j >> 2))) & 3;
    const float dl = h(__fmul_rn(d, (float)((lo | (hi << 4)) - 32)));
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int q = ((qs[32 * g + l + k] >> (2 * s)) & 3) - (((hm[l + k] >> hb) & 1) ? 0 : 4);
      v[k] = __fmul_rn(dl, (float)q);
    }
  } else if constexpr (TYPE == kQ4_K || TYPE == kQ5_K) {
    const float d = f16_at(p), dmin = f16_at(p + 2);
    const uint8_t* sc = p + 4;
    const uint8_t* qh = p + 16;
    const uint8_t* qs = p + (TYPE == kQ5_K ? 48 : 16);
    const int j = e >> 5, l = e & 31;
    int si, mi;
    k_scale_min(sc, j, &si, &mi);
    const float D = h(__fmul_rn(d, (float)si));
    const float M = h(__fmul_rn(dmin, (float)mi));
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      int q = (qs[32 * (j >> 1) + l + k] >> (4 * (j & 1))) & 15;
      if constexpr (TYPE == kQ5_K) q |= ((qh[l + k] >> j) & 1) << 4;
      v[k] = __fsub_rn(h(__fmul_rn(D, (float)q)), M);
    }
  } else if constexpr (TYPE == kQ6_K) {
    const uint8_t* ql = p;
    const uint8_t* qh = p + 128;
    const int8_t* sc = reinterpret_cast<const int8_t*>(p + 192);
    const float d = f16_at(p + 208);
    const int half_ = e >> 7, r = e & 127;
    const float S = h(__fmul_rn(d, (float)sc[e >> 4]));
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int lo = (ql[64 * half_ + ((r + k) & 63)] >> (4 * (r >> 6))) & 15;
      const int hi = (qh[32 * half_ + ((r + k) & 31)] >> (2 * (r >> 5))) & 3;
      v[k] = __fmul_rn(S, (float)((lo | (hi << 4)) - 32));
    }
  } else {  // BF16
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint8_t* q = p + 2 * k;
      v[k] = __uint_as_float(((uint32_t)q[0] | ((uint32_t)q[1] << 8)) << 16);
    }
  }
}

template <int TYPE>
__global__ void __launch_bounds__(kThreads) gguf_dequant_kernel(const uint8_t* __restrict__ src, long long n_elem,
                                                                __half* __restrict__ out, int vec16) {
  constexpr int BE = block_elems(TYPE), BB = block_bytes(TYPE);
  constexpr int kCtaBytes = kElemsPerCta / BE * BB;   // a multiple of 16 for every type
  static_assert(kCtaBytes % 16 == 0, "CTA byte range must keep the source alignment");
  __shared__ __align__(16) uint8_t s[kCtaBytes];
  const long long e_cta = (long long)blockIdx.x * kElemsPerCta;
  const long long byte0 = e_cta / BE * BB;
  const int nbytes = (int)min((long long)kCtaBytes, n_elem / BE * BB - byte0);
  const uint8_t* g = src + byte0;
  int done;
  if (vec16) {
    const int n16 = nbytes >> 4;
    for (int i = threadIdx.x; i < n16; i += kThreads)
      reinterpret_cast<uint4*>(s)[i] = __ldg(reinterpret_cast<const uint4*>(g) + i);
    done = n16 << 4;
  } else {
    const int n4 = nbytes >> 2;
    for (int i = threadIdx.x; i < n4; i += kThreads)
      reinterpret_cast<uint32_t*>(s)[i] = __ldg(reinterpret_cast<const uint32_t*>(g) + i);
    done = n4 << 2;
  }
  for (int i = done + threadIdx.x; i < nbytes; i += kThreads) s[i] = g[i];   // the tail of the last CTA
  __syncthreads();

  const int l = threadIdx.x * 8;               // first output of this thread, relative to the CTA
  const long long e0 = e_cta + l;
  if (e0 >= n_elem) return;
  float v[8];
  decode8<TYPE>(s + (l / BE) * BB, l % BE, v);
  if (e0 + 8 <= n_elem) {
    uint4 pack;
    __half2* ph = reinterpret_cast<__half2*>(&pack);
#pragma unroll
    for (int k = 0; k < 4; ++k) ph[k] = __halves2half2(__float2half_rn(v[2 * k]), __float2half_rn(v[2 * k + 1]));
    *reinterpret_cast<uint4*>(out + e0) = pack;
  } else {                                      // BF16 tensors whose element count is not a multiple of 8
    for (int k = 0; k < (int)(n_elem - e0); ++k) out[e0 + k] = __float2half_rn(v[k]);
  }
}

template <int TYPE>
void launch(const void* blocks, long long n, void* out, cudaStream_t s) {
  const long long grid = (n + kElemsPerCta - 1) / kElemsPerCta;
  const int vec16 = ((uintptr_t)blocks & 15) == 0;
  gguf_dequant_kernel<TYPE><<<(unsigned)grid, kThreads, 0, s>>>((const uint8_t*)blocks, n, (__half*)out, vec16);
}

}  // namespace
}  // namespace svr2

using namespace svr2;

extern "C" int svr2_gguf_type_size(int ggml_type, int* block_elems_out, int* block_bytes_out) {
  int e = 0, b = 0;
  if (!geometry(ggml_type, &e, &b)) {
    char buf[128];
    snprintf(buf, sizeof buf, "svr2_gguf_type_size: GGML type %d is not a block format the engine dequantizes",
             ggml_type);
    return set_error(SVR2_ERR_ARG, buf);
  }
  if (block_elems_out) *block_elems_out = e;
  if (block_bytes_out) *block_bytes_out = b;
  return SVR2_OK;
}

extern "C" int svr2_gguf_dequant_f16(int ggml_type, const void* blocks, int64_t n_elements, void* out, void* stream) {
  int be = 0, bb = 0;
  if (!geometry(ggml_type, &be, &bb)) {
    char buf[128];
    snprintf(buf, sizeof buf, "svr2_gguf_dequant_f16: GGML type %d is not a block format the engine dequantizes",
             ggml_type);
    return set_error(SVR2_ERR_ARG, buf);
  }
  if (n_elements <= 0) return set_error(SVR2_ERR_ARG, "svr2_gguf_dequant_f16: empty tensor");
  if (n_elements % be) return set_error(SVR2_ERR_ARG, "svr2_gguf_dequant_f16: n_elements is not a whole number of blocks");
  if ((n_elements + kElemsPerCta - 1) / kElemsPerCta >= ((int64_t)1 << 31))
    return set_error(SVR2_ERR_ARG, "svr2_gguf_dequant_f16: tensor too large");
  if (!blocks || !out) return set_error(SVR2_ERR_ARG, "svr2_gguf_dequant_f16: null tensor");
  if ((uintptr_t)blocks % 4) return set_error(SVR2_ERR_ARG, "svr2_gguf_dequant_f16: blocks must be 4-byte aligned");
  if ((uintptr_t)out % 16) return set_error(SVR2_ERR_ARG, "svr2_gguf_dequant_f16: out must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  switch (ggml_type) {
    case kQ4_0: launch<kQ4_0>(blocks, n_elements, out, s); break;
    case kQ4_1: launch<kQ4_1>(blocks, n_elements, out, s); break;
    case kQ5_0: launch<kQ5_0>(blocks, n_elements, out, s); break;
    case kQ5_1: launch<kQ5_1>(blocks, n_elements, out, s); break;
    case kQ8_0: launch<kQ8_0>(blocks, n_elements, out, s); break;
    case kQ2_K: launch<kQ2_K>(blocks, n_elements, out, s); break;
    case kQ3_K: launch<kQ3_K>(blocks, n_elements, out, s); break;
    case kQ4_K: launch<kQ4_K>(blocks, n_elements, out, s); break;
    case kQ5_K: launch<kQ5_K>(blocks, n_elements, out, s); break;
    case kQ6_K: launch<kQ6_K>(blocks, n_elements, out, s); break;
    default: launch<kBF16>(blocks, n_elements, out, s); break;
  }
  return check_launch("gguf_dequant");
}
