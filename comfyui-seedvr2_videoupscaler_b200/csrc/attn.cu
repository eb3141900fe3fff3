// K4 — varlen (windowed) self-attention for head_dim = 128 on wgmma (sm_90a).
//
// Drop-in for FlashAttentionVarlen.forward / pytorch_varlen_attention
// (reference dit_3b/attention.py:27-64, 114-148): for every sequence i (one Swin
// window + its 58 text tokens) and head h
//      O_i = softmax(Q_i K_i^T / sqrt(128)) V_i        (non-causal, no mask)
// on the packed (total, heads, 128) bf16 layout with int32 cu_seqlens.
//
// One CTA per work item (q-tile of 128 rows, head, sequence); 9 warps:
//   warps 0-7 : two consumer warpgroups, 64 query rows each:
//               S = Q K^T   wgmma m64n64k16, Q and K from 128B-swizzled smem (K-major), fp32 S in registers;
//               online softmax on the accumulator fragment (row max / sum over the 4 lanes sharing a row, exp2);
//               O += P V    wgmma m64n128k16 with P as the register A operand (bf16 pairs of the S fragment) and V
//                           straight from its row-major tile as an MN-major B operand; fp32 O in registers;
//               final 1/l and the scatter store through out_row_map
//   warp 8    : TMA producer (Q once, a 2-stage ring of K + V tiles)
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "ptx.cuh"
#include "svr2_internal.h"

namespace svr2 {

constexpr int ATT_BM = 128;      // q rows per CTA
constexpr int ATT_BN = 64;       // kv rows per tile
constexpr int ATT_D = 128;
constexpr int ATT_THREADS = 288;
constexpr int ATT_STAGES = 2;
constexpr int ATT_Q_BYTES = 128 * 128 * 2;          // 32 KB: two [128 x 64] swizzled halves
constexpr int ATT_QH_BYTES = ATT_Q_BYTES / 2;
constexpr int ATT_KV_BYTES = ATT_BN * 128 * 2;      // 16 KB: two [64 x 64] swizzled halves
constexpr int ATT_KVH_BYTES = ATT_KV_BYTES / 2;

struct AttnSmem {
  // offsets inside the 1024-aligned dynamic smem
  static constexpr int kQ = 0;
  static constexpr int kK = kQ + ATT_Q_BYTES;                      // ATT_STAGES K tiles
  static constexpr int kV = kK + ATT_STAGES * ATT_KV_BYTES;        // ATT_STAGES V tiles
  static constexpr int kBar = kV + ATT_STAGES * ATT_KV_BYTES;
  static constexpr int kTotal = kBar + 128 + 1024;
};

struct AttnParams {
  const int32_t* cu_seqlens;
  const int32_t* out_row_map;
  __nv_bfloat16* out;
  int heads;
  float scale_log2;  // softmax_scale * log2(e)
  int n_qt;          // q tiles per sequence (of the longest sequence)
};

__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_varlen_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                   const __grid_constant__ CUtensorMap tmap_v, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AttnSmem::kBar);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;                    // [ATT_STAGES]
  uint64_t* kv_empty = bars + 1 + ATT_STAGES;      // [ATT_STAGES]

  // work item -> (q tile, head, sequence); q tiles of one (sequence, head) are neighbours so that the CTAs running
  // at the same time share its K / V through L2
  const int w = blockIdx.x;
  const int qt = w % p.n_qt;
  const int rest = w / p.n_qt;
  const int head = rest % p.heads;
  const int seq = rest / p.heads;
  const int s_begin = p.cu_seqlens[seq];
  const int len = p.cu_seqlens[seq + 1] - s_begin;
  if (qt * ATT_BM >= len) return;                  // uniform over the CTA
  const int n_kv = (len + ATT_BN - 1) / ATT_BN;
  const int col0 = head * ATT_D;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < ATT_STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 2);                  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
      const int q_row0 = s_begin + qt * ATT_BM;
      mbar_expect_tx(q_full, ATT_Q_BYTES);
      tma_load_2d(smem + AttnSmem::kQ, &tmap_q, q_full, col0, q_row0);
      tma_load_2d(smem + AttnSmem::kQ + ATT_QH_BYTES, &tmap_q, q_full, col0 + 64, q_row0);
      for (int j = 0; j < n_kv; ++j) {
        const int s = j % ATT_STAGES;
        const int r0 = s_begin + j * ATT_BN;
        mbar_wait(&kv_empty[s], ((j / ATT_STAGES) & 1) ^ 1);
        mbar_expect_tx(&kv_full[s], 2 * ATT_KV_BYTES);
        uint8_t* k_dst = smem + AttnSmem::kK + s * ATT_KV_BYTES;
        uint8_t* v_dst = smem + AttnSmem::kV + s * ATT_KV_BYTES;
        tma_load_2d(k_dst, &tmap_k, &kv_full[s], col0, r0);
        tma_load_2d(k_dst + ATT_KVH_BYTES, &tmap_k, &kv_full[s], col0 + 64, r0);
        tma_load_2d(v_dst, &tmap_v, &kv_full[s], col0, r0);
        tma_load_2d(v_dst + ATT_KVH_BYTES, &tmap_v, &kv_full[s], col0 + 64, r0);
      }
    }
    return;
  }

  // ------------------------------ consumer warpgroups
  const int wg = warp >> 2;                        // rows [64 wg, 64 wg + 64) of the q tile
  const int quad = lane & 3;
  const int r_lo = wg * 64 + ((warp & 3) << 4) + (lane >> 2);   // this thread's rows: r_lo and r_lo + 8
  const float sc = p.scale_log2;
  const uint32_t q_addr = smem_u32(smem + AttnSmem::kQ) + wg * 64 * 128;
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  mbar_wait(q_full, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int s = j % ATT_STAGES;
    mbar_wait(&kv_full[s], (j / ATT_STAGES) & 1);
    const uint32_t k_addr = smem_u32(smem + AttnSmem::kK + s * ATT_KV_BYTES);
    const uint32_t v_addr = smem_u32(smem + AttnSmem::kV + s * ATT_KV_BYTES);
    float sv[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {                 // contraction over d = 128
      const uint64_t da = wgmma_desc_kmajor_sw128(q_addr + (kk >> 2) * ATT_QH_BYTES) + uint64_t((kk & 3) * 2);
      const uint64_t db = wgmma_desc_kmajor_sw128(k_addr + (kk >> 2) * ATT_KVH_BYTES) + uint64_t((kk & 3) * 2);
      wgmma_ss<ATT_BN>(sv, da, db, kk != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sv);

    const int kv_valid = len - j * ATT_BN;           // columns >= kv_valid are padding / the next sequence
    if (kv_valid < ATT_BN) {                         // only the last tile of a sequence is ragged
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if ((i >> 2) * 8 + 2 * quad + (i & 1) >= kv_valid) sv[i] = -INFINITY;
    }
    // row maxima (fragment rows: even register pairs -> r_lo, odd pairs -> r_lo + 8), reduced over the 4 lanes of a row
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 32; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sv[i]);
    float alpha[2], nmb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(m_run[h], mx[h]);
      alpha[h] = exp2_approx((m_run[h] - m_new) * sc);  // 0 on the first tile (m_run = -inf)
      nmb[h] = -m_new * sc;
      m_run[h] = m_new;
    }
    // P = exp2(s * sc - m * sc): fp32 row sums, bf16 pairs packed in the A-operand fragment order
    float ls[2] = {0.f, 0.f};
    uint32_t pa[16];
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int h = (i >> 1) & 1;
      const float e0 = exp2_approx(fmaf(sv[i], sc, nmb[h]));
      const float e1 = exp2_approx(fmaf(sv[i + 1], sc, nmb[h]));
      ls[h] += e0 + e1;
      pa[i >> 1] = pack_bf16x2(e0, e1);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * alpha[h] + ls[h];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] *= alpha[(i >> 1) & 1];

    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk) {       // contraction over the 64 kv rows (16 per MMA)
      const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
      const uint64_t db = wgmma_desc_mnmajor_sw128(v_addr + kk * 16 * 128, ATT_KVH_BYTES, 1024);
      wgmma_rs_tb<ATT_D>(o, a, db, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[s]);   // K_j / V_j fully read by this warpgroup
  }

  // ------------------------------ epilogue: O / l -> bf16 -> global
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float inv_l = 1.0f / l_run[h];
    const int q_idx = qt * ATT_BM + r_lo + 8 * h;
    if (q_idx >= len) continue;
    long long grow_ = (long long)(s_begin + q_idx);
    if (p.out_row_map) grow_ = p.out_row_map[grow_];
    __nv_bfloat16* orow = p.out + (grow_ * p.heads + head) * ATT_D;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const int i = 4 * c + 2 * h;
      *reinterpret_cast<uint32_t*>(orow + 8 * c + 2 * quad) = pack_bf16x2(o[i] * inv_l, o[i + 1] * inv_l);
    }
  }
}

}  // namespace svr2

using namespace svr2;

extern "C" int svr2_attn_varlen_bf16(const void* q, const void* k, const void* v, void* out,
                                     const int32_t* cu_seqlens, int n_seq, int total, int heads, int max_seqlen,
                                     const int32_t* out_row_map, void* stream) {
  if (n_seq <= 0 || total <= 0) return SVR2_OK;
  if (max_seqlen <= 0) return set_error(SVR2_ERR_ARG, "svr2_attn_varlen_bf16: max_seqlen must be > 0");
  static bool configured[64] = {};                // the attribute is per (function, device)
  auto kern = attn_varlen_kernel;
  const int dev = current_device();
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnSmem::kTotal);
    if (e != cudaSuccess) return set_error(SVR2_ERR_CUDA, cudaGetErrorString(e));
    configured[dev] = true;
  }
  CUtensorMap tq, tk, tv;
  uint64_t dims[2] = {(uint64_t)heads * ATT_D, (uint64_t)total};
  uint64_t strides[1] = {(uint64_t)heads * ATT_D * 2};
  uint32_t box_q[2] = {64, ATT_BM}, box_kv[2] = {64, ATT_BN};
  int rc = make_tmap_bf16(&tq, q, 2, dims, strides, box_q);
  if (rc) return rc;
  rc = make_tmap_bf16(&tk, k, 2, dims, strides, box_kv);
  if (rc) return rc;
  rc = make_tmap_bf16(&tv, v, 2, dims, strides, box_kv);
  if (rc) return rc;
  AttnParams p;
  p.cu_seqlens = cu_seqlens;
  p.out_row_map = out_row_map;
  p.out = (__nv_bfloat16*)out;
  p.heads = heads;
  p.scale_log2 = 1.4426950408889634f / sqrtf((float)ATT_D);
  p.n_qt = (max_seqlen + ATT_BM - 1) / ATT_BM;
  const long long n_work = (long long)p.n_qt * n_seq * heads;
  if (n_work > 0x7fffffffLL) return set_error(SVR2_ERR_ARG, "svr2_attn_varlen_bf16: too many work items");
  kern<<<(unsigned)n_work, ATT_THREADS, AttnSmem::kTotal, (cudaStream_t)stream>>>(tq, tk, tv, p);
  return check_launch("attn_varlen");
}
