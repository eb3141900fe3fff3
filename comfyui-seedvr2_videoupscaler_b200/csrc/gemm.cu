// K1/K6 — persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] = A[M,K] · B[N,K]^T   (bf16 x bf16 -> fp32 in registers -> fused epilogue)
//
// One kernel body serves the DiT Linear layers (A = activation rows, 2-D TMA)
// and the VAE causal Conv3d as an implicit GEMM (A = shifted NDHWC boxes fetched
// by 4-D/5-D TMA with out-of-bounds zero fill = spatial zero padding; the causal
// temporal halo is two real frames stored in front of every activation tensor).
//
// Roles (384 threads, 1 CTA / SM, grid = #SMs, static tile schedule):
//   warps 0,3  : TMA producers (even / odd k-blocks of a kStages-deep smem ring, 128B-swizzled K-major tiles;
//                SLAB convs: warp 0 a weight ring, warp 3 a ring of activation slabs, see SlabLayout)
//   warps 4-11 : two MMA warpgroups (wgmma m64 x BLOCK_N x 16, 64 tile rows each, fp32 accumulators in registers)
//   KIND_BF16  : the MMA warpgroups round bf16(acc + bias) into a dedicated bf16 tile and go on with the next tile's
//                MMAs; warps 1,2 run the rest of the epilogue from that tile (activation, gate, residual, GroupNorm
//                partial sums, row-contiguous 16-byte global stores, halo copies) under those MMAs
//   other kinds: warps 1,2 idle; the MMA warpgroups also run the epilogue (accumulators -> fp32 tile in shared memory
//                over the drained ring -> one row per thread -> fused math -> swizzled smem slab -> global stores), so
//                the next tile's loads wait for it
//
// Reference semantics replaced: nn.Linear (dit_3b/mmattn.py:56-59,173,269; mlp.py:56-61;
// patch_v1.py:37,62), InflatedCausalConv3d (causal_inflation_lib.py:213-305), Upsample3D's
// 1x1x1 conv + pixel shuffle (attn_video_vae.py:135-143), with the elementwise ops around
// them (bias, AdaSingle gate, residual add, SwiGLU, GELU) fused into the epilogue and
// rounded to bf16 at the same points as the reference's bf16 path (SURVEY.md §8 G3).
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <type_traits>

#include "ptx.cuh"
#include "svr2_internal.h"

namespace svr2 {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 B = one swizzle row
constexpr int WGMMA_K = 16;

struct GemmParams {
  int M, N, K;
  int num_m_tiles, num_n_tiles, num_k_blocks;
  int band_h;            // conv m-tile raster: tile rows per band (order: band, frame, row in band, column)
  int group_n;           // n-tiles per L2 raster group (tiles run group by group: for group: for m: for n in group)
  // ---- A addressing (conv) ----
  int a_mode;            // 0 linear (2-D [M,K]); 1 conv stride-1 (4-D C,W,H,T); 2 conv spatial stride-2 (5-D pair view)
  int tiles_w, tiles_h;  // M tiles per output frame
  int bw, bh;            // output pixels per tile: bw*bh == 128
  int taps_t, taps_h, taps_w;
  int cin_blocks;        // Cin / 64
  int cin;               // Cin (pair view channel offset)
  int extra_blocks;      // conv: trailing 64-channel k-blocks read from the SECOND activation tensor (tmap_a2) at the
                         // output pixel itself (a fused 1x1x1 conv_shortcut: [h ; x] . [W2 ; Wsc], attn_video_vae.py:311-362)
  int pad_h, pad_w;      // subtracted from the tap offset (1 for padding=1)
  int stride_t;          // temporal stride of the conv (1 or 2)
  int H_out, W_out, T_out;
  // ---- epilogue ----
  int epi;               // EPI_* flags
  int ldc;               // elements between consecutive output rows/pixels
  long long out_frame_stride;  // conv/shuffle: elements per output frame
  int out_t_pad;         // leading halo frames in the output tensor (0 or 2)
  int out_dup_head;      // also write frame 0 into the halo frames
  // ---- conv head fold (SVR2_EPI_FOLD_HEAD): output frames t_o < fold_t read a halo that replicates input frame 0 and
  // run t_o + 1 temporal taps with the folded weights in B rows [fold_n, fold_n + Cout)
  int fold_t, fold_n;
  int shuf_c, shuf_z;    // pixel shuffle: channels per output voxel, temporal factor
  int shuf_H, shuf_W;    // input H,W of the shuffle GEMM (rows are (f,h,w))
  int shuf_drop;         // drop the duplicated first output frame (first chunk)
  float out_scale;       // fp32 output scale
  const __nv_bfloat16* bias;      // [N] or null
  const float* gate;              // [N] or null
  const __nv_bfloat16* residual;  // same layout as out, or null
  void* out;
  float4* stat_partial;           // conv only: [frame][slot][N/8] (sum0, sq0, sum1, sq1) of the stored values, or null
  int stat_slots;                 // slots per frame (tiles per frame x warps covering distinct rows)
  // ---- single-pass attention probabilities (VAE mid-block attention without the duplicated Q K^T pass)
  const float* rowscale;          // EPI_ROWSCALE: acc * rowscale[m] before everything else (P~ V / l)
  float2* stat2;                  // KIND_PEXP: also emit per (row, column slot) (max of acc*out_scale, sum of the exponentials)
  int ld_stat;                    // float2 slots per row of stat2
  const int* run_if;              // launch is a no-op unless *run_if != 0 (device-side conditional fallback), or null
  // ---- KIND_QKV*: fused q/k RMSNorm + RoPE + window scatter (out = q, out2 = k, out3 = v, each [rows, inner])
  void* out2;
  void* out3;
  const int32_t* tok_dst;         // [M] destination row (window order) of every token
  const int32_t* tok_rope;        // [M,3] rows of the cos/sin tables per axis, or -1
  const float* rope_cos;          // [R, nfreq]
  const float* rope_sin;
  const float* qk_weight;         // [2][128]: q-norm weight, k-norm weight
  float qk_eps;
  int qkv_inner;                  // heads * 128
};

enum : int {
  EPI_BIAS = 1,
  EPI_GATE = 2,       // t = bf16(t * gate[n])
  EPI_RESIDUAL = 4,   // out = bf16(t + res)
  EPI_SWIGLU = 8,     // out[:, j] = bf16(bf16(silu(bf16 acc[j])) * bf16 acc[j + BLOCK_N/2]) per tile
  EPI_GELU = 16,      // t = gelu_tanh(t)
  EPI_F32 = 32,       // fp32 output = acc * out_scale (no rounding)
  EPI_SHUFFLE = 64,   // Upsample3D pixel shuffle store
  EPI_SILU = 128,     // t = bf16(silu(t))
  EPI_ROWSTAT = 256,  // out: per (row, n-tile half) partial (max, sum exp2) of acc*out_scale  (attention pass 1)
  EPI_PEXP = 512,     // out: bf16(exp2(acc*out_scale - rowvec[m]))                         (attention pass 2)
  EPI_ROWSCALE = 1024,  // acc *= rowscale[m] first (un-normalised probabilities x V, divided by the row sum)
};

// EPI_WG: the epilogue warps' bf16 tile, BLOCK_M x max(BLOCK_N, 32) (swap-AB: 256 pixels x 128 channels);
// otherwise the per-warp epilogue slabs, 8 warps x (32 rows x 128 B)
template <int BLOCK_N, bool EPI_WG>
struct SmemLayout {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kTileCols = BLOCK_N < 32 ? 32 : BLOCK_N;
  static constexpr int kStagingBytes = EPI_WG ? BLOCK_M * kTileCols * 2 : 8 * 4096;
  static constexpr int kBudget = 232448 - kStagingBytes - 256 - 1024;   // 227 KB max dynamic smem
  static constexpr int kStages = kBudget / kStageBytes > 8 ? 8 : kBudget / kStageBytes;
  static constexpr int kStagingOffset = kStages * kStageBytes;
  static constexpr int kBarOffset = kStagingOffset + kStagingBytes;
  static constexpr int kTotal = kBarOffset + 256 + 1024;  // barriers + alignment slack
};

// Slab mainloop (SLAB: stride-1 3x3 convs on the swap-AB and the 256-column tiles).  The taps kh = 0, 1, 2 of one
// (kt, kw, channel block) read the same bw x bh activation box shifted down by one image row each, so one bw x (bh + 2)
// box -- the slab -- holds all three: tap kh is the slab from row kh on, kh * bw * 128 bytes in, a whole number of
// 1024-byte swizzle atoms for every tile shape that takes this path.  The ring splits in two: a weight ring of one
// k-block's weight tile per stage and a slab ring of one slab per stage, both sized from SmemLayout's budget.  (The
// one-ring members it inherits only let the ring code, which a SLAB kernel never runs, compile.)
template <bool SWAP>
struct SlabLayout : SmemLayout<256, true> {
  using Base = SmemLayout<256, true>;
  static constexpr int kWBytes = (SWAP ? BLOCK_M : 256) * BLOCK_K * 2;          // 16 KB / 32 KB
  static constexpr int kSBytes = (SWAP ? 32 * 10 : 16 * 10) * BLOCK_K * 2;      // the widest slab: 32 x 10 / 16 x 10 px
  static constexpr int kSStages = SWAP ? 2 : 3;
  static constexpr int kWStages = (Base::kBudget - kSStages * kSBytes) / kWBytes;
  static constexpr int kStages = kWStages + kSStages;   // barriers: the weight stages, then the slab stages
  static constexpr int kSlabOffset = kWStages * kWBytes;
  static constexpr int kStagingOffset = kSlabOffset + kSStages * kSBytes;
  static constexpr int kBarOffset = kStagingOffset + Base::kStagingBytes;
  static constexpr int kTotal = kBarOffset + 256 + 1024;
  static_assert(kWStages >= 3 && kSBytes % 1024 == 0 && kTotal <= 232448, "slab rings do not fit");
};

// 32 consecutive fp32 accumulator columns of one row of the shared accumulator tile (idx: element offset, % 4 == 0)
__device__ __forceinline__ void acc_ld32(const float* acc, uint32_t idx, uint32_t (&v)[32]) {
  const float4* s = reinterpret_cast<const float4*>(acc + idx);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 t = s[i];
    v[4 * i] = __float_as_uint(t.x); v[4 * i + 1] = __float_as_uint(t.y);
    v[4 * i + 2] = __float_as_uint(t.z); v[4 * i + 3] = __float_as_uint(t.w);
  }
}

// per-lane GroupNorm partial sums of the 8 bf16 values a lane stores (channels 0-3 -> x/y, 4-7 -> z/w)
__device__ __forceinline__ void stat_acc(float4& a, const uint4& d) {
  const uint32_t w[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float lo = __uint_as_float(w[e] << 16), hi = __uint_as_float(w[e] & 0xffff0000u);
    if (e < 2) { a.x += lo + hi; a.y += lo * lo + hi * hi; }
    else { a.z += lo + hi; a.w += lo * lo + hi * hi; }
  }
}

// bf16(a + b) of 8 bf16 values (the residual add)
__device__ __forceinline__ uint4 add_bf16x8(const uint4& a, const uint4& b) {
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
  uint32_t o[4];
#pragma unroll
  for (int e = 0; e < 4; ++e)
    o[e] = pack_bf16x2(__uint_as_float(aw[e] << 16) + __uint_as_float(bw[e] << 16),
                       __uint_as_float(aw[e] & 0xffff0000u) + __uint_as_float(bw[e] & 0xffff0000u));
  return make_uint4(o[0], o[1], o[2], o[3]);
}

// Conv m-tile raster.  A causal 3x3x3 conv reads every input frame for three consecutive output frames; in
// frame-major tile order those three reads are a whole frame apart (GBs) and all miss L2.  Tiles are therefore
// ordered band-major: a band of `band_h` tile rows is swept over ALL output frames before the next band, so the
// three temporal taps (and the vertical 3x3 halo inside the band) hit L2.
__device__ __forceinline__ void conv_tile(const GemmParams& p, int m_blk, int& t_o, int& th, int& tw) {
  const int full = p.T_out * p.band_h * p.tiles_w;          // m-tiles in a full band
  const int band = m_blk / full;
  const int r = m_blk - band * full;
  const int rows_left = p.tiles_h - band * p.band_h;
  const int rows = rows_left < p.band_h ? rows_left : p.band_h;
  const int per = rows * p.tiles_w;                          // tiles of this band in one frame
  t_o = r / per;
  const int rr = r - t_o * per;
  const int trow = rr / p.tiles_w;
  th = band * p.band_h + trow;
  tw = rr - trow * p.tiles_w;
}

// k-blocks of a conv m-tile: with folded head taps, output frame 0 runs one temporal tap and frame 1 two
__device__ __forceinline__ int conv_k_blocks(const GemmParams& p, int m_blk) {
  if (p.fold_t == 0) return p.num_k_blocks;
  int t_o, th, tw;
  conv_tile(p, m_blk, t_o, th, tw);
  return t_o < p.fold_t ? p.num_k_blocks - (p.taps_t - 1 - t_o) * p.taps_h * p.taps_w * p.cin_blocks : p.num_k_blocks;
}

// L2-aware tile raster: the n-tiles are processed in groups of `g` columns of tiles; inside a group the order is
// m-major with n fastest, so a group's slice of B (g * BLOCK_N * K * 2 bytes, chosen <= ~16 MB by the host) stays
// L2-resident while A streams through once per group.  (Plain n-fastest order re-streams all of B from DRAM for
// every m-row once B exceeds L2 — 132 MB for the 4K VAE attention keys.)
__device__ __forceinline__ void tile_coords(int tile, int num_m, int num_n, int g, int& m, int& n) {
  const int per_group = g * num_m;
  const int ng = tile / per_group;
  const int r = tile - ng * per_group;
  const int n0 = ng * g;
  const int gsz = (num_n - n0) < g ? (num_n - n0) : g;
  m = r / gsz;
  n = n0 + (r - m * gsz);
}

enum : int { KIND_BF16 = 0, KIND_SWIGLU = 1, KIND_F32 = 2, KIND_ROWSTAT = 3, KIND_PEXP = 4,
             KIND_QKV21 = 5, KIND_QKV10 = 6,
             KIND_BF16_RS = 7,
             KIND_PEXP_STAT = 8 };   // KIND_PEXP that also emits per-slot (0, sum of exponentials)   // KIND_BF16 with a per-row scale on the accumulator (its own instantiation: a runtime test in
                                   // the shared per-element loop cost the pixel-shuffle store 50 %)   // QKV projection + q/k RMSNorm + RoPE (21 / 10 frequencies per axis) + window scatter

// KIND_BF16 epilogues start with bf16(acc + bias), and everything after it acts on that bf16 value: the MMA warpgroups
// compute it and hand a bf16 tile to the two epilogue warps.  The other kinds need the fp32 accumulators (or a
// row-wide first step) in the epilogue and keep it on the MMA warpgroups.
template <int KIND> constexpr bool kEpiWG = KIND == KIND_BF16;
constexpr int kNumThreads = 384;   // producer warpgroup (2 TMA warps, 2 epilogue warps for KIND_BF16) + 2 MMA warpgroups
constexpr int kEpiWarps = 2;       // KIND_BF16: warps 1 and 2, 64 tile rows each

// 16-byte chunk swizzle of the swap-AB bf16 tile (rows = pixels, 16 chunks of 8 channels): distinct for 8 consecutive
// pixels (stmatrix rows) and in different halves of the 8-chunk bank cycle for a pixel pair (the epilogue's reads)
__device__ __forceinline__ int swap_tile_swz(int pix) { return ((pix & 1) << 2) | ((pix >> 1) & 3); }

// One tile's output row of a thread: destination offset (elements), validity, halo duplication.
struct RowDest {
  long long off;
  int valid;
  int dup;
};

template <int BLOCK_N>
__device__ __forceinline__ RowDest row_dest(const GemmParams& p, int epi, int m_blk, int n_blk, int row, int n_cols) {
  RowDest d;
  d.dup = 0;
  if (epi & EPI_SHUFFLE) {
    const int m = m_blk * BLOCK_M + row;
    d.valid = m < p.M;
    const int hw = p.shuf_H * p.shuf_W;
    const int f = m / hw, rr = m - f * hw, h = rr / p.shuf_W, w = rr - h * p.shuf_W;
    // channel n = ((x*2 + y)*Z + z)*C + c ; a BLOCK_N tile never straddles a (x,y,z) group
    const int grp = (n_blk * BLOCK_N) / p.shuf_c;
    const int z = grp % p.shuf_z, y = (grp / p.shuf_z) & 1, x = grp / (p.shuf_z * 2);
    int t_out = f * p.shuf_z + z;
    if (p.shuf_drop) {
      // remove_head (causal_inflation_lib.py:412-419): keep (f=0,z=0), drop (f=0,z=1)
      if (f == 0 && z == 1) d.valid = 0;
      if (f > 0) t_out -= 1;
    }
    const int Wo = p.shuf_W * 2;
    const long long pix = (long long)(2 * h + x) * Wo + (2 * w + y);
    d.off = (long long)(t_out + p.out_t_pad) * p.out_frame_stride + pix * p.ldc + ((n_blk * BLOCK_N) % p.shuf_c);
    d.dup = (p.out_dup_head && t_out == 0 && d.valid) ? 1 : 0;
  } else if (p.a_mode == 0) {
    const int m = m_blk * BLOCK_M + row;
    d.valid = m < p.M;
    d.off = (long long)m * p.ldc + (long long)n_blk * n_cols;
  } else {
    int t_o, th, tw;
    conv_tile(p, m_blk, t_o, th, tw);
    const int rh = row / p.bw;
    const int h = th * p.bh + rh;
    const int w = tw * p.bw + (row - rh * p.bw);
    d.valid = (h < p.H_out) && (w < p.W_out);
    d.off = (long long)(t_o + p.out_t_pad) * p.out_frame_stride + ((long long)h * p.W_out + w) * p.ldc +
            (long long)n_blk * BLOCK_N;
    d.dup = (p.out_dup_head && t_o == 0 && d.valid) ? 1 : 0;
  }
  return d;
}

// SWAP (conv only, BLOCK_N = 256): operands exchanged so that M = 128 output channels (weights as A)
// and N = 256 output pixels (activation box as B).  Cout = 128 layers then run 128x256 tiles instead of
// 128x128 ones (half the weight traffic per output, twice the MMA work per k-block).
// EPI_CT >= 0: the epilogue flags are a compile-time constant (p.epi must equal it) — the per-element loops then carry
// no runtime flag tests.  A single such test cost the short-K pixel-shuffle GEMM 50 % (its epilogue, ~1 800 warp
// instructions per tile, is the whole kernel); EPI_CT = -1 keeps the generic runtime-flag epilogue.
// SLAB: the slab mainloop (SlabLayout); tmap_a then has the box (64, bw, bh + 2, 1).
template <int BLOCK_N, int KIND, bool SWAP = false, int EPI_CT = -1, bool SLAB = false>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_a2, const GemmParams p) {
  if (p.run_if != nullptr && *p.run_if == 0) return;     // conditional launch: every thread of every CTA sees the same flag
  constexpr bool EPI_WG = kEpiWG<KIND>;
  static_assert(EPI_WG || (!SWAP && EPI_CT < 0), "swap-AB and compile-time epilogues are KIND_BF16 only");
  static_assert(!SLAB || (KIND == KIND_BF16 && BLOCK_N == 256), "the slab mainloop is KIND_BF16 with 256-column tiles");
  using S = SlabLayout<SWAP>;
  using L = std::conditional_t<SLAB, S, SmemLayout<BLOCK_N, EPI_WG>>;
  constexpr int kStages = L::kStages;
  constexpr int ACC_STRIDE = BLOCK_N < 32 ? 32 : BLOCK_N;   // accumulator columns the epilogue addresses
  constexpr int ACC_LD = ACC_STRIDE + 4;                    // fp32 row pitch of the shared accumulator tile
  static_assert(EPI_WG || BLOCK_M * ACC_LD * 4 <= L::kStagingOffset, "the accumulator tile overlays the operand ring");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* acc_free = empty_bar + kStages;      // the epilogue is done with the accumulator tile (it overlays the ring)
  uint64_t* tile_full = acc_free + 1;            // EPI_WG: the MMA warpgroups have written the bf16 tile
  uint64_t* tile_empty = acc_free + 2;           // EPI_WG: the epilogue warps have read it
  const float* acc_s = reinterpret_cast<const float*>(smem);
  uint8_t* tile_s = smem + L::kStagingOffset;    // EPI_WG: the bf16 tile

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (p.extra_blocks) tma_prefetch_desc(&tmap_a2);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);                  // one arrive per consumer warpgroup
    }
    if constexpr (EPI_WG) {
      mbar_init(tile_full, 256);
      mbar_init(tile_empty, 32 * kEpiWarps);
    } else {
      mbar_init(acc_free, 256);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int num_n_tiles = p.num_n_tiles;
  const int num_m_tiles = p.num_m_tiles;
  const int num_tiles = num_m_tiles * num_n_tiles;
  const int tile0 = (int)blockIdx.x;
  const int tile_step = (int)gridDim.x;

  if (warp == 0 || warp == 3) {
    // ========================= TMA producers (2 warps) =========================
    if constexpr (SLAB) {
      // One thread of warp 0 feeds the weight ring (one stage per k-block), one thread of warp 3 the slab ring (one
      // stage per (kt, kw, channel block), then one per shortcut k-block, holding its bw x bh box).  A tile's k-blocks
      // run kt, kw, channel block, kh = 0, 1, 2; the weight column of a tap is ((kt 3 + kh) 3 + kw) Cin + 64 cb.
      if (lane == 0) {
        const bool wgt = warp == 0;
        const int n_st = wgt ? S::kWStages : S::kSStages;
        const int bar0 = wgt ? 0 : S::kWStages;
        const int st_bytes = wgt ? S::kWBytes : S::kSBytes;
        uint8_t* const ring = smem + (wgt ? 0 : S::kSlabOffset);
        int stage = 0;
        uint32_t phase = 0;
        auto acquire = [&](uint32_t bytes, uint64_t*& fb) -> uint8_t* {
          mbar_wait(&empty_bar[bar0 + stage], phase ^ 1);
          fb = &full_bar[bar0 + stage];
          mbar_expect_tx(fb, bytes);
          uint8_t* s = ring + stage * st_bytes;
          if (++stage == n_st) { stage = 0; phase ^= 1; }
          return s;
        };
        const int bw = p.bw, bh = p.bh, taps_t = p.taps_t, cin_blocks = p.cin_blocks, cin = p.cin;
        const uint32_t slab_bytes = bw * (bh + 2) * BLOCK_K * 2, box_bytes = bw * bh * BLOCK_K * 2;
        for (int tile = tile0; tile < num_tiles; tile += tile_step) {
          int m_blk, n_blk, t_o, th, tw;
          tile_coords(tile, num_m_tiles, num_n_tiles, p.group_n, m_blk, n_blk);
          conv_tile(p, m_blk, t_o, th, tw);
          const int h0 = th * bh, w0 = tw * bw;
          int n0 = n_blk * (SWAP ? BLOCK_M : BLOCK_N);
          int taps = taps_t, kcol = 0;
          if (t_o < p.fold_t) {      // folded head, as in the ring producer below
            taps = t_o + 1;
            kcol = t_o == 0 ? 2 * 9 * cin : 0;
            n0 += p.fold_n;
          }
          uint64_t* fb;
          for (int kt_ = 0; kt_ < taps; ++kt_) {
            const int t_in = t_o * p.stride_t + taps_t - taps + kt_;
            for (int kw_ = 0; kw_ < 3; ++kw_) {
              for (int cb = 0; cb < cin_blocks; ++cb) {
                if (wgt) {
                  for (int kh_ = 0; kh_ < 3; ++kh_) {
                    uint8_t* s = acquire(S::kWBytes, fb);
                    tma_load_2d(s, &tmap_b, fb, kcol + ((kt_ * 3 + kh_) * 3 + kw_) * cin + cb * BLOCK_K, n0);
                  }
                } else {
                  uint8_t* s = acquire(slab_bytes, fb);
                  tma_load_4d(s, &tmap_a, fb, cb * BLOCK_K, w0 + kw_ - p.pad_w, h0 - p.pad_h, t_in);
                }
              }
            }
          }
          kcol += taps * 9 * cin;
          for (int cb = 0; cb < p.extra_blocks; ++cb) {
            if (wgt) {
              uint8_t* s = acquire(S::kWBytes, fb);
              tma_load_2d(s, &tmap_b, fb, kcol + cb * BLOCK_K, n0);
            } else {
              uint8_t* s = acquire(box_bytes, fb);
              tma_load_4d(s, &tmap_a2, fb, cb * BLOCK_K, w0, h0, t_o);
            }
          }
        }
      }
    } else if (lane == 0) {
      // One thread of warp 0 feeds the even k-blocks of the ring, one thread of warp 3 the odd ones, so that the
      // per-k-block issue path (barrier poll, expect-tx, two TMA issues) of one thread never paces the MMAs.
      // Without the epilogue warps the shared accumulator tile of the epilogue overlays the ring: a tile's loads
      // start once the previous tile's epilogue has released it (acc_free).
      int stage = 0;
      uint32_t phase = 0;
      uint32_t g = (warp == 0) ? 0u : 1u;   // parity toggle: handle a k-block when (g & 1) == 0
      uint32_t it = 0;                      // tiles started by this CTA
      const int a_mode = p.a_mode;
      const int nkb = p.num_k_blocks;
      auto acquire = [&](uint8_t*& sa, uint64_t*& fb) -> bool {
        const bool mine = (g++ & 1u) == 0u;
        if (mine) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          sa = smem + stage * L::kStageBytes;
          fb = &full_bar[stage];
          mbar_expect_tx(fb, L::kStageBytes);
        }
        return mine;
      };
      auto advance = [&]() {
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      };
      auto tile_start = [&]() {
        if (!EPI_WG && it > 0) mbar_wait(acc_free, (it - 1) & 1u);
        ++it;
      };
      if (a_mode == 0) {
        for (int tile = tile0; tile < num_tiles; tile += tile_step) {
          int m_blk, n_blk;
          tile_coords(tile, num_m_tiles, num_n_tiles, p.group_n, m_blk, n_blk);
          tile_start();
          const int m0 = m_blk * BLOCK_M, n0 = n_blk * BLOCK_N;
          for (int kb = 0; kb < nkb; ++kb) {
            uint8_t* sa; uint64_t* fb;
            if (acquire(sa, fb)) {
              tma_load_2d(sa, &tmap_a, fb, kb * BLOCK_K, m0);
              tma_load_2d(sa + L::kABytes, &tmap_b, fb, kb * BLOCK_K, n0);
            }
            advance();
          }
        }
      } else {
        const int bw = p.bw, bh = p.bh, pad_h = p.pad_h, pad_w = p.pad_w, stride_t = p.stride_t;
        const int taps_t = p.taps_t, taps_h = p.taps_h, taps_w = p.taps_w, cin_blocks = p.cin_blocks, cin = p.cin;
        for (int tile = tile0; tile < num_tiles; tile += tile_step) {
          int m_blk, n_blk;
          tile_coords(tile, num_m_tiles, num_n_tiles, p.group_n, m_blk, n_blk);
          tile_start();
          int t_o, th, tw;
          conv_tile(p, m_blk, t_o, th, tw);
          const int h0 = th * bh, w0 = tw * bw;
          int n0 = n_blk * (SWAP ? BLOCK_M : BLOCK_N);
          int taps = taps_t, kcol = 0;
          if (t_o < p.fold_t) {
            // folded head: fold rows are [bf16(W0+W1) W2 | bf16(W0+W1+W2)], read from input frame 0 on
            taps = t_o + 1;
            kcol = t_o == 0 ? 2 * taps_h * taps_w * cin : 0;
            n0 += p.fold_n;
          }
          for (int kt_ = 0; kt_ < taps; ++kt_) {
            const int t_in = t_o * stride_t + taps_t - taps + kt_;
            for (int kh_ = 0; kh_ < taps_h; ++kh_) {
              for (int kw_ = 0; kw_ < taps_w; ++kw_) {
                for (int cb = 0; cb < cin_blocks; ++cb) {
                  uint8_t* sa; uint64_t* fb;
                  if (acquire(sa, fb)) {
                    uint8_t* s_act = SWAP ? sa + L::kABytes : sa;      // activation box
                    uint8_t* s_wgt = SWAP ? sa : sa + L::kABytes;      // weight rows
                    if (a_mode == 1) {
                      tma_load_4d(s_act, &tmap_a, fb, cb * BLOCK_K, w0 + kw_ - pad_w, h0 + kh_ - pad_h, t_in);
                    } else {
                      // pair view (2C, W/2, 2, H/2, T): input pixel 2*o + k -> pair o + k/2, phase k%2
                      tma_load_5d(s_act, &tmap_a, fb, (kw_ & 1) * cin + cb * BLOCK_K, w0 + (kw_ >> 1), kh_ & 1,
                                  h0 + (kh_ >> 1), t_in);
                    }
                    tma_load_2d(s_wgt, &tmap_b, fb, kcol, n0);
                  }
                  kcol += BLOCK_K;
                  advance();
                }
              }
            }
          }
          // fused 1x1x1 shortcut: extra k-blocks from the second tensor at the output pixels (no tap offset, no halo)
          for (int cb = 0; cb < p.extra_blocks; ++cb) {
            uint8_t* sa; uint64_t* fb;
            if (acquire(sa, fb)) {
              uint8_t* s_act = SWAP ? sa + L::kABytes : sa;
              uint8_t* s_wgt = SWAP ? sa : sa + L::kABytes;
              tma_load_4d(s_act, &tmap_a2, fb, cb * BLOCK_K, w0, h0, t_o);
              tma_load_2d(s_wgt, &tmap_b, fb, kcol, n0);
            }
            kcol += BLOCK_K;
            advance();
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ========================= MMA warpgroups (2) =========================
    // Mainloop: warpgroup wg owns tile rows [64 wg, 64 wg + 64): one wgmma m64 x BLOCK_N x 16 per 16 columns of K,
    // fp32 accumulators in registers, A and B straight from the 128B-swizzled stages.  The stage of k-block kb is
    // released once the MMAs of kb + 1 are issued and those of kb have retired (one MMA group in flight).
    // `tail` then takes the accumulators out of the registers.
    const int wg = (warp - 4) >> 2;
    int mstage = 0;
    uint32_t mphase = 0;
    uint32_t it = 0;
    auto mainloop = [&](int nkb, auto&& tail) {
      float d[BLOCK_N / 2];
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) d[i] = 0.f;
      const bool leader = (threadIdx.x & 127) == 0;
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[mstage], mphase);
        const uint32_t a_addr = smem_u32(smem + mstage * L::kStageBytes);
        const uint64_t a_desc = wgmma_desc_kmajor_sw128(a_addr + wg * 64 * 128);
        const uint64_t b_desc = wgmma_desc_kmajor_sw128(a_addr + L::kABytes);
        wgmma_fence_regs(d);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
          wgmma_ss<BLOCK_N>(d, a_desc + uint64_t(k * 2), b_desc + uint64_t(k * 2), (kb | k) != 0);
        wgmma_commit();
        wgmma_fence_regs(d);
        wgmma_wait<1>();
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = mstage;
        if (++mstage == kStages) { mstage = 0; mphase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
      tail(d);
    };
    // Slab mainloop: k-block kb waits on its weight stage and, at the first k-block of a slab, on the slab stage, and
    // reads the slab from row kh on.  A stage is released once the MMAs of the last k-block that reads it have retired
    // (the same one-group-in-flight rule, per ring).  The shortcut's k-blocks are one-use slabs read from row 0.
    int wstage = 0, sstage = 0;
    uint32_t wphase = 0, sphase = 0;
    auto mainloop_slab = [&](int nkb, auto&& tail) {
      float d[BLOCK_N / 2];
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) d[i] = 0.f;
      const bool leader = (threadIdx.x & 127) == 0;
      const int nkb_taps = nkb - p.extra_blocks;            // a multiple of 3: slabs of kh = 0, 1, 2
      const uint32_t row_bytes = p.bw * BLOCK_K * 2;
      const uint32_t w_ring = smem_u32(smem), s_ring = smem_u32(smem + S::kSlabOffset);
      int prev_w = -1, prev_s = -1, kh = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[wstage], wphase);
        if (kh == 0) mbar_wait(&full_bar[S::kWStages + sstage], sphase);
        const uint32_t w_addr = w_ring + wstage * S::kWBytes;
        const uint32_t s_addr = s_ring + sstage * S::kSBytes + kh * row_bytes;
        const uint64_t a_desc = wgmma_desc_kmajor_sw128((SWAP ? w_addr : s_addr) + wg * 64 * 128);
        const uint64_t b_desc = wgmma_desc_kmajor_sw128(SWAP ? s_addr : w_addr);
        wgmma_fence_regs(d);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
          wgmma_ss<BLOCK_N>(d, a_desc + uint64_t(k * 2), b_desc + uint64_t(k * 2), (kb | k) != 0);
        wgmma_commit();
        wgmma_fence_regs(d);
        wgmma_wait<1>();
        if (leader) {
          if (prev_w >= 0) mbar_arrive(&empty_bar[prev_w]);
          if (prev_s >= 0) mbar_arrive(&empty_bar[S::kWStages + prev_s]);
        }
        prev_w = wstage;
        if (++wstage == S::kWStages) { wstage = 0; wphase ^= 1; }
        prev_s = -1;
        if (kh == 2 || kb >= nkb_taps) {                    // the last k-block that reads this slab
          prev_s = sstage;
          if (++sstage == S::kSStages) { sstage = 0; sphase ^= 1; }
          kh = 0;
        } else {
          ++kh;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      if (leader) {
        if (prev_w >= 0) mbar_arrive(&empty_bar[prev_w]);
        if (prev_s >= 0) mbar_arrive(&empty_bar[S::kWStages + prev_s]);
      }
      tail(d);
    };
    const int epi = EPI_CT >= 0 ? EPI_CT : p.epi;
    const __nv_bfloat16* __restrict__ bias = p.bias;
    if constexpr (EPI_WG) {
      // bf16(acc + bias) -- the first rounding point of every KIND_BF16 epilogue, the same fp32 add and round to
      // nearest even -- into the bf16 tile with stmatrix, then on to the next tile.  A warp's fragment is 16 rows:
      // register group i..i+7 covers columns 16 (i / 8) .. +15, i.e. four 8x8 matrices (rows r0 / r0 + 8, column
      // halves), lanes 8j..8j+7 address the 16-byte rows of matrix j.  Row-major tile rows, 16-byte chunks XOR-swizzled
      // by (row % 8): conflict-free for the matrix stores and for the epilogue's 8-lane row reads.  Swap-AB: the rows
      // are output channels and the epilogue reads pixels, so the matrices are stored transposed into a pixel-major
      // tile [256 pixels][128 channels].
      const int r0 = wg * 64 + ((warp & 3) << 4);
      const uint32_t tbase = smem_u32(tile_s);
      const int lr = lane & 7, mj = lane >> 3;
      auto store_tile = [&](float (&d)[BLOCK_N / 2], int n_blk) {
        if (it > 0) mbar_wait(tile_empty, (it - 1) & 1u);   // the epilogue warps are done with the previous tile
        if constexpr (SWAP) {
          const int co = n_blk * BLOCK_M + r0 + (lane >> 2);
          const bool has_bias = (epi & EPI_BIAS) != 0;
          const float b0 = (has_bias && co < p.N) ? __bfloat162float(bias[co]) : 0.f;
          const float b1 = (has_bias && co + 8 < p.N) ? __bfloat162float(bias[co + 8]) : 0.f;
          const int chunk = (r0 >> 3) + (mj & 1);
#pragma unroll
          for (int i = 0; i < BLOCK_N / 2; i += 8) {
            const int pix = (i >> 3) * 16 + ((mj >> 1) << 3) + lr;
            stmatrix_x4_trans(tbase + pix * 256 + ((chunk ^ swap_tile_swz(pix)) << 4),
                              pack_bf16x2(d[i] + b0, d[i + 1] + b0), pack_bf16x2(d[i + 2] + b1, d[i + 3] + b1),
                              pack_bf16x2(d[i + 4] + b0, d[i + 5] + b0), pack_bf16x2(d[i + 6] + b1, d[i + 7] + b1));
          }
        } else {
          constexpr int ROW_B = L::kTileCols * 2;
          constexpr int SWZ = (L::kTileCols / 8 < 8 ? L::kTileCols / 8 : 8) - 1;
          const int row = r0 + ((mj & 1) << 3) + lr;
          const int cn0 = n_blk * BLOCK_N + 2 * (lane & 3);
#pragma unroll
          for (int i = 0; i < BLOCK_N / 2; i += 8) {
            float x[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) x[e] = d[i + e];
            if (epi & EPI_BIAS) {
              const int cn = cn0 + (i >> 3) * 16;
              const uint32_t bl = cn < p.N ? __ldg(reinterpret_cast<const unsigned int*>(bias + cn)) : 0u;
              const uint32_t bh = cn + 8 < p.N ? __ldg(reinterpret_cast<const unsigned int*>(bias + cn + 8)) : 0u;
              x[0] += __uint_as_float(bl << 16); x[1] += __uint_as_float(bl & 0xffff0000u);
              x[2] += __uint_as_float(bl << 16); x[3] += __uint_as_float(bl & 0xffff0000u);
              x[4] += __uint_as_float(bh << 16); x[5] += __uint_as_float(bh & 0xffff0000u);
              x[6] += __uint_as_float(bh << 16); x[7] += __uint_as_float(bh & 0xffff0000u);
            }
            const int chunk = (i >> 3) * 2 + (mj >> 1);
            stmatrix_x4(tbase + row * ROW_B + ((chunk ^ (row & SWZ)) << 4), pack_bf16x2(x[0], x[1]),
                        pack_bf16x2(x[2], x[3]), pack_bf16x2(x[4], x[5]), pack_bf16x2(x[6], x[7]));
          }
        }
        mbar_arrive(tile_full);
      };
      for (int tile = tile0; tile < num_tiles; tile += tile_step, ++it) {
        int m_blk, n_blk;
        tile_coords(tile, num_m_tiles, num_n_tiles, p.group_n, m_blk, n_blk);
        auto store = [&](float (&d)[BLOCK_N / 2]) { store_tile(d, n_blk); };
        if constexpr (SLAB) mainloop_slab(conv_k_blocks(p, m_blk), store);
        else mainloop(conv_k_blocks(p, m_blk), store);
      }
    } else {
      // The accumulators go to a row-major fp32 tile in shared memory (over the drained operand ring), and the
      // epilogue below reads its rows from there:
      // Two warps per 32-row quadrant (warp % 4), each owning half of the tile's columns.
      // Phase 1: a thread owns one accumulator row: 32 columns at a time, fused math, result
      //          (bf16 or fp32) into a per-warp XOR-swizzled staging slab (32 rows x 128 B).
      // Phase 2: the warp re-reads the slab row-major so that every global load/store instruction covers
      //          contiguous 128-byte row segments (16 B per lane); residual loads are issued in batches
      //          before use, then add + store.
      auto acc_to_smem = [&](float (&d)[BLOCK_N / 2]) {
        named_bar_sync(1, 256);                    // both warpgroups' MMAs have read their last operands
        float* acc_w = reinterpret_cast<float*>(smem);
        const int r0 = wg * 64 + ((warp & 3) << 4) + (lane >> 2);
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; i += 4) {
          const int col = (i >> 2) * 8 + 2 * (lane & 3);
          *reinterpret_cast<float2*>(acc_w + r0 * ACC_LD + col) = make_float2(d[i], d[i + 1]);
          *reinterpret_cast<float2*>(acc_w + (r0 + 8) * ACC_LD + col) = make_float2(d[i + 2], d[i + 3]);
        }
        named_bar_sync(1, 256);
      };
      constexpr bool IS_BF16 = KIND == KIND_BF16_RS;
      constexpr bool IS_PEXP = KIND == KIND_PEXP || KIND == KIND_PEXP_STAT;
      constexpr int N_COLS = KIND == KIND_SWIGLU ? ACC_STRIDE / 2 : ACC_STRIDE;   // output columns per tile
      constexpr int COLS_W = N_COLS >= 64 ? N_COLS / 2 : N_COLS;                 // columns per epilogue warp
      constexpr int PH_COLS = KIND == KIND_F32 ? 32 : (COLS_W < 64 ? COLS_W : 64);
      constexpr int CPR = KIND == KIND_F32 ? PH_COLS / 4 : PH_COLS / 8;    // 16-byte chunks per staged row
      constexpr int ROWS_PER_IT = 32 / CPR;
      constexpr int N_IT = 32 / ROWS_PER_IT;                                // warp-wide accesses per phase
      constexpr int kBatch = N_IT < 4 ? N_IT : 4;
      const int q = warp & 3;               // 32-row quadrant of the tile this warp's epilogue covers
      const int half = (warp - 4) >> 2;     // which half of the columns
      const int row = q * 32 + lane;        // tile row owned by this thread
      const bool active = (N_COLS >= 64) || (half == 0);
      const int col_lo = (N_COLS >= 64) ? half * COLS_W : 0;
      uint8_t* slab = smem + L::kStagingOffset + (warp - 4) * 4096;
      const int n_lim = KIND == KIND_SWIGLU ? p.N / 2 : p.N;
      const float* __restrict__ gate = p.gate;
      const __nv_bfloat16* __restrict__ resid = p.residual;
      for (int tile = tile0; tile < num_tiles; tile += tile_step) {
        int m_blk, n_blk;
        tile_coords(tile, num_m_tiles, num_n_tiles, p.group_n, m_blk, n_blk);
        if (it++ > 0) {                        // the previous tile's epilogue is done with the accumulator tile
          fence_proxy_async_smem();
          mbar_arrive(acc_free);
        }
        mainloop(conv_k_blocks(p, m_blk), acc_to_smem);
        RowDest dst = row_dest<BLOCK_N>(p, epi, m_blk, n_blk, row, N_COLS);
        const int n_base = n_blk * (KIND == KIND_SWIGLU ? BLOCK_N / 2 : BLOCK_N);   // first output column

        // Wide path (64-column phases): per-column operands live in lane registers (lane l holds columns 2l, 2l+1
        // of the phase) and are broadcast by shuffle in phase 1; they are fetched before the accumulator tile is read so
        // the global-load latency never sits on the epilogue's critical path.
        constexpr bool kWide = (IS_BF16 || IS_PEXP) && PH_COLS == 64;
        constexpr int N_PH = kWide ? COLS_W / 64 : 1;
        uint32_t bias_pk[N_PH];
        float2 gate2[N_PH];
        if constexpr (kWide && IS_BF16) {
#pragma unroll
          for (int ph = 0; ph < N_PH; ++ph) {
            const int cn = n_base + col_lo + ph * 64 + 2 * lane;
            const bool ok = cn < p.N;
            bias_pk[ph] = ((epi & EPI_BIAS) && ok) ? *reinterpret_cast<const uint32_t*>(bias + cn) : 0u;
            gate2[ph] = ((epi & EPI_GATE) && ok) ? *reinterpret_cast<const float2*>(gate + cn) : make_float2(0.f, 0.f);
          }
        }

        const uint32_t t_addr = row * ACC_LD;

        float row_lse = 0.f;
        float2 st_a = make_float2(0.f, 0.f), st_b = make_float2(0.f, 0.f);   // KIND_PEXP_STAT: this thread's row sum
        if constexpr (IS_PEXP) {
          const int m = m_blk * BLOCK_M + row;
          row_lse = (m < p.M) ? gate[m] : 0.f;
        }
        float row_scale = 1.f;
        if constexpr (KIND == KIND_BF16_RS) {
          const int m = m_blk * BLOCK_M + row;
          row_scale = (p.a_mode == 0 && m < p.M) ? p.rowscale[m] : 1.f;
        }
        if constexpr (KIND == KIND_QKV21 || KIND == KIND_QKV10) {
          // NaSwinAttention between the QKV projection and the attention call (mmattn.py:199-248, rope.py:116-176), in
          // the epilogue: a 256-column tile is two heads of q, of k or of v, so this warp's 128 columns are ONE head of
          // ONE row per thread — per-head RMSNorm is a thread-local sum, RoPE pairs are adjacent registers.  The bf16
          // rounding of the projection output comes first (the reference normalises the bf16 Linear output in fp32).
          static_assert(BLOCK_N == 256, "QKV epilogue needs 256-column tiles");
          constexpr int NF = KIND == KIND_QKV21 ? 21 : 10;
          const int tpw = p.qkv_inner / 256;               // n-tiles per q / k / v
          const int which = n_blk / tpw;                   // 0 q, 1 k, 2 v
          const int m = m_blk * BLOCK_M + row;
          const bool rvalid = (m < p.M);
          uint32_t pk[64];
#pragma unroll
          for (int c0 = 0; c0 < 128; c0 += 64) {
            uint32_t v0[32], v1[32];
            acc_ld32(acc_s, t_addr + col_lo + c0, v0);
            acc_ld32(acc_s, t_addr + col_lo + c0 + 32, v1);
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              pk[c0 / 2 + i] = pack_bf16x2(__uint_as_float(v0[2 * i]), __uint_as_float(v0[2 * i + 1]));
              pk[c0 / 2 + 16 + i] = pack_bf16x2(__uint_as_float(v1[2 * i]), __uint_as_float(v1[2 * i + 1]));
            }
          }
          if (which < 2) {
            float ss = 0.f;
#pragma unroll
            for (int i = 0; i < 64; ++i) {
              const float lo = __uint_as_float(pk[i] << 16), hi = __uint_as_float(pk[i] & 0xffff0000u);
              ss = fmaf(lo, lo, ss);
              ss = fmaf(hi, hi, ss);
            }
            const float rr = 1.0f / sqrtf(ss * (1.0f / 128.0f) + p.qk_eps);
            const float2* wn = reinterpret_cast<const float2*>(p.qk_weight + which * 128);
            int ri[3] = {-1, -1, -1};
            if (rvalid) {
              ri[0] = p.tok_rope[(long long)m * 3 + 0];
              ri[1] = p.tok_rope[(long long)m * 3 + 1];
              ri[2] = p.tok_rope[(long long)m * 3 + 2];
            }
#pragma unroll
            for (int i = 0; i < 64; ++i) {
              const float2 w2 = __ldg(wn + i);
              const float x0 = __uint_as_float(pk[i] << 16) * rr * w2.x;
              const float x1 = __uint_as_float(pk[i] & 0xffff0000u) * rr * w2.y;
              float y0 = x0, y1 = x1;
              if (i < 3 * NF) {                        // compile-time: pairs 3*NF..63 are not rotated
                const int tr = ri[i / NF];
                if (tr >= 0) {
                  const float c = __ldg(p.rope_cos + tr * NF + (i % NF)), sn = __ldg(p.rope_sin + tr * NF + (i % NF));
                  y0 = x0 * c - x1 * sn;               // interleaved pairs: (x0, x1) -> (x0 c - x1 s, x1 c + x0 s)
                  y1 = x1 * c + x0 * sn;
                }
              }
              pk[i] = pack_bf16x2(y0, y1);
            }
          }
          __nv_bfloat16* ob = reinterpret_cast<__nv_bfloat16*>(which == 0 ? p.out : (which == 1 ? p.out2 : p.out3));
          const long long roff = rvalid ? (long long)p.tok_dst[m] * p.qkv_inner + (long long)(n_blk - which * tpw) * 256 : 0;
#pragma unroll
          for (int ph = 0; ph < 2; ++ph) {
#pragma unroll
            for (int c = 0; c < 8; ++c)
              *reinterpret_cast<uint4*>(slab + lane * 128 + ((c ^ (lane & 7)) << 4)) =
                  make_uint4(pk[ph * 32 + 4 * c], pk[ph * 32 + 4 * c + 1], pk[ph * 32 + 4 * c + 2], pk[ph * 32 + 4 * c + 3]);
            __syncwarp();
            const int ch = lane & 7, rsub = lane >> 3;       // 8 x 16-byte chunks per staged row, 4 rows per access
#pragma unroll
            for (int it = 0; it < 8; ++it) {
              const int r = it * 4 + rsub;
              const long long off = __shfl_sync(0xffffffffu, roff, r);
              const int ok = __shfl_sync(0xffffffffu, (int)rvalid, r);
              if (ok) {
                const uint4 d = *reinterpret_cast<const uint4*>(slab + r * 128 + ((ch ^ (r & 7)) << 4));
                *reinterpret_cast<uint4*>(ob + off + col_lo + ph * 64 + ch * 8) = d;
              }
            }
            __syncwarp();
          }
        } else if constexpr (KIND == KIND_ROWSTAT) {
          // attention pass 1: thread-local online (max, sum exp2) over this warp's columns; no staging
          float mx = -INFINITY, sum = 0.f;
          if (active) {
            const float sc = p.out_scale;
            constexpr int RS = COLS_W >= 64 ? 64 : 32;      // columns in flight per step
#pragma unroll 1
            for (int c0 = col_lo; c0 < col_lo + COLS_W; c0 += RS) {
              uint32_t v[RS];
              acc_ld32(acc_s, t_addr + c0, *reinterpret_cast<uint32_t(*)[32]>(&v[0]));
              if constexpr (RS == 64) acc_ld32(acc_s, t_addr + c0 + 32, *reinterpret_cast<uint32_t(*)[32]>(&v[32]));
              const int n0 = n_base + c0;
              if (sc > 0.f && n0 + RS <= p.N) {
                // interior step: max on the raw accumulators, the scale folded into the exponent's FMA
                float cm = __uint_as_float(v[0]);
#pragma unroll
                for (int j = 1; j < RS; ++j) cm = fmaxf(cm, __uint_as_float(v[j]));
                const float m_new = fmaxf(mx, cm * sc);
                float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
                for (int j = 0; j < RS; j += 2) {
                  cs0 += exp2_approx(fmaf(__uint_as_float(v[j]), sc, -m_new));
                  cs1 += exp2_approx(fmaf(__uint_as_float(v[j + 1]), sc, -m_new));
                }
                sum = sum * exp2_approx(mx - m_new) + (cs0 + cs1);
                mx = m_new;
              } else {
                float cm = -INFINITY;
#pragma unroll
                for (int j = 0; j < RS; ++j) {
                  const float t = (n0 + j < p.N) ? __uint_as_float(v[j]) * sc : -INFINITY;
                  v[j] = __float_as_uint(t);
                  cm = fmaxf(cm, t);
                }
                const float m_new = fmaxf(mx, cm);
                if (m_new > -INFINITY) {
                  float cs = 0.f;
#pragma unroll
                  for (int j = 0; j < RS; ++j) cs += exp2_approx(__uint_as_float(v[j]) - m_new);
                  sum = sum * exp2_approx(mx - m_new) + cs;
                  mx = m_new;
                }
              }
            }
          }
          const int m = m_blk * BLOCK_M + row;
          if (active && m < p.M) {
            const int slot = (N_COLS >= 64) ? n_blk * 2 + half : n_blk;
            reinterpret_cast<float2*>(p.out)[(long long)m * p.ldc + slot] = make_float2(mx, sum);
          }
        } else if (active) {
#pragma unroll 1
          for (int ph0 = col_lo; ph0 < col_lo + COLS_W; ph0 += PH_COLS) {
            // ---------------- phase 1 ----------------
            if constexpr (kWide) {
              // both 32-column accumulator chunks of the phase loaded at once; every bf16 rounding point is one
              // cvt.rn.bf16x2 on a column pair (identical to bf16_rne, half the instructions), and the packed
              // pair is what gets staged
              uint32_t v0[32], v1[32];
              acc_ld32(acc_s, t_addr + ph0, v0);
              acc_ld32(acc_s, t_addr + ph0 + 32, v1);
              const int phi = (ph0 - col_lo) / 64;
              uint32_t pk[32];
              const float sc = p.out_scale;
              constexpr bool want_stats = KIND == KIND_PEXP_STAT;
              const bool stats_full = n_base + ph0 + 64 <= p.N;
              const bool plain = !(epi & (EPI_GELU | EPI_SILU | EPI_GATE));
              auto elements = [&](auto ragged) {
#pragma unroll
              for (int i = 0; i < 32; ++i) {
                float a = __uint_as_float(i < 16 ? v0[2 * (i & 15)] : v1[2 * (i & 15)]);
                float b = __uint_as_float(i < 16 ? v0[2 * (i & 15) + 1] : v1[2 * (i & 15) + 1]);
                if constexpr (IS_PEXP) {
                  // two of every five column pairs take their exp2 on the FMA pipe: the epilogue is MUFU-bound (128 ex2 per
                  // thread and tile = 2048 SM cycles against 1024 of MMA at K = 512)
                  const bool kPoly = (KIND == KIND_PEXP_STAT) && ((i % 5 == 1) || (i % 5 == 3));   // folds after unrolling
                  const float xa = fmaf(a, sc, -row_lse), xb = fmaf(b, sc, -row_lse);
                  const float ea = kPoly ? exp2_poly(xa) : exp2_approx(xa), eb = kPoly ? exp2_poly(xb) : exp2_approx(xb);
                  pk[i] = pack_bf16x2(ea, eb);
                  if constexpr (want_stats) {         // fp32 row sum of the exponentials (two packed chains)
                    if constexpr (decltype(ragged)::value) {   // last n-tile: zero-padded operand columns are not scores
                      const int cn = n_base + ph0 + 2 * i;
                      if (cn < p.N) st_a.x += ea;
                      if (cn + 1 < p.N) st_a.y += eb;
                    } else {
                      if (i & 1) st_b = fadd2(st_b, make_float2(ea, eb));
                      else st_a = fadd2(st_a, make_float2(ea, eb));
                    }
                  }
                } else {
                  if constexpr (KIND == KIND_BF16_RS) {
                    a *= row_scale;
                    b *= row_scale;
                  }
                  if (epi & EPI_BIAS) {
                    const uint32_t bw_ = __shfl_sync(0xffffffffu, bias_pk[phi], i);
                    a += __uint_as_float(bw_ << 16);
                    b += __uint_as_float(bw_ & 0xffff0000u);
                  }
                  uint32_t r = pack_bf16x2(a, b);
                  if (!plain) {
                    if (epi & EPI_GELU) {
                      r = pack_bf16x2(gelu_tanh_fast(__uint_as_float(r << 16)), gelu_tanh_fast(__uint_as_float(r & 0xffff0000u)));
                    }
                    if (epi & EPI_SILU) {
                      r = pack_bf16x2(silu_fast(__uint_as_float(r << 16)), silu_fast(__uint_as_float(r & 0xffff0000u)));
                    }
                    if (epi & EPI_GATE) {
                      const float g0 = __shfl_sync(0xffffffffu, gate2[phi].x, i);
                      const float g1 = __shfl_sync(0xffffffffu, gate2[phi].y, i);
                      r = pack_bf16x2(__uint_as_float(r << 16) * g0, __uint_as_float(r & 0xffff0000u) * g1);
                    }
                  }
                  pk[i] = r;
                }
              }
              };
              if (want_stats && !stats_full) elements(std::true_type{});
              else elements(std::false_type{});
#pragma unroll
              for (int c = 0; c < 8; ++c)
                *reinterpret_cast<uint4*>(slab + lane * 128 + ((c ^ (lane & 7)) << 4)) =
                    make_uint4(pk[4 * c], pk[4 * c + 1], pk[4 * c + 2], pk[4 * c + 3]);
            } else {
#pragma unroll 1
            for (int c0 = ph0; c0 < ph0 + PH_COLS; c0 += 32) {
              uint32_t v[32];
              acc_ld32(acc_s, t_addr + c0, v);
              if constexpr (KIND == KIND_SWIGLU) {
                uint32_t u[32];
                acc_ld32(acc_s, t_addr + ACC_STRIDE / 2 + c0, u);
                // rounding points of the reference's bf16 flow (gate, in, silu(gate), product), one
                // cvt.rn.bf16x2 per column pair each; v[0..15] end up holding the packed output pairs
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                  const uint32_t rg = pack_bf16x2(__uint_as_float(v[2 * i]), __uint_as_float(v[2 * i + 1]));
                  const uint32_t ru = pack_bf16x2(__uint_as_float(u[2 * i]), __uint_as_float(u[2 * i + 1]));
                  const uint32_t rs = pack_bf16x2(silu_fast(__uint_as_float(rg << 16)),
                                                  silu_fast(__uint_as_float(rg & 0xffff0000u)));
                  v[i] = pack_bf16x2(__uint_as_float(rs << 16) * __uint_as_float(ru << 16),
                                     __uint_as_float(rs & 0xffff0000u) * __uint_as_float(ru & 0xffff0000u));
                }
              } else if constexpr (KIND == KIND_F32) {
                const float sc = p.out_scale;
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = __float_as_uint(__uint_as_float(v[j]) * sc);
              } else {
                static_assert(IS_PEXP, "the bf16 kinds take the wide path");
                const float sc = p.out_scale;
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  v[j] = __float_as_uint(bf16_rne(exp2_approx(__uint_as_float(v[j]) * sc - row_lse)));
              }
              // stage: chunk index within the phase row, XOR-swizzled by the row
              if constexpr (KIND == KIND_F32) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                  const int ch = j ^ (lane & (CPR - 1));
                  *reinterpret_cast<uint4*>(slab + lane * 128 + ch * 16) =
                      make_uint4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                }
              } else if constexpr (KIND == KIND_SWIGLU) {
                const int cbase = (c0 - ph0) / 8;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const int ch = (cbase + j) ^ (lane & (CPR - 1));
                  *reinterpret_cast<uint4*>(slab + lane * 128 + ch * 16) =
                      make_uint4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                }
              } else {
                // values are already bf16-representable: packing is a byte permute (no conversion)
                const int cbase = (c0 - ph0) / 8;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const int ch = (cbase + j) ^ (lane & (CPR - 1));
                  *reinterpret_cast<uint4*>(slab + lane * 128 + ch * 16) =
                      make_uint4(__byte_perm(v[8 * j], v[8 * j + 1], 0x7632), __byte_perm(v[8 * j + 2], v[8 * j + 3], 0x7632),
                                 __byte_perm(v[8 * j + 4], v[8 * j + 5], 0x7632), __byte_perm(v[8 * j + 6], v[8 * j + 7], 0x7632));
                }
              }
            }
            }   // !kWide
            __syncwarp();
            // ---------------- phase 2 ----------------
            const int ch = lane % CPR, rsub = lane / CPR;
            const int col = ph0 + (KIND == KIND_F32 ? ch * 4 : ch * 8);
            const bool col_ok = (n_base + col) < n_lim;
#pragma unroll 1
            for (int b0 = 0; b0 < N_IT; b0 += kBatch) {
              long long off[kBatch];
              int flags[kBatch];
              uint4 rv[kBatch];
#pragma unroll
              for (int i = 0; i < kBatch; ++i) {
                const int r = (b0 + i) * ROWS_PER_IT + rsub;
                off[i] = __shfl_sync(0xffffffffu, dst.off, r);
                const int f = __shfl_sync(0xffffffffu, dst.valid | (dst.dup << 1), r);
                flags[i] = col_ok ? f : 0;
                if constexpr (IS_BF16) {
                  if ((epi & EPI_RESIDUAL) && (flags[i] & 1)) rv[i] = *reinterpret_cast<const uint4*>(resid + off[i] + col);
                }
              }
#pragma unroll
              for (int i = 0; i < kBatch; ++i) {
                if (!(flags[i] & 1)) continue;
                const int r = (b0 + i) * ROWS_PER_IT + rsub;
                uint4 d = *reinterpret_cast<const uint4*>(slab + r * 128 + ((ch ^ (r & (CPR - 1))) << 4));
                if constexpr (KIND == KIND_F32) {
                  *reinterpret_cast<uint4*>(reinterpret_cast<float*>(p.out) + off[i] + col) = d;
                } else {
                  __nv_bfloat16* ob = reinterpret_cast<__nv_bfloat16*>(p.out);
                  if constexpr (IS_BF16) {
                    if (epi & EPI_RESIDUAL) d = add_bf16x8(d, rv[i]);
                  }
                  *reinterpret_cast<uint4*>(ob + off[i] + col) = d;
                }
              }
            }
            __syncwarp();
          }
          if constexpr (KIND == KIND_PEXP_STAT) {
            if (p.stat2) {     // this thread's row over this warp's columns of the tile: (0, sum of exponentials)
              const int m = m_blk * BLOCK_M + row;
              if (m < p.M) {
                const int slot = (N_COLS >= 64) ? n_blk * 2 + half : n_blk;
                p.stat2[(long long)m * p.ld_stat + slot] = make_float2(0.f, (st_a.x + st_b.x) + (st_a.y + st_b.y));
              }
            }
          }
        }
      }
    }
  } else {
    if constexpr (EPI_WG) {
      // ========================= epilogue warps (KIND_BF16: warps 1, 2) =========================
      // Warp 1 + e owns the 32-row quadrants q = 2 e, 2 e + 1 of the tile; for each, rows [32 q, 32 q + 32) over all
      // columns, in 64-column phases (32-column phases below 128-column tiles).  Every global load / store instruction covers contiguous row segments, 16 bytes per
      // lane; residual loads are issued in batches before use.  The GroupNorm partial sums of a phase go to slot
      // (tile, q), summed in the same order as when two warps split a quadrant's columns.
      // Swap-AB: quadrant q is output channels [32 q, 32 q + 32) of the tile's 256 pixels, one pixel half (and
      // statistics slot) after the other.
      const int q0 = 2 * (warp - 1);
      const int epi = EPI_CT >= 0 ? EPI_CT : p.epi;
      const float* __restrict__ gate = p.gate;
      const __nv_bfloat16* __restrict__ resid = p.residual;
      __nv_bfloat16* ob = reinterpret_cast<__nv_bfloat16*>(p.out);
      uint32_t it = 0;
      for (int tile = tile0; tile < num_tiles; tile += tile_step, ++it) {
        int m_blk, n_blk;
        tile_coords(tile, num_m_tiles, num_n_tiles, p.group_n, m_blk, n_blk);
        mbar_wait(tile_full, it & 1u);
#pragma unroll 1
        for (int q = q0; q < q0 + 2; ++q) {
          const int row = q * 32 + lane;
          if constexpr (SWAP) {
            int t_o, th, tw;
            conv_tile(p, m_blk, t_o, th, tw);
            const int r = th * p.tiles_w + tw;                        // tile index within the frame (statistics slot)
            const int h0 = th * p.bh, w0 = tw * p.bw;
            const long long fbase = (long long)(t_o + p.out_t_pad) * p.out_frame_stride + n_blk * BLOCK_M + q * 32;
            const bool dup_t = p.out_dup_head && t_o == 0;
            const int chn = lane & 3, psub = lane >> 2;              // 4 lanes x 16 B per pixel, 8 pixels per access
            const bool ch_ok = n_blk * BLOCK_M + q * 32 + chn * 8 < p.N;
#pragma unroll 1
            for (int half = 0; half < 2; ++half) {
              float4 st = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
              for (int c0 = half * 128; c0 < half * 128 + 128; c0 += 32) {
                long long off[4];
                int flags[4];
                uint4 rv[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                  const int pj = c0 + i * 8 + psub;                  // pixel index within the tile
                  const int ph = pj / p.bw, pw = pj - ph * p.bw;
                  const int h = h0 + ph, w = w0 + pw;
                  const bool ok = (h < p.H_out) && (w < p.W_out) && ch_ok;
                  off[i] = fbase + ((long long)h * p.W_out + w) * p.ldc + chn * 8;
                  flags[i] = ok ? (dup_t ? 3 : 1) : 0;
                  if ((epi & EPI_RESIDUAL) && ok) rv[i] = *reinterpret_cast<const uint4*>(resid + off[i]);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                  if (!(flags[i] & 1)) continue;
                  const int pj = c0 + i * 8 + psub;
                  uint4 d = *reinterpret_cast<const uint4*>(tile_s + pj * 256 + (((q * 4 + chn) ^ swap_tile_swz(pj)) << 4));
                  if (epi & EPI_RESIDUAL) d = add_bf16x8(d, rv[i]);
                  *reinterpret_cast<uint4*>(ob + off[i]) = d;
                  if (p.stat_partial) stat_acc(st, d);
                  if (flags[i] & 2) {
                    *reinterpret_cast<uint4*>(ob + off[i] - p.out_frame_stride) = d;
                    *reinterpret_cast<uint4*>(ob + off[i] - 2 * p.out_frame_stride) = d;
                  }
                }
              }
              if (p.stat_partial) {
                // lanes with the same channel octet (lane & 3) hold different pixels: fixed-order xor tree
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
                  st.x += __shfl_xor_sync(0xffffffffu, st.x, o); st.y += __shfl_xor_sync(0xffffffffu, st.y, o);
                  st.z += __shfl_xor_sync(0xffffffffu, st.z, o); st.w += __shfl_xor_sync(0xffffffffu, st.w, o);
                }
                if (lane < 4 && t_o < p.T_out) {
                  const int octet = (n_blk * BLOCK_M + q * 32) / 8 + lane;
                  if (octet * 8 < p.N)
                    p.stat_partial[((long long)t_o * p.stat_slots + r * 2 + half) * (p.N / 8) + octet] = st;
                }
              }
            }
          } else {
            constexpr int PH_COLS = ACC_STRIDE >= 128 ? 64 : 32;
            constexpr int CPR = PH_COLS / 8;                         // 16-byte chunks per phase row
            constexpr int ROWS_PER_IT = 32 / CPR;
            constexpr int N_IT = 32 / ROWS_PER_IT;                   // warp-wide accesses per phase
            constexpr int kBatch = N_IT;   // a phase's residual loads all in flight: two warps cover the whole tile
            constexpr int ROW_B = L::kTileCols * 2;
            constexpr int SWZ = (L::kTileCols / 8 < 8 ? L::kTileCols / 8 : 8) - 1;
            const RowDest dst = row_dest<BLOCK_N>(p, epi, m_blk, n_blk, row, ACC_STRIDE);
            const int n_base = n_blk * BLOCK_N;
            const int ch = lane % CPR, rsub = lane / CPR;
            const bool plain = !(epi & (EPI_GELU | EPI_SILU | EPI_GATE));
            int t_o = 0, rt = 0;
            if (p.stat_partial && p.a_mode != 0) {
              int th, tw;
              conv_tile(p, m_blk, t_o, th, tw);
              rt = th * p.tiles_w + tw;
            }
#pragma unroll 1
            for (int ph0 = 0; ph0 < ACC_STRIDE; ph0 += PH_COLS) {
              const int col = ph0 + ch * 8;
              const bool col_ok = (n_base + col) < p.N;
              float gg[8];
              if (epi & EPI_GATE) {
                const float4 ga = col_ok ? *reinterpret_cast<const float4*>(gate + n_base + col) : make_float4(0, 0, 0, 0);
                const float4 gb = col_ok ? *reinterpret_cast<const float4*>(gate + n_base + col + 4) : make_float4(0, 0, 0, 0);
                gg[0] = ga.x; gg[1] = ga.y; gg[2] = ga.z; gg[3] = ga.w;
                gg[4] = gb.x; gg[5] = gb.y; gg[6] = gb.z; gg[7] = gb.w;
              }
              float4 st = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
              for (int b0 = 0; b0 < N_IT; b0 += kBatch) {
                long long off[kBatch];
                int flags[kBatch];
                uint4 rv[kBatch];
#pragma unroll
                for (int i = 0; i < kBatch; ++i) {
                  const int r = (b0 + i) * ROWS_PER_IT + rsub;
                  off[i] = __shfl_sync(0xffffffffu, dst.off, r);
                  const int f = __shfl_sync(0xffffffffu, dst.valid | (dst.dup << 1), r);
                  flags[i] = col_ok ? f : 0;
                  if ((epi & EPI_RESIDUAL) && (flags[i] & 1)) rv[i] = *reinterpret_cast<const uint4*>(resid + off[i] + col);
                }
#pragma unroll
                for (int i = 0; i < kBatch; ++i) {
                  if (!(flags[i] & 1)) continue;
                  const int tr = q * 32 + (b0 + i) * ROWS_PER_IT + rsub;
                  uint4 d = *reinterpret_cast<const uint4*>(tile_s + tr * ROW_B + (((col >> 3) ^ (tr & SWZ)) << 4));
                  if (!plain) {
                    uint32_t w[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                      if (epi & EPI_GELU)
                        w[e] = pack_bf16x2(gelu_tanh_fast(__uint_as_float(w[e] << 16)),
                                           gelu_tanh_fast(__uint_as_float(w[e] & 0xffff0000u)));
                      if (epi & EPI_SILU)
                        w[e] = pack_bf16x2(silu_fast(__uint_as_float(w[e] << 16)), silu_fast(__uint_as_float(w[e] & 0xffff0000u)));
                      if (epi & EPI_GATE)
                        w[e] = pack_bf16x2(__uint_as_float(w[e] << 16) * gg[2 * e],
                                           __uint_as_float(w[e] & 0xffff0000u) * gg[2 * e + 1]);
                    }
                    d = make_uint4(w[0], w[1], w[2], w[3]);
                  }
                  if (epi & EPI_RESIDUAL) d = add_bf16x8(d, rv[i]);
                  *reinterpret_cast<uint4*>(ob + off[i] + col) = d;
                  if (p.stat_partial) stat_acc(st, d);
                  if (flags[i] & 2) {
                    *reinterpret_cast<uint4*>(ob + off[i] - p.out_frame_stride + col) = d;
                    *reinterpret_cast<uint4*>(ob + off[i] - 2 * p.out_frame_stride + col) = d;
                  }
                }
              }
              if (p.stat_partial && p.a_mode != 0) {
                // lanes with equal (lane % CPR) own the same channel octet for different rows
#pragma unroll
                for (int o = CPR; o < 32; o <<= 1) {
                  st.x += __shfl_xor_sync(0xffffffffu, st.x, o); st.y += __shfl_xor_sync(0xffffffffu, st.y, o);
                  st.z += __shfl_xor_sync(0xffffffffu, st.z, o); st.w += __shfl_xor_sync(0xffffffffu, st.w, o);
                }
                if (lane < CPR && col_ok && m_blk < p.num_m_tiles)
                  p.stat_partial[((long long)t_o * p.stat_slots + rt * 4 + q) * (p.N / 8) + (n_base + col) / 8] = st;
              }
            }
          }
        }
        mbar_arrive(tile_empty);
      }
    }
  }
}

// ----------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

// rank-r bf16 tensor map, dims fastest-first, 128B swizzle, zero OOB fill
int make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(SVR2_ERR_CUDA, "cuTensorMapEncodeTiled entry point not found");
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[256];
    snprintf(msg, sizeof msg, "cuTensorMapEncodeTiled failed (%d) rank=%d dims=%llu,%llu,%llu box=%u,%u,%u", (int)r,
             rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
             (unsigned long long)(rank > 2 ? dims[2] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0);
    return set_error(SVR2_ERR_CUDA, msg);
  }
  return SVR2_OK;
}

// per-device caches: a host process may drive several GPUs (ComfyUI), so nothing here is cached per process
constexpr int kMaxDevices = 64;
int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}
static int g_num_sms[kMaxDevices] = {};
int num_sms() {
  const int dev = current_device();
  if (!g_num_sms[dev]) cudaDeviceGetAttribute(&g_num_sms[dev], cudaDevAttrMultiProcessorCount, dev);
  return g_num_sms[dev];
}

template <int BLOCK_N, int KIND, bool SWAP = false, int EPI_CT = -1, bool SLAB = false>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p_in, cudaStream_t stream,
                       const CUtensorMap* ta2_opt = nullptr) {
  const CUtensorMap& ta2 = ta2_opt ? *ta2_opt : ta;
  using L = std::conditional_t<SLAB, SlabLayout<SWAP>, SmemLayout<BLOCK_N, kEpiWG<KIND>>>;
  auto kern = gemm_wgmma_kernel<BLOCK_N, KIND, SWAP, EPI_CT, SLAB>;
  GemmParams p = p_in;
  {
    // raster group: keep the group's B slice around 16 MB (L2 = 50 MB, shared with A tiles and the output stream)
    const long long b_tile_bytes = (long long)(SWAP ? BLOCK_M : BLOCK_N) * p.num_k_blocks * BLOCK_K * 2;
    long long g = (16LL << 20) / (b_tile_bytes > 0 ? b_tile_bytes : 1);
    if (g < 1) g = 1;
    if (g > p.num_n_tiles) g = p.num_n_tiles;
    p.group_n = (int)g;
  }
  static bool configured[kMaxDevices] = {};       // the attribute is per (function, device)
  const int dev = current_device();
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
    if (e != cudaSuccess) return set_error(SVR2_ERR_CUDA, cudaGetErrorString(e));
    configured[dev] = true;
  }
  int tiles = p.num_m_tiles * p.num_n_tiles;
  int grid = tiles < num_sms() ? tiles : num_sms();
  if (grid <= 0) return SVR2_OK;
  kern<<<grid, kNumThreads, L::kTotal, stream>>>(ta, tb, ta2, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(SVR2_ERR_CUDA, cudaGetErrorString(e));
  return SVR2_OK;
}

static int dispatch_gemm(int block_n, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                         cudaStream_t s, const CUtensorMap* ta2 = nullptr) {
  if (ta2) {     // conv with a fused shortcut: plain bf16 epilogue only
    switch (block_n) {
      case 256: return launch_gemm<256, KIND_BF16>(ta, tb, p, s, ta2);
      case 128: return launch_gemm<128, KIND_BF16>(ta, tb, p, s, ta2);
    }
    return set_error(SVR2_ERR_ARG, "fused shortcut: Cout must be >= 128");
  }
  if (p.epi & EPI_ROWSCALE) {
    if (block_n == 256) return launch_gemm<256, KIND_BF16_RS>(ta, tb, p, s);
    if (block_n == 128) return launch_gemm<128, KIND_BF16_RS>(ta, tb, p, s);
    return set_error(SVR2_ERR_ARG, "EPI_ROWSCALE needs >= 128-column tiles");
  }
  if ((p.epi & EPI_PEXP) && p.stat2) {
    if (block_n != 256) return set_error(SVR2_ERR_ARG, "EPI_PEXP statistics need 256-column tiles");
    return launch_gemm<256, KIND_PEXP_STAT>(ta, tb, p, s);
  }
  if (p.epi & EPI_SWIGLU) {
    if (block_n == 256) return launch_gemm<256, KIND_SWIGLU>(ta, tb, p, s);
    return set_error(SVR2_ERR_ARG, "SwiGLU epilogue needs BLOCK_N = 256");
  }
  if (p.epi & EPI_ROWSTAT) {
    if (block_n == 256) return launch_gemm<256, KIND_ROWSTAT>(ta, tb, p, s);
    if (block_n == 128) return launch_gemm<128, KIND_ROWSTAT>(ta, tb, p, s);
    if (block_n == 64) return launch_gemm<64, KIND_ROWSTAT>(ta, tb, p, s);
    return launch_gemm<32, KIND_ROWSTAT>(ta, tb, p, s);
  }
  if (p.epi & EPI_PEXP) {
    if (block_n == 256) return launch_gemm<256, KIND_PEXP>(ta, tb, p, s);
    if (block_n == 128) return launch_gemm<128, KIND_PEXP>(ta, tb, p, s);
    if (block_n == 64) return launch_gemm<64, KIND_PEXP>(ta, tb, p, s);
    return launch_gemm<32, KIND_PEXP>(ta, tb, p, s);
  }
  if (p.epi & EPI_F32) {
    switch (block_n) {
      case 256: return launch_gemm<256, KIND_F32>(ta, tb, p, s);
      case 128: return launch_gemm<128, KIND_F32>(ta, tb, p, s);
      case 64: return launch_gemm<64, KIND_F32>(ta, tb, p, s);
      case 32: return launch_gemm<32, KIND_F32>(ta, tb, p, s);
      case 16: return launch_gemm<16, KIND_F32>(ta, tb, p, s);
    }
  }
  if (block_n == 256) {
    switch (p.epi) {      // the epilogue-bound shapes of the hot path get flag-free epilogues
      case EPI_SHUFFLE | EPI_BIAS: return launch_gemm<256, KIND_BF16, false, EPI_SHUFFLE | EPI_BIAS>(ta, tb, p, s);
      case EPI_BIAS | EPI_GATE | EPI_RESIDUAL: return launch_gemm<256, KIND_BF16, false, EPI_BIAS | EPI_GATE | EPI_RESIDUAL>(ta, tb, p, s);
      case EPI_GATE | EPI_RESIDUAL: return launch_gemm<256, KIND_BF16, false, EPI_GATE | EPI_RESIDUAL>(ta, tb, p, s);
      case EPI_BIAS: return launch_gemm<256, KIND_BF16, false, EPI_BIAS>(ta, tb, p, s);
      case 0: return launch_gemm<256, KIND_BF16, false, 0>(ta, tb, p, s);
    }
  }
  switch (block_n) {
    case 256: return launch_gemm<256, KIND_BF16>(ta, tb, p, s);
    case 128: return launch_gemm<128, KIND_BF16>(ta, tb, p, s);
    case 64: return launch_gemm<64, KIND_BF16>(ta, tb, p, s);
    case 32: return launch_gemm<32, KIND_BF16>(ta, tb, p, s);
    case 16: return launch_gemm<16, KIND_BF16>(ta, tb, p, s);
  }
  return set_error(SVR2_ERR_ARG, "unsupported BLOCK_N");
}

static int pick_block_n(int N, int epi) {
  if (epi & EPI_SWIGLU) return 256;
  if ((epi & (EPI_ROWSTAT | EPI_PEXP)) && N <= 32) return 32;
  if (N >= 256) return 256;
  if (N > 64) return 128;
  if (N > 32) return 64;
  if (N > 16) return 32;
  return 16;
}

}  // namespace svr2

using namespace svr2;

// ----------------------------------------------------------------------------
// C ABI
// ----------------------------------------------------------------------------
static int linear_impl(const void* a, int64_t lda, const void* w, int64_t ldw, int M, int N, int K, int epi_flags,
                       const void* bias, const float* gate, const void* residual, void* out, int64_t ldc, float out_scale,
                       const float* rowscale, void* stat_out, int64_t ld_stat, const int* run_if, void* stream);

extern "C" int svr2_linear_bf16(const void* a, int64_t lda, const void* w, int64_t ldw, int M, int N, int K,
                                int epi_flags, const void* bias, const float* gate, const void* residual, void* out,
                                int64_t ldc, float out_scale, void* stream) {
  return linear_impl(a, lda, w, ldw, M, N, K, epi_flags, bias, gate, residual, out, ldc, out_scale, nullptr, nullptr, 0,
                     nullptr, stream);
}

// svr2_linear_bf16 with the extras of the single-pass attention probabilities:
//   rowscale (with SVR2_EPI_ROWSCALE): acc * rowscale[m] before the rest of the epilogue;
//   stat_out (with SVR2_EPI_PEXP, N >= 256): float2 [M][ld_stat] = per (row, 128-column slot) (0, fp32 sum of the
//     exponentials written), ld_stat >= 2 * ceil(N / 256);
//   run_if: device flag — the launch does nothing unless *run_if != 0 (conditional fallback without a host sync).
extern "C" int svr2_linear_ex_bf16(const void* a, int64_t lda, const void* w, int64_t ldw, int M, int N, int K,
                                   int epi_flags, const void* bias, const float* gate, const void* residual, void* out,
                                   int64_t ldc, float out_scale, const float* rowscale, void* stat_out, int64_t ld_stat,
                                   const int* run_if, void* stream) {
  return linear_impl(a, lda, w, ldw, M, N, K, epi_flags, bias, gate, residual, out, ldc, out_scale, rowscale, stat_out,
                     ld_stat, run_if, stream);
}

static int linear_impl(const void* a, int64_t lda, const void* w, int64_t ldw, int M, int N, int K, int epi_flags,
                       const void* bias, const float* gate, const void* residual, void* out, int64_t ldc, float out_scale,
                       const float* rowscale, void* stat_out, int64_t ld_stat, const int* run_if, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0) return set_error(SVR2_ERR_ARG, "svr2_linear_bf16: empty problem");
  const bool f32 = (epi_flags & EPI_F32) != 0, rowstat = (epi_flags & EPI_ROWSTAT) != 0;
  if ((lda % 8) || (ldw % 8) || (!rowstat && ((ldc % (f32 ? 4 : 8)) || (N % (f32 ? 4 : 8)))))
    return set_error(SVR2_ERR_ARG, "svr2_linear_bf16: lda/ldw must be multiples of 8, ldc/N of 8 (4 for fp32 out)");
  if ((epi_flags & EPI_PEXP) && !gate) return set_error(SVR2_ERR_ARG, "EPI_PEXP needs the row log-sum-exp vector (gate)");
  if ((epi_flags & EPI_SWIGLU) && (N % 256)) return set_error(SVR2_ERR_ARG, "SwiGLU needs N % 256 == 0");
  int bn = pick_block_n(N, epi_flags);
  // Few-row problems (the 58 text tokens of every DiT layer, single images): with 256-column tiles only a handful of
  // CTAs would walk the whole K loop.  Narrower tiles spread the same work over up to half the SMs.
  if (!(epi_flags & (EPI_SWIGLU | EPI_ROWSTAT | EPI_PEXP))) {
    const long long m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
    const int bn_min = (epi_flags & EPI_ROWSCALE) ? 128 : 32;       // the row-scale epilogue lives in the wide path
    while (bn > bn_min && 2 * m_tiles * ((N + bn - 1) / bn) <= num_sms()) bn /= 2;
  }
  CUtensorMap ta, tb;
  uint64_t da[2] = {(uint64_t)K, (uint64_t)M}, sa[1] = {(uint64_t)lda * 2};
  uint32_t ba[2] = {BLOCK_K, BLOCK_M};
  int rc = make_tmap_bf16(&ta, a, 2, da, sa, ba);
  if (rc) return rc;
  uint64_t db[2] = {(uint64_t)K, (uint64_t)N}, sb[1] = {(uint64_t)ldw * 2};
  uint32_t bb[2] = {BLOCK_K, (uint32_t)bn};
  rc = make_tmap_bf16(&tb, w, 2, db, sb, bb);
  if (rc) return rc;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.num_m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  p.num_n_tiles = (N + bn - 1) / bn;
  p.num_k_blocks = (K + BLOCK_K - 1) / BLOCK_K;
  p.a_mode = 0;
  p.epi = epi_flags & ~EPI_SHUFFLE;
  p.ldc = (int)ldc;
  p.out_scale = out_scale;
  p.bias = (const __nv_bfloat16*)bias;
  p.gate = gate;
  p.residual = (const __nv_bfloat16*)residual;
  p.out = out;
  if ((p.epi & EPI_BIAS) && !bias) return set_error(SVR2_ERR_ARG, "EPI_BIAS without bias");
  if ((p.epi & EPI_GATE) && !gate) return set_error(SVR2_ERR_ARG, "EPI_GATE without gate");
  if (rowstat && ldc < (int64_t)p.num_n_tiles * (bn >= 64 ? 2 : 1))
    return set_error(SVR2_ERR_ARG, "EPI_ROWSTAT: ldc (float2 slots per row) must be >= svr2_rowstat_slots(N)");
  if ((p.epi & EPI_RESIDUAL) && !residual) return set_error(SVR2_ERR_ARG, "EPI_RESIDUAL without residual");
  if ((p.epi & EPI_ROWSCALE) && (!rowscale || bn < 128 || (p.epi & (EPI_SWIGLU | EPI_ROWSTAT | EPI_PEXP | EPI_F32))))
    return set_error(SVR2_ERR_ARG, "EPI_ROWSCALE needs rowscale, a plain bf16 epilogue and N > 64 (128-column tiles)");
  if (stat_out && (!(p.epi & EPI_PEXP) || bn != 256 || ld_stat < 2 * (int64_t)p.num_n_tiles))
    return set_error(SVR2_ERR_ARG, "stat_out needs EPI_PEXP, N >= 256 and ld_stat >= 2 * ceil(N / 256)");
  p.rowscale = rowscale;
  p.stat2 = reinterpret_cast<float2*>(stat_out);
  p.ld_stat = (int)ld_stat;
  p.run_if = run_if;
  return dispatch_gemm(bn, ta, tb, p, (cudaStream_t)stream);
}

// QKV projection with NaSwinAttention's q/k RMSNorm + RoPE + window partition fused into the epilogue
// (mmattn.py:173,199-248; rope.py:116-176): a [M, K] x w [3*heads*128, K]^T; token m's q/k/v rows land at row
// tok_dst[m] of q / k / v ([rows, heads*128], window order).  heads must be even (a 256-column tile = 2 heads).
extern "C" int svr2_linear_qkv_rope_bf16(const void* a, int64_t lda, const void* w, int64_t ldw, int M, int heads, int K,
                                         const int32_t* tok_dst, const int32_t* tok_rope, const float* cos_tab,
                                         const float* sin_tab, int nfreq, const float* qk_weight, float eps, void* q,
                                         void* k, void* v, void* stream) {
  if (M <= 0 || K <= 0 || heads <= 0) return set_error(SVR2_ERR_ARG, "svr2_linear_qkv_rope_bf16: empty problem");
  if (heads & 1) return set_error(SVR2_ERR_ARG, "svr2_linear_qkv_rope_bf16: heads must be even");
  if (nfreq != 21 && nfreq != 10) return set_error(SVR2_ERR_ARG, "svr2_linear_qkv_rope_bf16: nfreq must be 21 (3B) or 10 (7B)");
  if ((lda % 8) || (ldw % 8)) return set_error(SVR2_ERR_ARG, "svr2_linear_qkv_rope_bf16: lda/ldw must be multiples of 8");
  const int inner = heads * 128, N = 3 * inner, bn = 256;
  const int num_m = (M + BLOCK_M - 1) / BLOCK_M;
  CUtensorMap ta, tb;
  uint64_t da[2] = {(uint64_t)K, (uint64_t)M}, sa[1] = {(uint64_t)lda * 2};
  uint32_t ba[2] = {BLOCK_K, BLOCK_M};
  int rc = make_tmap_bf16(&ta, a, 2, da, sa, ba);
  if (rc) return rc;
  uint64_t db[2] = {(uint64_t)K, (uint64_t)N}, sb[1] = {(uint64_t)ldw * 2};
  uint32_t bb[2] = {BLOCK_K, (uint32_t)bn};
  rc = make_tmap_bf16(&tb, w, 2, db, sb, bb);
  if (rc) return rc;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.num_m_tiles = num_m;
  p.num_n_tiles = N / bn;
  p.num_k_blocks = (K + BLOCK_K - 1) / BLOCK_K;
  p.a_mode = 0;
  p.out = q; p.out2 = k; p.out3 = v;
  p.tok_dst = tok_dst; p.tok_rope = tok_rope;
  p.rope_cos = cos_tab; p.rope_sin = sin_tab;
  p.qk_weight = qk_weight; p.qk_eps = eps; p.qkv_inner = inner;
  cudaStream_t s = (cudaStream_t)stream;
  if (nfreq == 21) return launch_gemm<256, KIND_QKV21>(ta, tb, p, s);
  return launch_gemm<256, KIND_QKV10>(ta, tb, p, s);
}

// number of (max, sum) float2 partial slots per row that EPI_ROWSTAT writes for a given N
extern "C" int svr2_rowstat_slots(int N) {
  const int bn = pick_block_n(N, EPI_ROWSTAT);
  return ((N + bn - 1) / bn) * (bn >= 64 ? 2 : 1);
}

// Causal Conv3d as implicit GEMM.  x: NDHWC bf16 with `in_t_pad` halo frames in front
// (frames [0,in_t_pad) hold the causal context; the first real frame is at index in_t_pad).
// w: [Cout][kt][kh][kw][Cin] bf16 (K-major).  y: NDHWC bf16 with out_t_pad halo frames.
static int conv3d_impl(const void* x, int T_in_total, int H, int W, int Cin, const void* w, int Cout, int kt,
                       int kh, int kw, int stride_t, int stride_hw, int pad_hw, int T_out, int epi_flags,
                       const void* bias, const void* residual, void* y, int out_t_pad, int out_dup_head,
                       int ldc, void* stat_partial, int64_t stat_bytes, int* stat_slots_out, void* stream,
                       const void* x2 = nullptr, int C2 = 0);

extern "C" int svr2_conv3d_bf16(const void* x, int T_in_total, int H, int W, int Cin, const void* w, int Cout, int kt,
                                int kh, int kw, int stride_t, int stride_hw, int pad_hw, int T_out, int epi_flags,
                                const void* bias, const void* residual, void* y, int out_t_pad, int out_dup_head,
                                int ldc, void* stream) {
  return conv3d_impl(x, T_in_total, H, W, Cin, w, Cout, kt, kh, kw, stride_t, stride_hw, pad_hw, T_out, epi_flags, bias,
                     residual, y, out_t_pad, out_dup_head, ldc, nullptr, 0, nullptr, stream);
}

// Same conv, additionally emitting per-tile GroupNorm partial sums of the stored output
// (stat_partial: [T_out][slots][Cout/8] float4, slots returned in *stat_slots; see svr2_groupnorm_from_stats_bf16).
// Call with stat_partial == NULL to query *stat_slots / the required bytes (= T_out * slots * Cout/8 * 16).
extern "C" int svr2_conv3d_stats_bf16(const void* x, int T_in_total, int H, int W, int Cin, const void* w, int Cout,
                                      int kt, int kh, int kw, int stride_t, int stride_hw, int pad_hw, int T_out,
                                      int epi_flags, const void* bias, const void* residual, void* y, int out_t_pad,
                                      int out_dup_head, int ldc, void* stat_partial, int64_t stat_bytes,
                                      int* stat_slots, void* stream) {
  if (!stat_slots) return set_error(SVR2_ERR_ARG, "svr2_conv3d_stats_bf16: stat_slots must not be NULL");
  return conv3d_impl(x, T_in_total, H, W, Cin, w, Cout, kt, kh, kw, stride_t, stride_hw, pad_hw, T_out, epi_flags, bias,
                     residual, y, out_t_pad, out_dup_head, ldc, stat_partial, stat_bytes, stat_slots, stream);
}

// Same conv with a fused 1x1x1 conv_shortcut (ResnetBlock3D, attn_video_vae.py:311-362): y = conv(x; w[:, :K]) +
// x2 . w[:, K:]^T + bias, x2 = [T_out, H, W, C2] (no halo), w = [Cout][kt*kh*kw*Cin + C2], bias = conv bias + shortcut
// bias.  One fp32 accumulation, one rounding (the reference rounds the shortcut and the conv output separately).
extern "C" int svr2_conv3d_shortcut_stats_bf16(const void* x, int T_in_total, int H, int W, int Cin, const void* w,
                                               int Cout, int kt, int kh, int kw, int T_out, const void* bias,
                                               const void* x2, int C2, void* y, int out_t_pad, int out_dup_head,
                                               void* stat_partial, int64_t stat_bytes, int* stat_slots, void* stream) {
  if (!x2 || C2 <= 0 || (C2 % 64)) return set_error(SVR2_ERR_ARG, "svr2_conv3d_shortcut_stats_bf16: x2 / C2 % 64");
  if (Cout < 128) return set_error(SVR2_ERR_ARG, "svr2_conv3d_shortcut_stats_bf16: Cout must be >= 128");
  return conv3d_impl(x, T_in_total, H, W, Cin, w, Cout, kt, kh, kw, 1, 1, 1, T_out, EPI_BIAS, bias, nullptr, y,
                     out_t_pad, out_dup_head, Cout, stat_partial, stat_bytes, stat_slots, stream, x2, C2);
}

// Output tile of the implicit-GEMM conv.  Cout <= 128: swap operands (128 channels x 256 pixels per tile); else
// 128 pixels x up to 256 channels.  bw x bh output pixels (128, or 256 when swapped).
static void conv_tile_shape(int Cout, int H_out, int W_out, bool* swap_out, int* bw_out, int* bh_out) {
  const bool swap = (Cout > 64 && Cout <= 128) && (long long)H_out * W_out >= 256;
  int bw = 16, bh = 8;
  if (swap) {
    bw = 32; bh = 8;
    if (W_out <= 16) { bw = 16; bh = 16; }
    if (W_out <= 8) { bw = 8; bh = 32; }
  } else {
    if (W_out >= 128 && H_out < 8) { bw = 128; bh = 1; }
    else if (W_out <= 8) { bw = 8; bh = 16; }
  }
  *swap_out = swap; *bw_out = bw; *bh_out = bh;
}
// The slab mainloop (SlabLayout) serves stride-1 convs with 3x3 spatial taps and a temporal kernel on the swap-AB tiles
// and on the 256-column tiles of two or more tile rows; every other conv runs the one-ring mainloop.
static bool conv_slab(int Cout, int kt, int kh, int kw, int stride_hw, int H_out, int W_out) {
  bool swap;
  int bw, bh;
  conv_tile_shape(Cout, H_out, W_out, &swap, &bw, &bh);
  return stride_hw == 1 && kt > 1 && kh == 3 && kw == 3 && bh > 1 && (swap || pick_block_n(Cout, 0) == 256);
}
extern "C" int svr2_conv_mainloop(int Cin, int Cout, int kt, int kh, int kw, int stride_hw, int H, int W) {
  if (Cin <= 0 || Cin % 64 || Cout <= 0 || (stride_hw != 1 && stride_hw != 2))
    return set_error(SVR2_ERR_ARG, "svr2_conv_mainloop: Cin must be a positive multiple of 64, stride_hw 1 or 2");
  return conv_slab(Cout, kt, kh, kw, stride_hw, stride_hw == 1 ? H : H / 2, stride_hw == 1 ? W : W / 2) ? 1 : 0;
}
// GroupNorm partial-sum slots per frame a conv with statistics writes (the size query of svr2_conv3d_stats_bf16 without
// the tensor maps: workspace planning)
extern "C" int svr2_conv_stat_slots(int Cout, int H_out, int W_out) {
  bool swap;
  int bw, bh;
  conv_tile_shape(Cout, H_out, W_out, &swap, &bw, &bh);
  return ((W_out + bw - 1) / bw) * ((H_out + bh - 1) / bh) * (swap ? 2 : 4);
}

static int conv3d_impl(const void* x, int T_in_total, int H, int W, int Cin, const void* w, int Cout, int kt,
                       int kh, int kw, int stride_t, int stride_hw, int pad_hw, int T_out, int epi_flags,
                       const void* bias, const void* residual, void* y, int out_t_pad, int out_dup_head,
                       int ldc, void* stat_partial, int64_t stat_bytes, int* stat_slots_out, void* stream,
                       const void* x2, int C2) {
  if (Cin % 64) return set_error(SVR2_ERR_ARG, "svr2_conv3d_bf16: Cin must be a multiple of 64 (pad channels)");
  if (Cout % 8 || ldc % 8) return set_error(SVR2_ERR_ARG, "svr2_conv3d_bf16: Cout/ldc must be multiples of 8");
  if (stride_hw != 1 && stride_hw != 2) return set_error(SVR2_ERR_ARG, "stride_hw must be 1 or 2");
  if (out_dup_head && out_t_pad != 2)        // the epilogue copies frame 0 into exactly two halo frames
    return set_error(SVR2_ERR_ARG, "svr2_conv3d_bf16: out_dup_head needs out_t_pad == 2");
  const int H_out = stride_hw == 1 ? H : H / 2, W_out = stride_hw == 1 ? W : W / 2;
  if (stride_hw == 2 && ((H | W) & 1)) return set_error(SVR2_ERR_ARG, "stride-2 conv needs even H, W");
  bool swap;
  int bw, bh;
  conv_tile_shape(Cout, H_out, W_out, &swap, &bw, &bh);
  const int bn = swap ? 128 : pick_block_n(Cout, 0);
  const bool slab = conv_slab(Cout, kt, kh, kw, stride_hw, H_out, W_out);
  CUtensorMap ta, tb;
  int rc;
  if (stride_hw == 1) {
    uint64_t d[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)T_in_total};
    uint64_t s[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
    uint32_t b[4] = {BLOCK_K, (uint32_t)bw, (uint32_t)(slab ? bh + 2 : bh), 1};
    rc = make_tmap_bf16(&ta, x, 4, d, s, b);
  } else {
    uint64_t d[5] = {(uint64_t)Cin * 2, (uint64_t)W / 2, 2, (uint64_t)H / 2, (uint64_t)T_in_total};
    uint64_t s[4] = {(uint64_t)Cin * 4, (uint64_t)W * Cin * 2, (uint64_t)W * Cin * 4, (uint64_t)H * W * Cin * 2};
    uint32_t b[5] = {BLOCK_K, (uint32_t)bw, 1, (uint32_t)bh, 1};
    rc = make_tmap_bf16(&ta, x, 5, d, s, b);
  }
  if (rc) return rc;
  CUtensorMap ta2;
  if (x2) {   // second activation tensor: same pixel box, read at the output pixel
    uint64_t d[4] = {(uint64_t)C2, (uint64_t)W, (uint64_t)H, (uint64_t)T_out};
    uint64_t s2[3] = {(uint64_t)C2 * 2, (uint64_t)W * C2 * 2, (uint64_t)H * W * C2 * 2};
    uint32_t b[4] = {BLOCK_K, (uint32_t)bw, (uint32_t)bh, 1};
    rc = make_tmap_bf16(&ta2, x2, 4, d, s2, b);
    if (rc) return rc;
  }
  const int K = kt * kh * kw * Cin + (x2 ? C2 : 0);
  const bool fold = (epi_flags & SVR2_EPI_FOLD_HEAD) != 0;
  if (fold && (kt != 3 || x2 || Cout % bn))
    return set_error(SVR2_ERR_ARG, "svr2_conv3d_bf16: SVR2_EPI_FOLD_HEAD needs kt = 3, no shortcut and Cout a multiple of the n-tile");
  uint64_t db[2] = {(uint64_t)K, (uint64_t)(fold ? 2 * Cout : Cout)}, sb[1] = {(uint64_t)K * 2};
  uint32_t bb[2] = {BLOCK_K, (uint32_t)bn};
  rc = make_tmap_bf16(&tb, w, 2, db, sb, bb);
  if (rc) return rc;
  GemmParams p{};
  p.a_mode = stride_hw == 1 ? 1 : 2;
  p.bw = bw; p.bh = bh;
  p.tiles_w = (W_out + bw - 1) / bw;
  p.tiles_h = (H_out + bh - 1) / bh;
  p.taps_t = kt; p.taps_h = kh; p.taps_w = kw;
  p.cin_blocks = Cin / 64; p.cin = Cin;
  p.extra_blocks = x2 ? C2 / 64 : 0;
  p.pad_h = p.pad_w = pad_hw;
  p.stride_t = stride_t;
  p.H_out = H_out; p.W_out = W_out; p.T_out = T_out;
  {
    // band of tile rows whose input (all channels, 3 temporal taps) stays L2-resident: <= ~12 MB per frame
    const long long row_bytes = (long long)bh * stride_hw * W * Cin * 2;
    long long bhn = (12LL << 20) / (row_bytes > 0 ? row_bytes : 1);
    if (bhn < 1) bhn = 1;
    if (bhn > (H_out + bh - 1) / bh) bhn = (H_out + bh - 1) / bh;
    if (bh == 1 && (bw == 256 || bw == 128) && kh == 3) {     // one-row tiles: 8 MB of input rows per frame (12 MB measured 1.6 x the DRAM reads)
      bhn = (8LL << 20) / (row_bytes > 0 ? row_bytes : 1);
      if (bhn < 2) bhn = 2;
      if (bhn > H_out) bhn = H_out;
    }
    p.band_h = (kt > 1) ? (int)bhn : (H_out + bh - 1) / bh;   // no temporal reuse for kt = 1: plain frame-major order
  }
  p.M = T_out * p.tiles_w * p.tiles_h * BLOCK_M;
  p.N = Cout; p.K = K;
  p.num_m_tiles = T_out * p.tiles_w * p.tiles_h;
  p.num_n_tiles = (Cout + bn - 1) / bn;
  p.num_k_blocks = K / BLOCK_K;
  p.epi = epi_flags & (EPI_BIAS | EPI_RESIDUAL);
  p.ldc = ldc;
  p.out_frame_stride = (long long)H_out * W_out * ldc;
  p.out_t_pad = out_t_pad;
  p.out_dup_head = out_dup_head;
  if (fold) {
    p.fold_t = stride_t == 1 ? (T_out < 2 ? T_out : 2) : 1;
    p.fold_n = Cout;
  }
  p.bias = (const __nv_bfloat16*)bias;
  p.residual = (const __nv_bfloat16*)residual;
  p.out = y;
  if (stat_slots_out) {
    if (Cout % 8 || ldc != Cout) return set_error(SVR2_ERR_ARG, "conv stats: need Cout % 8 == 0 and ldc == Cout");
    const int slots = svr2_conv_stat_slots(Cout, H_out, W_out);
    *stat_slots_out = slots;
    if (!stat_partial) return SVR2_OK;   // size query only
    const int64_t need = (int64_t)T_out * slots * (Cout / 8) * 16;
    if (stat_bytes < need) return set_error(SVR2_ERR_ARG, "conv stats: stat_partial buffer too small");
    p.stat_partial = (float4*)stat_partial;
    p.stat_slots = slots;
  }
  const CUtensorMap* ta2p = x2 ? &ta2 : nullptr;
  if (slab) {
    if (swap) return launch_gemm<256, KIND_BF16, true, -1, true>(ta, tb, p, (cudaStream_t)stream, ta2p);
    if (p.epi == EPI_BIAS && !x2)
      return launch_gemm<256, KIND_BF16, false, EPI_BIAS, true>(ta, tb, p, (cudaStream_t)stream);
    return launch_gemm<256, KIND_BF16, false, -1, true>(ta, tb, p, (cudaStream_t)stream, ta2p);
  }
  if (swap) return launch_gemm<256, KIND_BF16, true>(ta, tb, p, (cudaStream_t)stream, x2 ? &ta2 : nullptr);
  return dispatch_gemm(bn, ta, tb, p, (cudaStream_t)stream, x2 ? &ta2 : nullptr);
}

// Upsample3D: 1x1x1 conv (GEMM over voxels) with the 3-D pixel shuffle fused into the store.
// x: [F,H,W,C] bf16 (no halo, contiguous rows); w: [r*C, C]; y: [(F*z - drop) (+pad), 2H, 2W, C].
extern "C" int svr2_upsample_shuffle_bf16(const void* x, int F, int H, int W, int C, const void* w, const void* bias,
                                          int temporal, int drop_head, void* y, int out_t_pad, int out_dup_head,
                                          void* stream) {
  const int z = temporal ? 2 : 1;
  const int N = 4 * z * C, M = F * H * W;
  const int bn = C >= 256 ? 256 : 128;
  if (C % bn) return set_error(SVR2_ERR_ARG, "svr2_upsample_shuffle_bf16: C must be a multiple of 128");
  if (out_dup_head && out_t_pad != 2)
    return set_error(SVR2_ERR_ARG, "svr2_upsample_shuffle_bf16: out_dup_head needs out_t_pad == 2");
  CUtensorMap ta, tb;
  uint64_t da[2] = {(uint64_t)C, (uint64_t)M}, sa[1] = {(uint64_t)C * 2};
  uint32_t ba[2] = {BLOCK_K, BLOCK_M};
  int rc = make_tmap_bf16(&ta, x, 2, da, sa, ba);
  if (rc) return rc;
  uint64_t db[2] = {(uint64_t)C, (uint64_t)N}, sb[1] = {(uint64_t)C * 2};
  uint32_t bb[2] = {BLOCK_K, (uint32_t)bn};
  rc = make_tmap_bf16(&tb, w, 2, db, sb, bb);
  if (rc) return rc;
  GemmParams p{};
  p.M = M; p.N = N; p.K = C;
  p.num_m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  p.num_n_tiles = N / bn;
  p.num_k_blocks = C / BLOCK_K;
  p.a_mode = 0;
  p.epi = EPI_SHUFFLE | (bias ? EPI_BIAS : 0);
  p.ldc = C;
  p.out_frame_stride = (long long)(2 * H) * (2 * W) * C;
  p.out_t_pad = out_t_pad;
  p.out_dup_head = out_dup_head;
  p.shuf_c = C; p.shuf_z = z; p.shuf_H = H; p.shuf_W = W;
  p.shuf_drop = (temporal && drop_head) ? 1 : 0;
  p.bias = (const __nv_bfloat16*)bias;
  p.out = y;
  return dispatch_gemm(bn, ta, tb, p, (cudaStream_t)stream);
}
