// Native host runtime of the causal 3-D conv video VAE behind the handle ABI (SURVEY.md §8(b) "C ABI to export":
// svr2_vae_encode / svr2_vae_decode / workspace query): the whole Encoder3D / Decoder3D kernel sequence, the temporal
// slicing with its per-layer conv memories and the activation arena run in C++ on a svr2_t handle — no Python and no
// torch allocation between the kernels.
//
// Replaces VideoAutoencoderKLWrapper.encode / .decode (attn_video_vae.py:1680-1698) with everything below it:
// Encoder3D.forward (:808-856), Decoder3D.forward (:983-1035), ResnetBlock3D (:311-362), Upsample3D (:110-174),
// Downsample3D (:226-250), UNetMidBlock3D + diffusers Attention (:656-668), causal_norm_wrapper and
// InflatedCausalConv3d incl. its `memory` across temporal slices (causal_inflation_lib.py:213-352, 354-409) and
// slicing_encode / slicing_decode (:1254-1300).
//
// Memory: every activation lives in ONE workspace (caller-provided or engine-owned).  The sequence is executed twice
// by the same code: a dry run (no launches) over an unbounded arena yields the exact peak = svr2_vae_workspace_bytes();
// the real run replays the identical first-fit decisions inside the workspace.  All work is stream-ordered on one
// stream, so a block is reusable as soon as the launch that last read it has been enqueued.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "engine_internal.h"

namespace svr2 {

struct VaeState {
  void* workspace = nullptr;
  size_t workspace_bytes = 0;
  std::vector<void*> retired;     // outgrown blocks: queued work / captured graphs may still use them
  int64_t last_launches = 0;
};

void vae_state_destroy(svr2_engine* e) {
  if (!e || !e->vae) return;
#ifndef SVR2_HOST_TEST
  if (e->vae->workspace) cudaFree(e->vae->workspace);
  for (void* p : e->vae->retired) cudaFree(p);
#endif
  delete e->vae;
  e->vae = nullptr;
}

namespace {

constexpr size_t NONE = ~(size_t)0;

// stream-ordered device copies / fills (host memory in the CPU test harness, tests/native/vae_trace.cu)
inline bool dev_copy(void* dst, const void* src, size_t bytes, void* stream) {
#ifdef SVR2_HOST_TEST
  memmove(dst, src, bytes);
  return true;
#else
  return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream) == cudaSuccess;
#endif
}
inline bool dev_zero(void* dst, size_t bytes, void* stream) {
#ifdef SVR2_HOST_TEST
  memset(dst, 0, bytes);
  return true;
#else
  return cudaMemsetAsync(dst, 0, bytes, (cudaStream_t)stream) == cudaSuccess;
#endif
}

// First-fit arena over [0, cap) with a persistent region growing down from the top (slicing state).
struct Arena {
  size_t cap = 0;                 // ~0/2 in a dry run
  size_t high = 0;                // high-water mark of the first-fit (low) end
  size_t top_used = 0;            // bytes taken from the top
  std::vector<std::pair<size_t, size_t>> free_list;   // (offset, size), sorted by offset, coalesced
  explicit Arena(size_t capacity) : cap(capacity) { free_list.push_back({0, capacity}); }
  size_t alloc(size_t bytes) {
    bytes = align_up(bytes ? bytes : 1);
    for (size_t i = 0; i < free_list.size(); ++i) {
      if (free_list[i].second < bytes) continue;
      const size_t off = free_list[i].first;
      if (off + bytes > cap - top_used) return NONE;
      if (free_list[i].second == bytes) free_list.erase(free_list.begin() + i);
      else { free_list[i].first += bytes; free_list[i].second -= bytes; }
      if (off + bytes > high) high = off + bytes;
      return off;
    }
    return NONE;
  }
  void release(size_t off, size_t bytes) {
    if (off == NONE) return;
    bytes = align_up(bytes ? bytes : 1);
    size_t i = 0;
    while (i < free_list.size() && free_list[i].first < off) ++i;
    free_list.insert(free_list.begin() + i, {off, bytes});
    if (i + 1 < free_list.size() && free_list[i].first + free_list[i].second == free_list[i + 1].first) {
      free_list[i].second += free_list[i + 1].second;
      free_list.erase(free_list.begin() + i + 1);
    }
    if (i > 0 && free_list[i - 1].first + free_list[i - 1].second == free_list[i].first) {
      free_list[i - 1].second += free_list[i].second;
      free_list.erase(free_list.begin() + i);
    }
  }
  size_t alloc_top(size_t bytes) {
    bytes = align_up(bytes ? bytes : 1);
    if (high + top_used + bytes > cap) return NONE;
    top_used += bytes;
    return cap - top_used;
  }
  size_t peak = 0;                // high + top_used before the last release_top()
  // the whole top region is free again (the next spatial tile starts its own slicing state)
  void release_top() {
    if (high + top_used > peak) peak = high + top_used;
    top_used = 0;
  }
  size_t need() const { return high + top_used > peak ? high + top_used : peak; }
};

// [pad + T, H, W, C] bf16 activation in the arena; `pad` halo frames in front replicate frame 0 (rep: its producer wrote
// them so, in the clip's first temporal slice) or hold the previous temporal slice's tail.  stat: GroupNorm partial sums
// written by the producing conv's epilogue.
struct Act {
  size_t off = NONE, bytes = 0;
  int T = 0, H = 0, W = 0, C = 0, pad = 0;
  bool rep = false;
  size_t stat_off = NONE, stat_bytes = 0;
  int slots = 0;
  size_t frame_bytes() const { return (size_t)H * W * C * 2; }
};

// The tile plan of tiled_encode / tiled_decode as vae.py's _tiled computes it.  encode: H x W sample pixels; decode:
// H x W latent pixels.  Tiles are latent rectangles [y0, y1) x [x0, x1) in row-major order.
struct TilePlan {
  bool encode = false, whole = false;     // whole: the frame fits one tile, the pass runs un-tiled
  int Hl = 0, Wl = 0, s = 1;              // latent frame; result pixels per latent pixel
  int ovh = 0, ovw = 0;                   // ramp lengths in result pixels
  std::vector<std::array<int, 4>> tiles;
};
TilePlan tile_plan(bool encode, int H, int W, int tile_h, int tile_w, int overlap_h, int overlap_w) {
  TilePlan p;
  const int f = 8;
  const int th = tile_h / f > 1 ? tile_h / f : 1, tw = tile_w / f > 1 ? tile_w / f : 1;
  p.encode = encode;
  p.whole = encode ? (H <= tile_h && W <= tile_w) : (H <= th && W <= tw);
  const int loh = std::max(0, std::min(overlap_h / f, th - 1)), low = std::max(0, std::min(overlap_w / f, tw - 1));
  const int sh = std::max(1, th - loh), sw = std::max(1, tw - low);
  p.Hl = encode ? (H + f - 1) / f : H;
  p.Wl = encode ? (W + f - 1) / f : W;
  p.s = encode ? 1 : f;
  p.ovh = encode ? loh : overlap_h;
  p.ovw = encode ? low : overlap_w;
  if (p.whole) return p;
  for (int y0 = 0; y0 < p.Hl; y0 += sh) {
    const int y1 = std::min(y0 + th, p.Hl);
    for (int x0 = 0; x0 < p.Wl; x0 += sw) {
      const int x1 = std::min(x0 + tw, p.Wl);
      if ((y0 > 0 && y1 - y0 <= loh) || (x0 > 0 && x1 - x0 <= low)) continue;    // inside the previous tile's overlap
      p.tiles.push_back({y0, y1, x0, x1});
    }
  }
  return p;
}

struct Run {
  svr2_engine* e;
  Arena A;
  char* base;          // nullptr: dry run (plan only)
  void* stream;
  bool slicing = false, first = true;
  bool tails = true;                                 // a later slice reads this slice's tails (false: the last decode slice)
  std::unordered_map<std::string, size_t> state;     // layer key -> top-region offset of the previous slice's tail
  int64_t launches = 0;
  int rc = SVR2_OK;
  // while a spatially tiled pass runs one tile: the input is a window of the clip (strides in elements) and the final
  // kernel is the seam variant, accumulating into the clip-sized result (seam.result: the tile's corner, frame 0)
  struct TileIO {
    int64_t in_cs, in_fs;
    int in_rs;
    Seam seam;
  };
  const TileIO* tile = nullptr;

  Run(svr2_engine* eng, size_t cap, char* b, void* st) : e(eng), A(cap), base(b), stream(st) {}
  bool dry() const { return base == nullptr; }
  bool ok() const { return rc == SVR2_OK; }
  char* P(size_t off) const { return base + off; }

  int err(int code, const char* msg) {
    if (rc == SVR2_OK) rc = fail(e, code, msg);
    return rc;
  }
  void ck(int r, int kernels = 1) {
    if (r && rc == SVR2_OK) {
      rc = r;
      snprintf(e->err, sizeof e->err, "%s", svr2_last_error());
    }
    launches += kernels;
  }
  size_t take(size_t bytes) {
    if (!ok()) return NONE;
    const size_t off = A.alloc(bytes);
    if (off == NONE) err(SVR2_ERR_ARG, "svr2_vae: workspace smaller than svr2_vae_workspace_bytes()");
    return off;
  }
  void give(size_t off, size_t bytes) { A.release(off, bytes); }
  Act act(int T, int H, int W, int C, int pad) {
    Act a;
    a.T = T; a.H = H; a.W = W; a.C = C; a.pad = pad;
    a.bytes = (size_t)(pad + T) * a.frame_bytes();
    a.off = take(a.bytes);
    return a;
  }
  void drop(Act& a) {
    give(a.off, a.bytes);
    give(a.stat_off, a.stat_bytes);
    a.off = a.stat_off = NONE;
  }
  const Tensor* weight(const std::string& name) {
    const Tensor* t = find(e, name);
    if (!t && ok()) {
      char buf[200];
      snprintf(buf, sizeof buf, "svr2_vae: weight '%s' not loaded", name.c_str());
      err(SVR2_ERR_ARG, buf);
    }
    return t;
  }
  bool has(const std::string& name) { return find(e, name) != nullptr; }

  // Slice boundary: the halo of a tensor that feeds a causal conv is the previous slice's tail at the same layer
  // (InflatedCausalConv3d.memory, causal_inflation_lib.py:306-352); remember this slice's tail unless no later slice
  // runs (the last decode slice).
  void halo(const Act& y, const std::string& key) {
    if (!slicing || y.pad == 0 || !ok()) return;
    const size_t bytes = (size_t)y.pad * y.frame_bytes();
    auto it = state.find(key);
    if (it != state.end()) {
      if (!dry() && !dev_copy(P(y.off), P(it->second), bytes, stream)) err(SVR2_ERR_CUDA, "svr2_vae: halo copy failed");
    } else if (tails) {
      const size_t off = A.alloc_top(bytes);
      if (off == NONE) { err(SVR2_ERR_ARG, "svr2_vae: workspace smaller than svr2_vae_workspace_bytes()"); return; }
      it = state.emplace(key, off).first;
    }
    if (tails && !dry() && ok()) {
      if (!dev_copy(P(it->second), P(y.off) + (size_t)y.T * y.frame_bytes(), bytes, stream))
        err(SVR2_ERR_CUDA, "svr2_vae: halo copy failed");
    }
  }

  // causal_norm_wrapper + SiLU (causal_inflation_lib.py:354-409): statistics from the producing conv's epilogue when
  // present, else the three-kernel path
  Act gn(const Act& x, const std::string& p, bool silu, int pad) {
    Act y = act(x.T, x.H, x.W, x.C, pad);
    const Tensor *g = weight(p + ".weight"), *b = weight(p + ".bias");
    if (!ok()) return y;
    const int dup = pad > 0 && first;
    y.rep = dup;
    if (x.stat_off != NONE) {
      const size_t cb = (size_t)x.T * x.C * 2 * 4;
      const size_t coef = take(cb);
      if (!dry() && ok())
        ck(svr2_groupnorm_from_stats_bf16(P(x.off) + (size_t)x.pad * x.frame_bytes(), P(y.off), x.T, x.H * x.W, x.C, g->ptr,
                                          b->ptr, 1e-6f, silu, pad, dup, P(x.stat_off), x.slots, P(coef), stream), 2);
      give(coef, cb);
    } else {
      const size_t sb = ((size_t)svr2_groupnorm_scratch_bytes(x.T, x.H * x.W, x.C) + 7) / 8 * 8;
      const size_t scratch = take(sb);
      if (!dry() && ok())
        ck(svr2_groupnorm_bf16(P(x.off) + (size_t)x.pad * x.frame_bytes(), P(y.off), x.T, x.H * x.W, x.C, g->ptr, b->ptr,
                               1e-6f, silu, pad, dup, (double*)P(scratch), (int64_t)sb, stream), 3);
      give(scratch, sb);
    }
    halo(y, p);
    return y;
  }

  // InflatedCausalConv3d (causal_inflation_lib.py:213-305); weight tensor [Cout, kt, kh, kw, Cin]
  Act conv(const Act& x, const std::string& p, int out_pad, const Act* residual, int stride_t, int stride_hw, bool stats) {
    const Tensor *w = weight(p + ".weight"), *b = weight(p + ".bias");
    if (!ok()) return Act();
    if (w->rank != 5) { err(SVR2_ERR_ARG, "svr2_vae: conv weights must be passed as [Cout, kt, kh, kw, Cin]"); return Act(); }
    const int Cout = (int)w->shape[0], kt = (int)w->shape[1], kh = (int)w->shape[2], kw = (int)w->shape[3];
    if (x.pad != kt - 1 || (int)w->shape[4] != x.C) { err(SVR2_ERR_ARG, "svr2_vae: conv input halo / channels do not match the weight"); return Act(); }
    size_t x_off = x.off;
    int T_in_total = x.pad + x.T, T_out;
    if (stride_t == 2 && !first) {
      // a later slice of a temporally strided conv continues the global stride phase: one frame of memory instead of two
      if (x.T % 2) { err(SVR2_ERR_ARG, "svr2_vae: temporal slices after the first must hold a multiple of 4 frames"); return Act(); }
      x_off += x.frame_bytes();
      T_in_total = x.pad - 1 + x.T;
      T_out = x.T / 2;
    } else {
      T_out = (x.T - 1) / stride_t + 1;
    }
    const int Ho = stride_hw == 1 ? x.H : x.H / 2, Wo = stride_hw == 1 ? x.W : x.W / 2;
    Act y = act(T_out, Ho, Wo, Cout, out_pad);
    y.rep = out_pad > 0 && first;
    const bool with_stats = stats && (Cout == 128 || Cout == 256 || Cout == 512);
    if (with_stats) {
      y.slots = svr2_conv_stat_slots(Cout, Ho, Wo);
      y.stat_bytes = (size_t)T_out * y.slots * (Cout / 8) * 16;
      y.stat_off = take(y.stat_bytes);
    }
    if (residual && (residual->T != T_out || residual->H != Ho || residual->W != Wo || residual->C != Cout)) {
      err(SVR2_ERR_ARG, "svr2_vae: residual shape mismatch");
      return y;
    }
    const Tensor* wf = x.rep ? head_weight(p + ".weight", kt, Cout, (int64_t)kt * kh * kw * x.C) : nullptr;
    if (dry() || !ok()) return finish_conv(y, p);
    // the kernel indexes the residual with the output's offsets (which include out_pad halo frames)
    const void* res = residual ? P(residual->off) + (size_t)residual->pad * residual->frame_bytes() - (size_t)out_pad * y.frame_bytes()
                               : nullptr;
    const int epi = SVR2_EPI_BIAS | (residual ? SVR2_EPI_RESIDUAL : 0) | (wf ? SVR2_EPI_FOLD_HEAD : 0);
    const int pad_hw = (stride_hw == 1 && kh == 3) ? 1 : 0;
    const int dup = out_pad > 0 && first;
    const void* wp = wf ? wf->ptr : w->ptr;
    if (with_stats) {
      int slots = 0;
      ck(svr2_conv3d_stats_bf16(P(x_off), T_in_total, x.H, x.W, x.C, wp, Cout, kt, kh, kw, stride_t, stride_hw, pad_hw,
                                T_out, epi, b->ptr, res, P(y.off), out_pad, dup, Cout, P(y.stat_off), (int64_t)y.stat_bytes,
                                &slots, stream));
      if (ok() && slots != y.slots) err(SVR2_ERR_ARG, "svr2_vae: statistics slot count differs from the plan");
    } else {
      ck(svr2_conv3d_bf16(P(x_off), T_in_total, x.H, x.W, x.C, wp, Cout, kt, kh, kw, stride_t, stride_hw, pad_hw, T_out,
                          epi, b->ptr, res, P(y.off), out_pad, dup, Cout, stream));
    }
    return finish_conv(y, p);
  }
  // When the halo in front of a kt = 3 conv's input replicates its frame 0 (Act::rep), output frames 0 and 1 run with the
  // taps over the copies folded into one weight (SVR2_EPI_FOLD_HEAD).  `name` + ":head" is that weight with the folded
  // rows appended ([2 Cout, K]); null when it was not loaded.
  const Tensor* head_weight(const std::string& name, int kt, int Cout, int64_t K) {
    if (kt != 3 || !ok()) return nullptr;
    const Tensor* t = find(e, name + ":head");
    if (t && (t->rank != 2 || t->shape[0] != 2 * (int64_t)Cout || t->shape[1] != K)) {
      err(SVR2_ERR_ARG, "svr2_vae: folded head weights must be [2 Cout, K]");
      return nullptr;
    }
    return t;
  }
  Act finish_conv(Act& y, const std::string& p) {
    halo(y, p + ":out");
    return y;
  }

  // conv2(h) + conv_shortcut(x) as one implicit GEMM over [h ; x]; statistics for the next GroupNorm
  Act conv_shortcut(const Act& h, const Act& x, const std::string& p, int out_pad) {
    const Tensor *w = weight(p + "conv2+shortcut.weight"), *b = weight(p + "conv2+shortcut.bias"), *w2 = weight(p + "conv2.weight");
    if (!ok()) return Act();
    const int Cout = (int)w->shape[0], kt = (int)w2->shape[1], kh = (int)w2->shape[2], kw = (int)w2->shape[3], C2 = x.C;
    if (h.pad != kt - 1 || h.T != x.T || h.H != x.H || h.W != x.W || h.C != Cout) { err(SVR2_ERR_ARG, "svr2_vae: fused shortcut shape mismatch"); return Act(); }
    Act y = act(h.T, h.H, h.W, Cout, out_pad);
    y.rep = out_pad > 0 && first;
    y.slots = svr2_conv_stat_slots(Cout, h.H, h.W);
    y.stat_bytes = (size_t)h.T * y.slots * (Cout / 8) * 16;
    y.stat_off = take(y.stat_bytes);
    if (!dry() && ok()) {
      int slots = 0;
      ck(svr2_conv3d_shortcut_stats_bf16(P(h.off), h.pad + h.T, h.H, h.W, h.C, w->ptr, Cout, kt, kh, kw, h.T, b->ptr,
                                         P(x.off) + (size_t)x.pad * x.frame_bytes(), C2, P(y.off), out_pad,
                                         out_pad > 0 && first, P(y.stat_off), (int64_t)y.stat_bytes, &slots, stream));
      if (ok() && slots != y.slots) err(SVR2_ERR_ARG, "svr2_vae: statistics slot count differs from the plan");
    }
    halo(y, p + "conv2:out");
    return y;
  }

  // ResnetBlock3D.forward (attn_video_vae.py:311-362); consumes x
  Act resnet(Act& x, const std::string& p, int out_pad) {
    Act h = gn(x, p + "norm1", true, 2);
    Act c1 = conv(h, p + "conv1", 0, nullptr, 1, 1, true);
    drop(h);
    Act h2 = gn(c1, p + "norm2", true, 2);
    drop(c1);
    Act y = has(p + "conv_shortcut.weight") ? conv_shortcut(h2, x, p, out_pad) : conv(h2, p + "conv2", out_pad, &x, 1, 1, true);
    drop(h2);
    drop(x);
    return y;
  }

  int linear(const void* a, int64_t lda, const void* w, int64_t ldw, int M, int N, int K, int epi, const void* bias,
             const float* gate, const void* residual, void* out, int64_t ldc, float out_scale, const float* rowscale = nullptr,
             void* stat_out = nullptr, int64_t ld_stat = 0, const int* run_if = nullptr) {
    if (!ok()) return rc;
    if (bias) epi |= SVR2_EPI_BIAS;
    if (gate && !(epi & SVR2_EPI_PEXP)) epi |= SVR2_EPI_GATE;
    if (residual) epi |= SVR2_EPI_RESIDUAL;
    if (rowscale || stat_out || run_if) {
      if (rowscale) epi |= SVR2_EPI_ROWSCALE;
      ck(svr2_linear_ex_bf16(a, lda, w, ldw, M, N, K, epi, bias, gate, residual, out, ldc, out_scale, rowscale, stat_out, ld_stat,
                             run_if, stream));
    } else {
      ck(svr2_linear_bf16(a, lda, w, ldw, M, N, K, epi, bias, gate, residual, out, ldc, out_scale, stream));
    }
    return rc;
  }

  // UNetMidBlock3D per-frame attention (attn_video_vae.py:656-668): GN -> q,k,v -> 1-head softmax(q k^T / sqrt(C)) v ->
  // out proj -> + x.  Consumes x.  One Q K^T pass with a sampled reference exponent, the exact two-pass launches
  // conditional on the device-side safety flag (see svr2.h "Single-pass variant").
  Act attention(Act& x, const std::string& p) {
    const int C = x.C, n = x.H * x.W, T = x.T;
    Act y = gn(x, p + "group_norm", false, 0);
    const Tensor *wq = weight(p + "to_q.weight"), *bq = weight(p + "to_q.bias"), *wk = weight(p + "to_k.weight"),
                 *bk = weight(p + "to_k.bias"), *wv = weight(p + "to_v.weight"), *bv = weight(p + "to_v.bias"),
                 *wo = weight(p + "to_out.0.weight"), *bo = weight(p + "to_out.0.bias");
    const size_t rowb = (size_t)C * 2, tn = (size_t)T * n;
    const size_t q_b = tn * rowb, k_b = (tn + 8) * rowb;
    const size_t q = take(q_b), kbuf = take(k_b), v = take(q_b);
    const int ldn = (n + 7) / 8 * 8;
    if (!dry() && ok()) {
      // K carries 8 spare zero rows: the exact pass 2 runs with N rounded up to a multiple of 8 (16-byte stores)
      if (!dev_zero(P(kbuf) + tn * rowb, 8 * rowb, stream)) err(SVR2_ERR_CUDA, "svr2_vae: memset failed");
      linear(P(y.off), C, wq->ptr, C, (int)tn, C, C, 0, bq->ptr, nullptr, nullptr, P(q), C, 1.f);
      linear(P(y.off), C, wk->ptr, C, (int)tn, C, C, 0, bk->ptr, nullptr, nullptr, P(kbuf), C, 1.f);
      linear(P(y.off), C, wv->ptr, C, (int)tn, C, C, 0, bv->ptr, nullptr, nullptr, P(v), C, 1.f);
    }
    drop(y);
    const long long wave_rows = 66 * 128;       // 66 m-tiles x 2 n-tiles (d = 512) = one full wave of 132 CTAs
    long long kk = (1LL << 32) / (wave_rows * ldn * 2);
    if (kk < 1) kk = 1;
    long long cq = wave_rows * kk;
    if (cq > (n + 127) / 128 * 128) cq = (n + 127) / 128 * 128;
    const int rows_max = (int)(cq < n ? cq : n);
    const int slots = svr2_rowstat_slots(n);
    const size_t vt_b = (size_t)C * ldn * 2, part_b = (size_t)rows_max * 2 * slots * 4, lse_b = (size_t)rows_max * 4,
                 P_b = (size_t)rows_max * ldn * 2;
    const size_t vt = take(vt_b), part = take(part_b), lse = take(lse_b), Pm = take(P_b), o = take(q_b);
    const float scale2 = (float)((1.0 / sqrt((double)C)) * 1.4426950408889634);
    const bool single = n >= 256 && n % 8 == 0;
    const int k_sub = 16, n_sub = (n + k_sub - 1) / k_sub;
    const int slots_s = single ? svr2_rowstat_slots(n_sub) : 0, slots_p = 2 * ((n + 255) / 256);
    const size_t ps_b = (size_t)rows_max * 2 * slots_s * 4, st_b = (size_t)rows_max * 2 * slots_p * 4;
    size_t part_s = NONE, stat = NONE, mhat = NONE, rscale = NONE, flag = NONE;
    if (single) {
      part_s = take(ps_b); stat = take(st_b); mhat = take(lse_b); rscale = take(lse_b); flag = take(4);
      if (!dry() && ok() && !dev_zero(P(flag), 4, stream)) err(SVR2_ERR_CUDA, "svr2_vae: memset failed");
    }
    if (!dry()) {
      for (int f = 0; f < T && ok(); ++f) {
        const char *qf = P(q) + (size_t)f * n * rowb, *kf = P(kbuf) + (size_t)f * n * rowb, *vf = P(v) + (size_t)f * n * rowb;
        ck(svr2_transpose_bf16(vf, C, P(vt), ldn, n, C, stream));
        for (long long r0 = 0; r0 < n && ok(); r0 += cq) {
          const int rows = (int)(cq < n - r0 ? cq : n - r0);
          const char* qc = qf + (size_t)r0 * rowb;
          char* oc = P(o) + ((size_t)f * n + r0) * rowb;
          const int* run_if = nullptr;
          if (single) {
            linear(qc, C, kf, (int64_t)k_sub * C, rows, n_sub, C, SVR2_EPI_ROWSTAT, nullptr, nullptr, nullptr, P(part_s), slots_s, scale2);
            ck(svr2_rowstat_max(P(part_s), slots_s, slots_s, (float*)P(mhat), rows, (int*)P(flag), stream));
            linear(qc, C, kf, C, rows, n, C, SVR2_EPI_PEXP, nullptr, (const float*)P(mhat), nullptr, P(Pm), ldn, scale2, nullptr,
                   P(stat), slots_p);
            ck(svr2_pexp_stat_combine(P(stat), slots_p, slots_p, (const float*)P(mhat), (float*)P(rscale), rows, (int*)P(flag), stream));
            linear(P(Pm), ldn, P(vt), ldn, rows, C, n, 0, nullptr, nullptr, nullptr, oc, C, 1.f, (const float*)P(rscale));
            run_if = (const int*)P(flag);
          }
          // exact path: unconditional, or the device-side fallback (no-ops while the flag is clear)
          linear(qc, C, kf, C, rows, n, C, SVR2_EPI_ROWSTAT, nullptr, nullptr, nullptr, P(part), slots, scale2, nullptr, nullptr, 0, run_if);
          ck(svr2_rowstat_combine(P(part), slots, slots, (float*)P(lse), rows, stream));
          linear(qc, C, kf, C, rows, ldn, C, SVR2_EPI_PEXP, nullptr, (const float*)P(lse), nullptr, P(Pm), ldn, scale2, nullptr, nullptr, 0, run_if);
          linear(P(Pm), ldn, P(vt), ldn, rows, C, n, 0, nullptr, nullptr, nullptr, oc, C, 1.f, nullptr, nullptr, 0, run_if);
        }
      }
    }
    give(part_s, ps_b); give(stat, st_b); give(mhat, lse_b); give(rscale, lse_b); give(flag, 4);
    give(vt, vt_b); give(part, part_b); give(lse, lse_b); give(Pm, P_b);
    give(q, q_b); give(kbuf, k_b); give(v, q_b);
    Act out = act(T, x.H, x.W, C, 0);
    if (!dry() && ok())
      linear(P(o), C, wo->ptr, C, (int)tn, C, C, 0, bo->ptr, nullptr, P(x.off) + (size_t)x.pad * x.frame_bytes(), P(out.off), C, 1.f);
    give(o, q_b);
    drop(x);
    return out;
  }

  Act mid(Act& x, const std::string& p) {
    Act a = resnet(x, p + "resnets.0.", 0);
    Act b = attention(a, p + "attentions.0.");
    return resnet(b, p + "resnets.1.", 0);
  }

  // Upsample3D.forward (attn_video_vae.py:110-174); consumes x.  keep > 0: only the first `keep` shuffled frames are
  // wanted — every layer after the decoder's last temporal upsampler is causal frame by frame, so the conv and
  // everything after it run on those frames alone (the block keeps its full size: it is released whole)
  Act upsample(Act& x, const std::string& p, bool temporal, int keep = 0) {
    const Tensor *w = weight(p + "upscale_conv.weight"), *b = weight(p + "upscale_conv.bias");
    const int z = temporal ? 2 : 1;
    const int T_out = x.T * z - (temporal && first ? 1 : 0);      // remove_head only drops (f=0, z=1) of the clip's first slice
    Act y = act(T_out, 2 * x.H, 2 * x.W, x.C, 2);
    y.rep = first;
    if (!dry() && ok())
      ck(svr2_upsample_shuffle_bf16(P(x.off) + (size_t)x.pad * x.frame_bytes(), x.T, x.H, x.W, x.C, w->ptr, b->ptr, temporal, first,
                                    P(y.off), 2, first, stream));
    drop(x);
    if (keep > 0 && keep < y.T) y.T = keep;
    halo(y, p + "shuffle");
    Act c = conv(y, p + "conv", 0, nullptr, 1, 1, true);
    drop(y);
    return c;
  }

  // One temporal slice of Decoder3D.forward: z (16 channels, T frames of h x w, channel stride zin_cs elements) ->
  // out (3 channels, the first `keep` of the slice's T' frames of 8h x 8w written at out, channel stride out_cs);
  // T' = 4T-3 for the first slice, else 4T
  void decode_slice(const void* zin, int dt, int64_t zin_cs, int T, int h, int w, void* out, int64_t out_cs, int keep) {
    Act x = act(T, h, w, 64, 2);
    x.rep = first;
    if (!dry() && ok()) ck(read_input(zin, dt, 16, T, h, w, zin_cs, P(x.off), 64));
    halo(x, "decoder.in");
    Act c = conv(x, "decoder.conv_in", 0, nullptr, 1, 1, true);
    drop(x);
    Act m = mid(c, "decoder.mid_block.");
    char name[96];
    for (int i = 0; i < 4 && ok(); ++i) {
      for (int j = 0; j < 3; ++j) {
        snprintf(name, sizeof name, "decoder.up_blocks.%d.resnets.%d.", i, j);
        m = resnet(m, name, 0);
      }
      if (i < 3) {
        snprintf(name, sizeof name, "decoder.up_blocks.%d.upsamplers.0.", i);
        m = upsample(m, name, i < 2, i == 1 ? keep : 0);
      }
    }
    Act g = gn(m, "decoder.conv_norm_out", true, 2);
    drop(m);
    if (ok() && g.T != keep) err(SVR2_ERR_ARG, "svr2_vae_decode: decoded frame count differs from the plan");
    // conv_out (128 -> 3): per-tap channel contraction as ONE GEMM over all input pixels (x read once, not 27 times),
    // fp32 z[tap*3+co][pixel], then the 27-tap gather writes NCDHW directly
    const Tensor *wt = weight("decoder.conv_out.weight"), *bo = weight("decoder.conv_out.bias");
    const long long npix = (long long)(g.pad + g.T) * g.H * g.W;
    const long long ldz = (npix + 3) / 4 * 4;
    const size_t z_b = (size_t)81 * ldz * 4;
    const size_t z = take(z_b);
    if (!dry() && ok()) {
      if (npix > 0x7fffffffLL) err(SVR2_ERR_ARG, "svr2_vae_decode: slice too large (pixels per slice must fit 31 bits)");
      linear(wt->ptr, g.C, P(g.off), g.C, 81, (int)npix, g.C, SVR2_EPI_F32, nullptr, nullptr, nullptr, P(z), ldz, 1.f);
      if (ok() && tile) ck(conv_tap_gather_seam((const float*)P(z), ldz, 3, bo->ptr, g.T, g.H, g.W, seam_at(out), stream));
      else if (ok()) ck(conv_tap_gather_strided((const float*)P(z), ldz, 3, bo->ptr, g.T, g.H, g.W, out, 1, out_cs, stream));
    }
    give(z, z_b);
    drop(g);
  }

  // One temporal slice of Encoder3D.forward + posterior mode: x (3 channels, T frames H x W) -> 16 x T' x H/8 x W/8;
  // T = 1 + 4k for the first slice (T' = k + 1), 4k afterwards (T' = k)
  void encode_slice(const void* xin, int dt, int64_t xin_cs, int T, int H, int W, void* out, int64_t out_cs) {
    Act x8 = act(T, H, W, 8, 2);
    if (!dry() && ok()) ck(read_input(xin, dt, 3, T, H, W, xin_cs, P(x8.off), 8));
    halo(x8, "encoder.in");
    const size_t col_b = (size_t)T * H * W * 128 * 2;
    const size_t col = take(col_b);
    const Tensor *wi = weight("encoder.conv_in.weight"), *bi = weight("encoder.conv_in.bias");
    Act h = act(T, H, W, 128, 0);
    if (!dry() && ok()) {
      ck(svr2_im2col3_bf16(P(x8.off), T, H, W, 3, 8, P(col), 128, stream));
      linear(P(col), 128, wi->ptr, 128, T * H * W, 128, 128, 0, bi->ptr, nullptr, nullptr, P(h.off), 128, 1.f);
    }
    give(col, col_b);
    drop(x8);
    char name[96];
    for (int i = 0; i < 4 && ok(); ++i) {
      const bool temporal = i == 1 || i == 2;
      snprintf(name, sizeof name, "encoder.down_blocks.%d.resnets.0.", i);
      h = resnet(h, name, 0);
      snprintf(name, sizeof name, "encoder.down_blocks.%d.resnets.1.", i);
      h = resnet(h, name, (i < 3 && temporal) ? 2 : 0);
      if (i < 3) {
        snprintf(name, sizeof name, "encoder.down_blocks.%d.downsamplers.0.conv", i);
        Act d = conv(h, name, 0, nullptr, temporal ? 2 : 1, 2, true);
        drop(h);
        h = d;
      }
    }
    h = mid(h, "encoder.mid_block.");
    Act g = gn(h, "encoder.conv_norm_out", true, 2);
    drop(h);
    Act c = conv(g, "encoder.conv_out", 0, nullptr, 1, 1, false);
    drop(g);
    if (!dry() && ok() && tile) ck(ndhwc_to_ncdhw_seam(P(c.off), c.C, 16, c.T, c.H, c.W, seam_at(out), stream));
    else if (!dry() && ok()) ck(ndhwc_to_ncdhw_strided(P(c.off), c.C, 16, c.T, c.H, c.W, out, 1, out_cs, stream));
    drop(c);
  }

  // the input conversion of a slice: the whole clip's frames, or the current tile's window of them
  int read_input(const void* in, int dt, int C, int T, int H, int W, int64_t cs, void* out, int C_pad) {
    if (tile) return ncdhw_to_ndhwc_window(in, dt, C, T, H, W, cs, tile->in_fs, tile->in_rs, out, C_pad, 2, 1.0f, stream);
    return ncdhw_to_ndhwc_strided(in, dt, C, T, H, W, cs, out, C_pad, 2, 1.0f, stream);
  }
  // the current tile's seam at `out` (this slice's first frame); the count plane takes each pixel's weight once, in the
  // first slice
  Seam seam_at(void* out) const {
    Seam s = tile->seam;
    s.result = out;
    if (!first) s.count = nullptr;
    return s;
  }

  // slicing_decode (attn_video_vae.py:1279-1300): the first slice is latent frame 0 plus `size` frames, then `size` each.
  // Only the first `frames` (1 .. 4T-3) output frames are computed: the decoder is causal in time, so the reference's
  // decode-then-crop returns the same values.  Slices past them do not run, the last one that does is trimmed.
  void decode(const void* z, int dt, int T, int h, int w, int size, int frames, void* out) {
    const int esz = dt == 0 ? 4 : 2;
    const int64_t zin_cs = tile ? tile->in_cs : (int64_t)T * h * w, out_cs = (int64_t)frames * 64 * h * w;
    const int64_t in_fs = tile ? tile->in_fs : (int64_t)h * w, out_fs = tile ? tile->seam.fs : (int64_t)64 * h * w;
    if (size <= 0 || T - 1 <= size) {
      decode_slice(z, dt, zin_cs, T, h, w, out, out_cs, frames);
      return;
    }
    slicing = true;
    for (int a = 0, b = 1 + size; a < T && ok(); a = b, b = (b + size < T ? b + size : T)) {
      first = a == 0;
      const int o0 = a == 0 ? 0 : 4 * a - 3, n_out = 4 * (b - a) - (first ? 3 : 0);
      const int keep = frames - o0 < n_out ? frames - o0 : n_out;
      if (keep <= 0) break;                // this and every later slice lie past the wanted frames
      tails = o0 + n_out < frames;         // a later slice runs and continues from this one's tails
      decode_slice((const char*)z + (size_t)a * in_fs * esz, dt, zin_cs, b - a, h, w, (char*)out + (size_t)o0 * out_fs * 2,
                   out_cs, keep);
    }
  }

  // slicing_encode (attn_video_vae.py:1254-1277): frame 0 plus `size` sample frames (a multiple of 4), then `size` each;
  // only clips of 4n+1 frames continue the stride-2 phase of the temporal downsamplers across slices
  void encode(const void* x, int dt, int T, int H, int W, int size, void* out) {
    const int esz = dt == 0 ? 4 : 2;
    const int T_lat = (T - 1) / 4 + 1;
    const int64_t xin_cs = tile ? tile->in_cs : (int64_t)T * H * W, out_cs = (int64_t)T_lat * (H / 8) * (W / 8);
    const int64_t in_fs = tile ? tile->in_fs : (int64_t)H * W, out_fs = tile ? tile->seam.fs : (int64_t)(H / 8) * (W / 8);
    if (size <= 0 || T - 1 <= size || (T - 1) % 4 != 0) {
      encode_slice(x, dt, xin_cs, T, H, W, out, out_cs);
      return;
    }
    if (size % 4) { err(SVR2_ERR_ARG, "svr2_vae_encode: slice_frames must be a multiple of 4"); return; }
    slicing = true;
    for (int a = 0, b = 1 + size; a < T && ok(); a = b, b = (b + size < T ? b + size : T)) {
      first = a == 0;
      const int64_t o0 = a == 0 ? 0 : (a - 1) / 4 + 1;
      encode_slice((const char*)x + (size_t)a * in_fs * esz, dt, xin_cs, b - a, H, W, (char*)out + (size_t)o0 * out_fs * 2,
                   out_cs);
    }
  }

  // tiled_encode / tiled_decode (attn_video_vae.py:1302-1630) in vae.py _tiled's order: the frame is cut into latent
  // tiles of tile // 8 stepping by tile // 8 - overlap // 8, a tile wholly inside the previous one's overlap is skipped;
  // each tile runs the whole (temporally sliced) encoder / decoder with its own slicing state on a window of the clip,
  // and its final kernel accumulates it into `out` with the edge weights; `out` is normalised by the count plane at the
  // end.  encode: x [3, T, H, W] -> [16, T', H/8, W/8]; decode: z [16, T, H, W] -> [3, frames, 8H, 8W].
  void tiled(const TilePlan& p, const void* in, int dt, int T, int H, int W, int size, int frames, void* out) {
    const int esz = dt == 0 ? 4 : 2, f = p.encode ? 8 : 1;        // input pixels per latent pixel
    const int C = p.encode ? 16 : 3, T_out = p.encode ? (T - 1) / 4 + 1 : frames;
    const int Hr = p.Hl * p.s, Wr = p.Wl * p.s;
    const size_t plane = (size_t)Hr * Wr, count_b = plane * 2;
    const size_t count = take(count_b);
    const size_t rh_b = (size_t)4 * p.ovh, rw_b = (size_t)4 * p.ovw;
    const size_t rh = p.ovh > 0 ? take(rh_b) : NONE, rw = p.ovw > 0 ? take(rw_b) : NONE;
    if (!dry() && ok()) {
      if (!dev_zero(out, (size_t)C * T_out * count_b, stream) || !dev_zero(P(count), count_b, stream))
        err(SVR2_ERR_CUDA, "svr2_vae: memset failed");
      ck(tile_ramp(rh == NONE ? nullptr : P(rh), p.ovh, rw == NONE ? nullptr : P(rw), p.ovw, stream));
    }
    for (const auto& r : p.tiles) {
      if (!ok()) break;
      const int y0 = r[0], y1 = r[1], x0 = r[2], x1 = r[3];
      const size_t corner = ((size_t)y0 * p.s * Wr + (size_t)x0 * p.s) * 2;
      TileIO io;
      io.in_cs = (int64_t)T * H * W;
      io.in_fs = (int64_t)H * W;
      io.in_rs = W;
      io.seam = Seam{(char*)out + corner, (int64_t)T_out * (int64_t)plane, (int64_t)plane, Wr, dry() ? nullptr : P(count) + corner,
                     rh == NONE ? nullptr : P(rh), rw == NONE ? nullptr : P(rw), p.ovh, p.ovw,
                     (y0 > 0 ? SVR2_SEAM_TOP : 0) | (y1 < p.Hl ? SVR2_SEAM_BOTTOM : 0) | (x0 > 0 ? SVR2_SEAM_LEFT : 0) |
                         (x1 < p.Wl ? SVR2_SEAM_RIGHT : 0)};
      tile = &io;
      slicing = false;
      first = tails = true;
      state.clear();
      A.release_top();
      const char* src = (const char*)in + ((size_t)y0 * f * W + (size_t)x0 * f) * esz;
      if (p.encode) encode(src, dt, T, (y1 - y0) * 8, (x1 - x0) * 8, size, io.seam.result);
      else decode(src, dt, T, y1 - y0, x1 - x0, size, frames, io.seam.result);
      tile = nullptr;
    }
    if (!dry() && ok()) ck(svr2_tile_normalize_bf16(out, P(count), C * T_out, (int64_t)plane, stream));
    give(rw, rw_b);
    give(rh, rh_b);
    give(count, count_b);
  }
};

int check_args(svr2_engine* e, const char* what, int T, int H, int W, int mult) {
  char buf[160];
  if (!e) return set_error(SVR2_ERR_ARG, "svr2_vae: null handle");
  if (e->desc.variant != 2) {
    snprintf(buf, sizeof buf, "%s: the handle was not created as a VAE (svr2_model_desc.variant == 2)", what);
    return fail(e, SVR2_ERR_ARG, buf);
  }
  if (T <= 0 || H <= 0 || W <= 0 || H % mult || W % mult) {
    snprintf(buf, sizeof buf, "%s: T, H, W > 0 and H, W multiples of %d", what, mult);
    return fail(e, SVR2_ERR_ARG, buf);
  }
  return SVR2_OK;
}

// decode: the number of output frames wanted, 1 .. 4T-3
int check_frames(svr2_engine* e, const char* what, int T, int frames) {
  if (frames >= 1 && frames <= 4 * T - 3) return SVR2_OK;
  char buf[160];
  snprintf(buf, sizeof buf, "%s: frames = %d, a decode of %d latent frames returns 1 .. %d frames", what, frames, T, 4 * T - 3);
  return fail(e, SVR2_ERR_ARG, buf);
}

// a spatial tile of at least one pixel, overlaps >= 0
int check_tiles(svr2_engine* e, const char* what, int tile_h, int tile_w, int overlap_h, int overlap_w) {
  if (tile_h >= 1 && tile_w >= 1 && overlap_h >= 0 && overlap_w >= 0) return SVR2_OK;
  char buf[160];
  snprintf(buf, sizeof buf, "%s: tile sizes >= 1 and overlaps >= 0 (got %d x %d, %d x %d)", what, tile_h, tile_w, overlap_h,
           overlap_w);
  return fail(e, SVR2_ERR_ARG, buf);
}

// the whole pass on one Run: spatially tiled when `tiles` cuts the frame, else un-tiled
void sequence(Run& r, const TilePlan* tiles, int encode, const void* in, int dt, int T, int H, int W, int slice_frames,
              int frames, void* out) {
  if (tiles && !tiles->whole) r.tiled(*tiles, in, dt, T, H, W, slice_frames, frames, out);
  else if (encode) r.encode(in, dt, T, H, W, slice_frames, out);
  else r.decode(in, dt, T, H, W, slice_frames, frames, out);
}

// frames: output frames of a decode (ignored by an encode)
size_t plan_bytes(svr2_engine* e, int encode, int T, int H, int W, int slice_frames, int frames, const TilePlan* tiles = nullptr) {
  Run r(e, ~(size_t)0 / 2, nullptr, nullptr);
  sequence(r, tiles, encode, nullptr, 1, T, H, W, slice_frames, frames, nullptr);
  return r.ok() ? r.A.need() : 0;
}

int run(svr2_engine* e, int encode, const void* in, int dt, int T, int H, int W, int slice_frames, int frames, void* out,
        void* ws, size_t ws_bytes, void* stream, const TilePlan* tiles = nullptr) {
  const char* what = tiles ? (encode ? "svr2_vae_encode_tiled" : "svr2_vae_decode_tiled")
                           : (encode ? "svr2_vae_encode" : "svr2_vae_decode");
  int rc = check_args(e, what, T, H, W, encode ? 8 : 1);
  if (!rc && !encode) rc = check_frames(e, what, T, frames);
  if (rc) return rc;
  if (!in || !out) return fail(e, SVR2_ERR_ARG, "svr2_vae: null input / output");
  if (dt < 0 || dt > 2) return fail(e, SVR2_ERR_ARG, "svr2_vae: dtype must be 0 (f32), 1 (bf16) or 2 (f16)");
#ifndef SVR2_HOST_TEST
  int cur = 0;
  cudaGetDevice(&cur);
  if (cur != e->device) return fail(e, SVR2_ERR_ARG, "svr2_vae: the handle's device is not the current device");
#endif
  const size_t need = plan_bytes(e, encode, T, H, W, slice_frames, frames, tiles);
  if (!need) return SVR2_ERR_ARG;      // message already recorded
  if (!e->vae) e->vae = new VaeState();
  char* base;
  if (ws) {
    if (ws_bytes < need) return fail(e, SVR2_ERR_ARG, "svr2_vae: workspace smaller than svr2_vae_workspace_bytes()");
    if ((uintptr_t)ws % 256) return fail(e, SVR2_ERR_ARG, "svr2_vae: workspace must be 256-byte aligned");
    base = (char*)ws;
  } else {
    VaeState* v = e->vae;
    if (need > v->workspace_bytes) {
      if (v->workspace) v->retired.push_back(v->workspace);
      v->workspace = nullptr;
      v->workspace_bytes = 0;
#ifdef SVR2_HOST_TEST
      return fail(e, SVR2_ERR_CUDA, "svr2_vae: host test needs a caller workspace");
#else
      if (cudaMalloc(&v->workspace, need) != cudaSuccess) return fail(e, SVR2_ERR_CUDA, "svr2_vae: workspace allocation failed");
#endif
      v->workspace_bytes = need;
    }
    base = (char*)v->workspace;
  }
  Run r(e, need, base, stream);
  sequence(r, tiles, encode, in, dt, T, H, W, slice_frames, frames, out);
  e->vae->last_launches = r.launches;
  return r.rc;
}

}  // namespace
}  // namespace svr2

using namespace svr2;

// Bytes of workspace one encode (direction 0: T sample frames of H x W) or decode (direction 1: T latent frames of
// H x W latent pixels) uses with temporal slices of `slice_frames` (0 = un-sliced).  Exact: the dry run of the same code.
extern "C" size_t svr2_vae_workspace_bytes(svr2_t* e, int direction, int T, int H, int W, int slice_frames) {
  if (check_args(e, "svr2_vae_workspace_bytes", T, H, W, direction == 0 ? 8 : 1)) return 0;
  return plan_bytes(e, direction == 0, T, H, W, slice_frames, 4 * T - 3);
}

// Bytes of workspace one decode of T latent frames that returns only the first `frames` output frames uses.  Exact.
extern "C" size_t svr2_vae_decode_frames_workspace_bytes(svr2_t* e, int T, int h, int w, int slice_frames, int frames) {
  const char* what = "svr2_vae_decode_frames_workspace_bytes";
  if (check_args(e, what, T, h, w, 1) || check_frames(e, what, T, frames)) return 0;
  return plan_bytes(e, 0, T, h, w, slice_frames, frames);
}

extern "C" int svr2_vae_encode(svr2_t* e, const void* x, int x_dtype, int T, int H, int W, int slice_frames, void* latent,
                               void* workspace, size_t workspace_bytes, void* stream) {
  return run(e, 1, x, x_dtype, T, H, W, slice_frames, 0, latent, workspace, workspace_bytes, stream);
}

extern "C" int svr2_vae_decode(svr2_t* e, const void* z, int z_dtype, int T, int h, int w, int slice_frames, void* sample,
                               void* workspace, size_t workspace_bytes, void* stream) {
  return run(e, 0, z, z_dtype, T, h, w, slice_frames, 4 * T - 3, sample, workspace, workspace_bytes, stream);
}

extern "C" int svr2_vae_decode_frames(svr2_t* e, const void* z, int z_dtype, int T, int h, int w, int slice_frames, int frames,
                                      void* sample, void* workspace, size_t workspace_bytes, void* stream) {
  return run(e, 0, z, z_dtype, T, h, w, slice_frames, frames, sample, workspace, workspace_bytes, stream);
}

// Spatially tiled passes (see svr2.h): the same arguments as the un-tiled ones plus the tile plan's four settings
extern "C" size_t svr2_vae_tiled_workspace_bytes(svr2_t* e, int direction, int T, int H, int W, int tile_h, int tile_w,
                                                 int overlap_h, int overlap_w, int slice_frames, int frames) {
  const char* what = "svr2_vae_tiled_workspace_bytes";
  if (check_args(e, what, T, H, W, direction == 0 ? 8 : 1) || check_tiles(e, what, tile_h, tile_w, overlap_h, overlap_w) ||
      (direction != 0 && check_frames(e, what, T, frames)))
    return 0;
  const TilePlan p = tile_plan(direction == 0, H, W, tile_h, tile_w, overlap_h, overlap_w);
  return plan_bytes(e, direction == 0, T, H, W, slice_frames, frames, &p);
}

extern "C" int svr2_vae_encode_tiled(svr2_t* e, const void* x, int x_dtype, int T, int H, int W, int tile_h, int tile_w,
                                     int overlap_h, int overlap_w, int slice_frames, void* latent, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  if (int rc = check_tiles(e, "svr2_vae_encode_tiled", tile_h, tile_w, overlap_h, overlap_w)) return rc;
  const TilePlan p = tile_plan(true, H, W, tile_h, tile_w, overlap_h, overlap_w);
  return run(e, 1, x, x_dtype, T, H, W, slice_frames, 0, latent, workspace, workspace_bytes, stream, &p);
}

extern "C" int svr2_vae_decode_tiled(svr2_t* e, const void* z, int z_dtype, int T, int h, int w, int tile_h, int tile_w,
                                     int overlap_h, int overlap_w, int slice_frames, int frames, void* sample,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_tiles(e, "svr2_vae_decode_tiled", tile_h, tile_w, overlap_h, overlap_w)) return rc;
  const TilePlan p = tile_plan(false, h, w, tile_h, tile_w, overlap_h, overlap_w);
  return run(e, 0, z, z_dtype, T, h, w, slice_frames, frames, sample, workspace, workspace_bytes, stream, &p);
}

// kernels launched by the last svr2_vae_encode / svr2_vae_decode of this handle (bench.py's gpu_launches)
extern "C" int64_t svr2_vae_last_launches(svr2_t* e) { return e && e->vae ? e->vae->last_launches : 0; }
