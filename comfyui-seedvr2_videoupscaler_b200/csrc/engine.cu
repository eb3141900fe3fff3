// Handle-based C ABI (SURVEY.md §8(b) "C ABI to export") and the native host runtime behind it: the whole NaDiT
// forward — window / RoPE geometry, workspace plan and the kernel sequence — runs in C++ on a svr2_t handle that owns
// (or borrows) the weights and owns its workspace.  The per-op entry points of this library are the building blocks;
// nothing here touches Python or torch.
//
// Replaces, for b = 1 and the one-step sampler (t == 1000): NaDiT.forward (dit_3b/nadit.py:190-248,
// dit_7b/nadit.py:152-190) with everything below it (mmsr_block.py:84-128, mmattn.py:161-271, attention.py:114-148,
// modulation.py:65-118, normalization.py:88-109, mlp.py:46-62, patch_v1.py:76-127), and the index bookkeeping of
// window.py:28-83, na.py:320-424,583-641, rope.py:130-176.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "engine_internal.h"

namespace svr2 {

// One window layout (regular or shifted) of a clip geometry, device-resident index tables.
struct Layout {
  int n_win = 0, total = 0, max_len = 0, n_txt_rows = 0;
  int32_t *cu_seqlens = nullptr, *row_src = nullptr, *row_rope = nullptr, *out_row_map = nullptr;
  int32_t *tok_dst = nullptr, *tok_rope = nullptr, *txt_rows = nullptr;
};
struct RopeTable {
  float *cos = nullptr, *sin = nullptr;
  int rows = 0;
};
struct Geometry {
  Layout lay[2];
  std::vector<int> table_of_layer;   // layer -> index into tables
  std::vector<RopeTable> tables;
  int nfreq = 0;
  std::vector<void*> allocs;
};

namespace {

struct Box {
  int t0, t1, h0, h1, w0, w1;
};

// make_720Pwindows_bysize / make_shifted_720Pwindows_bysize (dit_3b/window.py:28-83), num_windows = (4,3,3);
// enumeration order w-major, then h, then t.  Python's round() is round-half-even = nearbyint in the default mode.
std::vector<Box> window_boxes(int t, int h, int w, bool shifted) {
  const int rnt = 4, rnh = 3, rnw = 3;
  const double scale = sqrt((45.0 * 80.0) / ((double)h * w));
  const double rh = nearbyint(h * scale), rw = nearbyint(w * scale);
  const int wh = (int)ceil(rh / rnh), ww = (int)ceil(rw / rnw);
  const int wt = (int)ceil((double)(t < 30 ? t : 30) / rnt);
  std::vector<Box> out;
  if (!shifted) {
    const int nt = (t + wt - 1) / wt, nh = (h + wh - 1) / wh, nw = (w + ww - 1) / ww;
    for (int iw = 0; iw < nw; ++iw)
      for (int ih = 0; ih < nh; ++ih)
        for (int it = 0; it < nt; ++it) {
          Box b{it * wt, (it + 1) * wt < t ? (it + 1) * wt : t, ih * wh, (ih + 1) * wh < h ? (ih + 1) * wh : h, iw * ww,
                (iw + 1) * ww < w ? (iw + 1) * ww : w};
          if (b.t1 > b.t0 && b.h1 > b.h0 && b.w1 > b.w0) out.push_back(b);
        }
    return out;
  }
  const double st = wt < t ? 0.5 : 0.0, sh = wh < h ? 0.5 : 0.0, sw = ww < w ? 0.5 : 0.0;
  int nt = (int)ceil((t - st) / wt), nh = (int)ceil((h - sh) / wh), nw = (int)ceil((w - sw) / ww);
  nt = st > 0 ? nt + 1 : 1;
  nh = sh > 0 ? nh + 1 : 1;
  nw = sw > 0 ? nw + 1 : 1;
  auto lo = [](int i, double s, int win) { int v = (int)((i - s) * win); return v > 0 ? v : 0; };
  auto hi = [](int i, double s, int win, int ext) { int v = (int)((i - s + 1) * win); return v < ext ? v : ext; };
  for (int iw = 0; iw < nw; ++iw) {
    const int w0 = lo(iw, sw, ww), w1 = hi(iw, sw, ww, w);
    if (w1 <= w0) continue;
    for (int ih = 0; ih < nh; ++ih) {
      const int h0 = lo(ih, sh, wh), h1 = hi(ih, sh, wh, h);
      if (h1 <= h0) continue;
      for (int it = 0; it < nt; ++it) {
        const int t0 = lo(it, st, wt), t1 = hi(it, st, wt, t);
        if (t1 <= t0) continue;
        out.push_back(Box{t0, t1, h0, h1, w0, w1});
      }
    }
  }
  return out;
}

// value of a RoPE frequency / position in the dtype of the checkpoint's `freqs` buffer (SURVEY.md §8 G4):
// rotary_embedding_torch computes pos.type(freqs.dtype) * freqs and cos / sin in that dtype.
inline float round_to(float x, int dtype) {
  if (dtype == 2) return __half2float(__float2half_rn(x));
  if (dtype == 1) return __bfloat162float(__float2bfloat16_rn(x));
  return x;
}

}  // namespace
}  // namespace svr2

using namespace svr2;


namespace svr2 {
namespace {

template <typename T>
T* upload(Geometry* g, const std::vector<T>& host) {
  void* d = nullptr;
  if (host.empty()) return nullptr;
#ifdef SVR2_HOST_TEST      // geometry unit tests on a box without a GPU: tables stay in host memory
  d = malloc(host.size() * sizeof(T));
  memcpy(d, host.data(), host.size() * sizeof(T));
  g->allocs.push_back(d);
  return reinterpret_cast<T*>(d);
#endif
  if (cudaMalloc(&d, host.size() * sizeof(T)) != cudaSuccess) return nullptr;
  cudaMemcpy(d, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice);
  g->allocs.push_back(d);
  return reinterpret_cast<T*>(d);
}

// build_layout (na.window_idx + repeat_concat_idx, na.py:320-424,583-641; RoPE positions rope.py:172-173,
// dit_7b/rope.py:73-111) for one layout; size_rows: 7B table offset of every distinct window-axis size.
bool build_layout(Geometry* g, Layout& L, int T, int Hp, int Wp, int l, bool shifted, bool is7,
                  std::vector<std::pair<int, int>>& size_rows, int& max_rope_row) {
  const std::vector<Box> boxes = window_boxes(T, Hp, Wp, shifted);
  const int Ltok = T * Hp * Wp;
  auto size_row = [&](int n) -> int {
    for (auto& kv : size_rows)
      if (kv.first == n) return kv.second;
    return -1;
  };
  if (is7) {
    int off = 0;
    for (auto& kv : size_rows) off = off > kv.second + kv.first ? off : kv.second + kv.first;
    for (const Box& b : boxes)
      for (int n : {b.t1 - b.t0, b.h1 - b.h0, b.w1 - b.w0})
        if (size_row(n) < 0) {
          size_rows.push_back({n, off});
          off += n;
        }
  }
  std::vector<int32_t> src, rope, omap, cu(1, 0), tok_dst(Ltok, -1), tok_rope((size_t)Ltok * 3, -1), txt_rows;
  int max_len = 0;
  for (size_t wi = 0; wi < boxes.size(); ++wi) {
    const Box& b = boxes[wi];
    for (int t = b.t0; t < b.t1; ++t)
      for (int h = b.h0; h < b.h1; ++h)
        for (int w = b.w0; w < b.w1; ++w) {
          const int tok = (t * Hp + h) * Wp + w;
          int r0, r1, r2;
          if (!is7) {
            r0 = t - b.t0 + l; r1 = h - b.h0; r2 = w - b.w0;
          } else {
            r0 = t - b.t0 + size_row(b.t1 - b.t0); r1 = h - b.h0 + size_row(b.h1 - b.h0); r2 = w - b.w0 + size_row(b.w1 - b.w0);
          }
          tok_dst[tok] = (int32_t)src.size();
          tok_rope[(size_t)tok * 3 + 0] = r0; tok_rope[(size_t)tok * 3 + 1] = r1; tok_rope[(size_t)tok * 3 + 2] = r2;
          src.push_back(tok);
          rope.push_back(r0); rope.push_back(r1); rope.push_back(r2);
          omap.push_back(tok);
          const int m = r0 > r1 ? (r0 > r2 ? r0 : r2) : (r1 > r2 ? r1 : r2);
          if (m > max_rope_row) max_rope_row = m;
        }
    for (int j = 0; j < l; ++j) {
      txt_rows.push_back((int32_t)src.size());
      src.push_back(-(j + 1));
      const int r = is7 ? -1 : j;
      rope.push_back(r); rope.push_back(r); rope.push_back(r);
      omap.push_back(Ltok + (int)wi * l + j);
      if (r > max_rope_row) max_rope_row = r;
    }
    const int len = (b.t1 - b.t0) * (b.h1 - b.h0) * (b.w1 - b.w0) + l;
    cu.push_back(cu.back() + len);
    if (len > max_len) max_len = len;
  }
  L.n_win = (int)boxes.size();
  L.total = (int)src.size();
  L.max_len = max_len;
  L.n_txt_rows = (int)txt_rows.size();
  L.cu_seqlens = upload(g, cu);
  L.row_src = upload(g, src);
  L.row_rope = upload(g, rope);
  L.out_row_map = upload(g, omap);
  L.tok_dst = upload(g, tok_dst);
  L.tok_rope = upload(g, tok_rope);
  L.txt_rows = upload(g, txt_rows);
  return L.cu_seqlens && L.row_src && L.row_rope && L.out_row_map && L.tok_dst && L.tok_rope && L.txt_rows;
}

// cos / sin tables [rows, nfreq] fp32 from the layer's frequency buffer (host copy), evaluated in the buffer's dtype
bool build_rope_table(Geometry* g, RopeTable& tab, const std::vector<float>& freqs, int fdtype, bool is7, int rows,
                      const std::vector<std::pair<int, int>>& size_rows) {
  const int nf = (int)freqs.size();
  std::vector<float> pos(rows, 0.f);
  if (!is7) {
    for (int p = 0; p < rows; ++p) pos[p] = round_to((float)p, fdtype);
  } else {
    for (auto& kv : size_rows) {       // torch.linspace(-1, 1, n): fp32, symmetric halves
      const int n = kv.first, off = kv.second;
      const float step = n > 1 ? 2.0f / (float)(n - 1) : 0.f;
      for (int i = 0; i < n && off + i < rows; ++i) {
        // torch's CPU linspace evaluates both halves with a fused multiply-add (the centre of an odd-length axis is
        // -2^-24, not 0)
        const float v = i < n / 2 ? fmaf(step, (float)i, -1.0f) : fmaf(-step, (float)(n - 1 - i), 1.0f);
        pos[off + i] = round_to(n > 1 ? v : -1.0f, fdtype);
      }
    }
  }
  std::vector<float> c((size_t)rows * nf), s((size_t)rows * nf);
  for (int p = 0; p < rows; ++p)
    for (int j = 0; j < nf; ++j) {
      const float ang = round_to(pos[p] * freqs[j], fdtype);
      c[(size_t)p * nf + j] = round_to(cosf(ang), fdtype);
      s[(size_t)p * nf + j] = round_to(sinf(ang), fdtype);
    }
  tab.rows = rows;
  tab.cos = upload(g, c);
  tab.sin = upload(g, s);
  return tab.cos && tab.sin;
}

std::vector<float> host_copy_as_float(const Tensor& t) {
  const int64_t n = t.numel();
  std::vector<float> out(n);
  if (t.dtype == 0) {
    cudaMemcpy(out.data(), t.ptr, n * 4, cudaMemcpyDefault);
  } else {
    std::vector<uint16_t> raw(n);
    cudaMemcpy(raw.data(), t.ptr, n * 2, cudaMemcpyDefault);
    for (int64_t i = 0; i < n; ++i) {
      if (t.dtype == 2) {
        __half h;
        memcpy(&h, &raw[i], 2);
        out[i] = __half2float(h);
      } else {
        uint32_t u = (uint32_t)raw[i] << 16;
        memcpy(&out[i], &u, 4);
      }
    }
  }
  return out;
}

Geometry* geometry(svr2_engine* e, int T, int Hp, int Wp, int l) {
  const std::vector<int> key{T, Hp, Wp, l};
  auto it = e->geo.find(key);
  if (it != e->geo.end()) return it->second;
  const bool is7 = e->desc.variant == 1;
  Geometry* g = new Geometry();
  std::vector<std::pair<int, int>> size_rows[2];
  int max_row[2] = {0, 0};
  bool ok = true;
  for (int s = 0; s < 2 && ok; ++s) ok = build_layout(g, g->lay[s], T, Hp, Wp, l, s == 1, is7, size_rows[s], max_row[s]);
  // one table per distinct (layout parity, frequency buffer): layers that share both share the table
  std::vector<std::pair<int, std::vector<float>>> seen;
  std::vector<int> seen_dtype;
  for (int i = 0; i < e->desc.layers && ok; ++i) {
    char name[64];
    snprintf(name, sizeof name, "%d.rope_freqs", i);
    const Tensor* ft = find(e, name);
    if (!ft) { ok = false; break; }
    std::vector<float> fr = host_copy_as_float(*ft);
    g->nfreq = (int)fr.size();
    int idx = -1;
    for (size_t k = 0; k < seen.size(); ++k)
      if (seen[k].first == (i & 1) && seen_dtype[k] == ft->dtype && seen[k].second == fr) idx = (int)k;
    if (idx < 0) {
      RopeTable tab;
      int rows = max_row[i & 1] + 1;
      if (is7)
        for (auto& kv : size_rows[i & 1]) rows = rows > kv.first + kv.second ? rows : kv.first + kv.second;
      ok = build_rope_table(g, tab, fr, ft->dtype, is7, rows, size_rows[i & 1]);
      g->tables.push_back(tab);
      seen.push_back({i & 1, fr});
      seen_dtype.push_back(ft->dtype);
      idx = (int)seen.size() - 1;
    }
    g->table_of_layer.push_back(idx);
  }
  if (!ok) {
    for (void* p : g->allocs) cudaFree(p);
    delete g;
    return nullptr;
  }
  e->geo[key] = g;
  return g;
}

// bytes a tensor of the handle occupies: dense, or whole blocks of a compressed format
size_t tensor_bytes(const Tensor& t) {
  int be = 0, bb = 0;
  if (t.dtype >= 3 && weight_format_size(t.dtype, &be, &bb)) return (size_t)(t.numel() / be) * bb;
  return (size_t)t.numel() * dtype_size(t.dtype);
}

// The staging slot (svr2.h, "compressed matrices"): which matrices of every block are expanded before the block runs,
// where they land in the slot, and the slot's size.  A matrix whose sources are those of an earlier matrix of the same
// block (the 3B layers whose video and text streams share weights) shares its bytes.
bool build_slot_plan(svr2_engine* e, char* err, size_t err_len) {
  e->slot_plan.clear();
  e->slot_bytes = 0;
  if (e->desc.variant == 2) return true;
  e->slot_plan.resize(e->desc.layers > 0 ? e->desc.layers : 0);
  for (int i = 0; i < e->desc.layers; ++i) {
    std::vector<SlotMatrix>& slots = e->slot_plan[i];
    size_t off = 0;
    for (const char* s : {"vid", "txt"})
      for (const char* n : {"qkv.w", "out.w", "mlp_in.w", "mlp_out.w"}) {
        SlotMatrix m;
        m.name = std::to_string(i) + "." + s + "." + n;
        const Tensor* whole = find(e, m.name);
        const Tensor *gate = nullptr, *in = nullptr;
        if (whole && whole->dtype >= 3) {
          if (whole->rank != 2) {
            snprintf(err, err_len, "svr2_load_weights: compressed matrix '%s' must have rank 2", m.name.c_str());
            return false;
          }
          m.cols = whole->shape[1];
          m.parts.push_back({whole->ptr, whole->dtype, whole->shape[0], whole->shape[0], whole->shape[0], 0});
        } else if (!whole && (gate = find(e, m.name + ".gate")) && (in = find(e, m.name + ".in"))) {
          if (gate->dtype < 2 || in->dtype < 2 || gate->rank != 2 || in->rank != 2 || gate->shape[0] != in->shape[0] ||
              gate->shape[1] != in->shape[1] || gate->shape[0] % 128) {
            snprintf(err, err_len, "svr2_load_weights: '%s.gate' / '.in' must be fp16, fp8_e4m3fn or GGML matrices of one "
                     "shape with a multiple of 128 rows", m.name.c_str());
            return false;
          }
          m.cols = gate->shape[1];
          m.parts.push_back({gate->ptr, gate->dtype, gate->shape[0], 128, 256, 0});
          m.parts.push_back({in->ptr, in->dtype, in->shape[0], 128, 256, 128});
        } else {
          continue;
        }
        int64_t rows = 0;
        for (const SlotPart& p : m.parts) {
          int be = 0, bb = 0;
          weight_format_size(p.format, &be, &bb);
          if (p.rows <= 0 || m.cols <= 0 || m.cols % (be > 8 ? be : 8)) {
            snprintf(err, err_len, "svr2_load_weights: compressed matrix '%s' must have a row length that is a multiple "
                     "of its block size and of 8", m.name.c_str());
            return false;
          }
          rows += p.rows;
        }
        for (const SlotMatrix& prev : slots)
          if (prev.parts.size() == m.parts.size() && prev.parts[0].src == m.parts[0].src &&
              prev.parts.back().src == m.parts.back().src) {
            m.off = prev.off;
            m.parts.clear();
            break;
          }
        if (!m.parts.empty()) {
          m.off = off;
          off += align_up((size_t)rows * m.cols * 2);
        }
        slots.push_back(m);
      }
    e->slot_bytes = e->slot_bytes > off ? e->slot_bytes : off;
  }
  return true;
}

// workspace plan of one forward (bump allocation, bytes)
struct Plan {
  size_t xp, x, t, a_v, a_t, qkv_t, qkv_v, q, k, v, o_all, o_t, h_v, h_t, mm, z, zt, v64, slot, total;
};
Plan make_plan(const svr2_model_desc& d, int T, int H, int W, int l, int max_total, int max_rows, bool fuse_qkv,
               size_t slot_bytes) {
  const size_t L = (size_t)T * (H / 2) * (W / 2), dim = d.dim, inner = (size_t)d.heads * 128;
  const size_t hid = d.mlp_kind == 0 ? (size_t)d.mlp_hidden : (size_t)d.mlp_hidden;
  Plan p{};
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes); return o; };
  p.xp = take(L * 192 * 2);
  p.x = take(L * dim * 2);
  p.t = take((size_t)l * dim * 2);
  p.a_v = take(L * dim * 2);
  p.a_t = take((size_t)l * dim * 2);
  p.qkv_t = take((size_t)l * 3 * inner * 2);
  p.qkv_v = fuse_qkv ? 0 : take(L * 3 * inner * 2);
  p.q = take((size_t)max_total * inner * 2);
  p.k = take((size_t)max_total * inner * 2);
  p.v = take((size_t)max_total * inner * 2);
  p.o_all = take((size_t)max_rows * inner * 2);
  p.o_t = take((size_t)l * inner * 2);
  p.h_v = take(L * dim * 2);
  p.h_t = take((size_t)l * dim * 2);
  p.mm = take(L * dim * 2);
  p.z = take(L * hid * 2);
  p.zt = take((size_t)l * hid * 2);
  p.v64 = take(L * (size_t)d.out_ch * 4 * 2);
  p.slot = take(slot_bytes);       // 0 bytes when every matrix is resident bf16: the plan is the same as without it
  p.total = off;
  return p;
}

bool fuse_qkv_ok(svr2_engine* e, int nfreq) { return (e->desc.heads % 2 == 0) && (nfreq == 21 || nfreq == 10); }

}  // namespace
}  // namespace svr2

// ------------------------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------------------------
extern "C" int svr2_create(svr2_t** out, int device, const svr2_model_desc* desc) {
  if (!out || !desc) return set_error(SVR2_ERR_ARG, "svr2_create: null argument");
  if (desc->variant < 0 || desc->variant > 2)
    return set_error(SVR2_ERR_ARG, "svr2_create: variant 0 (NaDiT 3B), 1 (NaDiT 7B) or 2 (video VAE)");
  if (desc->variant != 2 && (desc->heads <= 0 || desc->dim != desc->heads * 128))
    return set_error(SVR2_ERR_ARG, "svr2_create: dim must equal heads * 128 (head_dim 128)");
  int cur = 0;
  cudaGetDevice(&cur);
  if (cudaSetDevice(device) != cudaSuccess) return set_error(SVR2_ERR_CUDA, "svr2_create: cudaSetDevice failed");
  int sm = 0, maj = 0, mnr = 0;
  int rc = svr2_device_check(&sm, &maj, &mnr);
  cudaSetDevice(cur);
  if (rc) return rc;
  svr2_engine* e = new svr2_engine();
  e->device = device;
  e->desc = *desc;
  *out = e;
  return SVR2_OK;
}

extern "C" void svr2_destroy(svr2_t* e) {
  if (!e) return;
  for (auto& kv : e->w)
    if (kv.second.owned) cudaFree(kv.second.ptr);
  for (auto& kv : e->geo) {
    for (void* p : kv.second->allocs) cudaFree(p);
    delete kv.second;
  }
  if (e->workspace) cudaFree(e->workspace);
  for (void* p : e->retired_workspaces) cudaFree(p);
  vae_state_destroy(e);
  delete e;
}

extern "C" const char* svr2_engine_last_error(svr2_t* e) { return e ? e->err : svr2_last_error(); }

// Tensors in the ENGINE layout (the names / shapes `B200NaDiT` registers: K-major bf16 matrices, SwiGLU gate/in rows
// interleaved per 128, folded AdaSingle fp32 vectors, per-layer "<i>.rope_freqs" in the checkpoint dtype).
// copy != 0: the engine allocates device memory and copies (host or device source) — the caller keeps ownership of the
// source; copy == 0: the engine borrows a device pointer that must outlive the handle (nn.Module buffers).
extern "C" int svr2_load_weights(svr2_t* e, const svr2_tensor_desc* tensors, size_t n, int copy) {
  if (!e || (!tensors && n)) return set_error(SVR2_ERR_ARG, "svr2_load_weights: null argument");
  int cur = 0;
  cudaGetDevice(&cur);
  cudaSetDevice(e->device);
  int rc = SVR2_OK;
  for (size_t i = 0; i < n && rc == SVR2_OK; ++i) {
    const svr2_tensor_desc& d = tensors[i];
    int be = 0, bb = 0;
    if (!d.name || !d.data || d.rank < 1 || d.rank > 5 || d.dtype < 0 ||
        (d.dtype > 2 && !weight_format_size(d.dtype, &be, &bb))) {
      rc = fail(e, SVR2_ERR_ARG, "svr2_load_weights: bad tensor descriptor");
      break;
    }
    Tensor t;
    t.dtype = d.dtype;
    t.rank = d.rank;
    for (int k = 0; k < d.rank; ++k) t.shape[k] = d.shape[k];
    auto old = e->w.find(d.name);
    if (old != e->w.end() && old->second.owned) cudaFree(old->second.ptr);
    if (copy) {
      const size_t bytes = tensor_bytes(t);
      if (cudaMalloc(&t.ptr, bytes ? bytes : 1) != cudaSuccess ||
          cudaMemcpy(t.ptr, d.data, bytes, cudaMemcpyDefault) != cudaSuccess) {
        rc = fail(e, SVR2_ERR_CUDA, "svr2_load_weights: allocation / copy failed");
        break;
      }
      t.owned = true;
    } else {
      t.ptr = const_cast<void*>(d.data);
    }
    e->w[d.name] = t;
  }
  // geometry tables depend on the frequency buffers: rebuild lazily
  for (auto& kv : e->geo) {
    for (void* p : kv.second->allocs) cudaFree(p);
    delete kv.second;
  }
  e->geo.clear();
  char msg[256];
  if (rc == SVR2_OK && !build_slot_plan(e, msg, sizeof msg)) rc = fail(e, SVR2_ERR_ARG, msg);
  cudaSetDevice(cur);
  return rc;
}

// bytes of engine-owned workspace one svr2_dit_forward of this geometry uses (allocated / grown on first use)
extern "C" size_t svr2_workspace_bytes(svr2_t* e, int T, int H, int W, int txt_len) {
  if (!e || e->desc.variant == 2 || T <= 0 || H <= 0 || W <= 0 || (H & 1) || (W & 1) || txt_len <= 0) return 0;
  const int Hp = H / 2, Wp = W / 2;
  size_t max_total = 0, max_win = 0;
  for (int s = 0; s < 2; ++s) {
    const std::vector<Box> b = window_boxes(T, Hp, Wp, s == 1);
    size_t tot = (size_t)T * Hp * Wp + b.size() * (size_t)txt_len;
    max_total = max_total > tot ? max_total : tot;
    max_win = max_win > b.size() ? max_win : b.size();
  }
  const size_t max_rows = (size_t)T * Hp * Wp + max_win * txt_len;
  const int nfreq = e->desc.variant == 1 ? 10 : 21;
  return make_plan(e->desc, T, H, W, txt_len, (int)max_total, (int)max_rows, fuse_qkv_ok(e, nfreq), e->slot_bytes).total;
}

// The tables svr2_dit_forward reads for one layer, built (on first use) by the same geometry() call
extern "C" int svr2_dit_geometry(svr2_t* e, int T, int H, int W, int txt_len, int layer, svr2_dit_geometry_desc* out) {
  if (!e || !out) return set_error(SVR2_ERR_ARG, "svr2_dit_geometry: null argument");
  if (T <= 0 || H <= 0 || W <= 0 || (H & 1) || (W & 1) || txt_len <= 0)
    return fail(e, SVR2_ERR_ARG, "svr2_dit_geometry: T, H, W > 0, H and W even, txt_len > 0");
  int cur = 0;
  cudaGetDevice(&cur);
  if (cur != e->device) return fail(e, SVR2_ERR_ARG, "svr2_dit_geometry: the handle's device is not the current device");
  if (e->desc.variant == 2) return fail(e, SVR2_ERR_ARG, "svr2_dit_geometry: the handle was created as a VAE (variant 2)");
  if (layer < 0 || layer >= e->desc.layers) return fail(e, SVR2_ERR_ARG, "svr2_dit_geometry: layer outside [0, layers)");
  const Geometry* g = geometry(e, T, H / 2, W / 2, txt_len);
  if (!g) return fail(e, SVR2_ERR_ARG, "svr2_dit_geometry: geometry tables could not be built (missing '<i>.rope_freqs'?)");
  const Layout& lay = g->lay[layer & 1];
  const RopeTable& tab = g->tables[g->table_of_layer[layer]];
  *out = svr2_dit_geometry_desc{lay.n_win, lay.total, lay.max_len, lay.n_txt_rows, g->nfreq, tab.rows,
                                fuse_qkv_ok(e, g->nfreq) ? 1 : 0, lay.cu_seqlens, lay.row_src, lay.row_rope,
                                lay.out_row_map, lay.tok_dst, lay.tok_rope, lay.txt_rows, tab.cos, tab.sin};
  return SVR2_OK;
}

// One NaDiT forward: vid [T*H*W, in_ch] bf16 (latent pixels, channels last), txt [txt_len, txt_in_dim] bf16 ->
// out [T*H*W, out_ch] bf16 (= NaDiTOutput.vid_sample).  Stream-ordered; the first call for a geometry builds and
// uploads its index tables (synchronous copies) and may grow the workspace (cudaMalloc) — warm up before a graph capture.
static int dit_forward_impl(svr2_t* e, const void* vid, const void* txt, int T, int H, int W, int txt_len, void* out,
                            void* ext_ws, size_t ext_ws_bytes, void* stream);

extern "C" int svr2_dit_forward(svr2_t* e, const void* vid, const void* txt, int T, int H, int W, int txt_len, void* out,
                                void* stream) {
  return dit_forward_impl(e, vid, txt, T, H, W, txt_len, out, nullptr, 0, stream);
}

// Same forward in a CALLER-provided workspace of at least svr2_workspace_bytes(...) bytes (256-byte aligned): nothing is
// allocated or retained by the engine, so a host that pools device memory (PyTorch's caching allocator, a CUDA-graph
// capture pool) gets the bytes back for the next phase — at 550 800 tokens (65-frame 4K clip) that is 35 GB.
extern "C" int svr2_dit_forward_ws(svr2_t* e, const void* vid, const void* txt, int T, int H, int W, int txt_len,
                                   void* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (!workspace) return set_error(SVR2_ERR_ARG, "svr2_dit_forward_ws: workspace must not be NULL");
  return dit_forward_impl(e, vid, txt, T, H, W, txt_len, out, workspace, workspace_bytes, stream);
}

static int dit_forward_impl(svr2_t* e, const void* vid, const void* txt, int T, int H, int W, int txt_len, void* out,
                            void* ext_ws, size_t ext_ws_bytes, void* stream) {
  if (!e || !vid || !txt || !out) return set_error(SVR2_ERR_ARG, "svr2_dit_forward: null argument");
  if (T <= 0 || H <= 0 || W <= 0 || (H & 1) || (W & 1) || txt_len <= 0)
    return fail(e, SVR2_ERR_ARG, "svr2_dit_forward: T, H, W > 0, H and W even, txt_len > 0");
  int cur = 0;
  cudaGetDevice(&cur);
  if (cur != e->device) return fail(e, SVR2_ERR_ARG, "svr2_dit_forward: the handle's device is not the current device");
  const svr2_model_desc& D = e->desc;
  if (D.variant == 2) return fail(e, SVR2_ERR_ARG, "svr2_dit_forward: the handle was created as a VAE (variant 2)");
  const int Hp = H / 2, Wp = W / 2, l = txt_len, d = D.dim, heads = D.heads, inner = heads * 128;
  const int L = T * Hp * Wp;
  Geometry* g = geometry(e, T, Hp, Wp, l);
  if (!g) return fail(e, SVR2_ERR_ARG, "svr2_dit_forward: geometry tables could not be built (missing '<i>.rope_freqs'?)");
  const bool fuse = fuse_qkv_ok(e, g->nfreq);
  const int max_total = g->lay[0].total > g->lay[1].total ? g->lay[0].total : g->lay[1].total;
  const int max_win = g->lay[0].n_win > g->lay[1].n_win ? g->lay[0].n_win : g->lay[1].n_win;
  const Plan P = make_plan(D, T, H, W, l, max_total, L + max_win * l, fuse, e->slot_bytes);
  if (ext_ws) {
    if (ext_ws_bytes < P.total) return fail(e, SVR2_ERR_ARG, "svr2_dit_forward_ws: workspace smaller than svr2_workspace_bytes()");
  } else if (P.total > e->workspace_bytes) {
    // grow: the outgrown block is kept until svr2_destroy — work already queued, or a captured CUDA graph of a smaller
    // geometry, may still use it (freeing it would hand its address to someone else)
    if (e->workspace) e->retired_workspaces.push_back(e->workspace);
    e->workspace = nullptr;
    e->workspace_bytes = 0;
    if (cudaMalloc(&e->workspace, P.total) != cudaSuccess) return fail(e, SVR2_ERR_CUDA, "svr2_dit_forward: workspace allocation failed");
    e->workspace_bytes = P.total;
  }
  char* ws = reinterpret_cast<char*>(ext_ws ? ext_ws : e->workspace);
  auto B = [&](size_t off) { return reinterpret_cast<void*>(ws + off); };
  char name[96];
  auto Wt = [&](const char* fmt, int i, const char* s, const char* n) -> const void* {
    if (i >= 0) snprintf(name, sizeof name, fmt, i, s, n); else snprintf(name, sizeof name, "%s", n);
    const Tensor* t = find(e, name);
    return t ? t->ptr : nullptr;
  };
  auto need = [&](const void* p) { return p != nullptr; };
  int rc;
#define CK(call) do { rc = (call); if (rc) { snprintf(e->err, sizeof e->err, "%s", svr2_last_error()); return rc; } } while (0)
#define NEED(ptr, what) do { if (!need(ptr)) { snprintf(e->err, sizeof e->err, "svr2_dit_forward: weight '%s' not loaded", what); return set_error(SVR2_ERR_ARG, e->err); } } while (0)
  const int EPI_B = SVR2_EPI_BIAS, EPI_G = SVR2_EPI_GATE, EPI_R = SVR2_EPI_RESIDUAL;
  // ---- stem (nadit.py:199-218)
  const void *w_in = Wt("", -1, "", "vid_in.w"), *b_in = Wt("", -1, "", "vid_in.b");
  const void *w_ti = Wt("", -1, "", "txt_in.w"), *b_ti = Wt("", -1, "", "txt_in.b");
  NEED(w_in, "vid_in.w"); NEED(b_in, "vid_in.b"); NEED(w_ti, "txt_in.w"); NEED(b_ti, "txt_in.b");
  CK(svr2_patchify_bf16(vid, B(P.xp), T, H, W, D.in_ch, 192, stream));
  CK(svr2_linear_bf16(B(P.xp), 192, w_in, 192, L, d, 192, EPI_B, b_in, nullptr, nullptr, B(P.x), d, 1.f, stream));
  CK(svr2_linear_bf16(txt, D.txt_in_dim, w_ti, D.txt_in_dim, l, d, D.txt_in_dim, EPI_B, b_ti, nullptr, nullptr, B(P.t), d, 1.f, stream));
  void *x = B(P.x), *t = B(P.t), *h_v = B(P.h_v), *h_t = B(P.h_t);
  const int hid = D.mlp_hidden;
  for (int i = 0; i < D.layers; ++i) {
    const bool last = D.last_vid_only && i == D.layers - 1;
    const Layout& lay = g->lay[i & 1];
    const RopeTable& tab = g->tables[g->table_of_layer[i]];
    auto Wl = [&](const char* s, const char* n) { return Wt("%d.%s.%s", i, s, n); };
    // compressed matrices of this block: expanded to bf16 into the slot now (stream order puts this after the previous
    // block's GEMMs, which read the same slot); Wm finds a block matrix there, or resident among the weights
    static const std::vector<SlotMatrix> none;
    const std::vector<SlotMatrix>& slots = (size_t)i < e->slot_plan.size() ? e->slot_plan[i] : none;
    char* slot = ws + P.slot;
    for (const SlotMatrix& m : slots)
      for (const SlotPart& p : m.parts)
        CK(svr2_weight_expand_bf16(p.format, p.src, p.rows, m.cols, slot + m.off, p.group, p.stride, p.offset, stream));
    auto Wm = [&](const char* s, const char* n) -> const void* {
      snprintf(name, sizeof name, "%d.%s.%s", i, s, n);
      for (const SlotMatrix& m : slots)
        if (m.name == name) return slot + m.off;
      const Tensor* t = find(e, name);
      return t ? t->ptr : nullptr;
    };
    // ---- attention branch (mmsr_block.py:107-114)
    const void *sc_v = Wl("vid", "attn_scale"), *sh_v = Wl("vid", "attn_shift");
    const void *sc_t = Wl("txt", "attn_scale"), *sh_t = Wl("txt", "attn_shift");
    NEED(sc_v, "<i>.vid.attn_scale"); NEED(sh_v, "<i>.vid.attn_shift"); NEED(sc_t, "<i>.txt.attn_scale"); NEED(sh_t, "<i>.txt.attn_shift");
    CK(svr2_rmsnorm_ada_bf16(x, B(P.a_v), L, d, D.eps, nullptr, (const float*)sc_v, (const float*)sh_v, 0, stream));
    CK(svr2_rmsnorm_ada_bf16(t, B(P.a_t), l, d, D.eps, nullptr, (const float*)sc_t, (const float*)sh_t, 0, stream));
    const void *wqkv_v = Wm("vid", "qkv.w"), *wqkv_t = Wm("txt", "qkv.w");
    const void *nq_v = Wl("vid", "nq"), *nk_v = Wl("vid", "nk"), *nq_t = Wl("txt", "nq"), *nk_t = Wl("txt", "nk");
    const void* nqk_v = Wl("vid", "nqk");
    NEED(wqkv_v, "<i>.vid.qkv.w"); NEED(wqkv_t, "<i>.txt.qkv.w"); NEED(nq_v, "<i>.vid.nq"); NEED(nk_v, "<i>.vid.nk");
    NEED(nq_t, "<i>.txt.nq"); NEED(nk_t, "<i>.txt.nk"); NEED(nqk_v, "<i>.vid.nqk");
    CK(svr2_linear_bf16(B(P.a_t), d, wqkv_t, d, l, 3 * inner, d, 0, nullptr, nullptr, nullptr, B(P.qkv_t), 3 * inner, 1.f, stream));
    if (fuse) {
      CK(svr2_linear_qkv_rope_bf16(B(P.a_v), d, wqkv_v, d, L, heads, d, lay.tok_dst, lay.tok_rope, tab.cos, tab.sin, g->nfreq,
                                   (const float*)nqk_v, D.eps, B(P.q), B(P.k), B(P.v), stream));
      CK(svr2_qk_norm_rope_rows_bf16(nullptr, B(P.qkv_t), lay.row_src, lay.row_rope, tab.cos, tab.sin, g->nfreq,
                                     (const float*)nq_v, (const float*)nk_v, (const float*)nq_t, (const float*)nk_t, D.eps,
                                     lay.txt_rows, lay.n_txt_rows, heads, B(P.q), B(P.k), B(P.v), stream));
    } else {
      CK(svr2_linear_bf16(B(P.a_v), d, wqkv_v, d, L, 3 * inner, d, 0, nullptr, nullptr, nullptr, B(P.qkv_v), 3 * inner, 1.f, stream));
      CK(svr2_qk_norm_rope_window_bf16(B(P.qkv_v), B(P.qkv_t), lay.row_src, lay.row_rope, tab.cos, tab.sin, g->nfreq,
                                       (const float*)nq_v, (const float*)nk_v, (const float*)nq_t, (const float*)nk_t, D.eps,
                                       lay.total, heads, B(P.q), B(P.k), B(P.v), stream));
    }
    CK(svr2_attn_varlen_bf16(B(P.q), B(P.k), B(P.v), B(P.o_all), lay.cu_seqlens, lay.n_win, lay.total, heads, lay.max_len,
                             lay.out_row_map, stream));
    char* o_txt = reinterpret_cast<char*>(B(P.o_all)) + (size_t)L * inner * 2;
    CK(svr2_txt_window_mean_bf16(o_txt, B(P.o_t), lay.n_win, l, inner, stream));
    const void *wo_v = Wm("vid", "out.w"), *bo_v = Wl("vid", "out.b"), *wo_t = Wm("txt", "out.w"), *bo_t = Wl("txt", "out.b");
    const void *ga_v = Wl("vid", "attn_gate"), *ga_t = last ? nullptr : Wl("txt", "attn_gate");
    NEED(wo_v, "<i>.vid.out.w"); NEED(bo_v, "<i>.vid.out.b"); NEED(wo_t, "<i>.txt.out.w"); NEED(bo_t, "<i>.txt.out.b"); NEED(ga_v, "<i>.vid.attn_gate");
    if (!last) NEED(ga_t, "<i>.txt.attn_gate");
    CK(svr2_linear_bf16(B(P.o_all), inner, wo_v, inner, L, d, inner, EPI_B | EPI_G | EPI_R, bo_v, (const float*)ga_v, x, h_v, d, 1.f, stream));
    CK(svr2_linear_bf16(B(P.o_t), inner, wo_t, inner, l, d, inner, EPI_B | (last ? 0 : EPI_G) | EPI_R, bo_t, (const float*)ga_t, t, h_t, d, 1.f, stream));
    // ---- MLP branch (mmsr_block.py:116-126); the outputs land in the buffers that held this layer's inputs
    auto mlp = [&](const char* s, void* hh, void* yy, int rows, void* zbuf) -> int {
      const void *msc = Wl(s, "mlp_scale"), *msh = Wl(s, "mlp_shift"), *mg = Wl(s, "mlp_gate");
      const void *w1 = Wm(s, "mlp_in.w"), *w2 = Wm(s, "mlp_out.w");
      if (!msc || !msh || !mg || !w1 || !w2) { snprintf(e->err, sizeof e->err, "svr2_dit_forward: MLP weights of layer %d (%s) not loaded", i, s); return set_error(SVR2_ERR_ARG, e->err); }
      int r = svr2_rmsnorm_ada_bf16(hh, B(P.mm), rows, d, D.eps, nullptr, (const float*)msc, (const float*)msh, 1, stream);
      if (r) return r;
      if (D.mlp_kind == 0) {     // SwiGLU: interleaved [gate ; in] rows, N = 2 * hidden, output hidden
        r = svr2_linear_bf16(B(P.mm), d, w1, d, rows, 2 * hid, d, SVR2_EPI_SWIGLU, nullptr, nullptr, nullptr, zbuf, hid, 1.f, stream);
        if (r) return r;
        return svr2_linear_bf16(zbuf, hid, w2, hid, rows, d, hid, EPI_G | EPI_R, nullptr, (const float*)mg, hh, yy, d, 1.f, stream);
      }
      const void *b1 = Wl(s, "mlp_in.b"), *b2 = Wl(s, "mlp_out.b");
      if (!b1 || !b2) { snprintf(e->err, sizeof e->err, "svr2_dit_forward: MLP biases of layer %d not loaded", i); return set_error(SVR2_ERR_ARG, e->err); }
      r = svr2_linear_bf16(B(P.mm), d, w1, d, rows, hid, d, EPI_B | SVR2_EPI_GELU, b1, nullptr, nullptr, zbuf, hid, 1.f, stream);
      if (r) return r;
      return svr2_linear_bf16(zbuf, hid, w2, hid, rows, d, hid, EPI_B | EPI_G | EPI_R, b2, (const float*)mg, hh, yy, d, 1.f, stream);
    };
    CK(mlp("vid", h_v, x, L, B(P.z)));
    if (last) {                 // vid_only: the text stream's output is unused downstream
      void* tmp = t; t = h_t; h_t = tmp;
    } else {
      CK(mlp("txt", h_t, t, l, B(P.zt)));
    }
  }
  // ---- head (nadit.py:234-247)
  const void* xo = x;
  if (D.out_norm) {
    const void *osc = Wt("", -1, "", "out_scale"), *osh = Wt("", -1, "", "out_shift"), *ow = Wt("", -1, "", "out_weight");
    NEED(osc, "out_scale"); NEED(osh, "out_shift"); NEED(ow, "out_weight");
    CK(svr2_rmsnorm_ada_bf16(x, B(P.a_v), L, d, D.eps, (const float*)ow, (const float*)osc, (const float*)osh, 0, stream));
    xo = B(P.a_v);
  }
  const void *w_out = Wt("", -1, "", "vid_out.w"), *b_out = Wt("", -1, "", "vid_out.b");
  NEED(w_out, "vid_out.w"); NEED(b_out, "vid_out.b");
  const int n64 = D.out_ch * 4;
  CK(svr2_linear_bf16(xo, d, w_out, d, L, n64, d, EPI_B, b_out, nullptr, nullptr, B(P.v64), n64, 1.f, stream));
  CK(svr2_unpatchify_bf16(B(P.v64), n64, out, T, H, W, D.out_ch, stream));
#undef CK
#undef NEED
  return SVR2_OK;
}
