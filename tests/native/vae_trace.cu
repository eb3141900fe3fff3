// Test harness (CPU): the native VAE runtime (csrc/vae_engine.cu) compiled with SVR2_HOST_TEST — host memory as the
// workspace, every kernel entry point replaced by a stub that prints its name and scalar arguments (pointers as p0 / p1
// = NULL / not NULL).  The tests compare the trace with the op sequence of the Python module (vae.py) on the same clip,
// and the dry-run workspace size with the extent the real run touches.
// usage: vae_trace fuzz
//        vae_trace <weights manifest> enc|dec T H W slice_frames                  svr2_vae_encode / svr2_vae_decode
//        vae_trace <weights manifest> frames T h w slice_frames frames [plan]     svr2_vae_decode_frames
//        vae_trace <weights manifest> tiled enc|dec T H W tile_h tile_w overlap_h overlap_w slice_frames frames [plan]
//                                                                                 svr2_vae_encode_tiled / _decode_tiled
//   A pass prints the trace, then "# workspace <bytes> touched_max_offset <bytes> launches <n>" ("plan": only
//   "# workspace <bytes>").  A refused plan exits 3: "plan failed: <message>" on stderr for enc|dec, "refused: <message>"
//   for tiled, and for frames "refused: <query's message> | <decode's message>" when the decode refuses as well.
//   A seam line ends with "| <offset of the tile's corner in the result, elements> <channel stride> <frame stride>
//   <row stride> <count p0/p1> <ramp lengths> <edges>"; a windowed conversion with "| <channel, frame, row strides>
//   <offset of the window in the input, elements>".
#define SVR2_HOST_TEST 1
#include "../../comfyui-seedvr2_videoupscaler_b200/csrc/vae_engine.cu"
#include <stdarg.h>
#include <stdlib.h>

#include <fstream>
#include <sstream>

namespace svr2 {
static char g_msg[512];
int set_error(int code, const char* m) { snprintf(g_msg, sizeof g_msg, "%s", m ? m : ""); return code; }
}
static char* g_lo = nullptr;
static char* g_hi = nullptr;       // workspace bounds: every non-NULL pointer into it must stay inside
static size_t g_touch = 0;
static const char* g_in = nullptr;  // a tiled pass's input and result (bf16): windows and seams print offsets into them
static const char* g_out = nullptr;
static const char* P_(const void* p) {
  if (p && (const char*)p >= g_lo && (const char*)p < g_hi) {
    const size_t off = (const char*)p - g_lo;
    if (off > g_touch) g_touch = off;
  }
  return p ? "p1" : "p0";
}
extern "C" {
const char* svr2_last_error(void) { return svr2::g_msg; }
int svr2_groupnorm_from_stats_bf16(const void* x, void* y, int frames, int hw, int C, const void* gamma, const void* beta,
                                   float eps, int silu, int out_t_pad, int out_dup_head, const void* stat_partial,
                                   int stat_slots, void* coef_scratch, void* stream) {
  printf("svr2_groupnorm_from_stats_bf16 %s %s %d %d %d %s %s %.5g %d %d %d %s %d %s %s\n", P_(x), P_(y), frames, hw, C, P_(gamma),
         P_(beta), eps, silu, out_t_pad, out_dup_head, P_(stat_partial), stat_slots, P_(coef_scratch), P_(stream));
  return 0;
}
int svr2_groupnorm_bf16(const void* x, void* y, int frames, int hw, int C, const void* gamma, const void* beta, float eps,
                        int silu, int out_t_pad, int out_dup_head, double* scratch, int64_t scratch_bytes, void* stream) {
  printf("svr2_groupnorm_bf16 %s %s %d %d %d %s %s %.5g %d %d %d %s %lld %s\n", P_(x), P_(y), frames, hw, C, P_(gamma), P_(beta), eps,
         silu, out_t_pad, out_dup_head, P_(scratch), (long long)scratch_bytes, P_(stream));
  return 0;
}
int svr2_conv3d_bf16(const void* x, int T_in_total, int H, int W, int Cin, const void* w, int Cout, int kt, int kh, int kw,
                     int stride_t, int stride_hw, int pad_hw, int T_out, int epi_flags, const void* bias, const void* residual,
                     void* y, int out_t_pad, int out_dup_head, int ldc, void* stream) {
  printf("svr2_conv3d_bf16 %s %d %d %d %d %s %d %d %d %d %d %d %d %d %d %s %s %s %d %d %d %s\n", P_(x), T_in_total, H, W, Cin, P_(w),
         Cout, kt, kh, kw, stride_t, stride_hw, pad_hw, T_out, epi_flags, P_(bias), P_(residual), P_(y), out_t_pad, out_dup_head,
         ldc, P_(stream));
  return 0;
}
int svr2_conv3d_stats_bf16(const void* x, int T_in_total, int H, int W, int Cin, const void* w, int Cout, int kt, int kh,
                           int kw, int stride_t, int stride_hw, int pad_hw, int T_out, int epi_flags, const void* bias,
                           const void* residual, void* y, int out_t_pad, int out_dup_head, int ldc, void* stat_partial,
                           int64_t stat_bytes, int* stat_slots, void* stream) {
  printf("svr2_conv3d_stats_bf16 %s %d %d %d %d %s %d %d %d %d %d %d %d %d %d %s %s %s %d %d %d %s %lld %s %s\n", P_(x), T_in_total, H,
         W, Cin, P_(w), Cout, kt, kh, kw, stride_t, stride_hw, pad_hw, T_out, epi_flags, P_(bias), P_(residual), P_(y), out_t_pad,
         out_dup_head, ldc, P_(stat_partial), (long long)stat_bytes, P_(stat_slots), P_(stream));
  *stat_slots = svr2_conv_stat_slots(Cout, stride_hw == 1 ? H : H / 2, stride_hw == 1 ? W : W / 2);
  return 0;
}
int svr2_conv3d_shortcut_stats_bf16(const void* x, int T_in_total, int H, int W, int Cin, const void* w, int Cout, int kt,
                                    int kh, int kw, int T_out, const void* bias, const void* x2, int C2, void* y,
                                    int out_t_pad, int out_dup_head, void* stat_partial, int64_t stat_bytes,
                                    int* stat_slots, void* stream) {
  printf("svr2_conv3d_shortcut_stats_bf16 %s %d %d %d %d %s %d %d %d %d %d %s %s %d %s %d %d %s %lld %s %s\n", P_(x), T_in_total, H, W,
         Cin, P_(w), Cout, kt, kh, kw, T_out, P_(bias), P_(x2), C2, P_(y), out_t_pad, out_dup_head, P_(stat_partial),
         (long long)stat_bytes, P_(stat_slots), P_(stream));
  *stat_slots = svr2_conv_stat_slots(Cout, H, W);
  return 0;
}
int svr2_upsample_shuffle_bf16(const void* x, int F, int H, int W, int C, const void* w, const void* bias, int temporal,
                               int drop_head, void* y, int out_t_pad, int out_dup_head, void* stream) {
  printf("svr2_upsample_shuffle_bf16 %s %d %d %d %d %s %s %d %d %s %d %d %s\n", P_(x), F, H, W, C, P_(w), P_(bias), temporal, drop_head,
         P_(y), out_t_pad, out_dup_head, P_(stream));
  return 0;
}
int svr2_linear_bf16(const void* a, int64_t lda, const void* w, int64_t ldw, int M, int N, int K, int epi_flags,
                     const void* bias, const float* gate, const void* residual, void* out, int64_t ldc, float out_scale,
                     void* stream) {
  printf("svr2_linear_bf16 %s %lld %s %lld %d %d %d %d %s %s %s %s %lld %.5g %s\n", P_(a), (long long)lda, P_(w), (long long)ldw, M, N, K,
         epi_flags, P_(bias), P_(gate), P_(residual), P_(out), (long long)ldc, out_scale, P_(stream));
  return 0;
}
int svr2_linear_ex_bf16(const void* a, int64_t lda, const void* w, int64_t ldw, int M, int N, int K, int epi_flags,
                        const void* bias, const float* gate, const void* residual, void* out, int64_t ldc, float out_scale,
                        const float* rowscale, void* stat_out, int64_t ld_stat, const int* run_if, void* stream) {
  printf("svr2_linear_ex_bf16 %s %lld %s %lld %d %d %d %d %s %s %s %s %lld %.5g %s %s %lld %s %s\n", P_(a), (long long)lda, P_(w),
         (long long)ldw, M, N, K, epi_flags, P_(bias), P_(gate), P_(residual), P_(out), (long long)ldc, out_scale, P_(rowscale),
         P_(stat_out), (long long)ld_stat, P_(run_if), P_(stream));
  return 0;
}
int svr2_rowstat_max(const void* partial, int slots, int64_t ld, float* mhat, int rows, int* flag_reset, void* stream) {
  printf("svr2_rowstat_max %s %d %lld %s %d %s %s\n", P_(partial), slots, (long long)ld, P_(mhat), rows, P_(flag_reset), P_(stream));
  return 0;
}
int svr2_pexp_stat_combine(const void* partial, int slots, int64_t ld, const float* mhat, float* rowscale, int rows, int* flag,
                           void* stream) {
  printf("svr2_pexp_stat_combine %s %d %lld %s %s %d %s %s\n", P_(partial), slots, (long long)ld, P_(mhat), P_(rowscale), rows, P_(flag),
         P_(stream));
  return 0;
}
int svr2_rowstat_combine(const void* partial, int slots, int64_t ld, float* lse, int rows, void* stream) {
  printf("svr2_rowstat_combine %s %d %lld %s %d %s\n", P_(partial), slots, (long long)ld, P_(lse), rows, P_(stream));
  return 0;
}
int svr2_transpose_bf16(const void* in, int64_t ld_in, void* out, int64_t ld_out, int rows, int cols, void* stream) {
  printf("svr2_transpose_bf16 %s %lld %s %lld %d %d %s\n", P_(in), (long long)ld_in, P_(out), (long long)ld_out, rows, cols, P_(stream));
  return 0;
}
int svr2_im2col3_bf16(const void* x, int T, int H, int W, int C, int ld_in, void* out, int ld_out, void* stream) {
  printf("svr2_im2col3_bf16 %s %d %d %d %d %d %s %d %s\n", P_(x), T, H, W, C, ld_in, P_(out), ld_out, P_(stream));
  return 0;
}
}
namespace svr2 {
// the channel stride is the one argument the public entry points (what vae.py calls) do not carry: printed last, after '|'
int ncdhw_to_ndhwc_strided(const void* in, int in_dtype, int C, int T, int H, int W, int64_t cs, void* out, int C_pad,
                           int out_t_pad, float div, void* stream) {
  printf("svr2_ncdhw_to_ndhwc_bf16 %s %d %d %d %d %d %s %d %d %.5g %s | %lld\n", P_(in), in_dtype, C, T, H, W, P_(out), C_pad, out_t_pad,
         div, P_(stream), (long long)cs);
  return 0;
}
int ndhwc_to_ncdhw_strided(const void* in, int ld_in, int C, int T, int H, int W, void* out, int out_dtype, int64_t cs,
                           void* stream) {
  printf("svr2_ndhwc_to_ncdhw %s %d %d %d %d %d %s %d %s | %lld\n", P_(in), ld_in, C, T, H, W, P_(out), out_dtype, P_(stream), (long long)cs);
  return 0;
}
int conv_tap_gather_strided(const float* z, int64_t ldz, int co_n, const void* bias, int T, int H, int W, void* out,
                            int out_dtype, int64_t cs, void* stream) {
  printf("svr2_conv_tap_gather %s %lld %d %s %d %d %d %s %d %s | %lld\n", P_(z), (long long)ldz, co_n, P_(bias), T, H, W, P_(out), out_dtype,
         P_(stream), (long long)cs);
  return 0;
}
// the tiled passes' own launches: the windowed input conversion, the seam variants of the final kernels, the ramp tables
int ncdhw_to_ndhwc_window(const void* in, int in_dtype, int C, int T, int H, int W, int64_t cs, int64_t fs, int rs, void* out,
                          int C_pad, int out_t_pad, float div, void* stream) {
  printf("svr2_ncdhw_to_ndhwc_window %s %d %d %d %d %d %s %d %d %.5g %s | %lld %lld %d %lld\n", P_(in), in_dtype, C, T, H, W, P_(out),
         C_pad, out_t_pad, div, P_(stream), (long long)cs, (long long)fs, rs, (long long)(((const char*)in - g_in) / 2));
  return 0;
}
static void seam_suffix(const Seam& s) {
  printf(" | %lld %lld %lld %d %s %d %d %d\n", (long long)(((const char*)s.result - g_out) / 2), (long long)s.cs, (long long)s.fs,
         s.rs, P_(s.count), s.len_h, s.len_w, s.edges);
  P_(s.ramp_h);
  P_(s.ramp_w);
}
int conv_tap_gather_seam(const float* z, int64_t ldz, int co_n, const void* bias, int T, int H, int W, const Seam& s, void* stream) {
  printf("svr2_conv_tap_gather_seam %s %lld %d %s %d %d %d %s", P_(z), (long long)ldz, co_n, P_(bias), T, H, W, P_(stream));
  seam_suffix(s);
  return 0;
}
int ndhwc_to_ncdhw_seam(const void* in, int ld_in, int C, int T, int H, int W, const Seam& s, void* stream) {
  printf("svr2_ndhwc_to_ncdhw_seam %s %d %d %d %d %d %s", P_(in), ld_in, C, T, H, W, P_(stream));
  seam_suffix(s);
  return 0;
}
int tile_ramp(void* ramp_h, int len_h, void* ramp_w, int len_w, void* stream) {
  printf("svr2_tile_ramp_bf16 %s %d %s %d %s\n", P_(ramp_h), len_h, P_(ramp_w), len_w, P_(stream));
  return 0;
}
}  // namespace svr2
extern "C" int svr2_tile_normalize_bf16(void* result, const void* count, int planes, int64_t hw, void* stream) {
  printf("svr2_tile_normalize_bf16 %s %s %d %lld %s\n", result ? "p1" : "p0", P_(count), planes, (long long)hw, P_(stream));
  return 0;
}

// Arena fuzz: a random alloc / release / alloc_top sequence replayed on an unbounded arena (the dry run) and on one capped
// at the dry run's need() must make identical placement decisions, never overlap two live blocks and stay inside the cap.
static int arena_fuzz(unsigned seed, int ops) {
  struct Blk { size_t off, bytes; };
  auto rnd = [&]() { seed = seed * 1664525u + 1013904223u; return seed >> 8; };
  std::vector<int> script;           // >0: alloc of that many bytes; 0: release a pseudo-random live block; <0: alloc_top
  std::vector<size_t> pick;
  for (int i = 0; i < ops; ++i) {
    const unsigned r = rnd() % 100;
    if (r < 55) script.push_back(1 + (int)(rnd() % (1 << (4 + rnd() % 18))));
    else if (r < 95) script.push_back(0);
    else script.push_back(-(1 + (int)(rnd() % 100000)));
    pick.push_back(rnd());
  }
  auto replay = [&](Arena& A, std::vector<size_t>* trace) -> bool {
    std::vector<Blk> live, top;
    for (size_t i = 0; i < script.size(); ++i) {
      const int op = script[i];
      if (op > 0) {
        const size_t off = A.alloc((size_t)op);
        if (off == NONE) return false;
        const size_t bytes = align_up((size_t)op);
        for (const Blk& b : live)
          if (off < b.off + b.bytes && b.off < off + bytes) return false;          // overlap with a live block
        if (off + bytes > A.cap - A.top_used) return false;
        live.push_back({off, bytes});
        trace->push_back(off);
      } else if (op == 0) {
        if (live.empty()) continue;
        const size_t k = pick[i] % live.size();
        A.release(live[k].off, live[k].bytes);
        live.erase(live.begin() + k);
      } else {
        const size_t off = A.alloc_top((size_t)(-op));
        if (off == NONE) return false;
        trace->push_back(A.top_used);
        for (const Blk& b : live)
          if (b.off + b.bytes > A.cap - A.top_used) return false;                   // the top region ran into a live block
      }
    }
    return true;
  };
  Arena dry(~(size_t)0 / 2);
  std::vector<size_t> t0, t1;
  if (!replay(dry, &t0)) return 1;
  Arena real(dry.need());
  if (!replay(real, &t1)) return 2;
  if (t0 != t1) return 3;
  if (real.need() != dry.need()) return 4;
  return 0;
}

// One traced pass: given its exact plan `need`, prints only that ("plan"), or runs the pass in a host workspace of that size
// with a result of `out_bytes`, checks that a workspace 256 bytes short is refused and prints the summary line.
// pass(ws, ws_bytes, out) calls the entry point under test.
template <class Pass>
static int trace(svr2_engine& eng, size_t need, bool plan_only, size_t out_bytes, Pass pass) {
  if (plan_only) {
    printf("# workspace %zu\n", need);
    return 0;
  }
  std::vector<char> out(out_bytes);
  g_out = out.data();
  void* ws = nullptr;
  if (posix_memalign(&ws, 256, need)) return 4;
  g_lo = (char*)ws;
  g_hi = g_lo + need;
  if (const int rc = pass(ws, need, out.data())) { fprintf(stderr, "run failed (%d): %s\n", rc, eng.err); return 5; }
  const int64_t launches = svr2_vae_last_launches(&eng);
  if (pass(ws, need - 256, out.data()) == 0) return 6;
  printf("# workspace %zu touched_max_offset %zu launches %lld\n", need, g_touch, (long long)launches);
  free(ws);
  vae_state_destroy(&eng);
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 2 && std::string(argv[1]) == "fuzz") {
    for (unsigned seed = 1; seed <= 200; ++seed) {
      const int rc = arena_fuzz(seed, 400);
      if (rc) { fprintf(stderr, "arena fuzz seed %u failed (%d)\n", seed, rc); return 10 + rc; }
    }
    printf("arena fuzz ok\n");
    return 0;
  }
  if (argc < 7) return 2;
  svr2_engine eng;
  eng.desc.variant = 2;
  std::ifstream f(argv[1]);
  std::string line;
  while (std::getline(f, line)) {       // name rank d0 d1 ...
    std::istringstream is(line);
    std::string name;
    Tensor t;
    is >> name >> t.rank;
    for (int i = 0; i < t.rank; ++i) is >> t.shape[i];
    t.ptr = (void*)0x1000;
    eng.w[name] = t;
  }
  const std::string mode = argv[2];
  auto arg = [&](int i) { return atoi(argv[i]); };
  auto plan_only = [&](int i) { return argc > i && std::string(argv[i]) == "plan"; };
  static char in[16];
  g_in = in;
  if (mode == "enc" || mode == "dec") {
    const bool enc = mode == "enc";
    const int T = arg(3), H = arg(4), W = arg(5), slice = arg(6);
    const size_t need = svr2_vae_workspace_bytes(&eng, enc ? 0 : 1, T, H, W, slice);
    if (!need) { fprintf(stderr, "plan failed: %s\n", eng.err); return 3; }
    return trace(eng, need, false, 16, [&](void* ws, size_t bytes, void* out) {
      return enc ? svr2_vae_encode(&eng, in, 1, T, H, W, slice, out, ws, bytes, nullptr)
                 : svr2_vae_decode(&eng, in, 1, T, H, W, slice, out, ws, bytes, nullptr);
    });
  }
  if (mode == "frames" && argc >= 8) {
    const int T = arg(3), h = arg(4), w = arg(5), slice = arg(6), frames = arg(7);
    const size_t need = svr2_vae_decode_frames_workspace_bytes(&eng, T, h, w, slice, frames);
    if (!need) {        // the decode itself must refuse `frames` too
      const std::string msg = eng.err;
      static char small_ws[1 << 12] __attribute__((aligned(256)));
      static char out[16];
      if (svr2_vae_decode_frames(&eng, in, 1, T, h, w, slice, frames, out, small_ws, sizeof small_ws, nullptr) == 0) return 8;
      fprintf(stderr, "refused: %s | %s\n", msg.c_str(), eng.err);
      return 3;
    }
    return trace(eng, need, plan_only(8), 16, [&](void* ws, size_t bytes, void* out) {
      return svr2_vae_decode_frames(&eng, in, 1, T, h, w, slice, frames, out, ws, bytes, nullptr);
    });
  }
  if (mode == "tiled" && argc >= 13) {
    const bool enc = std::string(argv[3]) == "enc";
    const int T = arg(4), H = arg(5), W = arg(6), th = arg(7), tw = arg(8), oh = arg(9), ow = arg(10), slice = arg(11),
              frames = arg(12);
    const size_t need = svr2_vae_tiled_workspace_bytes(&eng, enc ? 0 : 1, T, H, W, th, tw, oh, ow, slice, frames);
    if (!need) { fprintf(stderr, "refused: %s\n", eng.err); return 3; }
    // the result is zeroed on the host before the tiles accumulate into it: it needs its real size
    const size_t out_bytes = enc ? (size_t)16 * ((T - 1) / 4 + 1) * (H / 8) * (W / 8) * 2 : (size_t)3 * frames * 64 * H * W * 2;
    return trace(eng, need, plan_only(13), out_bytes, [&](void* ws, size_t bytes, void* out) {
      return enc ? svr2_vae_encode_tiled(&eng, in, 1, T, H, W, th, tw, oh, ow, slice, out, ws, bytes, nullptr)
                 : svr2_vae_decode_tiled(&eng, in, 1, T, H, W, th, tw, oh, ow, slice, frames, out, ws, bytes, nullptr);
    });
  }
  return 2;
}
