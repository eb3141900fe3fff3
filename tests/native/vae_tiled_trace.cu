// Test harness (CPU): the native VAE runtime's spatially tiled passes (svr2_vae_encode_tiled / svr2_vae_decode_tiled),
// traced through vae_trace.cu's kernel stubs on a host-memory workspace, plus stubs for the tiled passes' own launches:
// the windowed input conversion, the seam variants of the final kernels, the ramp tables and the normalisation.
// tests/test_vae_tiled_cpu.py compares the trace with the Python module's tile-by-tile sequence (vae.py _tiled).
// usage: vae_tiled_trace <weights manifest> enc|dec T H W tile_h tile_w overlap_h overlap_w slice_frames frames [plan]
//   prints the trace, then "# workspace <bytes> touched_max_offset <bytes> launches <n>" ("plan": only "# workspace
//   <bytes>").  A seam line ends with "| <offset of the tile's corner in the result, elements> <channel stride> <frame
//   stride> <row stride> <count p0/p1> <ramp lengths> <edges>"; a windowed conversion with "| <channel, frame, row
//   strides> <offset of the window in the input, elements>".
#define main vae_trace_main
#include "vae_trace.cu"
#undef main

static const char* g_in = nullptr;
static const char* g_out = nullptr;
static int g_in_esz = 2;

namespace svr2 {
int ncdhw_to_ndhwc_window(const void* in, int in_dtype, int C, int T, int H, int W, int64_t cs, int64_t fs, int rs, void* out,
                          int C_pad, int out_t_pad, float div, void* stream) {
  printf("svr2_ncdhw_to_ndhwc_window %s %d %d %d %d %d %s %d %d %.5g %s | %lld %lld %d %lld\n", P_(in), in_dtype, C, T, H, W, P_(out),
         C_pad, out_t_pad, div, P_(stream), (long long)cs, (long long)fs, rs, (long long)(((const char*)in - g_in) / g_in_esz));
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

int main(int argc, char** argv) {
  if (argc < 12) return 2;
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
  const bool enc = std::string(argv[2]) == "enc";
  const int T = atoi(argv[3]), H = atoi(argv[4]), W = atoi(argv[5]), th = atoi(argv[6]), tw = atoi(argv[7]), oh = atoi(argv[8]),
            ow = atoi(argv[9]), slice = atoi(argv[10]), frames = atoi(argv[11]);
  const size_t need = svr2_vae_tiled_workspace_bytes(&eng, enc ? 0 : 1, T, H, W, th, tw, oh, ow, slice, frames);
  if (!need) { fprintf(stderr, "refused: %s\n", eng.err); return 3; }
  if (argc >= 13 && std::string(argv[12]) == "plan") {
    printf("# workspace %zu\n", need);
    return 0;
  }
  // the result is zeroed on the host before the tiles accumulate into it: it needs its real size
  const size_t out_bytes = enc ? (size_t)16 * ((T - 1) / 4 + 1) * (H / 8) * (W / 8) * 2 : (size_t)3 * frames * 64 * H * W * 2;
  char* out = (char*)malloc(out_bytes);
  static char in_buf[16];
  g_in = in_buf;
  g_out = out;
  void* ws = nullptr;
  if (!out || posix_memalign(&ws, 256, need)) return 4;
  g_lo = (char*)ws;
  g_hi = g_lo + need;
  const int rc = enc ? svr2_vae_encode_tiled(&eng, in_buf, 1, T, H, W, th, tw, oh, ow, slice, out, ws, need, nullptr)
                     : svr2_vae_decode_tiled(&eng, in_buf, 1, T, H, W, th, tw, oh, ow, slice, frames, out, ws, need, nullptr);
  if (rc) { fprintf(stderr, "run failed (%d): %s\n", rc, eng.err); return 5; }
  const int64_t launches = svr2_vae_last_launches(&eng);
  // a workspace 256 bytes short of the plan must be refused
  if ((enc ? svr2_vae_encode_tiled(&eng, in_buf, 1, T, H, W, th, tw, oh, ow, slice, out, ws, need - 256, nullptr)
           : svr2_vae_decode_tiled(&eng, in_buf, 1, T, H, W, th, tw, oh, ow, slice, frames, out, ws, need - 256, nullptr)) == 0)
    return 6;
  printf("# workspace %zu touched_max_offset %zu launches %lld\n", need, g_touch, (long long)launches);
  free(ws);
  free(out);
  vae_state_destroy(&eng);
  return 0;
}
