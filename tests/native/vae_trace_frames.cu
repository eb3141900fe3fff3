// Test harness (CPU): the native VAE runtime's decode that returns only the first `frames` output frames
// (svr2_vae_decode_frames), traced through vae_trace.cu's kernel stubs on a host-memory workspace.
// tests/test_vae_decode_frames_cpu.py compares the trace with the Python module's (vae.py) decode(frames=...).
// usage: vae_trace_frames <weights manifest> T h w slice_frames frames [plan]
//   prints the trace, then "# workspace <bytes> touched_max_offset <bytes> launches <n>" ("plan": only "# workspace
//   <bytes>"); exit 3 with "refused: <message>" on stderr when both the workspace query and the decode refuse `frames`.
#define main vae_trace_main
#include "vae_trace.cu"
#undef main

int main(int argc, char** argv) {
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
  const int T = atoi(argv[2]), h = atoi(argv[3]), w = atoi(argv[4]), slice = atoi(argv[5]), frames = atoi(argv[6]);
  static char in_buf[16], out_buf[16];
  const size_t need = svr2_vae_decode_frames_workspace_bytes(&eng, T, h, w, slice, frames);
  if (!need) {
    std::string msg = eng.err;
    static char small_ws[1 << 12] __attribute__((aligned(256)));
    if (svr2_vae_decode_frames(&eng, in_buf, 1, T, h, w, slice, frames, out_buf, small_ws, sizeof small_ws, nullptr) == 0) return 8;
    fprintf(stderr, "refused: %s | %s\n", msg.c_str(), eng.err);
    return 3;
  }
  if (argc >= 8 && std::string(argv[7]) == "plan") {      // the exact workspace only (shapes too large to trace)
    printf("# workspace %zu\n", need);
    return 0;
  }
  void* ws = nullptr;
  if (posix_memalign(&ws, 256, need)) return 4;
  g_lo = (char*)ws;
  g_hi = g_lo + need;
  const int rc = svr2_vae_decode_frames(&eng, in_buf, 1, T, h, w, slice, frames, out_buf, ws, need, nullptr);
  if (rc) { fprintf(stderr, "run failed (%d): %s\n", rc, eng.err); return 5; }
  // a workspace 256 bytes short of the plan must be refused
  if (svr2_vae_decode_frames(&eng, in_buf, 1, T, h, w, slice, frames, out_buf, ws, need - 256, nullptr) == 0) return 6;
  printf("# workspace %zu touched_max_offset %zu launches %lld\n", need, g_touch, (long long)svr2_vae_last_launches(&eng));
  free(ws);
  vae_state_destroy(&eng);
  return 0;
}
