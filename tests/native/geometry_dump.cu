// Test harness (CPU): the native runtime's geometry code (csrc/engine.cu) compiled with SVR2_HOST_TEST so that its
// tables stay in host memory; dumps them as text for tests/test_native_geometry_cpu.py to compare with the oracle.
// usage: geometry_dump T Hp Wp l is7 fdtype nfreq f0 f1 ... > out.txt
#define SVR2_HOST_TEST 1
#include "../../comfyui-seedvr2_videoupscaler_b200/csrc/engine.cu"
#include <stdlib.h>
namespace svr2 {
int set_error(int code, const char*) { return code; }
}
extern "C" {
const char* svr2_last_error(void) { return ""; }
int svr2_device_check(int*, int*, int*) { return -3; }
#define STUB(name) int name(...) { return -1; }
}
int main(int argc, char** argv) {
  if (argc < 8) return 2;
  const int T = atoi(argv[1]), Hp = atoi(argv[2]), Wp = atoi(argv[3]), l = atoi(argv[4]);
  const bool is7 = atoi(argv[5]) != 0;
  const int fdtype = atoi(argv[6]), nf = atoi(argv[7]);
  std::vector<float> fr(nf);
  for (int j = 0; j < nf; ++j) fr[j] = (float)atof(argv[8 + j]);
  Geometry g;
  for (int s = 0; s < 2; ++s) {
    std::vector<std::pair<int, int>> size_rows;
    int max_row = 0;
    if (!build_layout(&g, g.lay[s], T, Hp, Wp, l, s == 1, is7, size_rows, max_row)) return 3;
    const Layout& L = g.lay[s];
    printf("layout %d %d %d %d %d\n", s, L.n_win, L.total, L.max_len, L.n_txt_rows);
    auto dump = [&](const char* name, const int32_t* p, int n) {
      printf("%s", name);
      for (int i = 0; i < n; ++i) printf(" %d", p[i]);
      printf("\n");
    };
    dump("cu_seqlens", L.cu_seqlens, L.n_win + 1);
    dump("row_src", L.row_src, L.total);
    dump("row_rope", L.row_rope, L.total * 3);
    dump("out_row_map", L.out_row_map, L.total);
    dump("tok_dst", L.tok_dst, T * Hp * Wp);
    dump("tok_rope", L.tok_rope, T * Hp * Wp * 3);
    dump("txt_rows", L.txt_rows, L.n_txt_rows);
    int rows = max_row + 1;
    if (is7)
      for (auto& kv : size_rows) rows = rows > kv.first + kv.second ? rows : kv.first + kv.second;
    RopeTable tab;
    if (!build_rope_table(&g, tab, fr, fdtype, is7, rows, size_rows)) return 4;
    printf("table %d\n", rows);
    for (int i = 0; i < rows * nf; ++i) printf("%.9g %.9g\n", tab.cos[i], tab.sin[i]);
  }
  return 0;
}
