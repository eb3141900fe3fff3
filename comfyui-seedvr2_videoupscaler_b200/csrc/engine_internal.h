// Internal (non-ABI): the svr2_t handle shared by the native host runtimes (engine.cu: NaDiT, vae_engine.cu: video VAE).
#pragma once
#include <stdint.h>

#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "svr2_internal.h"

namespace svr2 {

struct Tensor {
  void* ptr = nullptr;
  int dtype = 1;          // svr2_tensor_desc.dtype: 0 f32, 1 bf16, 2 f16; 3 fp8_e4m3fn or 16 + GGML type: a compressed matrix
  int rank = 0;
  int64_t shape[5] = {0, 0, 0, 0, 0};
  bool owned = false;
  int64_t numel() const {
    int64_t n = 1;
    for (int i = 0; i < rank; ++i) n *= shape[i];
    return n;
  }
};

inline size_t dtype_size(int dt) { return dt == 0 ? 4 : 2; }
inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }
// gguf.cu: elements and bytes per block of a storage format svr2_weight_expand_bf16 reads (dtype codes 2, 3, 16 + t)
bool weight_format_size(int format, int* block_elems, int* block_bytes);

// One matrix of a transformer block that svr2_dit_forward expands into the staging slot before the block runs.
// parts: the source tensors (one; gate and in for a SwiGLU input matrix) with their destination row maps.
struct SlotPart {
  const void* src;
  int format;
  int64_t rows, group, stride, offset;
};
struct SlotMatrix {
  std::string name;       // engine-layout name the block's GEMM asks for, e.g. "3.vid.mlp_in.w"
  size_t off = 0;         // byte offset in the slot
  int64_t cols = 0;
  std::vector<SlotPart> parts;   // empty: the matrix shares the bytes of an earlier entry (3B layers with shared weights)
};

struct Geometry;      // window / RoPE index tables of one clip geometry (engine.cu)
struct VaeState;      // engine-owned VAE workspace bookkeeping (vae_engine.cu)

}  // namespace svr2

struct svr2_engine {
  int device = 0;
  svr2_model_desc desc{};
  std::unordered_map<std::string, svr2::Tensor> w;
  std::vector<std::vector<svr2::SlotMatrix>> slot_plan;   // per layer: the compressed matrices (rebuilt by svr2_load_weights)
  size_t slot_bytes = 0;                                  // largest per-layer sum of their bf16 sizes; 0: all resident
  std::map<std::vector<int>, svr2::Geometry*> geo;      // (T, Hp, Wp, l) -> tables
  void* workspace = nullptr;
  size_t workspace_bytes = 0;
  std::vector<void*> retired_workspaces;          // outgrown blocks: a captured CUDA graph may still replay into them
  svr2::VaeState* vae = nullptr;                  // VAE handles (desc.variant == 2): engine-owned workspace state
  char err[256] = "";
};

namespace svr2 {
inline int fail(svr2_engine* e, int code, const char* msg) {
  if (e) snprintf(e->err, sizeof e->err, "%s", msg);
  return set_error(code, msg);
}
inline const Tensor* find(svr2_engine* e, const std::string& name) {
  auto it = e->w.find(name);
  return it == e->w.end() ? nullptr : &it->second;
}
void vae_state_destroy(svr2_engine* e);          // vae_engine.cu
}  // namespace svr2
