// Internal (non-ABI) declarations shared by the .cu files of libsvr2.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/svr2.h"

namespace svr2 {
int set_error(int code, const char* msg);  // records the message for svr2_last_error(), returns code
int num_sms();          // of the current device
int current_device();   // cudaGetDevice, clamped to the per-device cache size
int make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box);
// elementwise.cu: layout converters / conv_out gather with an explicit NCDHW channel stride (temporal slices of a clip)
int ncdhw_to_ndhwc_strided(const void* in, int in_dtype, int C, int T, int H, int W, int64_t chan_stride, void* out,
                           int C_pad, int out_t_pad, float div, void* stream);
int ndhwc_to_ncdhw_strided(const void* in, int ld_in, int C, int T, int H, int W, void* out, int out_dtype,
                           int64_t chan_stride, void* stream);
int conv_tap_gather_strided(const float* z, int64_t ldz, int co_n, const void* bias, int T, int H, int W, void* out,
                            int out_dtype, int64_t chan_stride, void* stream);
// the input conversion reading a rectangle of a clip (frame / row strides of the NCDHW side in elements)
int ncdhw_to_ndhwc_window(const void* in, int in_dtype, int C, int T, int H, int W, int64_t chan_stride,
                          int64_t frame_stride, int row_stride, void* out, int C_pad, int out_t_pad, float div, void* stream);
// One tile's destination in a spatially tiled VAE pass (see svr2_conv_tap_gather_seam_bf16 in svr2.h)
struct Seam {
  void* result;                     // bf16 clip-sized result at the tile's top-left corner, frame 0 of the call
  int64_t cs, fs;                   // its channel and frame strides (elements)
  int rs;                           // its row stride, also the count plane's
  void* count;                      // count plane at the tile's corner; NULL: not updated (a later temporal slice)
  const void *ramp_h, *ramp_w;      // svr2_tile_ramp_bf16 tables [r | 1 - r] of len_h / len_w entries each
  int len_h, len_w;
  int edges;                        // SVR2_SEAM_* sides with a neighbouring tile
};
int conv_tap_gather_seam(const float* z, int64_t ldz, int co_n, const void* bias, int T, int H, int W, const Seam& s,
                         void* stream);
int ndhwc_to_ncdhw_seam(const void* in, int ld_in, int C, int T, int H, int W, const Seam& s, void* stream);
int tile_ramp(void* ramp_h, int len_h, void* ramp_w, int len_w, void* stream);
inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    char buf[256];
    snprintf(buf, sizeof buf, "%s: %s", what, cudaGetErrorString(e));
    return set_error(SVR2_ERR_CUDA, buf);
  }
  return SVR2_OK;
}
}  // namespace svr2
