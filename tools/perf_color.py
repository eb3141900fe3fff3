"""Times the six colour-correction modes at the 4K shard shape (5 x 3 x 2160 x 3840 bf16 content and style) with CUDA
events, as color_fix runs them, and for comparison the fp32 torch restatements of hsv / wavelet_adaptive
(oracle/hsv_oracle.py, the reference's own algorithm with its boolean-mask gathers and sorts) on the same GPU.

Algorithmic bytes per pixel of the hsv path (csrc/hsv.cu; bf16 rgb = 6 B, fp32 = 4 B, sort entries u64 key + u32 pixel):
  bins 6 + 6 read, 4 (matched saturation) + 2 x 8 + 2 x 4 (content pairs) + 2 x 8 (style keys) written   = 56
  content pair sort over 34 key bits: a histogram read (2 x 8) + 5 passes reading and writing 2 x 12     = 256
  style key sort: 2 x 8 + 5 x 2 x 2 x 8                                                                 = 176
  match: 2 x 12 content entries + 2 x 8 style keys read (gathered), 4 written                          = 44
  compose: 6 + 4 read, 6 written                                                                        = 16
  hsv = 548 B;  wavelet_adaptive = 548 + 18 (style, fp32 wavelet read) + the fp32 wavelet pyramid: content levels
  (4 + 4 + 8: img read, low written, high read + written) x 5, style levels (4 + 4) x 4, last 4 + 4 + 4  = 690 B
The other modes are listed for reference (lab and adain as the engine runs them; wavelet in bf16)."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))  # repo root (this file lives in tools/)
sys.path.insert(0, ROOT)
from svr2_import import load_package  # noqa: E402

load_package()
from oracle import hsv_oracle as ho  # noqa: E402
from oracle.make_golden import color_inputs  # noqa: E402

cf = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.color_fix")
HBM = 3.35e12                        # H100 SXM HBM3, data sheet
BYTES_PER_PX = {"hsv": 548, "wavelet_adaptive": 690}


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    T, H, W = args.frames, 2160, 3840
    n = T * H * W
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    content, style = color_inputs(T, H, W, seed=11)
    c, s = content.cuda(), style.cuda()
    res = {"gpu": gpu, "shape": f"{T}x3x{H}x{W}"}
    modes = {"none": lambda: cf.apply_color_correction(c, s, "none"),
             "lab": lambda: cf.apply_color_correction(c, s, "lab"),
             "wavelet": lambda: cf.apply_color_correction(c, s, "wavelet"),
             "adain": lambda: cf.apply_color_correction(c, s, "adain"),
             "hsv": lambda: cf.hsv_saturation_histogram_match(c, s),
             "wavelet_adaptive": lambda: cf.apply_color_correction(c, s, "wavelet_adaptive")}
    oracles = {"hsv": lambda: ho.hsv_saturation_histogram_match(c, s),
               "wavelet_adaptive": lambda: ho.wavelet_adaptive_color_correction(c, s)}
    for mode, fn in modes.items():
        ms = timed(fn, args.reps)
        r = {"ms": round(ms, 3)}
        line = f"{mode:17s}: {ms:8.3f} ms"
        if mode in oracles:
            nbytes = BYTES_PER_PX[mode] * n
            ms_oracle = timed(oracles[mode], 2)
            r.update(GB=round(nbytes / 1e9, 2), frac_of_3_35TBps=round(nbytes / (ms * 1e-3) / HBM, 3),
                     torch_fp32_ms=round(ms_oracle, 2), speedup_vs_torch=round(ms_oracle / ms, 1))
            line += (f"  {nbytes / 1e9:.1f} GB algorithmic -> {nbytes / (ms * 1e-3) / 1e12:.2f} TB/s "
                     f"({100 * nbytes / (ms * 1e-3) / HBM:.0f} % of 3.35 TB/s);  torch fp32 restatement {ms_oracle:.1f} ms")
        res[mode] = r
        print(line)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
