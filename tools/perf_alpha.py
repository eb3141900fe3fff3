"""Times the alpha path of RGBA clips at the 4K shard shape (5 frames, 720p alpha -> 2160 x 3840) with CUDA events:
svr2_alpha_upscale writing channel 3 of the RGBA image, as the engine runs it, and for comparison the fp32 torch
restatement of the reference (oracle/alpha_oracle.py) on the same GPU (its edges in integer / fp64 torch ops instead of
the reference's host OpenCV loop, so it is faster than the reference itself).

Algorithmic bytes: the HBM traffic of the kernel sequence per output pixel (bf16 guide = 6 B, fp32 planes = 4 B):
statistics 6 (guide read) | resize 4 (base written) | Sobel 6 + 4 (guide read, gx^2+gy^2 written) |
guided filter A 6 + 4 + 8 (guide, base read; a, b written) | B 8 + 6 + 4 + 2 (a, b, guide, gx^2+gy^2 read; bf16 alpha
written) = 58 B, plus the input alpha read twice (statistics, resize)."""
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
from oracle import alpha_oracle as ao  # noqa: E402

am = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.alpha")
HBM = 3.35e12                        # H100 SXM HBM3, data sheet
BYTES_PER_PX = 58


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
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    T, h, w, H, W = args.frames, 720, 1280, 2160, 3840
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "shape": f"{T}x{h}x{w} -> {T}x{H}x{W}"}
    for kind in ("binary", "gradient"):
        alpha, rgb = ao.make_inputs(T, h, w, H, W, kind, seed=11)
        rgb = rgb.cuda()
        frames = torch.zeros(T, h, w, 4, device="cuda", dtype=torch.bfloat16)
        frames[..., 3] = alpha[:, 0].cuda()
        image = torch.empty(T, H, W, 4, device="cuda", dtype=torch.bfloat16)
        ms = timed(lambda: am.upscale_into_image(frames, rgb, image), args.reps)
        nbytes = BYTES_PER_PX * T * H * W + 2 * frames.numel() * 2 // 4
        a32 = alpha.cuda().float()
        ms_oracle = timed(lambda: ao.edge_guided_alpha_upscale(a32, rgb), max(2, args.reps // 5))
        res[kind] = {"ms": round(ms, 3), "GB": round(nbytes / 1e9, 3), "frac_of_3.35TBps": round(nbytes / (ms * 1e-3) / HBM, 3),
                     "torch_fp32_ms": round(ms_oracle, 2), "speedup_vs_torch": round(ms_oracle / ms, 1)}
        print(f"{kind:8s}: {ms:7.3f} ms  {nbytes / 1e9:.2f} GB algorithmic -> {nbytes / (ms * 1e-3) / 1e12:.2f} TB/s "
              f"({100 * nbytes / (ms * 1e-3) / HBM:.0f} % of 3.35 TB/s);  torch fp32 restatement {ms_oracle:.1f} ms")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
