"""Streams a long clip through SeedVR2Engine.stream_video at the 4K shard shape (720p source -> 2160 x 3840, batches of
5, the synthetic 3B engine) and prints the card, its power limit and max SM clock, and one JSON line:

  stream      frames/s of stream_video (8-bit output, pinned host frames handed to a consumer that touches them), the
              input read from pinned host uint8 frames in chunks of 4, against the summed upscale_clip time of the same
              batches (bf16 on the device, each ended by a device synchronise): the cost of streaming
  memory      peak device memory above the resident state at --frames / 2 against --frames (max_memory_allocated)
  kernel      svr2_sample_to_image_u8 on one 5-frame 4K sample, RGB and RGBA, CUDA events over --reps launches:
              ms and share of 3.35 TB/s (H100 SXM data sheet); algorithmic bytes: bf16 sample read and bytes
              written (9 B per pixel), plus the bf16 alpha read and its byte (12 B per pixel) for RGBA
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))  # repo root (this file lives in tools/)
sys.path.insert(0, ROOT)
from svr2_import import load_package  # noqa: E402

load_package()
pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
color_fix = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.color_fix")
HBM = 3.35e12                        # H100 SXM HBM3, data sheet


def event_ms(fn, reps):
    for _ in range(3):
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
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--batch", type=int, default=5)
    ap.add_argument("--overlap", type=int, default=0)
    ap.add_argument("--color-correction", default="lab")
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    H, W, h, w = 2160, 3840, 720, 1280
    res = {"gpu": card, "shape": f"{h}x{w} -> {H}x{W}", "frames": args.frames, "batch": args.batch,
           "overlap": args.overlap, "color_correction": args.color_correction}

    # ---- the uint8 formatting kernel on one batch
    g = torch.Generator(device="cuda").manual_seed(3)
    sample = (torch.rand(args.batch, 3, H, W, device="cuda", generator=g) * 2.2 - 1.1).to(torch.bfloat16)
    image = torch.rand(args.batch, H, W, 4, device="cuda", generator=g).to(torch.bfloat16)
    px = args.batch * H * W
    for name, fn, nbytes in (("u8_rgb", lambda: color_fix.sample_to_image_u8(sample), 9.0 * px),
                             ("u8_rgba", lambda: color_fix.sample_to_image_u8(sample, image), 12.0 * px),
                             ("bf16_rgb", lambda: color_fix.sample_to_image(sample), 12.0 * px)):
        ms = event_ms(fn, args.reps)
        res[name] = {"ms": round(ms, 4), "GB": round(nbytes / 1e9, 3), "frac_of_3.35TBps": round(nbytes / (ms * 1e-3) / HBM, 3)}
        print(f"{name:8s}: {ms:.4f} ms, {nbytes / 1e9:.3f} GB -> {nbytes / (ms * 1e-3) / 1e12:.2f} TB/s "
              f"({100 * nbytes / (ms * 1e-3) / HBM:.0f} % of 3.35 TB/s)")
    del sample, image

    # ---- the engine over a long clip
    eng = pipeline.build_synthetic_engine("3b", device="cuda")
    cpu = torch.Generator().manual_seed(42)
    frames = torch.randint(0, 256, (args.frames, h, w, 3), dtype=torch.uint8, generator=cpu).pin_memory()
    kw = dict(batch_size=args.batch, temporal_overlap=args.overlap, seed=42, color_correction=args.color_correction,
              resolution=H)

    def stream(n):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        got, checksum = 0, 0
        for first, t in eng.stream_video(iter(frames[:n].split(4)), **kw):
            assert first == got
            got += t.shape[0]
            checksum += int(t[:, ::97, ::89].sum())          # the consumer reads what it was handed
        torch.cuda.synchronize()
        return time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base, got

    stream(args.batch)                                       # warm-up: tables, kernels, the resident workspace
    # upscale_clip over the same batches, each timed to a device synchronise
    ranges, _ = pipeline.batch_ranges(args.frames, args.batch, args.overlap)
    clip_s = 0.0
    for a, b in ranges:
        x = frames[a:b].cuda()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.upscale_clip(x, seed=42, color_correction=args.color_correction, resolution=H)
        torch.cuda.synchronize()
        clip_s += time.perf_counter() - t0
    half_s, half_peak, n_half = stream(args.frames // 2)
    full_s, full_peak, n_full = stream(args.frames)
    assert n_full == args.frames and n_half == args.frames // 2
    res["stream"] = {"s": round(full_s, 3), "frames_per_s": round(args.frames / full_s, 4),
                     "upscale_clip_sum_s": round(clip_s, 3), "upscale_clip_frames_per_s": round(args.frames / clip_s, 4),
                     "overhead": round(full_s / clip_s - 1, 4)}
    res["memory"] = {f"peak_GiB_{args.frames // 2}": round(half_peak / 2 ** 30, 3),
                     f"peak_GiB_{args.frames}": round(full_peak / 2 ** 30, 3),
                     "growth_MiB": round((full_peak - half_peak) / 2 ** 20, 1)}
    print(f"stream_video: {args.frames} frames in {full_s:.2f} s = {args.frames / full_s:.3f} frames/s; summed "
          f"upscale_clip of the same batches {clip_s:.2f} s ({100 * (full_s / clip_s - 1):+.2f} %)")
    print(f"peak device memory above the resident state: {args.frames // 2} frames {half_peak / 2 ** 30:.2f} GiB, "
          f"{args.frames} frames {full_peak / 2 ** 30:.2f} GiB")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
