"""Streams one video over N ranks with shard.stream_shard (the synthetic 3B engine, batches of 5, 8-bit output) and
prints the card, its power limit and max SM clock, and one JSON line from rank 0.  Run it under torchrun, one process
per GPU (NCCL):

  torchrun --nproc-per-node N tools/perf_stream_multi.py --frames F [--shape 1080p|4k] [--reps R]

  stream   frames/s of the whole video (from a barrier before the first rank starts to a barrier after the last rank
           has handed its last frame to a consumer that touches it), --reps runs alternated between the shapes asked
           for; median, min and max, and every rank's peak device memory above its resident state (max over runs)
  kernel   svr2_blend_overlap_u8 at 2160 x 3840 x 3, overlap --overlap (rank 0): the fp32 + uint8 outputs, uint8 only and
           fp32 only alternated over --kernel-reps rounds of 20 launches each (CUDA events); median ms, spread, and the
           algorithmic bytes (fp32 tail and bf16 head read, the outputs written) over time against 3.35 TB/s (H100 SXM
           data sheet)
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))  # repo root (this file lives in tools/)
sys.path.insert(0, ROOT)
from svr2_import import load_package  # noqa: E402

load_package()
pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
HBM = 3.35e12                        # H100 SXM HBM3, data sheet
SHAPES = {"1080p": 1080, "4k": 2160}


def spread(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4), "n": len(xs)}


def kernel(overlap, rounds):
    H, W, C = 2160, 3840, 3
    g = torch.Generator(device="cuda").manual_seed(1)
    prev = torch.rand(overlap, H, W, C, device="cuda", generator=g)
    cur = torch.rand(overlap, H, W, C, device="cuda", generator=g).to(torch.bfloat16)
    n = prev.numel()
    modes = {"f32+u8": (True, True, 11.0 * n), "u8": (False, True, 7.0 * n), "f32": (True, False, 10.0 * n)}
    ms = {m: [] for m in modes}
    for _ in range(3):
        for f32, u8, _b in modes.values():
            shard.blend_seam(prev, cur, f32=f32, u8=u8)
    for _ in range(rounds):                                      # the modes alternate round by round
        for m, (f32, u8, _b) in modes.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                shard.blend_seam(prev, cur, f32=f32, u8=u8)
            e1.record()
            torch.cuda.synchronize()
            ms[m].append(e0.elapsed_time(e1) / 20)
    out = {}
    for m, (_f, _u, nbytes) in modes.items():
        med = statistics.median(ms[m])
        out[m] = dict(ms=spread(ms[m]), GB=round(nbytes / 1e9, 3), TBps=round(nbytes / (med * 1e-3) / 1e12, 3),
                      frac_of_3_35TBps=round(nbytes / (med * 1e-3) / HBM, 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40, help="frames of the whole video")
    ap.add_argument("--shape", default="1080p,4k", help="output shapes, comma-separated: 1080p, 4k")
    ap.add_argument("--overlap", type=int, default=4)
    ap.add_argument("--batch", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=10)
    ap.add_argument("--color-correction", default="lab")
    args = ap.parse_args()
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl" if "RANK" in os.environ else "gloo", device_id=dev if "RANK" in os.environ else None,
                            **({} if "RANK" in os.environ else dict(rank=0, world_size=1, init_method="tcp://127.0.0.1:29650")))
    rank, world = dist.get_rank(), dist.get_world_size()
    card = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": card, "world": world, "frames": args.frames, "batch": args.batch, "overlap": args.overlap,
           "color_correction": args.color_correction, "source": "720x1280 uint8, chunks of 4"}
    if rank == 0:
        print(f"card: {card}; ranks: {world}")
        res["kernel"] = kernel(args.overlap, args.kernel_reps)
    eng = pipeline.build_synthetic_engine("3b", device=dev)
    cpu = torch.Generator().manual_seed(42)
    src = torch.randint(0, 256, (args.frames, 720, 1280, 3), dtype=torch.uint8, generator=cpu)
    shapes = args.shape.split(",")

    def run(shape, frames):
        kw = dict(batch_size=args.batch, temporal_overlap=args.overlap, seed=42, color_correction=args.color_correction,
                  resolution=SHAPES[shape])
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        dist.barrier()
        t0 = time.perf_counter()
        got, checksum = 0, 0
        for _, t in shard.stream_shard(eng, lambda s, e: iter(src[s:e].split(4)), total=frames, **kw):
            got += t.shape[0]
            checksum += int(t[:, ::97, ::89].sum())              # the consumer reads what it was handed
        torch.cuda.synchronize()
        dist.barrier()
        return time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base, got

    for shape in shapes:                                         # warm-up: tables, kernels, the resident workspace
        run(shape, min(args.frames, world * (args.batch + args.overlap)))
    secs = {s: [] for s in shapes}
    peaks = {s: 0 for s in shapes}
    for _ in range(args.reps):
        for s in shapes:
            dt, peak, got = run(s, args.frames)
            secs[s].append(dt)
            peaks[s] = max(peaks[s], peak)
    gathered = [None] * world
    dist.all_gather_object(gathered, {s: peaks[s] for s in shapes})
    for s in shapes:
        fps = [args.frames / t for t in secs[s]]
        res[s] = {"frames_per_s": spread(fps), "seconds": spread(secs[s]),
                  "peak_GiB_per_rank": [round(g[s] / 2 ** 30, 3) for g in gathered]}
        if rank == 0:
            print(f"{s}: {args.frames} frames on {world} rank(s): {statistics.median(fps):.3f} frames/s "
                  f"(min {min(fps):.3f}, max {max(fps):.3f}); peak per rank "
                  f"{[round(g[s] / 2 ** 30, 2) for g in gathered]} GiB")
    if rank == 0:
        print(json.dumps(res))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
