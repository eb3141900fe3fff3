"""Spatially tiled VAE at 4K (720p source -> 2160 x 3840, the synthetic 3B engine): prints the card, its power limit and
max SM clock, and one JSON line:

  tiled_clip   a 9-frame batch upscaled by upscale_clip with encode_tiled and decode_tiled at --tile / --overlap:
               frames/s (host clock around calls ended by a device synchronise) and peak device memory
               (max_memory_reserved: the clip's one workspace, weights and torch's tensors)
  shard        the 5-frame (4 real frames) un-tiled batch of bench.py's 4k_shard workload in the same run, for scale
  decode       the tiled decode of the 9-frame batch's latent (3 x 270 x 480) on the native runtime
               (svr2_vae_decode_tiled) against the tile-by-tile loop in Python over the same tiles (vae.py _tiled, each
               tile one native decode, its output stored and accumulated): ms per call, CUDA events
  workspace    exact needs of the DiT at the 9-frame latent and of both tiled VAE passes
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
lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps, out


def event_ms(fn, reps):
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
    ap.add_argument("--tile", type=int, default=1024)
    ap.add_argument("--overlap", type=int, default=128)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    tiling = dict(encode_tiled=True, encode_tile_size=args.tile, encode_tile_overlap=args.overlap, decode_tiled=True,
                  decode_tile_size=args.tile, decode_tile_overlap=args.overlap)
    res = {"gpu": card, "shape": "720x1280 -> 2160x3840", "tile": args.tile, "overlap": args.overlap}
    eng = pipeline.build_synthetic_engine("3b")
    g = torch.Generator().manual_seed(1)
    res["workspace_gb"] = {
        "dit_3x270x480": eng.dit.workspace_bytes(3, 270, 480, eng.txt.shape[0]) / 1e9,
        "encode_tiled_9x2160x3840": eng.vae.workspace_bytes(True, 9, 2160, 3840, tiles=(args.tile,) * 2 + (args.overlap,) * 2) / 1e9,
        "decode_tiled_3x270x480": eng.vae.workspace_bytes(False, 3, 270, 480, frames=9,
                                                          tiles=(args.tile,) * 2 + (args.overlap,) * 2) / 1e9}

    # ---- the 5-frame un-tiled shard, then the 9-frame tiled clip
    shard = torch.rand(4, 720, 1280, 3, generator=g).cuda()
    s, _ = timed(lambda: eng.upscale_clip(shard, resolution=2160), args.reps)
    res["shard"] = {"frames": 4, "s_per_clip": s, "frames_per_s": 4 / s}
    lib.release_workspace()
    torch.cuda.empty_cache()
    clip = torch.rand(9, 720, 1280, 3, generator=g).cuda()
    torch.cuda.reset_peak_memory_stats()
    s, out = timed(lambda: eng.upscale_clip(clip, resolution=2160, **tiling), args.reps)
    assert out.shape == (9, 2160, 3840, 3)
    res["tiled_clip"] = {"frames": 9, "s_per_clip": s, "frames_per_s": 9 / s,
                         "peak_reserved_gb": torch.cuda.max_memory_reserved() / 1e9}
    del out
    lib.release_workspace()
    torch.cuda.empty_cache()

    # ---- tiled decode: native runtime vs the Python tile loop (each tile one native decode)
    z = torch.randn(1, 16, 3, 270, 480, generator=g).cuda()
    vae = eng.vae
    native = event_ms(lambda: vae.decode(z, tiled=True, tile_size=args.tile, tile_overlap=args.overlap), args.reps)
    loop = event_ms(lambda: vae._tiled(z, False, (args.tile,) * 2, (args.overlap,) * 2), args.reps)
    same = torch.equal(vae.decode(z, tiled=True, tile_size=args.tile, tile_overlap=args.overlap).sample,
                       vae._tiled(z, False, (args.tile,) * 2, (args.overlap,) * 2))
    res["decode"] = {"latent": "3x270x480", "native_ms": native, "python_loop_ms": loop, "speedup": loop / native,
                     "bit_identical": same}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
