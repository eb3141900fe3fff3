"""Times the generation-noise kernels (csrc/noise.cu) at the 4K shard: the input-noise blend on a 3x5x2160x3840 clip
with the draw in each of its three memory orders (6 B per value: clip and draw read, output written) and the DiT-input pass on the 2x270x480x16 latent, with and without
the latent augmentation.  Prints the card, its power limit and one JSON line per case.

    python tools/perf_noise.py [--iters 50]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))   # repo root
from svr2_import import load_package  # noqa: E402

load_package()


def timed(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_noise needs a GPU")
    import importlib
    nz = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.noise")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.rand(3, 5, 2160, 3840, device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)
    nbytes = 6.0 * x.numel()
    for layout, name in ((nz.TCHW, "t c h w"), (nz.CTHW, "c t h w"), (nz.THWC, "t h w c")):
        n = nz.draw_input_noise(x.shape, g, "cuda", layout)
        ms = timed(lambda: nz.add_input_noise(x, n, 0.5), args.iters)
        print(json.dumps(dict(case=f"input_noise 3x5x2160x3840, noise memory {name}", ms=round(ms, 4),
                              algorithmic_MB=round(nbytes / 1e6, 1), GBps=round(nbytes / ms / 1e6, 1),
                              share_of_3350GBps=round(nbytes / ms / 1e6 / 3350, 3))))
    shape = (2, 270, 480, 16)
    latent = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    noise = torch.randn(shape, device="cuda", generator=g, dtype=torch.bfloat16)
    r = nz.draw_latent_noise(shape, g, "cuda")
    rows = 2 * 270 * 480
    for aug in (False, True):
        coef = nz.latent_noise_coefficients(0.3, shape, "cuda") if aug else None
        ms = timed(lambda: nz.sr_condition(noise, latent, r if aug else None, coef), args.iters)
        nbytes = 2.0 * rows * 33 + 2.0 * rows * 16 * (3 if aug else 2)
        print(json.dumps(dict(case=f"sr_condition 2x270x480x16 aug={aug}", ms=round(ms, 4),
                              algorithmic_MB=round(nbytes / 1e6, 1), GBps=round(nbytes / ms / 1e6, 1))))
        if aug:
            ms = timed(lambda: nz.latent_noise_coefficients(0.3, shape, "cuda"), args.iters)
            print(json.dumps(dict(case="latent_noise_coefficients (torch ops)", ms=round(ms, 4))))


if __name__ == "__main__":
    main()
