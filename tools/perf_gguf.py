"""GGUF dequantization (csrc/gguf.cu) on the GPU:

1. svr2_gguf_dequant_f16 per type at the 7B weight shapes (12288x3072, 3072x12288, 9216x3072): ms and GB/s of the
   algorithmic traffic (raw blocks read + fp16 written) against 3.35 TB/s;
2. a 7B Q4_K_M-like weight set (Q4_K, Q6_K for the MLP output projections) dequantized by the kernel and by the torch
   fp16 restatement of the reference's block functions (what the reference repeats on every DiT forward);
3. wall clock of loading a DiT of 7B width (``--layers`` of its 36 blocks) from a GGUF file and from the same weights as
   fp16 safetensors, both written to a temporary directory first (so both are read from the page cache).

Prints the card, its power limit and max SM clock, and one JSON line per result.

    python tools/perf_gguf.py [--iters 20] [--layers 12]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from svr2_import import load_package  # noqa: E402

pkg = load_package()
import importlib  # noqa: E402

from oracle import gguf_oracle as go  # noqa: E402

lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
SHAPES = ((12288, 3072), (3072, 12288), (9216, 3072))
HBM = 3.35e12


def timed(fn, iters):
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def random_raw(name, rows, cols, gen):
    """Random blocks with finite fp16 scales (|d| < 1), on the GPU."""
    tid, be, bb = go.TYPES[name]
    n = rows * cols // be
    raw = torch.randint(0, 256, (n, bb), dtype=torch.uint8, device="cuda", generator=gen)
    d_off, m_off = go._D_OFF.get(name, (None, None))
    for off in (d_off, m_off):
        if off is not None:
            s = (torch.rand(n, 1, device="cuda", generator=gen) * 0.02 - 0.01).half()
            raw[:, off:off + 2] = s.view(torch.uint8)
    return raw


def kernel(tid, raw, n, out):
    lib.call("svr2_gguf_dequant_f16", tid, lib.ptr(raw), n, lib.ptr(out), lib.stream())


def weight_set(cfg):
    """(key, shape, type name) of the 2-D weights of a 7B DiT with a Q4_K_M-like type mix; 1-D tensors stay F32."""
    d, L = cfg["dim"], cfg["layers"]
    out = []
    for i in range(L):
        for s in ("vid", "txt"):
            p = f"blocks.{i}."
            out += [(p + f"attn.proj_qkv.{s}.weight", (3 * d, d), "Q4_K"),
                    (p + f"attn.proj_out.{s}.weight", (d, d), "Q4_K"),
                    (p + f"mlp.{s}.proj_in.weight", (4 * d, d), "Q4_K"),
                    (p + f"mlp.{s}.proj_out.weight", (d, 4 * d), "Q6_K")]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--layers", type=int, default=12, help="blocks of the 7B DiT in the load-time comparison")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_gguf needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True).stdout.strip()
    print(card)
    gen = torch.Generator(device="cuda").manual_seed(0)

    # 1. per type and shape
    for name, (tid, be, bb) in go.TYPES.items():
        for rows, cols in SHAPES:
            raw = random_raw(name, rows, cols, gen)
            n = rows * cols
            out = torch.empty(n, dtype=torch.float16, device="cuda")
            ms = timed(lambda: kernel(tid, raw, n, out), args.iters)
            nbytes = raw.numel() + 2 * n
            print(json.dumps(dict(case="kernel", type=name, shape=[rows, cols], ms=round(ms, 4),
                                  gb_per_s=round(nbytes / ms / 1e6, 1), hbm_share=round(nbytes / ms / 1e-3 / HBM, 3))))
            del raw, out

    # 2. a whole 7B Q4_K_M-like weight set: the kernel once (engine, at load) vs the torch fp16 restatement
    cfg = dit.dit_config("7b")
    ws = weight_set(cfg)
    raws = [(go.TYPES[t][0], t, shape, random_raw(t, *shape, gen)) for _, shape, t in ws]
    total_raw = sum(r.numel() for *_, r in raws)
    n_el = sum(shape[0] * shape[1] for _, shape, _ in ws)
    biggest = max(shape[0] * shape[1] for _, shape, _ in ws)
    out = torch.empty(biggest, dtype=torch.float16, device="cuda")

    def all_kernel():
        for tid, _, shape, r in raws:
            kernel(tid, r, shape[0] * shape[1], out)

    def all_oracle():
        for _, t, shape, r in raws:
            go.dequantize(t, r)

    ms_k = timed(all_kernel, 3)
    ms_o = timed(all_oracle, 1)
    nbytes = total_raw + 2 * n_el
    print(json.dumps(dict(case="7b_q4_k_m_weight_set", tensors=len(ws), elements=n_el, raw_gb=round(total_raw / 1e9, 3),
                          kernel_ms=round(ms_k, 2), kernel_gb_per_s=round(nbytes / ms_k / 1e6, 1),
                          torch_fp16_ms=round(ms_o, 1), ratio=round(ms_o / ms_k, 1))))
    del raws, out
    torch.cuda.empty_cache()

    # 3. load wall clock: the same weights as GGUF and as fp16 safetensors
    from safetensors.torch import save_file
    cfg = dit.dit_config("7b", layers=args.layers, mm_layers=args.layers)
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=1, dtype=torch.float16, device="cuda")
    mix = {k: t for k, _, t in weight_set(cfg)}
    with tempfile.TemporaryDirectory() as tmp:
        tensors, dense = [], {}
        for k, v in sd.items():
            if k in mix:
                raw = go.encode(mix[k], v)
                dense[k] = go.dequantize(mix[k], raw).reshape(v.shape).cpu()
                tensors.append(("model.diffusion_model." + k, go.TYPES[mix[k]][0], list(reversed(v.shape)),
                                raw.cpu().numpy().reshape(-1)))
            else:
                t = go.F32 if v.ndim == 1 else go.F16
                a = (v.float() if t == go.F32 else v).cpu()
                dense[k] = a
                tensors.append(("model.diffusion_model." + k, t, list(reversed(v.shape)), a.numpy().view(np.uint8)))
        del sd
        p_gguf, p_st = os.path.join(tmp, "dit.gguf"), os.path.join(tmp, "dit_fp16.safetensors")
        go.write_gguf(p_gguf, tensors)
        del tensors
        save_file({k: v.contiguous() for k, v in dense.items()}, p_st)
        del dense
        times = {}
        for label, load in (("gguf", lambda: pkg.weights.load_gguf(p_gguf)),
                            ("safetensors_fp16", lambda: pkg.weights.load_state_dict(p_st)),
                            ("gguf_again", lambda: pkg.weights.load_gguf(p_gguf))):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m = dit.B200NaDiT(cfg, load())
            torch.cuda.synchronize()
            times[label] = time.perf_counter() - t0
            del m
            torch.cuda.empty_cache()
        print(json.dumps(dict(case="load_dit", layers=args.layers, gguf_gb=round(os.path.getsize(p_gguf) / 1e9, 2),
                              safetensors_gb=round(os.path.getsize(p_st) / 1e9, 2),
                              **{k + "_s": round(v, 2) for k, v in times.items()})))


if __name__ == "__main__":
    main()
