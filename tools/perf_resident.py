"""DiT weights kept compressed in device memory (``B200NaDiT(resident="compressed")``) on the GPU, for the 3B and 7B
widths with a Q4_K_M-like GGUF mix (Q4_K, Q6_K for the MLP output projections) and with fp8_e4m3fn block matrices:

1. resident weight bytes in both modes and the staging slot;
2. svr2_weight_expand_bf16 at each distinct matrix shape of the model: ms and the algorithmic traffic (stored bytes read
   + 2 B per value written) against 3.35 TB/s;
3. the expansion launches of one whole forward (every block's matrices into one slot), alone: median ms;
4. one DiT forward (native runtime, caller-provided workspace) in both modes, alternating them in this process:
   median ms, and whether the two outputs are bit-identical.

The weights are random (random blocks with small finite scales), which the timings do not depend on.  Prints the card,
its power limit and max SM clock, and one JSON line per result.

    python tools/perf_resident.py [--variants 3b,7b] [--storages gguf,fp8] [--iters 5] [--thw 2,270,480]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from svr2_import import load_package  # noqa: E402

pkg = load_package()
import importlib  # noqa: E402

from oracle import gguf_oracle as go  # noqa: E402

lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
HBM = 3.35e12


class StoredBlocks(torch.Tensor):
    """GGUF blocks on the GPU with the attributes of the reference's GGUFTensor."""

    @staticmethod
    def __new__(cls, raw, tensor_type, tensor_shape):
        t = torch.Tensor._make_subclass(cls, raw)
        t.tensor_type, t.tensor_shape = tensor_type, torch.Size(tensor_shape)
        return t


def random_raw(name, rows, cols, gen):
    """Random blocks with finite fp16 scales (|d| < 0.01), on the GPU."""
    tid, be, bb = go.TYPES[name]
    n = rows * cols // be
    raw = torch.randint(0, 256, (n, bb), dtype=torch.uint8, device="cuda", generator=gen)
    for off in go._D_OFF[name]:
        if off is not None:
            s = (torch.rand(n, 1, device="cuda", generator=gen) * 0.02 - 0.01).half()
            raw[:, off:off + 2] = s.view(torch.uint8)
    return raw


def stored_state_dict(cfg, storage, gen):
    """Synthetic weights with the block matrices replaced, one at a time, by their stored form."""
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=1, dtype=torch.float16, device="cuda")
    for k in list(sd):
        v = sd[k]
        if not (k.startswith("blocks.") and v.ndim == 2 and (".attn.proj_" in k or ".mlp." in k)):
            continue
        if storage == "fp8":
            sd[k] = v.to(torch.float8_e4m3fn)
        else:
            name = "Q6_K" if ".proj_out." in k and ".mlp." in k else "Q4_K"
            sd[k] = StoredBlocks(random_raw(name, *v.shape, gen).reshape(v.shape[0], -1), go.TYPES[name][0], v.shape)
        del v
    return sd


def median_ms(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times), min(times), max(times)


def parts_of(m, name):
    """(entry, buffer-name suffix) of a compressed matrix: one, or the gate and in halves of a SwiGLU input matrix"""
    parts = m._plan[name]
    return zip(parts, ("",) if len(parts) == 1 else (".gate", ".in"))


def expand_part(m, name, part, suffix, dst):
    lib.call("svr2_weight_expand_bf16", part.format, lib.ptr(m.C[name + suffix]), part.rows, part.cols, lib.ptr(dst),
             part.row_group, part.group_stride, part.row_offset, lib.stream())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", default="3b,7b")
    ap.add_argument("--storages", default="gguf,fp8")
    ap.add_argument("--iters", type=int, default=5, help="timed forwards per mode")
    ap.add_argument("--thw", default="2,270,480", help="latent frames, rows, columns (default: the 5-frame 4K shard)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_resident needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True).stdout.strip()
    print(card)
    T, H, W = (int(x) for x in args.thw.split(","))
    gen = torch.Generator(device="cuda").manual_seed(0)
    for variant in args.variants.split(","):
        cfg = dit.dit_config(variant)
        g = torch.Generator(device="cuda").manual_seed(3)
        vid = torch.randn(T * H * W, cfg["in_ch"], generator=g, device="cuda", dtype=torch.bfloat16)
        txt = torch.randn(58, cfg["txt_in_dim"], generator=g, device="cuda", dtype=torch.bfloat16)
        for storage in args.storages.split(","):
            tag = dict(variant=variant, storage=storage)
            sd = stored_state_dict(cfg, storage, gen)
            mods = {r: dit.B200NaDiT(cfg, sd, resident=r) for r in dit.RESIDENT_MODES}
            del sd
            gc.collect()
            torch.cuda.empty_cache()
            m = mods["compressed"]
            held = {r: sum(b.numel() * b.element_size() for b in mm.buffers()) for r, mm in mods.items()}
            n_launch = sum(len(p) for p in m._plan.values())
            print(json.dumps(dict(case="resident_bytes", **tag, expanded_gb=round(held["expanded"] / 1e9, 3),
                                  compressed_gb=round(held["compressed"] / 1e9, 3), slot_mb=round(m.slot_bytes / 1e6, 1),
                                  expansion_launches_per_forward=n_launch)))

            # 2. the kernel at every distinct (format, shape) of the model
            stage = torch.empty(m.slot_bytes // 2, device="cuda", dtype=torch.bfloat16)
            seen = set()
            for name, parts in m._plan.items():
                for part, suffix in parts_of(m, name):
                    key = (part.format, part.rows, part.cols, part.row_offset)
                    if key in seen:
                        continue
                    seen.add(key)
                    dst = stage[: sum(p.rows for p in parts) * part.cols]
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    for _ in range(3):
                        expand_part(m, name, part, suffix, dst)
                    e0.record()
                    for _ in range(50):
                        expand_part(m, name, part, suffix, dst)
                    e1.record()
                    torch.cuda.synchronize()
                    ms = e0.elapsed_time(e1) / 50
                    nbytes = m.C[name + suffix].numel() + 2 * part.rows * part.cols
                    print(json.dumps(dict(case="kernel", **tag, format=part.format, shape=[part.rows, part.cols],
                                          row_map=[part.row_group, part.group_stride, part.row_offset],
                                          ms=round(ms, 4), gb_per_s=round(nbytes / ms / 1e6, 1),
                                          hbm_share=round(nbytes / ms / 1e-3 / HBM, 3))))

            # 3. the expansion launches of one forward, alone
            def expand_all():
                for i, offsets in enumerate(m._slot_offsets):
                    for name, off in offsets.items():
                        for part, suffix in parts_of(m, name):
                            expand_part(m, name, part, suffix, stage[off // 2:])

            med, lo, hi = median_ms(expand_all, 10)
            total = sum(m.C[n + sfx].numel() + 2 * p.rows * p.cols for n in m._plan for p, sfx in parts_of(m, n))
            print(json.dumps(dict(case="expansion_per_forward", **tag, launches=n_launch, median_ms=round(med, 3),
                                  min_ms=round(lo, 3), max_ms=round(hi, 3), algorithmic_gb=round(total / 1e9, 3),
                                  hbm_share=round(total / med / 1e-3 / HBM, 3))))
            del stage

            # 4. one forward per mode, alternating
            ws = torch.empty(max(mm.workspace_bytes(T, H, W, 58) for mm in mods.values()), device="cuda", dtype=torch.uint8)
            outs, times = {}, {r: [] for r in mods}
            for r, mm in mods.items():
                for _ in range(2):
                    outs[r] = mm(vid, txt, [[T, H, W]], [[58]], workspace=ws).vid_sample
            for _ in range(args.iters):
                for r, mm in mods.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    mm(vid, txt, [[T, H, W]], [[58]], workspace=ws)
                    e1.record()
                    torch.cuda.synchronize()
                    times[r].append(e0.elapsed_time(e1))
            med = {r: statistics.median(t) for r, t in times.items()}
            print(json.dumps(dict(case="dit_forward", **tag, thw=[T, H, W], iters=args.iters,
                                  expanded_ms=round(med["expanded"], 2), compressed_ms=round(med["compressed"], 2),
                                  expanded_range_ms=[round(min(times["expanded"]), 2), round(max(times["expanded"]), 2)],
                                  compressed_range_ms=[round(min(times["compressed"]), 2), round(max(times["compressed"]), 2)],
                                  extra_percent=round(100 * (med["compressed"] / med["expanded"] - 1), 2),
                                  bit_identical=bool(torch.equal(outs["expanded"].view(torch.int16),
                                                                 outs["compressed"].view(torch.int16))))))
            del mods, m, ws, outs
            gc.collect()
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
