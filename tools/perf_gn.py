"""GroupNorm(32)+SiLU at the 4K shard's shapes: the stand-alone path (statistics pass + finalize + apply) and the fused
path (finalize from conv-epilogue partials + apply), on ordinary data and on an all-flat frame (constant + a one-pixel
border ring, where the fused finalize sums every group again from x).  SVR2_LIB=<other build> times another library.
CUDA events around 10 launches after 3 warm-up launches; prints one line per (path, data)."""
import os, sys, importlib, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))  # repo root (this file lives in tools/)
sys.path.insert(0, ROOT)
from svr2_import import load_package
load_package()
lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
dev = "cuda"
frames, H, W, C = 2, 2160, 3840, 128
hw = H * W
slots = lib.load().svr2_conv_stat_slots(C, H, W)
g = torch.ones(C, device=dev, dtype=torch.bfloat16); b = torch.zeros(C, device=dev, dtype=torch.bfloat16)
y = torch.empty(2 + frames, hw, C, device=dev, dtype=torch.bfloat16)
need = lib.load().svr2_groupnorm_scratch_bytes(frames, hw, C)
st = torch.empty(need // 8 + 8, device=dev, dtype=torch.float64)
coef = torch.empty(frames * C * 2, device=dev)


def data(kind):
    if kind == "normal":
        x = torch.randn(frames, hw, C, device=dev, dtype=torch.bfloat16)
    else:
        x = torch.full((frames, H, W, C), 1.7, device=dev)
        x[:, 0] += 0.05; x[:, -1] += 0.05; x[:, :, 0] += 0.05; x[:, :, -1] += 0.05
        x = x.to(torch.bfloat16).view(frames, hw, C)
    # per-slot partials of even pixel runs, as a conv epilogue leaves them (fp32 sums)
    xs = x.float().view(frames, slots, -1, C // 8, 2, 4) if hw % slots == 0 else None
    assert xs is not None, "the 4K frame splits evenly into its slots"
    part = torch.stack([xs.sum((2, 5)), (xs * xs).sum((2, 5))], -1).contiguous()
    return x, part


print(torch.cuda.get_device_name(), "power limit (W):",
      os.popen("nvidia-smi --query-gpu=power.limit --format=csv,noheader").read().strip())
for kind in ("normal", "flat"):
    x, part = data(kind)
    runs = {
        "stand-alone": lambda: lib.call("svr2_groupnorm_bf16", lib.ptr(x), lib.ptr(y), frames, hw, C, lib.ptr(g),
                                        lib.ptr(b), 1e-6, 1, 2, 1, lib.ptr(st), st.numel() * 8, lib.stream()),
        "fused": lambda: lib.call("svr2_groupnorm_from_stats_bf16", lib.ptr(x), lib.ptr(y), frames, hw, C, lib.ptr(g),
                                  lib.ptr(b), 1e-6, 1, 2, 1, lib.ptr(part), slots, lib.ptr(coef), lib.stream()),
    }
    for name, run in runs.items():
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            run()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        nb = (6.0 if name == "stand-alone" else 4.0) * x.numel()
        print(f"groupnorm {name:11s} {kind:6s} {frames}x{H}x{W}x{C}: {ms:.3f} ms, {nb / ms / 1e6:.0f} GB/s "
              f"({nb / x.numel():.0f} B/elem)")
    del x, part
