"""Micro-benchmark of the wgmma GEMM / implicit-conv kernel on representative shapes
(used for ncu captures and kernel tuning; not a pytest)."""
import os, sys, importlib
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))  # repo root (this file lives in tools/)
sys.path.insert(0, ROOT)
from svr2_import import load_package
load_package()
lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
dev = "cuda"
only = sys.argv[1] if len(sys.argv) > 1 else ""
iters = int(os.environ.get("ITERS", "5"))

def timeit(fn, flops, name):
    for _ in range(2): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): fn()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    print(f"{name:44s} {ms:9.3f} ms  {flops / ms / 1e9:8.1f} TFLOP/s", flush=True)

def rnd(*s): return torch.randn(*s, device=dev, dtype=torch.bfloat16)

cases = []
# DiT linears at cfg2 (L = 40800)
L = 40800
for nm, N, K, epi in (("qkv", 7680, 2560, 0), ("out", 2560, 2560, 7), ("swiglu_in", 13824, 2560, 8), ("mlp_out", 2560, 6912, 6)):
    def mk(N=N, K=K, epi=epi):
        a, w = rnd(L, K), rnd(N, K)
        bias, gate = rnd(N), torch.randn(N, device=dev)
        res = rnd(L, N) if epi & 4 else None
        return lambda: lib.linear(a, w, bias=bias if epi & 1 else None, gate=gate if epi & 2 else None, residual=res,
                                  epi=epi & 8)
    cases.append((f"linear_{nm} {L}x{N}x{K}", mk, 2.0 * L * N * K))
# VAE convs (3x3x3), T frames at HxW
for nm, C_in, C_out, T, H, W in (("c128_720p", 128, 128, 3, 720, 1280), ("c256_720p", 256, 256, 2, 720, 1280),
                                  ("c256to128_720p", 256, 128, 3, 720, 1280),
                                  ("c512_360p", 512, 512, 3, 360, 640), ("c512_lat", 512, 512, 3, 136, 240)):
    def mk(C_in=C_in, C_out=C_out, T=T, H=H, W=W):
        x = rnd(T + 2, H, W, C_in); w = rnd(C_out, 27 * C_in); b = rnd(C_out)
        y = torch.empty(T, H, W, C_out, device=dev, dtype=torch.bfloat16)
        return lambda: lib.conv3d(x, T + 2, H, W, C_in, w, C_out, (3, 3, 3), 1, 1, 1, T, y, bias=b)
    cases.append((f"conv3d_{nm} {T}x{H}x{W}", mk, 2.0 * T * H * W * C_out * 27 * C_in))
# upsample shuffle 512 -> 4096 at 272x480
def mk_up():
    F_, H, W, C = 3, 272, 480, 512
    x = rnd(F_, H, W, C); w = rnd(8 * C, C); b = rnd(8 * C)
    y = torch.empty(2 + 2 * F_ - 1, 2 * H, 2 * W, C, device=dev, dtype=torch.bfloat16)
    return lambda: lib.call("svr2_upsample_shuffle_bf16", lib.ptr(x), F_, H, W, C, lib.ptr(w), lib.ptr(b), 1, 1,
                            lib.ptr(y), 2, 1, lib.stream())
cases.append(("upsample_512 3x272x480", mk_up, 2.0 * 3 * 272 * 480 * 512 * 4096))
# attention scores (VAE) : S = Q K^T fp32, n = 32640
def mk_s():
    n = 32640
    q, k = rnd(8192, 512), rnd(n, 512)
    S = torch.empty(8192, n, device=dev, dtype=torch.float32)
    return lambda: lib.linear(q, k, epi=lib.EPI_F32, out=S, out_scale=0.044)
cases.append(("vae_attn_S 8192x32640x512", mk_s, 2.0 * 8192 * 32640 * 512))
# DiT attention cfg2: 75 windows of 810+58
def mk_attn():
    lens = [868] * 75; heads = 20; total = sum(lens)
    q, k, v = rnd(total, heads, 128), rnd(total, heads, 128), rnd(total, heads, 128)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=dev)
    o = torch.empty_like(q)
    return lambda: lib.attn_varlen(q, k, v, cu, 868, out=o)
cases.append(("attn 75x868 h20", mk_attn, 75 * 20 * 4.0 * 868 * 868 * 128))
for name, mk, flops in cases:
    if only and only not in name: continue
    fn = mk()
    timeit(fn, flops, name)
    del fn
    torch.cuda.empty_cache()
