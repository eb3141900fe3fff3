"""Isolation timings of the epilogue-sensitive GEMM shapes of the 4K shard (short-K tiles, attention passes,
shuffle store).  SVR2_AB_LIB=<path to another libsvr2.so> loads that build next to the in-tree one and times the two
alternately in this process, ROUNDS times per case (default 3), so that both see the same clocks and neighbours."""
import os, sys, importlib
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from svr2_import import load_package
load_package()
lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
builds = [("tree", lib.load())]
if os.environ.get("SVR2_AB_LIB"):
    tree_path, lib._lib = lib.LIB_PATH, None
    lib.LIB_PATH = os.path.abspath(os.environ["SVR2_AB_LIB"])
    builds.append(("ab", lib.load()))
    lib.LIB_PATH = tree_path
rounds = int(os.environ.get("ROUNDS", "3" if len(builds) > 1 else "1"))
dev = "cuda"
only = sys.argv[1] if len(sys.argv) > 1 else ""
iters = int(os.environ.get("ITERS", "4"))
flush = torch.empty(256 << 20, device=dev, dtype=torch.uint8)

def timeit(fn, flops, name):
    for r in range(rounds):
        for tag, handle in builds:
            lib._lib = handle                   # lib.call dispatches through lib.load()
            for _ in range(2): fn()
            torch.cuda.synchronize()
            tot = 0.0
            for _ in range(iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); fn(); e1.record(); torch.cuda.synchronize()
                tot += e0.elapsed_time(e1)
            ms = tot / iters
            label = f"{name} [{tag} {r}]" if len(builds) > 1 else name
            print(f"{label:48s} {ms:9.3f} ms  {flops / ms / 1e9:8.1f} TFLOP/s", flush=True)
    lib._lib = builds[0][1]

def rnd(*s): return torch.randn(*s, device=dev, dtype=torch.bfloat16)

cases = []
L = 97200
for nm, N, K, epi in (("qkv_e0", 7680, 2560, 0), ("out_e7", 2560, 2560, 7), ("swiglu_e8", 13824, 2560, 8),
                      ("mlpout_e6", 2560, 6912, 6)):
    def mk(N=N, K=K, epi=epi):
        a, w = rnd(L, K), rnd(N, K) * 0.02
        bias, gate = rnd(N), torch.randn(N, device=dev)
        res = rnd(L, N) if epi & 4 else None
        return lambda: lib.linear(a, w, bias=bias if epi & 1 else None, gate=gate if epi & 2 else None, residual=res,
                                  epi=epi & 8)
    cases.append((f"linear_{nm} {L}x{N}x{K}", mk, 2.0 * L * N * K))
# VAE mid-block attention passes at the 4K latent (n = 129600, one 9472-row query chunk)
n, rows, C = 129600, 9472, 512
def mk_rowstat():
    q, k = rnd(rows, C), rnd(n, C)
    slots = lib.load().svr2_rowstat_slots(n)
    part = torch.empty(rows, 2 * slots, device=dev, dtype=torch.float32)
    return lambda: lib.linear(q, k, epi=lib.EPI_ROWSTAT, out=part, out_scale=0.0637)
def mk_pexp():
    q, k = rnd(rows, C), rnd(n + 8, C)
    lse = torch.full((rows,), 12.0, device=dev)
    P = torch.empty(rows, n, device=dev, dtype=torch.bfloat16)
    return lambda: lib.linear(q, k[:n], epi=lib.EPI_PEXP, gate=lse, out=P, out_scale=0.0637)
def mk_pexp_stat():                      # the single-pass probabilities: un-normalised exp2 + per-slot row sums
    q, k = rnd(rows, C), rnd(n, C)
    mhat = torch.full((rows,), 12.0, device=dev)
    P = torch.empty(rows, n, device=dev, dtype=torch.bfloat16)
    stat = torch.empty(rows, 2 * 2 * ((n + 255) // 256), device=dev)
    return lambda: lib.linear(q, k, epi=lib.EPI_PEXP, gate=mhat, out=P, out_scale=0.0637, stat_out=stat)
def mk_pv():
    P, vt = rnd(rows, n), rnd(C, n)
    return lambda: lib.linear(P, vt)
cases.append(("attn_rowstat_e256 9472x129600x512", mk_rowstat, 2.0 * rows * n * C))
cases.append(("attn_pexp_e512 9472x129600x512", mk_pexp, 2.0 * rows * n * C))
cases.append(("attn_pexp_stat_e512 9472x129600x512", mk_pexp_stat, 2.0 * rows * n * C))
cases.append(("attn_pv 9472x512x129600", mk_pv, 2.0 * rows * n * C))
def mk_up():
    T, H, W, C = 2, 1080, 1920, 256
    x = rnd(T, H, W, C); w = rnd(4 * C, C) * 0.05; b = rnd(4 * C)
    y = torch.empty(T + 2, 2 * H, 2 * W, C, device=dev, dtype=torch.bfloat16)
    return lambda: lib.call("svr2_upsample_shuffle_bf16", lib.ptr(x), T, H, W, C, lib.ptr(w), lib.ptr(b), 0, 1,
                            lib.ptr(y), 2, 1, lib.stream())
cases.append(("upsample_256 2x1080x1920", mk_up, 2.0 * 2 * 1080 * 1920 * 256 * 1024))
for nm, Cin, Cout, k3, T, H, W in (("sc256to128", 256, 128, 1, 2, 2160, 3840), ("sc512to256", 512, 256, 1, 4, 1080, 1920),
                                    ("c256", 256, 256, 3, 2, 1080, 1920), ("c128", 128, 128, 3, 2, 2160, 3840),
                                    ("c512", 512, 512, 3, 2, 540, 960)):   # longest K (13824): 3-stage ring
    def mk(Cin=Cin, Cout=Cout, k3=k3, T=T, H=H, W=W):
        pad = k3 - 1
        x = rnd(T + pad, H, W, Cin); w = rnd(Cout, k3 ** 3 * Cin) * 0.02; b = rnd(Cout)
        y = torch.empty(T, H, W, Cout, device=dev, dtype=torch.bfloat16)
        return lambda: lib.conv3d(x, T + pad, H, W, Cin, w, Cout, (k3, k3, k3), 1, 1, 1 if k3 == 3 else 0, T, y, bias=b)
    cases.append((f"conv_{nm} k{k3} {T}x{H}x{W}", mk, 2.0 * T * H * W * Cout * k3 ** 3 * Cin))
for name, mk, flops in cases:
    if only and only not in name: continue
    fn = mk()
    timeit(fn, flops, name)
    del fn
    torch.cuda.empty_cache()
