"""Can an HBM-bound GroupNorm run concurrently with the persistent wgmma conv kernel (2 streams)?"""
import os, sys, importlib, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from svr2_import import load_package
load_package()
lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
dev = "cuda"
def rnd(*s): return torch.randn(*s, device=dev, dtype=torch.bfloat16)
T, H, W, C = 2, 1080, 1920, 256
x = rnd(T + 2, H, W, C); w = rnd(C, 27 * C) * 0.01; b = rnd(C); y = torch.empty(T, H, W, C, device=dev, dtype=torch.bfloat16)
conv = lambda: lib.conv3d(x, T + 2, H, W, C, w, C, (3, 3, 3), 1, 1, 1, T, y, bias=b)
frames, hw, Cg = 2, 2160 * 3840, 128
gx = rnd(frames, hw, Cg); gy = torch.empty(2 + frames, hw, Cg, device=dev, dtype=torch.bfloat16)
g = torch.ones(Cg, device=dev, dtype=torch.bfloat16); bb = torch.zeros(Cg, device=dev, dtype=torch.bfloat16)
need = lib.load().svr2_groupnorm_scratch_bytes(frames, hw, Cg)
st = torch.empty(need // 8 + 8, device=dev, dtype=torch.float64)
gn = lambda: lib.call("svr2_groupnorm_bf16", lib.ptr(gx), lib.ptr(gy), frames, hw, Cg, lib.ptr(g), lib.ptr(bb), 1e-6, 1, 2, 1, lib.ptr(st), st.numel() * 8, lib.stream())
s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
def timed(fn, n=5):
    for _ in range(2): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
def both_serial(): conv(); gn()
def both_conc():
    cur = torch.cuda.current_stream()
    s1.wait_stream(cur); s2.wait_stream(cur)
    with torch.cuda.stream(s1): conv()
    with torch.cuda.stream(s2): gn()
    cur.wait_stream(s1); cur.wait_stream(s2)
def both_conc_gn_first():
    cur = torch.cuda.current_stream()
    s1.wait_stream(cur); s2.wait_stream(cur)
    with torch.cuda.stream(s2): gn()
    with torch.cuda.stream(s1): conv()
    cur.wait_stream(s1); cur.wait_stream(s2)
print(f"conv alone {timed(conv):.2f} ms | gn alone {timed(gn):.2f} ms | serial {timed(both_serial):.2f} ms | "
      f"concurrent (conv first) {timed(both_conc):.2f} ms | concurrent (gn first) {timed(both_conc_gn_first):.2f} ms")
