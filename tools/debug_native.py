"""Bisect a native-runtime (svr2_dit_forward) vs Python-sequenced mismatch over config switches (GPU box)."""
import importlib, os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from svr2_import import load_package
pkg = load_package()
dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")


def run(label, variant, **over):
    cfg = dit.dit_config(variant, **over)
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=1234, dtype=torch.float16)
    g = torch.Generator().manual_seed(42)
    T, H, W, l = 3, 40, 72, 58
    vid, txt = torch.randn(T * H * W, cfg["in_ch"], generator=g).cuda(), torch.randn(l, cfg["txt_in_dim"], generator=g).cuda()
    eng = dit.B200NaDiT(cfg, sd)
    eng.native = True
    a = eng(vid, txt, [[T, H, W]], [[l]]).vid_sample.float().clone()
    a2 = eng(vid, txt, [[T, H, W]], [[l]]).vid_sample.float().clone()
    eng.native = False
    b = eng(vid, txt, [[T, H, W]], [[l]]).vid_sample.float()
    d = (a - b).abs()
    fuse = lib.dit_geometry(eng.native_handle(), T, H, W, l, 0).fuse_qkv
    print(f"{label:44s} equal={torch.equal(a, b)} native-deterministic={torch.equal(a, a2)} max|d|={d.max().item():.4f} "
          f"frac_diff={(d > 0).float().mean().item():.4f} fuse={fuse}", flush=True)


base = dict(dim=256, heads=2, layers=3, mm_layers=1, txt_in_dim=64)
run("3b base (heads 2)", "3b", **base)
run("3b heads=3 dim=384", "3b", **{**base, "dim": 384, "heads": 3})
run("3b mm_layers=3", "3b", **{**base, "mm_layers": 3})
run("3b mlp=gelu", "3b", **{**base, "mlp": "gelu"})
run("3b out_norm=False", "3b", **{**base, "out_norm": False})
run("3b last_vid_only=False", "3b", **{**base, "last_vid_only": False})
run("7b heads 2 dim 256", "7b", **{**base, "mm_layers": 3})
run("7b heads 3 dim 384 (golden config)", "7b", dim=384, heads=3, layers=3, mm_layers=3, txt_in_dim=64)
run("7b heads 3, 1 layer", "7b", dim=384, heads=3, layers=1, mm_layers=1, txt_in_dim=64)
run("7b rope but 3b-like rest", "7b", **{**base, "mlp": "swiglu", "out_norm": True, "last_vid_only": True})
