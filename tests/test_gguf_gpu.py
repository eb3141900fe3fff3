"""-m gpu: svr2_gguf_dequant_f16 (csrc/gguf.cu) bit for bit against the reference's decoded blocks and against the
fp16 restatement run on the same GPU; GGUF DiT checkpoints through B200NaDiT and build_engine."""
import gc
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import gguf_oracle as go
from oracle.make_gguf_golden import random_blocks

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
PREFIX = "model.diffusion_model."
CTA_ELEMS = 2048                      # outputs per CTA in gguf.cu


def kernel(svr2lib, ttype, raw: torch.Tensor, n: int) -> torch.Tensor:
    out = torch.empty(n, dtype=torch.float16, device="cuda")
    svr2lib.call("svr2_gguf_dequant_f16", ttype, svr2lib.ptr(raw), n, svr2lib.ptr(out), svr2lib.stream())
    return out


def same(a: torch.Tensor, b: torch.Tensor) -> bool:
    """bit-identical, NaN equal to NaN"""
    a, b = a.reshape(-1), b.reshape(-1)
    nan = torch.isnan(a) & torch.isnan(b)
    return bool(((a.view(torch.int16) == b.view(torch.int16)) | nan).all())


def test_kernel_reproduces_the_reference_blocks(svr2lib):
    g = np.load(os.path.join(GOLD, "gguf_blocks.npz"))
    for name, (tid, be, bb) in go.TYPES.items():
        blocks = torch.from_numpy(g[f"{name}_blocks"]).cuda()
        want = torch.from_numpy(g[f"{name}_out"].view(np.int16)).cuda().view(torch.float16)
        assert same(kernel(svr2lib, tid, blocks, blocks.shape[0] * be), want), name


@pytest.mark.parametrize("name", list(go.TYPES))
def test_kernel_equals_oracle_on_the_gpu(svr2lib, name):
    """12288x3072, one block, a block count that is not a whole number of CTAs, a 4- but not 16-byte aligned source."""
    tid, be, bb = go.TYPES[name]
    full = torch.from_numpy(random_blocks(name, 12288 * 3072 // be, seed=tid)).cuda()
    cta_blocks = CTA_ELEMS // be
    cases = [full, full[:1], full[:3 * cta_blocks + 5], full[:cta_blocks - 1]]
    for blocks in cases:
        n = blocks.shape[0] * be
        want = go.dequantize(name, blocks)
        assert same(kernel(svr2lib, tid, blocks.contiguous(), n), want), (name, blocks.shape[0])
        # the same bytes 4 bytes past a 16-byte boundary
        buf = torch.empty(blocks.numel() + 16, dtype=torch.uint8, device="cuda")
        shifted = buf[4:4 + blocks.numel()]
        shifted.copy_(blocks.reshape(-1))
        assert shifted.data_ptr() % 16 == 4
        assert same(kernel(svr2lib, tid, shifted, n), want), (name, blocks.shape[0], "offset 4")
    if name == "BF16":                                   # element counts that are not a multiple of 8
        for n in (1, 7, 2048 + 3):
            assert same(kernel(svr2lib, tid, full[:n].contiguous(), n), go.dequantize(name, full[:n])), n


# ---- whole model -------------------------------------------------------------------------------------------------
CONFIGS = {"dit3b_tiny_img": ("3b", dict(dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64), (1, 64, 64)),
           "dit7b_tiny_t3": ("7b", dict(dim=384, heads=3, layers=3, mm_layers=3, txt_in_dim=64), (3, 40, 72))}
K_MIX = ("Q4_K", "Q6_K", "Q5_K")


def write_model_gguf(path, sd):
    """A `_M`-like mix: K-quants where rows are whole 256-element blocks, Q8_0 where they are whole 32-element blocks,
    F16 for other matrices (vid_in has 132 columns), F32 for 1-D tensors.  Returns {key: (type, raw uint8, shape)}."""
    tensors, meta = [], {}
    for i, (k, v) in enumerate(sd.items()):
        if v.ndim == 1:
            t, raw = go.F32, v.float().numpy().view(np.uint8)
        elif v.shape[-1] % 256 == 0:
            name = K_MIX[i % 3]
            t, raw = go.TYPES[name][0], go.encode(name, v).numpy().reshape(-1)
        elif v.shape[-1] % 32 == 0:
            t, raw = 8, go.encode("Q8_0", v).numpy().reshape(-1)
        else:
            t, raw = go.F16, v.half().numpy().view(np.uint8).reshape(-1)
        tensors.append((PREFIX + k, t, list(reversed(v.shape)), raw))
        meta[k] = (t, raw, tuple(v.shape))
    go.write_gguf(path, tensors)
    return meta


class RefStyleGGUFTensor(torch.Tensor):
    @staticmethod
    def __new__(cls, raw, tensor_type, tensor_shape):
        t = torch.Tensor._make_subclass(cls, raw)
        t.tensor_type, t.tensor_shape = tensor_type, torch.Size(tensor_shape)
        return t

    @property
    def shape(self):
        return self.tensor_shape

    def size(self, *args):
        return self.tensor_shape if not args else self.tensor_shape[args[0]]

    def numel(self):
        return int(np.prod(self.tensor_shape))


def three_inputs(pkg, meta, path):
    """load_gguf(path); reference-style GGUFTensor entries (bytes on the GPU, as the reference loads them); the dense
    dict with every quantized entry replaced by the oracle's fp16 dequantization (on the CPU)."""
    ref_style, dense = {}, {}
    for k, (t, raw, shape) in meta.items():
        r = torch.from_numpy(raw.copy())
        if t == go.F32:
            ref_style[k] = dense[k] = r.view(torch.float32).reshape(shape)
        elif t == go.F16:
            ref_style[k] = dense[k] = r.view(torch.float16).reshape(shape)
        else:
            ref_style[k] = RefStyleGGUFTensor(r.reshape(shape[0], -1).cuda(), t, shape)
            dense[k] = go.dequantize_tensor(t, r, shape)
    return pkg.weights.load_gguf(path), ref_style, dense


@pytest.mark.parametrize("name", list(CONFIGS))
def test_gguf_dit_equals_dense_dit(pkg, tmp_path, name):
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    variant, over, (T, H, W) = CONFIGS[name]
    cfg = dit.dit_config(variant, **over)
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=5)
    path = str(tmp_path / f"{name}.gguf")
    meta = write_model_gguf(path, sd)
    assert {t for t, _, _ in meta.values()} >= {12, 8, go.F16, go.F32}
    g = torch.Generator().manual_seed(3)
    vid = torch.randn(T * H * W, 33, generator=g).cuda()
    txt = torch.randn(58, 64, generator=g).cuda()
    outs = {}
    for label, src in zip(("gguf", "ref", "dense"), three_inputs(pkg, meta, path)):
        m = dit.B200NaDiT(cfg, src)
        for native in (True, False):
            m.native = native
            outs[label, native] = m(vid, txt, [[T, H, W]], [[58]]).vid_sample.clone()
        del m
    # per sequencing (the two agree except where their RoPE tables round an fp16 tie differently, see
    # test_dit_native_runtime_equals_python_sequencing)
    for (label, native), v in outs.items():
        base = outs["dense", native]
        assert torch.isfinite(base.float()).all()
        assert torch.equal(v, base), (label, native)


def test_gguf_load_holds_one_temporary(pkg, tmp_path):
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    variant, over, _ = CONFIGS["dit7b_tiny_t3"]
    cfg = dit.dit_config(variant, **over)
    path = str(tmp_path / "m.gguf")
    meta = write_model_gguf(path, pkg.weights.synth_dit_state_dict(cfg, seed=6))
    ck, _, dense = three_inputs(pkg, meta, path)

    def peak(src):
        gc.collect()                   # modules of earlier tests sit in reference cycles: free them before the baseline
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        m = dit.B200NaDiT(cfg, src)
        torch.cuda.synchronize()
        p = torch.cuda.max_memory_allocated() - base
        del m
        gc.collect()
        return p

    p_dense, p_gguf = peak(dense), peak(ck)
    assert p_dense > 0
    q = [(int(np.prod(s)) * 2 + raw.nbytes) for t, raw, s in meta.values() if t not in (go.F32, go.F16)]
    assert p_gguf - p_dense <= max(q) + 2 * 512, (p_gguf, p_dense, max(q))


def test_build_engine_from_gguf(pkg, tmp_path, monkeypatch):
    from safetensors.torch import save_file
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    variant, over, _ = CONFIGS["dit3b_tiny_img"]
    cfg = dit.dit_config(variant, **over)
    path = str(tmp_path / "dit.gguf")
    meta = write_model_gguf(path, pkg.weights.synth_dit_state_dict(cfg, seed=7))
    _, _, dense = three_inputs(pkg, meta, path)
    vae_path = str(tmp_path / "vae.safetensors")
    save_file({k: v.contiguous() for k, v in pkg.weights.synth_vae_state_dict(seed=8).items()}, vae_path)
    txt = torch.randn(58, 64, generator=torch.Generator().manual_seed(9))
    # the tiny width is not one of the two shipped variants: hand build_engine its config
    monkeypatch.setattr(pkg.weights, "detect_dit_variant", lambda sd: variant)
    monkeypatch.setattr(pipeline, "dit_config", lambda v: cfg)
    eng = pipeline.build_engine(path, vae_path, txt)
    frames = torch.rand(5, 36, 52, 3, generator=torch.Generator().manual_seed(3)).cuda()
    out = eng.upscale_clip(frames, seed=11, resolution=72)
    graphed = eng.graphed(frames, seed=11, resolution=72)(frames, clone=True)
    del eng
    ref = pipeline.SeedVR2Engine(cfg, dense, pkg.weights.load_state_dict(vae_path), txt)
    want = ref.upscale_clip(frames, seed=11, resolution=72)
    assert torch.equal(out, want) and torch.equal(graphed, want)
