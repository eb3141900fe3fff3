"""-m gpu: weights that stay compressed in device memory (resident="compressed") — svr2_weight_expand_bf16 bit for bit
against the torch restatement, the DiT bit for bit against the expanded mode for GGUF and fp8 sources in both
sequencings, the memory it saves, the caller-provided workspace and CUDA-graph paths, and the module lifecycle."""
import gc
import importlib

import numpy as np
import pytest
import torch

from oracle import gguf_oracle as go
from oracle import resident_oracle as ro
from oracle.make_gguf_golden import random_blocks

pytestmark = pytest.mark.gpu
PREFIX = "model.diffusion_model."
CTA_ELEMS = 2048                      # outputs per CTA in gguf.cu
FORMATS = {name: ro.FMT_GGML + tid for name, (tid, _, _) in go.TYPES.items()}
FORMATS.update(F8_E4M3=ro.FMT_F8_E4M3, F16=ro.FMT_F16)


def same(a: torch.Tensor, b: torch.Tensor) -> bool:
    """bit-identical, NaN equal to NaN"""
    a, b = a.reshape(-1), b.reshape(-1)
    nan = torch.isnan(a) & torch.isnan(b)
    return bool(((a.view(torch.int16) == b.view(torch.int16)) | nan).all())


def stored_matrix(name: str, rows: int, cols: int, seed: int) -> torch.Tensor:
    """Random bytes of a rows x cols matrix in the named format, on the GPU."""
    fmt = FORMATS[name]
    if fmt >= ro.FMT_GGML:
        be = go.TYPES[name][1]
        return torch.from_numpy(random_blocks(name, rows * cols // be, seed=seed)).reshape(-1).cuda()
    g = torch.Generator().manual_seed(seed)
    if fmt == ro.FMT_F16:
        x = torch.randn(rows, cols, generator=g) * torch.exp(torch.rand(rows, cols, generator=g) * 40 - 30)
        x.view(-1)[:4] = torch.tensor([65504.0, -7e4, float("inf"), -0.0])      # fp16 max, overflow to inf, inf, -0
        return x.half().view(torch.uint8).reshape(-1).cuda()
    return torch.randint(0, 256, (rows * cols,), dtype=torch.uint8, generator=g).cuda()


def expand(svr2lib, fmt, raw, rows, cols, dst, group, stride, offset):
    svr2lib.call("svr2_weight_expand_bf16", fmt, svr2lib.ptr(raw), rows, cols, svr2lib.ptr(dst), group, stride, offset,
                 svr2lib.stream())


@pytest.mark.parametrize("name", list(FORMATS))
def test_kernel_equals_oracle(svr2lib, name):
    fmt = FORMATS[name]
    # identity row map: whole CTAs, fewer outputs than one CTA, and a size that is not a multiple of a CTA's outputs
    for rows, cols in ((384, 512), (3, 256), (7, 768)):
        raw = stored_matrix(name, rows, cols, seed=fmt)
        want = ro.expand(fmt, raw, rows, cols)
        for shift in (0, 4):              # the same bytes 4 bytes past a 16-byte boundary
            buf = torch.empty(raw.numel() + 16, dtype=torch.uint8, device="cuda")
            src = buf[shift:shift + raw.numel()]
            src.copy_(raw)
            assert src.data_ptr() % 16 == shift
            got = torch.full((rows, cols), 7.0, dtype=torch.bfloat16, device="cuda")
            expand(svr2lib, fmt, src, rows, cols, got, rows, rows, 0)
            assert same(got, want), (name, rows, cols, shift)
    assert (7 * 768) % CTA_ELEMS and 3 * 256 < CTA_ELEMS
    # the two SwiGLU maps: gate rows to [256 j, 256 j + 128), proj_in rows to [256 j + 128, 256 j + 256)
    hid, cols = 384, 256
    gate, up = stored_matrix(name, hid, cols, seed=fmt + 100), stored_matrix(name, hid, cols, seed=fmt + 200)
    g_bf, u_bf = ro.expand(fmt, gate, hid, cols), ro.expand(fmt, up, hid, cols)
    want = torch.stack([g_bf.view(hid // 128, 128, cols), u_bf.view(hid // 128, 128, cols)], 1).reshape(2 * hid, cols)
    assert same(ro.swiglu_matrix(g_bf, u_bf), want)
    got = torch.full((2 * hid, cols), 7.0, dtype=torch.bfloat16, device="cuda")
    expand(svr2lib, fmt, gate, hid, cols, got, 128, 256, 0)
    assert same(got[:128], want[:128]) and bool((got[128:256] == 7.0).all())      # only the gate rows are written
    expand(svr2lib, fmt, up, hid, cols, got, 128, 256, 128)
    assert same(got, want), name


def test_fp8_all_byte_values(svr2lib):
    raw = torch.arange(256, dtype=torch.uint8).repeat(8).cuda()                  # 8 x 256: every value in every row
    got = torch.empty(8, 256, dtype=torch.bfloat16, device="cuda")
    expand(svr2lib, ro.FMT_F8_E4M3, raw, 8, 256, got, 8, 8, 0)
    want = raw.view(torch.float8_e4m3fn).reshape(8, 256).to(torch.bfloat16)
    assert same(got, want)
    assert torch.isnan(got[0, 0x7F]) and torch.isnan(got[0, 0xFF]) and int(torch.isnan(got).sum()) == 16
    finite = ~torch.isnan(want)
    assert torch.equal(got[finite].float(), raw.view(torch.float8_e4m3fn).reshape(8, 256)[finite].float())   # exact


def test_bad_arguments_launch_nothing(svr2lib):
    lib = svr2lib.load()
    raw = torch.zeros(4 * 144, dtype=torch.uint8, device="cuda")
    dst = torch.full((4, 256), 7.0, dtype=torch.bfloat16, device="cuda")
    args = lambda fmt, rows, cols, group: (fmt, svr2lib.ptr(raw), rows, cols, svr2lib.ptr(dst), group, group, 0,
                                           svr2lib.stream())
    assert lib.svr2_weight_expand_bf16(*args(ro.FMT_GGML + 12, 4, 128, 4)) == -1       # cols not a whole Q4_K block
    assert lib.svr2_weight_expand_bf16(*args(ro.FMT_GGML + 20, 4, 256, 4)) == -1       # IQ4_NL
    assert lib.svr2_weight_expand_bf16(*args(1, 4, 256, 4)) == -1                      # bf16 is not a storage format
    assert lib.svr2_weight_expand_bf16(*args(ro.FMT_GGML + 12, 4, 256, 3)) == -1       # group does not divide rows
    torch.cuda.synchronize()
    assert bool((dst == 7.0).all())


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
    """Stand-in for the reference's GGUFTensor: raw block bytes whose shape / size() / numel() report the logical shape."""

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


def is_block_matrix(key, v) -> bool:
    return key.startswith("blocks.") and key.endswith(".weight") and len(v.shape) == 2 and \
        (".attn.proj_" in key or ".mlp." in key)


def sources(pkg, sd, meta, path):
    """The three storage forms of one model: the GGUF file, reference-style GGUFTensor entries with their bytes on the
    GPU, and a state dict whose block matrices are float8_e4m3fn."""
    ref_style = {}
    for k, (t, raw, shape) in meta.items():
        r = torch.from_numpy(raw.copy())
        if t in (go.F32, go.F16):
            ref_style[k] = r.view(torch.float32 if t == go.F32 else torch.float16).reshape(shape)
        else:
            ref_style[k] = RefStyleGGUFTensor(r.reshape(shape[0], -1).cuda(), t, shape)
    fp8 = {k: (v.to(torch.float8_e4m3fn) if is_block_matrix(k, v) else v) for k, v in sd.items()}
    return {"gguf": pkg.weights.load_gguf(path), "ref": ref_style, "fp8": fp8}


def model(pkg, tmp_path, name, seed=5):
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    variant, over, thw = CONFIGS[name]
    cfg = dit.dit_config(variant, **over)
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=seed)
    path = str(tmp_path / f"{name}.gguf")
    meta = write_model_gguf(path, sd)
    return dit, cfg, sd, meta, path, thw


def inputs(T, H, W):
    g = torch.Generator().manual_seed(3)
    return torch.randn(T * H * W, 33, generator=g).cuda(), torch.randn(58, 64, generator=g).cuda()


@pytest.mark.parametrize("name", list(CONFIGS))
def test_compressed_equals_expanded(pkg, tmp_path, name):
    dit, cfg, sd, meta, path, (T, H, W) = model(pkg, tmp_path, name)
    assert {t for t, _, _ in meta.values()} >= {12, 8, go.F16, go.F32}
    vid, txt = inputs(T, H, W)
    for label, src in sources(pkg, sd, meta, path).items():
        outs = {}
        for resident in ("expanded", "compressed"):
            m = dit.B200NaDiT(cfg, src, resident=resident)
            assert (len(list(m.C.keys())) > 0) == (resident == "compressed") and (m.slot_bytes > 0) == (resident == "compressed")
            for native in (True, False):
                m.native = native
                outs[resident, native] = m(vid, txt, [[T, H, W]], [[58]]).vid_sample.clone()
            del m
        for native in (True, False):          # per sequencing, as the two sequencings' RoPE tables may round a tie apart
            assert torch.isfinite(outs["expanded", native].float()).all()
            assert torch.equal(outs["compressed", native], outs["expanded", native]), (label, native)


def held_by(make):
    gc.collect()                       # modules of earlier tests sit in reference cycles: free them before the baseline
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    m = make()
    m.native_handle()
    torch.cuda.synchronize()
    gc.collect()
    return m, torch.cuda.memory_allocated() - base


@pytest.mark.parametrize("name", list(CONFIGS))
def test_compressed_mode_saves_the_memory(pkg, tmp_path, name):
    dit, cfg, sd, meta, path, (T, H, W) = model(pkg, tmp_path, name, seed=6)
    ck = pkg.weights.load_gguf(path)
    m_e, held_e = held_by(lambda: dit.B200NaDiT(cfg, ck))
    ws_e = m_e.workspace_bytes(T, H, W, 58)
    n_buffers = len(list(m_e.buffers()))
    del m_e
    m_c, held_c = held_by(lambda: dit.B200NaDiT(cfg, ck, resident="compressed"))
    # independently of the module: the block matrices of the file, as stored and as bf16 (shared layers hold one set)
    raw_bytes = sum(raw.nbytes for k, (t, raw, shape) in meta.items() if is_block_matrix(k, sd[k]))
    bf16_bytes = sum(2 * sd[k].numel() for k in meta if is_block_matrix(k, sd[k]))
    assert all(meta[k][0] not in (go.F32, go.F16) for k in meta if is_block_matrix(k, sd[k]))
    assert held_e >= sum(2 * v.numel() for k, v in sd.items() if v.ndim == 2 and k.startswith("blocks."))
    slack = 512 * (n_buffers + 16)         # the allocator rounds every tensor up to 512 bytes
    assert held_c <= held_e - bf16_bytes + raw_bytes + slack, (held_c, held_e, bf16_bytes, raw_bytes)
    assert bf16_bytes > 3 * raw_bytes // 2 and held_c < held_e
    # the staging slot: the largest block's matrices in bf16, each a multiple of 256 bytes here
    d, inner = cfg["dim"], cfg["heads"] * 128
    hid = pkg.weights.swiglu_hidden(d) if cfg["mlp"] == "swiglu" else 4 * d
    stream = 2 * (3 * inner * d + d * inner + (2 if cfg["mlp"] == "swiglu" else 1) * hid * d + d * hid)
    slot = 2 * stream                      # layer 0 has separate video and text weights in both configs
    assert slot % 256 == 0 and m_c.slot_bytes == slot
    assert m_c.workspace_bytes(T, H, W, 58) - ws_e == slot
    del m_c
    dense = {k: v for k, v in sd.items()}
    m_d = dit.B200NaDiT(cfg, dense, resident="compressed")
    assert len(list(m_d.C.keys())) == 0 and m_d.workspace_bytes(T, H, W, 58) == ws_e


def test_engine_workspace_and_cuda_graph(pkg, tmp_path, monkeypatch):
    from safetensors.torch import save_file
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    dit, cfg, sd, meta, path, _ = model(pkg, tmp_path, "dit3b_tiny_img", seed=7)
    vae_path = str(tmp_path / "vae.safetensors")
    save_file({k: v.contiguous() for k, v in pkg.weights.synth_vae_state_dict(seed=8).items()}, vae_path)
    txt = torch.randn(58, 64, generator=torch.Generator().manual_seed(9))
    # the tiny width is not one of the two shipped variants: hand build_engine its config
    monkeypatch.setattr(pkg.weights, "detect_dit_variant", lambda sd: "3b")
    monkeypatch.setattr(pipeline, "dit_config", lambda v: cfg)
    frames = torch.rand(5, 36, 52, 3, generator=torch.Generator().manual_seed(3)).cuda()
    other = torch.rand(5, 36, 52, 3, generator=torch.Generator().manual_seed(4)).cuda()
    eng = pipeline.build_engine(path, vae_path, txt)
    assert eng.dit.resident == "expanded"
    want, want_other = (eng.upscale_clip(f, seed=11, resolution=72) for f in (frames, other))
    del eng
    eng = pipeline.build_engine(path, vae_path, txt, dit_resident="compressed")
    assert eng.dit.resident == "compressed" and eng.dit.slot_bytes > 0
    assert torch.equal(eng.upscale_clip(frames, seed=11, resolution=72), want)
    graphed = eng.graphed(frames, seed=11, resolution=72)
    assert torch.equal(graphed(frames, clone=True), want)
    assert torch.equal(graphed(other, clone=True), want_other)          # the slot is filled again on every replay
    assert torch.equal(graphed(frames, clone=True), want)


def test_lifecycle(pkg, svr2lib, tmp_path):
    dit, cfg, sd, meta, path, (T, H, W) = model(pkg, tmp_path, "dit3b_tiny_img", seed=8)
    vid, txt = inputs(T, H, W)
    m = dit.B200NaDiT(cfg, pkg.weights.load_gguf(path), resident="compressed")
    run = lambda: m(vid, txt, [[T, H, W]], [[58]]).vid_sample.clone()
    want = run()
    stored = {k: m.C[k] for k in m.C.keys()}
    assert stored and all(b.dtype == torch.uint8 and b.is_cuda for b in stored.values())
    assert all(any(b is c for b in m.buffers()) for c in stored.values())        # buffers(): the lifecycle reaches them
    assert m.half() is m and m.to(torch.float16) is m and m.float() is m           # dtype casts are refused
    assert all(m.C[k].dtype == torch.uint8 for k in m.C.keys())
    m.to("cpu")
    assert all(not m.C[k].is_cuda for k in m.C.keys())
    with pytest.raises(svr2lib.Svr2Error):
        run()
    m.to("cuda")
    assert torch.equal(run(), want)
    m.native = False
    python_seq = run()
    m.to("cpu").to("cuda")                                                        # the staging tensor is rebuilt
    assert torch.equal(run(), python_seq)
    m.native = True
    for t in list(m.parameters()) + list(m.buffers()):                            # a release: every tensor loses its storage
        t.data = torch.empty(0, dtype=t.dtype, device=t.device)
    assert all(m.C[k].numel() == 0 for k in m.C.keys())
    with pytest.raises(svr2lib.Svr2Error):
        run()
