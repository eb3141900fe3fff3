"""CPU: resident="compressed" without a device — the oracle's row map against a plain interleave, which state-dict
entries stay compressed for 3B- and 7B-like tiny models, the staging slot's size, the refusal of an unknown mode, and
the new entry point in the header and the library."""
import ctypes
import importlib
import os
import re

import pytest
import torch

from oracle import resident_oracle as ro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = {"3b": dict(dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64),
           "7b": dict(dim=384, heads=3, layers=3, mm_layers=3, txt_in_dim=64)}
Q4_K, Q8_0 = 12, 8


class Quantized:
    """A state-dict entry with the two attributes the loader recognises a GGUF-quantized tensor by."""

    def __init__(self, tensor_type, shape):
        self.tensor_type, self.tensor_shape = tensor_type, torch.Size(shape)


@pytest.fixture(scope="module")
def dit(pkg):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")


def test_oracle_row_map_is_the_swiglu_interleave():
    g = torch.Generator().manual_seed(0)
    hid, d = 384, 64
    gate, up = torch.randn(hid, d, generator=g).bfloat16(), torch.randn(hid, d, generator=g).bfloat16()
    want = torch.stack([gate.view(hid // 128, 128, d), up.view(hid // 128, 128, d)], 1).reshape(2 * hid, d)
    assert torch.equal(ro.swiglu_matrix(gate, up), want)
    assert torch.equal(ro.row_map(5, 5, 5, 0), torch.arange(5))                       # the identity
    assert ro.row_map(256, 128, 256, 128).tolist() == list(range(128, 256)) + list(range(384, 512))
    x = torch.randn(6, 8, generator=g).bfloat16()
    assert torch.equal(ro.place(torch.zeros(6, 8, dtype=torch.bfloat16), x, 6, 6, 0), x)


def block_matrix_keys(cfg):
    """engine name -> state-dict keys, written out from the model's structure"""
    out = {}
    for i in range(cfg["layers"]):
        shared = i >= cfg["mm_layers"]
        last = cfg["last_vid_only"] and i == cfg["layers"] - 1
        for s in (("vid",) if shared else ("vid", "txt")):
            k, p = ("all" if shared else s), f"blocks.{i}."
            out[f"{i}.{s}.qkv.w"] = [p + f"attn.proj_qkv.{k}.weight"]
            out[f"{i}.{s}.out.w"] = [p + f"attn.proj_out.{k}.weight"]
            if last and s == "txt":
                continue
            out[f"{i}.{s}.mlp_in.w"] = ([p + f"mlp.{k}.proj_in_gate.weight"] if cfg["mlp"] == "swiglu" else []) + \
                [p + f"mlp.{k}.proj_in.weight"]
            out[f"{i}.{s}.mlp_out.w"] = [p + f"mlp.{k}.proj_out.weight"]
    return out


@pytest.mark.parametrize("variant", ["3b", "7b"])
@pytest.mark.parametrize("storage", ["fp8", "gguf"])
def test_compressed_mode_selects_the_block_matrices(pkg, dit, svr2lib, variant, storage):
    cfg = dit.dit_config(variant, **CONFIGS[variant])
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=1)
    assert dit.compressed_matrices(cfg, sd) == {}                  # a dense checkpoint has nothing to keep compressed
    stored = {}
    for k, v in sd.items():                                         # every matrix of the file, not only the blocks'
        if v.ndim == 2 and v.shape[1] % 32 == 0:
            if storage == "fp8":
                stored[k] = v.to(torch.float8_e4m3fn)
            else:
                stored[k] = Quantized(Q4_K if v.shape[1] % 256 == 0 else Q8_0, v.shape)
        else:
            stored[k] = v
    assert dit.storage_format(stored["txt_in.weight"]) is not None  # compressible, but not a block matrix
    plan = dit.compressed_matrices(cfg, stored)
    want = block_matrix_keys(cfg)
    assert {n: [p.key for p in parts] for n, parts in plan.items()} == want
    n_shared = cfg["layers"] - cfg["mm_layers"]
    assert sum(n.split(".")[1] == "txt" for n in plan) == (4 * cfg["mm_layers"] if variant == "7b" else 4)
    assert all(f"{i}.txt.qkv.w" not in plan for i in range(cfg["mm_layers"], cfg["layers"])) and n_shared == (variant == "3b")
    for name, parts in plan.items():
        for j, p in enumerate(parts):
            v = stored[p.key]
            assert (p.rows, p.cols) == tuple(v.tensor_shape if storage == "gguf" else v.shape)
            if storage == "fp8":
                assert p.format == svr2lib.FMT_F8_E4M3
            else:
                assert p.format == svr2lib.FMT_GGML + v.tensor_type
            if len(parts) == 2:
                assert (p.row_group, p.group_stride, p.row_offset) == (128, 256, 128 * j)
            else:
                assert (p.row_group, p.group_stride, p.row_offset) == (p.rows, p.rows, 0)


def test_mixed_swiglu_halves(pkg, dit, svr2lib):
    """A quantized gate with an fp16 proj_in stays compressed (fp16 expands to the same bf16); with an fp32 one the
    matrix is loaded expanded; a GGML type the kernel does not decode is left to the load-time path's refusal."""
    cfg = dit.dit_config("3b", **CONFIGS["3b"])
    sd = dict(pkg.weights.synth_dit_state_dict(cfg, seed=1))
    gate, up = "blocks.0.mlp.vid.proj_in_gate.weight", "blocks.0.mlp.vid.proj_in.weight"
    sd[gate] = Quantized(Q4_K, sd[gate].shape)
    plan = dit.compressed_matrices(cfg, sd)
    assert list(plan) == ["0.vid.mlp_in.w"]
    assert [p.format for p in plan["0.vid.mlp_in.w"]] == [svr2lib.FMT_GGML + Q4_K, svr2lib.FMT_F16]
    sd[up] = sd[up].float()
    assert dit.compressed_matrices(cfg, sd) == {}
    sd[gate] = Quantized(20, sd[up].shape)                          # IQ4_NL
    assert dit.storage_format(sd[gate]) is None and dit.compressed_matrices(cfg, sd) == {}


@pytest.mark.parametrize("variant", ["3b", "7b"])
def test_slot_is_the_largest_block(pkg, dit, variant):
    cfg = dit.dit_config(variant, **CONFIGS[variant])
    sd = {k: (v.to(torch.float8_e4m3fn) if v.ndim == 2 else v)
          for k, v in pkg.weights.synth_dit_state_dict(cfg, seed=1).items()}
    plan = dit.compressed_matrices(cfg, sd)
    offsets, slot = dit.slot_layout(cfg, plan)
    d, inner = cfg["dim"], cfg["heads"] * 128
    hid = pkg.weights.swiglu_hidden(d) if cfg["mlp"] == "swiglu" else 4 * d
    stream = 2 * (3 * inner * d + d * inner + (2 if cfg["mlp"] == "swiglu" else 1) * hid * d + d * hid)
    assert stream % 256 == 0 and slot == 2 * stream                # a layer with separate video and text weights
    assert dit.slot_layout(cfg, {}) == ([{} for _ in range(cfg["layers"])], 0)
    for i, layer in enumerate(offsets):
        assert set(layer) == {n for n in plan if n.startswith(f"{i}.")}
        ends = sorted((off, off + sum(p.rows for p in plan[n]) * plan[n][0].cols * 2) for n, off in layer.items())
        assert ends[0][0] == 0 and all(a[1] == b[0] for a, b in zip(ends, ends[1:])) and ends[-1][1] <= slot
    if variant == "3b":                                             # the shared, video-only last layer needs one stream
        assert max(o for o in offsets[1].values()) < stream
    # sizes that are not multiples of 256 bytes are rounded up, per matrix
    part = dit.MatrixPart("k", 3, 3, 40, 3, 3, 0)
    assert dit.slot_layout(dict(layers=1), {"0.vid.qkv.w": [part], "0.vid.out.w": [part]}) == \
        ([{"0.vid.qkv.w": 0, "0.vid.out.w": 256}], 512)


def test_unknown_resident_mode_is_refused(pkg, dit):
    cfg = dit.dit_config("3b", **CONFIGS["3b"])
    with pytest.raises(ValueError, match="resident"):
        dit.B200NaDiT(cfg, {}, device="cpu", resident="quantized")
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    with pytest.raises(ValueError, match="resident"):
        pipeline.SeedVR2Engine(cfg, {}, {}, torch.zeros(58, 64), device="cpu", dit_resident="fp8")


def test_entry_point_is_declared_bound_and_exported(svr2lib):
    hdr = open(os.path.join(ROOT, "include", "svr2.h")).read()
    assert re.search(r"\bint svr2_weight_expand_bf16\s*\(int format, const void\* src, int64_t rows, int64_t cols", hdr)
    assert "svr2_weight_expand_bf16" in svr2lib.SIGNATURES
    lib = svr2lib.load()
    fn = lib.svr2_weight_expand_bf16
    P = ctypes.c_void_p
    assert fn(svr2lib.FMT_GGML + Q4_K, P(16), 4, 100, P(16), 4, 4, 0, None) == -1      # cols not whole blocks
    assert "cols" in lib.svr2_last_error().decode()
    assert fn(svr2lib.FMT_F8_E4M3, P(16), 4, 12, P(16), 4, 4, 0, None) == -1           # 8 outputs would cross a row
    for fmt in (0, 1, 4, 15, 16 + 0, 16 + 1, 16 + 20, -1):                             # dense codes, F32 / F16 / IQ4_NL
        assert fn(fmt, P(16), 4, 256, P(16), 4, 4, 0, None) == -1, fmt
        assert f"format {fmt} " in lib.svr2_last_error().decode()
    assert fn(svr2lib.FMT_F16, P(16), 6, 256, P(16), 4, 4, 0, None) == -1              # group does not divide rows
    assert fn(svr2lib.FMT_F16, P(16), 256, 256, P(16), 128, 256, 192, None) == -1      # group overruns its stride
    assert fn(svr2lib.FMT_F16, P(18), 4, 256, P(16), 4, 4, 0, None) == -1              # source 2-byte aligned
    assert fn(svr2lib.FMT_F16, P(16), 4, 256, P(8), 4, 4, 0, None) == -1               # destination not 16-byte aligned
