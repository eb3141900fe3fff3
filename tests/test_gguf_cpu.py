"""CPU: the GGUF reader against what gguf.GGUFReader recorded for tests/golden/gguf_fixture.gguf, its refusals, the
fp16 restatement against the reference's decoded blocks, the lazy dequantizing mapping and build_engine's routing
(kernel and engines stubbed), and the library's block-geometry table."""
import ctypes
import importlib
import os
import shutil
import struct

import numpy as np
import pytest
import torch

from oracle import gguf_oracle as go

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FIXTURE = os.path.join(GOLD, "gguf_fixture.gguf")
PREFIX = "model.diffusion_model."


def test_reader_matches_gguf_reader(pkg):
    ref = np.load(os.path.join(GOLD, "gguf_fixture.npz"))
    ck = pkg.weights.load_gguf(FIXTURE)
    want = {}
    for name, t, shape, rank, off, nb in zip(ref["names"], ref["types"], ref["shapes"], ref["ranks"], ref["offsets"],
                                             ref["nbytes"]):
        name = str(name)
        if name.startswith(PREFIX):                         # the prefix rule drops the unprefixed tensor
            want[name[len(PREFIX):]] = (name, int(t), tuple(int(s) for s in shape[:rank]), int(off), int(nb))
    assert len(want) == len(ref["names"]) - 1
    assert set(ck) == set(want) and len(ck) == len(want)
    for key, (name, t, shape, off, nb) in want.items():
        got_name, got_t, got_shape, got_off, got_nb = ck.infos[key]
        assert (got_name, got_t, tuple(got_shape), got_off) == (name, t, shape, off), key
        assert got_nb == (nb if t != 20 else None), key   # IQ4_NL: a type the engine does not decode
        v = ck[key]
        if t in (go.F32, go.F16):
            assert isinstance(v, torch.Tensor) and tuple(v.shape) == shape
            raw = np.fromfile(FIXTURE, dtype=np.uint8)[off:off + nb].view(np.float32 if t == go.F32 else np.float16)
            assert torch.equal(v, torch.from_numpy(raw.copy()).reshape(shape))
        else:
            assert (v.tensor_type, tuple(v.tensor_shape), tuple(v.shape)) == (t, shape, shape)
            if t != 20:
                assert v.data.tobytes() == np.fromfile(FIXTURE, dtype=np.uint8)[off:off + nb].tobytes()
    # orig_shape overrides the reversed GGUF dimensions (4 rows of 256 elements)
    assert tuple(ck["conv.weight"].tensor_shape) == (4, 4, 4, 4, 4)
    with pytest.raises(NotImplementedError, match="blocks.iq4_nl.weight"):
        ck["blocks.iq4_nl.weight"].data


def _copy(tmp_path, name, edit=None, size=None):
    p = str(tmp_path / name)
    shutil.copy(FIXTURE, p)
    data = bytearray(open(p, "rb").read())
    if edit:
        edit(data)
    open(p, "wb").write(bytes(data[:size] if size else data))
    return p


def test_reader_refusals(pkg, tmp_path):
    w = pkg.weights

    def bad_magic(d):
        d[0:4] = b"GGML"

    def v1(d):
        d[4:8] = struct.pack("<I", 1)

    with pytest.raises(ValueError, match="bad magic") as e:
        w.load_gguf(_copy(tmp_path, "magic.gguf", bad_magic))
    assert "magic.gguf" in str(e.value)
    with pytest.raises(ValueError, match="version 1") as e:
        w.load_gguf(_copy(tmp_path, "v1.gguf", v1))
    assert "v1.gguf" in str(e.value)
    last = max(w.load_gguf(FIXTURE).infos.values(), key=lambda i: i[3] + (i[4] or 0))
    with pytest.raises(ValueError, match="truncated") as e:
        w.load_gguf(_copy(tmp_path, "cut.gguf", size=last[3] + last[4] - 1))
    assert "cut.gguf" in str(e.value) and last[0] in str(e.value)
    # a Q4_K tensor whose rows hold 100 elements (not a whole number of 256-element blocks)
    p = str(tmp_path / "rows.gguf")
    go.write_gguf(p, [(PREFIX + "a.weight", 12, [100, 2], np.zeros(144, np.uint8))])
    with pytest.raises(ValueError, match="a.weight") as e:
        w.load_gguf(p)
    assert "rows.gguf" in str(e.value) and "block size 256" in str(e.value)


def test_reader_without_prefix_keeps_every_tensor(pkg, tmp_path):
    p = str(tmp_path / "plain.gguf")
    x = go.encode("Q8_0", torch.randn(2, 64)).numpy()
    go.write_gguf(p, [("w", 8, [64, 2], x), ("b", go.F32, [3], np.arange(3, dtype=np.float32).view(np.uint8))],
                  alignment=128, orig_shapes={"w": [1, 2, 64]})
    ck = pkg.weights.load_gguf(p)
    assert set(ck) == {"w", "b"} and tuple(ck["w"].tensor_shape) == (1, 2, 64)
    assert torch.equal(ck["b"], torch.arange(3, dtype=torch.float32))
    assert ck.infos["w"][3] % 128 == 0


def test_oracle_reproduces_the_reference_blocks():
    g = np.load(os.path.join(GOLD, "gguf_blocks.npz"))
    for name, (tid, be, bb) in go.TYPES.items():
        blocks = torch.from_numpy(g[f"{name}_blocks"])
        want = torch.from_numpy(g[f"{name}_out"].view(np.int16)).reshape(blocks.shape[0], be)
        got = go.dequantize(name, blocks).view(torch.int16)
        assert torch.equal(got, want), name


class RefStyleGGUFTensor(torch.Tensor):
    """Stand-in for the reference's GGUFTensor (model_loader.py:242-284): raw block bytes whose shape / size() /
    numel() report the logical shape."""

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


@pytest.fixture
def fake_kernel(svr2lib, monkeypatch):
    calls = []

    def call(name, *args, **kw):
        if name != "svr2_gguf_dequant_f16":
            raise AssertionError(name)
        ttype, src, n, out, _ = args
        calls.append((ttype, n, src.numel(), src.dtype))
        out.view(-1).copy_(go.dequantize(go.BY_ID[ttype], src.reshape(-1, go.TYPES[go.BY_ID[ttype]][2])).reshape(-1))

    monkeypatch.setattr(svr2lib, "call", call)
    monkeypatch.setattr(svr2lib, "ptr", lambda t: t)
    monkeypatch.setattr(svr2lib, "stream", lambda: None)
    return calls


def test_dequantizing_mapping(pkg, fake_kernel):
    w = pkg.weights
    ck = w.load_gguf(FIXTURE)
    sd = w.dequantizing(ck, "cpu")
    assert set(sd) == set(ck) and len(sd) == len(ck)
    for key in ("vid_in.proj.weight", "vid_in.proj.bias"):
        assert torch.equal(sd[key], ck[key])
    assert fake_kernel == []                                       # F32 / F16 never reach the kernel
    for key, (name, t, shape, off, nb) in ck.infos.items():
        if t in (go.F32, go.F16) or nb is None:
            continue
        before = len(fake_kernel)
        out = sd[key]
        assert fake_kernel[before:] == [(t, int(np.prod(shape)), nb, torch.uint8)], key
        assert out.dtype == torch.float16 and tuple(out.shape) == tuple(shape)
        raw = torch.from_numpy(np.fromfile(FIXTURE, dtype=np.uint8)[off:off + nb].copy())
        assert torch.equal(out, go.dequantize_tensor(t, raw, shape))
    with pytest.raises(NotImplementedError, match="iq4_nl"):
        sd["blocks.iq4_nl.weight"]
    assert sd.get("missing") is None


def test_dequantizing_reference_gguf_tensor(pkg, fake_kernel):
    raw = go.encode("Q4_K", torch.randn(6, 512)).reshape(6, -1)     # 6 rows of 2 blocks = 1728 bytes
    ref = RefStyleGGUFTensor(raw, 12, (6, 512))
    assert tuple(ref.shape) == (6, 512) and ref.numel() == 3072     # the logical view the reference reports
    sd = pkg.weights.dequantizing({"w": ref, "b": torch.ones(3)}, "cpu")
    out = sd["w"]
    assert fake_kernel == [(12, 3072, 6 * 2 * 144, torch.uint8)]
    assert torch.equal(out, go.dequantize_tensor(12, raw.reshape(-1), (6, 512)))
    assert torch.equal(sd["b"], torch.ones(3)) and len(fake_kernel) == 1


def test_build_engine_routes_gguf_through_load_gguf(pkg, monkeypatch, tmp_path):
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    w = pkg.weights
    seen = []
    monkeypatch.setattr(w, "load_gguf", lambda p: seen.append(("gguf", p)) or {"vid_in.proj.weight": torch.empty(3072, 132)})
    monkeypatch.setattr(w, "load_state_dict",
                        lambda p: seen.append(("dense", p)) or {"vid_in.proj.weight": torch.empty(2560, 132)})
    monkeypatch.setattr(pipeline, "SeedVR2Engine", lambda cfg, dit_sd, vae_sd, txt, device: (cfg["variant"], dit_sd))
    txt = torch.zeros(1, 58, 4096)
    v, sd = pipeline.build_engine("m/seedvr2_ema_7b-Q4_K_M.GGUF", "m/ema_vae_fp16.safetensors", txt)
    assert v == "7b" and seen == [("gguf", "m/seedvr2_ema_7b-Q4_K_M.GGUF"), ("dense", "m/ema_vae_fp16.safetensors")]
    for path in ("m/seedvr2_ema_3b_fp16.safetensors", "m/dit.pth"):
        seen.clear()
        v, _ = pipeline.build_engine(path, "m/ema_vae_fp16.safetensors", txt)
        assert v == "3b" and seen == [("dense", path), ("dense", "m/ema_vae_fp16.safetensors")]


def test_library_block_geometry(svr2lib):
    lib = svr2lib.load()
    e, b = ctypes.c_int(), ctypes.c_int()
    for name, (tid, be, bb) in go.TYPES.items():
        assert lib.svr2_gguf_type_size(tid, ctypes.byref(e), ctypes.byref(b)) == 0, name
        assert (e.value, b.value) == (be, bb), name
    for tid in (0, 1, 9, 15, 16, 20, 23, 29, 31, 34, 39, -1, 1000):    # F32, F16, Q8_1, Q8_K, IQ*, TQ*, MXFP4, ...
        assert lib.svr2_gguf_type_size(tid, ctypes.byref(e), ctypes.byref(b)) == -1, tid
        assert f"type {tid} " in lib.svr2_last_error().decode()
    assert lib.svr2_gguf_dequant_f16(20, None, 32, None, None) == -1
    assert "type 20" in lib.svr2_last_error().decode()
    assert lib.svr2_gguf_dequant_f16(12, ctypes.c_void_p(16), 100, ctypes.c_void_p(16), None) == -1   # not whole blocks
    assert lib.svr2_gguf_dequant_f16(8, ctypes.c_void_p(18), 32, ctypes.c_void_p(16), None) == -1    # 2-byte aligned
    assert lib.svr2_gguf_dequant_f16(8, ctypes.c_void_p(16), 32, ctypes.c_void_p(8), None) == -1     # out not 16-B
    assert lib.svr2_gguf_dequant_f16(8, ctypes.c_void_p(16), 0, ctypes.c_void_p(16), None) == -1
