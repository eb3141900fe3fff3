"""Writes the GGUF fixtures under tests/golden/ (CPU; needs the reference tree and the `gguf` package).

1. For each of the eleven block types, random blocks — fp16 scales that are subnormal, negative or zero, every
   nibble / bit pattern at the block edges, BF16 values beyond the fp16 range — are decoded by the reference's own
   ``dequantize`` (``gguf_dequant.py:70-143``, ``dtype=torch.float16``, then ``.to(float16)`` as ``dequantize_tensor``
   does) and by ``oracle/gguf_oracle.py``; the two must agree bit for bit.  A few hundred blocks per type and the
   reference's fp16 output bits go to ``gguf_blocks.npz``.
2. ``gguf_fixture.gguf`` is written by ``gguf.GGUFWriter``: every supported type, F32 and F16 tensors, one type the
   engine does not decode (IQ4_NL), one tensor outside the ``model.diffusion_model.`` prefix, one
   ``comfy.gguf.orig_shape`` entry and a 64-byte alignment.  ``gguf_fixture.npz`` holds the tensor table that
   ``gguf.GGUFReader`` reports for it (name, type, logical shape as ``_get_tensor_logical_shape`` derives it, absolute
   byte offset, byte length).

Run: python -m oracle.make_gguf_golden
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import gguf_oracle as go  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
N_GOLDEN = {32: 256, 256: 64, 1: 4096}        # blocks per type in gguf_blocks.npz
FIXTURE_ALIGNMENT = 64
PREFIX = "model.diffusion_model."


def _scale_pool(g: np.random.Generator, n: int) -> np.ndarray:
    """fp16 scale bit patterns: normal values of either sign, subnormals, +-0; all finite and |x| <= 2."""
    kind = g.integers(0, 4, n)
    normal = (g.standard_normal(n) * 0.3).clip(-2, 2).astype(np.float16).view(np.uint16)
    sub = g.integers(1, 0x400, n).astype(np.uint16) | (g.integers(0, 2, n).astype(np.uint16) << 15)
    zero = (g.integers(0, 2, n).astype(np.uint16) << 15)
    neg = (-np.abs(g.standard_normal(n) * 0.05)).astype(np.float16).view(np.uint16)
    return np.select([kind == 0, kind == 1, kind == 2], [normal, sub, zero], neg).astype(np.uint16)


def random_blocks(name: str, n: int, seed: int) -> np.ndarray:
    """n blocks of `name`: random quant bytes (the first two blocks all zero / all one bits), valid fp16 scales."""
    tid, be, bb = go.TYPES[name]
    g = np.random.default_rng(seed)
    if name == "BF16":
        v = np.concatenate([g.standard_normal(n - 16) * np.exp(g.uniform(-30, 30, n - 16)),
                            [7e4, -7e4, 65504.0, 65520.0, 1e38, -3e38, 1e-8, -1e-9, 6e-8, 0.0, -0.0, np.inf, -np.inf,
                             1.0, -2.0, 3e-5]])
        return torch.from_numpy(v.astype(np.float32)).to(torch.bfloat16).view(torch.uint8).numpy().reshape(n, 2)
    b = g.integers(0, 256, (n, bb), dtype=np.uint8)
    b[0], b[1] = 0, 255
    d_off, m_off = go._D_OFF[name]
    for off in (d_off, m_off):
        if off is not None:
            b[:, off:off + 2] = _scale_pool(g, n).view(np.uint8).reshape(n, 2)
    return b


def reference_dequant(gd, gguf, name: str, blocks: np.ndarray) -> torch.Tensor:
    tid, be, bb = go.TYPES[name]
    data = torch.from_numpy(blocks.copy())
    out = gd.dequantize(data, gguf.GGMLQuantizationType(tid), (blocks.shape[0] * be,), dtype=torch.float16)
    return out.to(torch.float16)


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.dtype == b.dtype and torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def make_blocks(gd, gguf):
    arrays = {}
    for i, (name, (tid, be, bb)) in enumerate(go.TYPES.items()):
        big = random_blocks(name, 8192 if be > 1 else 65536, seed=100 + i)
        ref = reference_dequant(gd, gguf, name, big).reshape(big.shape[0], be)
        ours = go.dequantize(name, torch.from_numpy(big))
        assert not torch.isnan(ref).any(), name
        assert same_bits(ours, ref), f"{name}: oracle differs from the reference"
        n = N_GOLDEN[be]
        keep = np.concatenate([big[:2], big[-(n - 2):]])
        arrays[f"{name}_blocks"] = keep
        arrays[f"{name}_out"] = reference_dequant(gd, gguf, name, keep).view(torch.int16).numpy().view(np.uint16)
        print(f"{name:5s} id {tid:2d}: oracle == reference on {big.shape[0]} blocks; golden {n} blocks")
    np.savez_compressed(os.path.join(GOLD, "gguf_blocks.npz"), **arrays)


def make_fixture(gguf):
    """Every supported type as one 2-D tensor (rows of 256 elements), plus F32 / F16 / IQ4_NL / unprefixed tensors."""
    path = os.path.join(GOLD, "gguf_fixture.gguf")
    w = gguf.GGUFWriter(path, arch="seedvr2")
    w.data_alignment = FIXTURE_ALIGNMENT
    w.add_custom_alignment(FIXTURE_ALIGNMENT)
    g = torch.Generator().manual_seed(7)
    rows = 3
    for name, (tid, be, bb) in go.TYPES.items():
        x = torch.randn(rows, 256, generator=g)
        raw = go.encode(name, x).numpy().reshape(rows, -1)
        w.add_tensor(f"{PREFIX}blocks.{name.lower()}.weight", raw, raw_dtype=gguf.GGMLQuantizationType(tid))
    w.add_tensor(f"{PREFIX}vid_in.proj.weight", torch.randn(8, 132, generator=g).half().numpy(),
                 raw_dtype=gguf.GGMLQuantizationType.F16)
    w.add_tensor(f"{PREFIX}vid_in.proj.bias", torch.randn(8, generator=g).numpy(), raw_dtype=gguf.GGMLQuantizationType.F32)
    # a 5-D convolution-style weight stored as 2-D rows of 256, its logical shape in the metadata
    name5 = f"{PREFIX}conv.weight"
    raw5 = go.encode("Q8_0", torch.randn(4, 256, generator=g)).numpy().reshape(4, -1)
    w.add_tensor(name5, raw5, raw_dtype=gguf.GGMLQuantizationType.Q8_0)
    w.add_array(f"comfy.gguf.orig_shape.{name5}", [4, 4, 4, 4, 4])
    # IQ4_NL (type 20, 32 elements in 18 bytes): a block format the reference's table does not have
    w.add_tensor(f"{PREFIX}blocks.iq4_nl.weight", np.zeros((2, 2 * 18), dtype=np.uint8),
                 raw_dtype=gguf.GGMLQuantizationType.IQ4_NL)
    w.add_tensor("text_encoder.weight", torch.randn(4, 32, generator=g).numpy(), raw_dtype=gguf.GGMLQuantizationType.F32)
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()

    r = gguf.GGUFReader(path)
    names, types, shapes, offsets, nbytes = [], [], [], [], []
    for t in r.tensors:
        f = r.get_field(f"comfy.gguf.orig_shape.{t.name}")
        shape = [int(f.parts[i][0]) for i in f.data] if f is not None else [int(v) for v in reversed(t.shape)]
        names.append(t.name)
        types.append(int(t.tensor_type))
        shapes.append(shape + [0] * (5 - len(shape)))
        offsets.append(int(t.data_offset))
        nbytes.append(int(t.n_bytes))
    np.savez(os.path.join(GOLD, "gguf_fixture.npz"), names=np.array(names), types=np.array(types),
             shapes=np.array(shapes, dtype=np.int64), ranks=np.array([len(s) - s.count(0) for s in shapes]),
             offsets=np.array(offsets, dtype=np.int64), nbytes=np.array(nbytes, dtype=np.int64),
             alignment=np.array(r.alignment))
    print(f"{path}: {len(names)} tensors, alignment {r.alignment}, {os.path.getsize(path)} bytes")


def main():
    from oracle import ref_import
    ref_import.install_stubs()
    import gguf
    from src.optimization import gguf_dequant as gd
    make_blocks(gd, gguf)
    make_fixture(gguf)


if __name__ == "__main__":
    main()
