"""TEST INFRASTRUCTURE ONLY — GGUF block dequantization restated in torch fp16, plus an encoder and a GGUF writer to
build test checkpoints.

The reference dequantizes with ``dtype=torch.float16`` (``gguf_dequant.py:146-342``, called from
``GGUFQuantizedLinear`` at ``gguf_ops.py:110-136``): every torch op there is one Half op, computed in fp32 and rounded
to fp16.  ``dequantize`` below states each format as per-element bit fields (byte index, shift, width) gathered out of
the block, then runs the same sequence of fp16 ops on the blocks' device.  ``oracle/make_gguf_golden.py`` checks it
bit for bit against the reference's own functions; the committed ``tests/golden/gguf_blocks.npz`` pins it.

``encode`` is a plain round-to-nearest quantizer per type (any valid bytes would do: what the tests pin is the
decoding); it writes its fields through the same bit-field tables.  ``write_gguf`` writes a minimal GGUF v3 file.
"""
from __future__ import annotations

import struct
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

# name -> (GGML id, elements per block, bytes per block)
TYPES: Dict[str, Tuple[int, int, int]] = {
    "BF16": (30, 1, 2), "Q8_0": (8, 32, 34), "Q5_1": (7, 32, 24), "Q5_0": (6, 32, 22), "Q4_1": (3, 32, 20),
    "Q4_0": (2, 32, 18), "Q6_K": (14, 256, 210), "Q5_K": (13, 256, 176), "Q4_K": (12, 256, 144),
    "Q3_K": (11, 256, 110), "Q2_K": (10, 256, 84),
}
BY_ID = {v[0]: k for k, v in TYPES.items()}
F32, F16 = 0, 1

_E32 = np.arange(32)
_E256 = np.arange(256)


def _fields(name: str) -> Dict[str, Tuple[np.ndarray, np.ndarray, int]]:
    """Per-element bit fields of one block: field -> (byte index [BE], shift [BE], width in bits)."""
    E = _E32 if TYPES[name][1] == 32 else _E256
    if name in ("Q4_0", "Q4_1", "Q5_0", "Q5_1"):
        qs = {"Q4_0": 2, "Q4_1": 4, "Q5_0": 6, "Q5_1": 8}[name]
        f = {"lo": (qs + E % 16, 4 * (E // 16), 4)}
        if name in ("Q5_0", "Q5_1"):
            f["hi"] = (qs - 4 + E // 8, E % 8, 1)                       # bit E of the little-endian u32 before qs
        return f
    if name == "Q8_0":
        return {"lo": (2 + E, 0 * E, 8)}
    if name == "Q2_K":                                                  # 128g + 32s + l -> q[32g + l] >> 2s
        return {"lo": (16 + 32 * (E // 128) + E % 32, 2 * ((E // 32) % 4), 2)}
    if name == "Q3_K":
        return {"lo": (32 + 32 * (E // 128) + E % 32, 2 * ((E // 32) % 4), 2),
                "hi": (E % 32, E // 32, 1)}                             # high-mask bit (E/32) of byte E%32
    if name in ("Q4_K", "Q5_K"):                                        # sub-block j = E/32: q[32(j/2) + l] >> 4(j%2)
        qs = 16 if name == "Q4_K" else 48
        f = {"lo": (qs + 32 * (E // 64) + E % 32, 4 * ((E // 32) % 2), 4)}
        if name == "Q5_K":
            f["hi"] = (16 + E % 32, E // 32, 1)
        return f
    if name == "Q6_K":
        return {"lo": (64 * (E // 128) + E % 64, 4 * ((E // 64) % 2), 4),
                "hi": (128 + 32 * (E // 128) + E % 32, 2 * ((E // 32) % 4), 2)}
    raise KeyError(name)


def _scale_fields(name: str) -> Dict[str, List[Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]]]:
    """Sub-block scale codes: field -> parts (byte index [J], shift in the byte [J], shift in the code [J], mask [J]).
    A code is the OR of its parts; a part with mask 0 is absent for that sub-block."""
    if name == "Q2_K":
        j = np.arange(16)
        return {"sc": [(j, 0 * j, 0 * j, 0 * j + 15)], "m": [(j, 0 * j + 4, 0 * j, 0 * j + 15)]}
    if name == "Q3_K":                     # low 4 bits: nibble j/8 of byte j%8; high 2 bits: pair j/4 of byte 8 + j%4
        j = np.arange(16)
        return {"sc": [(96 + j % 8, 4 * (j // 8), 0 * j, 0 * j + 15), (104 + j % 4, 2 * (j // 4), 0 * j + 4, 0 * j + 3)]}
    if name in ("Q4_K", "Q5_K"):           # 12 bytes: j < 4 six bits each; j >= 4 four bits + the top bits of j - 4
        j = np.arange(8)
        lo = j < 4
        hi_byte = np.where(lo, 4, 4 + j - 4)
        return {"sc": [(np.where(lo, 4 + j, 8 + j), 0 * j, 0 * j, np.where(lo, 63, 15)),
                       (hi_byte, 0 * j + 6, 0 * j + 4, np.where(lo, 0, 3))],
                "m": [(8 + j, np.where(lo, 0, 4), 0 * j, np.where(lo, 63, 15)),
                      (np.where(lo, 4, 4 + j), 0 * j + 6, 0 * j + 4, np.where(lo, 0, 3))]}
    if name == "Q6_K":
        j = np.arange(16)
        return {"sc": [(192 + j, 0 * j, 0 * j, 0 * j + 255)]}
    return {}


_D_OFF = {"Q8_0": (0, None), "Q4_0": (0, None), "Q4_1": (0, 2), "Q5_0": (0, None), "Q5_1": (0, 2),
          "Q2_K": (80, 82), "Q3_K": (108, None), "Q4_K": (0, 2), "Q5_K": (0, 2), "Q6_K": (208, None)}


def _i32(a, dev) -> torch.Tensor:
    return torch.as_tensor(np.asarray(a), device=dev).to(torch.int32)


def _gather(blocks: torch.Tensor, byte, shift, width) -> torch.Tensor:
    """Element fields: width in bits (an int)."""
    b = blocks[:, torch.as_tensor(np.asarray(byte), device=blocks.device)].to(torch.int32)
    return (b >> _i32(shift, blocks.device)) & ((1 << width) - 1)


def _code(blocks: torch.Tensor, parts) -> torch.Tensor:
    v = 0
    for byte, sh, vsh, mask in parts:
        b = blocks[:, torch.as_tensor(byte, device=blocks.device)].to(torch.int32)
        v = v | (((b >> _i32(sh, blocks.device)) & _i32(mask, blocks.device)) << _i32(vsh, blocks.device))
    return v


def _f16(blocks: torch.Tensor, off: int) -> torch.Tensor:
    return blocks[:, off:off + 2].contiguous().view(torch.float16)      # [n, 1]


def dequantize(name: str, blocks: torch.Tensor) -> torch.Tensor:
    """blocks [n, bytes] uint8 (any device) -> [n, elements] fp16, in the reference's fp16 op sequence."""
    assert blocks.dtype == torch.uint8 and blocks.shape[1] == TYPES[name][2]
    half = torch.float16
    if name == "BF16":
        bits = blocks.contiguous().view(torch.int16).to(torch.int32) << 16
        return bits.view(torch.float32).to(half)
    f = _fields(name)
    q = _gather(blocks, *f["lo"])
    if "hi" in f:
        hb = _gather(blocks, *f["hi"])
    d_off, m_off = _D_OFF[name]
    d = _f16(blocks, d_off)
    if name == "Q8_0":
        return d * q.to(torch.uint8).view(torch.int8).to(half)
    if name in ("Q4_0", "Q5_0"):
        qv = (q | (hb << 4)) - 16 if name == "Q5_0" else q - 8
        return d * qv.to(half)
    if name in ("Q4_1", "Q5_1"):
        qv = q | (hb << 4) if name == "Q5_1" else q
        return (d * qv.to(half)) + _f16(blocks, m_off)
    sf = _scale_fields(name)
    E = torch.arange(256, device=blocks.device)
    if name == "Q2_K":
        j = E // 16
        dl = (d * _code(blocks, sf["sc"]).to(half))[:, j]
        ml = (_f16(blocks, m_off) * _code(blocks, sf["m"]).to(half))[:, j]
        return (dl * q.to(half)) - ml
    if name == "Q3_K":
        dl = (d * (_code(blocks, sf["sc"]) - 32).to(half))[:, E // 16]
        return dl * (q - 4 * (1 - hb)).to(half)
    if name in ("Q4_K", "Q5_K"):
        j = E // 32
        D = (d * _code(blocks, sf["sc"]).to(half))[:, j]
        M = (_f16(blocks, m_off) * _code(blocks, sf["m"]).to(half))[:, j]
        qv = q | (hb << 4) if name == "Q5_K" else q
        return (D * qv.to(half)) - M
    if name == "Q6_K":
        S = (d * _code(blocks, sf["sc"]).to(torch.uint8).view(torch.int8).to(half))[:, E // 16]
        return S * ((q | (hb << 4)) - 32).to(half)
    raise KeyError(name)


def dequantize_tensor(ggml_type: int, raw: torch.Tensor, shape: Sequence[int]) -> torch.Tensor:
    name = BY_ID[int(ggml_type)]
    _, be, bb = TYPES[name]
    return dequantize(name, raw.reshape(-1, bb)).reshape(tuple(shape))


# ---------------------------------------------------------------------------------------------------------------------
# encoder (round to nearest; any valid bytes would do)
def _put(out: torch.Tensor, byte, shift, vals: torch.Tensor):
    """OR vals << shift into the bytes of out [n, bytes] (int32 accumulator); fields never overlap."""
    idx = torch.as_tensor(np.asarray(byte), device=out.device).expand(vals.shape[0], -1)
    out.scatter_add_(1, idx, vals.to(torch.int32) << _i32(shift, out.device))


def _put_code(out, parts, code: torch.Tensor):
    for byte, sh, vsh, mask in parts:
        _put(out, byte, sh, (code >> _i32(vsh, out.device)) & _i32(mask, out.device))


def _put_f16(out, off, v: torch.Tensor):
    b = v.to(torch.float16).reshape(-1, 1).view(torch.int16).to(torch.int32) & 0xFFFF
    out[:, off] += b[:, 0] & 0xFF
    out[:, off + 1] += b[:, 0] >> 8


def encode(name: str, x: torch.Tensor) -> torch.Tensor:
    """x [..., n*elements] float -> [n, bytes] uint8 blocks of type `name` (rows are consecutive blocks)."""
    _, be, bb = TYPES[name]
    x = x.float().reshape(-1, be)
    if name == "BF16":
        return x.to(torch.bfloat16).view(torch.uint8).reshape(-1, 2)
    n, dev = x.shape[0], x.device
    out = torch.zeros(n, bb, dtype=torch.int32, device=dev)
    f = _fields(name)
    d_off, m_off = _D_OFF[name]
    tiny = 1e-8

    def h(v):
        return v.to(torch.float16).float()

    if name in ("Q8_0", "Q4_0", "Q5_0"):
        lim = {"Q8_0": 127, "Q4_0": 8, "Q5_0": 16}[name]
        d = h(x.abs().amax(1, keepdim=True) / lim)
        q = torch.round(x / d.clamp_min(tiny)).clamp(-lim, lim if name == "Q8_0" else lim - 1).to(torch.int32)
        if name == "Q8_0":
            _put(out, *f["lo"][:2], q & 0xFF)
        else:
            u = q + lim
            _put(out, *f["lo"][:2], u & 15)
            if "hi" in f:
                _put(out, *f["hi"][:2], u >> 4)
        _put_f16(out, d_off, d)
    elif name in ("Q4_1", "Q5_1"):
        top = 15 if name == "Q4_1" else 31
        lo, hi = x.amin(1, keepdim=True), x.amax(1, keepdim=True)
        m, d = h(lo), h((hi - lo) / top)
        u = torch.round((x - m) / d.clamp_min(tiny)).clamp(0, top).to(torch.int32)
        _put(out, *f["lo"][:2], u & 15)
        if "hi" in f:
            _put(out, *f["hi"][:2], u >> 4)
        _put_f16(out, d_off, d)
        _put_f16(out, m_off, m)
    else:
        sf = _scale_fields(name)
        sub = {"Q2_K": 16, "Q3_K": 16, "Q4_K": 32, "Q5_K": 32, "Q6_K": 16}[name]
        xs = x.reshape(n, -1, sub)
        if name in ("Q2_K", "Q4_K", "Q5_K"):
            top = {"Q2_K": 3, "Q4_K": 15, "Q5_K": 31}[name]
            cmax = 15 if name == "Q2_K" else 63
            mn = (-xs.amin(2)).clamp_min(0)                              # value = D*q - M, M >= 0
            rng = (xs.amax(2) + mn) / top
            d, dmin = h(rng.amax(1, keepdim=True) / cmax), h(mn.amax(1, keepdim=True) / cmax)
            sc = torch.round(rng / d.clamp_min(tiny)).clamp(0, cmax).to(torch.int32)
            mc = torch.round(mn / dmin.clamp_min(tiny)).clamp(0, cmax).to(torch.int32)
            D, M = h(d * sc), h(dmin * mc)
            u = torch.round((xs + M[..., None]) / D[..., None].clamp_min(tiny)).clamp(0, top).to(torch.int32)
            u = u.reshape(n, -1)
            _put(out, *f["lo"][:2], u & (3 if name == "Q2_K" else 15))
            if "hi" in f:
                _put(out, *f["hi"][:2], u >> 4)
            _put_code(out, sf["sc"], sc)
            _put_code(out, sf["m"], mc)
            _put_f16(out, d_off, d)
            _put_f16(out, m_off, dmin)
        else:                                                            # Q3_K / Q6_K: symmetric, signed scales
            qlim, clim = (4, 32) if name == "Q3_K" else (32, 128)
            amax = xs.abs().amax(2)
            d = h(amax.amax(1, keepdim=True) / (qlim * (clim - 1)))
            sc = torch.round(amax / qlim / d.clamp_min(tiny)).clamp(-clim, clim - 1).to(torch.int32)
            S = h(d * sc)
            q = torch.round(xs / S[..., None].clamp_min(tiny)).clamp(-qlim, qlim - 1).to(torch.int32).reshape(n, -1)
            u = q + qlim
            if name == "Q3_K":
                _put(out, *f["lo"][:2], u & 3)
                _put(out, *f["hi"][:2], u >> 2)
                _put_code(out, sf["sc"], sc + 32)
            else:
                _put(out, *f["lo"][:2], u & 15)
                _put(out, *f["hi"][:2], u >> 4)
                _put_code(out, sf["sc"], sc & 0xFF)
            _put_f16(out, d_off, d)
    return out.to(torch.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# minimal GGUF v3 writer
def _s(x: str) -> bytes:
    b = x.encode()
    return struct.pack("<Q", len(b)) + b


def write_gguf(path: str, tensors: List[Tuple[str, int, Sequence[int], np.ndarray]], alignment: int = 32,
               orig_shapes: Optional[Dict[str, Sequence[int]]] = None) -> None:
    """tensors: (name, GGML type, GGUF dimensions innermost first, raw bytes).  orig_shapes: tensor name -> logical
    shape written as ``comfy.gguf.orig_shape.<name>`` (an ARRAY of INT32)."""
    kv = [_s("general.alignment") + struct.pack("<II", 4, alignment)]
    for name, shp in (orig_shapes or {}).items():
        kv.append(_s(f"comfy.gguf.orig_shape.{name}") + struct.pack("<IIQ", 9, 5, len(shp))
                  + struct.pack(f"<{len(shp)}i", *shp))
    infos, off = [], 0
    for name, ttype, dims, raw in tensors:
        infos.append(_s(name) + struct.pack("<I", len(dims)) + struct.pack(f"<{len(dims)}Q", *dims)
                     + struct.pack("<IQ", ttype, off))
        off = (off + raw.nbytes + alignment - 1) // alignment * alignment
    head = b"GGUF" + struct.pack("<IQQ", 3, len(tensors), len(kv)) + b"".join(kv) + b"".join(infos)
    with open(path, "wb") as fh:
        fh.write(head + b"\0" * (-len(head) % alignment))
        for _, _, _, raw in tensors:
            fh.write(np.ascontiguousarray(raw).view(np.uint8).tobytes())
            fh.write(b"\0" * (-raw.nbytes % alignment))
