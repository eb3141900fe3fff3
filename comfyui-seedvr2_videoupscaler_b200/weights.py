"""Deterministic synthetic checkpoints with the key layout of the real files.

No network and no real weights exist in the build/bench environment
(BASELINE.json: "random-init weights of that architecture"), so tests, the
benchmark and the golden-vector generator all draw weights from here.  Key
names/shapes are those of ``seedvr2_ema_{3b,7b}_fp16.safetensors`` and
``ema_vae_fp16.safetensors`` as produced by the reference module constructors
(SURVEY.md §8(a) "Synthetic-checkpoint key layout"; reference
``src/models/dit_3b/nadit.py:49-186``, ``src/models/video_vae_v3/modules/attn_video_vae.py:671-1035``).

Initialisation is *not* the reference's default init: gates / projections are
scaled so every block contributes O(1) to the residual stream — otherwise a
parity test would only exercise the skip path.
"""
from __future__ import annotations

import contextlib
import math
import struct
from collections.abc import Mapping
from typing import Dict, Optional, Tuple

import numpy as np
import torch


def _gen(seed: int, device="cpu") -> torch.Generator:
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    return g


class _Maker:
    def __init__(self, seed: int, dtype: torch.dtype, device: str):
        self.g = _gen(seed, device)
        self.dtype = dtype
        self.device = device
        self.sd: Dict[str, torch.Tensor] = {}

    def randn(self, *shape, std=1.0, mean=0.0):
        x = torch.randn(*shape, generator=self.g, device=self.device, dtype=torch.float32)
        return (x * std + mean).to(self.dtype)

    def linear(self, name: str, out_f: int, in_f: int, bias: bool = True, gain: float = 1.0):
        self.sd[name + ".weight"] = self.randn(out_f, in_f, std=gain / math.sqrt(in_f))
        if bias:
            self.sd[name + ".bias"] = self.randn(out_f, std=0.1)

    def conv(self, name: str, out_c: int, in_c: int, k=(3, 3, 3), gain: float = 1.0):
        fan_in = in_c * k[0] * k[1] * k[2]
        self.sd[name + ".weight"] = self.randn(out_c, in_c, *k, std=gain / math.sqrt(fan_in))
        self.sd[name + ".bias"] = self.randn(out_c, std=0.05)

    def norm(self, name: str, c: int):
        self.sd[name + ".weight"] = self.randn(c, std=0.1, mean=1.0)
        self.sd[name + ".bias"] = self.randn(c, std=0.1)


def swiglu_hidden(dim: int, expand_ratio: int = 4, multiple_of: int = 256) -> int:
    h = int(2 * dim * expand_ratio / 3)
    return multiple_of * ((h + multiple_of - 1) // multiple_of)


def synth_dit_state_dict(cfg: dict, seed: int = 1234, dtype=torch.float16, device="cpu") -> Dict[str, torch.Tensor]:
    """cfg: see ``dit.dit_config``; keys as the reference NaDiT.state_dict()."""
    m = _Maker(seed, dtype, device)
    d, heads, hd = cfg["dim"], cfg["heads"], cfg["head_dim"]
    inner = heads * hd
    is7 = cfg["variant"] == "7b"
    m.linear("vid_in.proj", d, cfg["in_ch"] * 4)
    m.linear("txt_in", d, cfg["txt_in_dim"])
    m.linear("emb_in.proj_in", d, 256)
    m.linear("emb_in.proj_hid", d, d)
    m.linear("emb_in.proj_out", 6 * d, d, gain=0.5)
    nfreq = (hd // 2 // 3) // 2 if is7 else (hd // 3) // 2
    if is7:
        freqs = torch.linspace(1.0, 256 / 2, nfreq) * math.pi          # freqs_for="pixel", max_freq=256
    else:
        rd = hd // 3
        freqs = 1.0 / (10000 ** (torch.arange(0, rd, 2)[: rd // 2].float() / rd))  # freqs_for="lang"
    for i in range(cfg["layers"]):
        shared = i >= cfg["mm_layers"]
        last = cfg.get("last_vid_only", False) and i == cfg["layers"] - 1
        p = f"blocks.{i}."
        for s in (("all",) if shared else ("vid", "txt")):
            m.linear(p + f"attn.proj_qkv.{s}", 3 * inner, d, bias=False)
            m.linear(p + f"attn.proj_out.{s}", d, inner)
            m.sd[p + f"attn.norm_q.{s}.weight"] = m.randn(hd, std=0.1, mean=1.0)
            m.sd[p + f"attn.norm_k.{s}.weight"] = m.randn(hd, std=0.1, mean=1.0)
        m.sd[p + "attn.rope.rope.freqs"] = freqs.to(dtype).to(device)
        for s in (("all",) if shared else (("vid",) if last else ("vid", "txt"))):
            if cfg["mlp"] == "swiglu":
                hid = swiglu_hidden(d)
                m.linear(p + f"mlp.{s}.proj_in_gate", hid, d, bias=False, gain=1.5)
                m.linear(p + f"mlp.{s}.proj_out", d, hid, bias=False)
                m.linear(p + f"mlp.{s}.proj_in", hid, d, bias=False)
            else:
                m.linear(p + f"mlp.{s}.proj_in", 4 * d, d, gain=1.5)
                m.linear(p + f"mlp.{s}.proj_out", d, 4 * d)
            for layer in ("attn", "mlp"):
                m.sd[p + f"ada.{s}.{layer}_shift"] = m.randn(d, std=0.1)
                m.sd[p + f"ada.{s}.{layer}_scale"] = m.randn(d, std=0.1, mean=1.0)
                m.sd[p + f"ada.{s}.{layer}_gate"] = m.randn(d, std=0.3)
    if cfg["out_norm"]:
        m.sd["vid_out_norm.weight"] = m.randn(d, std=0.1, mean=1.0)
        m.sd["vid_out_ada.out_shift"] = m.randn(d, std=0.1)
        m.sd["vid_out_ada.out_scale"] = m.randn(d, std=0.1, mean=1.0)
    m.linear("vid_out.proj", cfg["out_ch"] * 4, d)
    return m.sd


VAE_CHANNELS = (128, 256, 512, 512)


def synth_vae_state_dict(seed: int = 4321, dtype=torch.float16, device="cpu",
                         channels=VAE_CHANNELS, latent: int = 16) -> Dict[str, torch.Tensor]:
    """Keys of VideoAutoencoderKLWrapper.state_dict() for
    s8_c16_t4_inflation_sd3.yaml (attn_video_vae.py:671-1035)."""
    m = _Maker(seed, dtype, device)
    c = list(channels)

    def resnet(p, ci, co):
        m.norm(p + "norm1", ci)
        m.conv(p + "conv1", co, ci, gain=1.4)
        m.norm(p + "norm2", co)
        m.conv(p + "conv2", co, co, gain=0.7)
        if ci != co:
            m.conv(p + "conv_shortcut", co, ci, k=(1, 1, 1))

    def mid(p, ch):
        resnet(p + "resnets.0.", ch, ch)
        a = p + "attentions.0."
        m.norm(a + "group_norm", ch)
        for n in ("to_q", "to_k", "to_v"):
            m.linear(a + n, ch, ch, gain=1.5 if n != "to_v" else 1.0)
        m.linear(a + "to_out.0", ch, ch, gain=0.7)
        resnet(p + "resnets.1.", ch, ch)

    # encoder
    m.conv("encoder.conv_in", c[0], 3)
    ci = c[0]
    for i, co in enumerate(c):
        for j in range(2):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}.", ci if j == 0 else co, co)
        ci = co
        if i < len(c) - 1:
            temporal = i >= len(c) - 2 - 1      # Encoder3D: is_temporal_down_block
            k = (3, 3, 3) if temporal else (1, 3, 3)
            m.conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", co, co, k=k)
    mid("encoder.mid_block.", c[-1])
    m.norm("encoder.conv_norm_out", c[-1])
    m.conv("encoder.conv_out", 2 * latent, c[-1])
    # decoder
    rc = list(reversed(c))
    m.conv("decoder.conv_in", rc[0], latent)
    mid("decoder.mid_block.", rc[0])
    ci = rc[0]
    for i, co in enumerate(rc):
        for j in range(3):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}.", ci if j == 0 else co, co)
        ci = co
        if i < len(rc) - 1:
            temporal = i < 2
            r = 8 if temporal else 4
            p = f"decoder.up_blocks.{i}.upsamplers.0."
            eye = torch.eye(co, device=device).repeat(r, 1).reshape(co * r, co, 1, 1, 1)
            w = eye + torch.randn(co * r, co, 1, 1, 1, generator=m.g, device=device) * (0.3 / math.sqrt(co))
            m.sd[p + "upscale_conv.weight"] = w.to(dtype)
            m.sd[p + "upscale_conv.bias"] = m.randn(co * r, std=0.05)
            m.conv(p + "conv", co, co)
    m.norm("decoder.conv_norm_out", rc[-1])
    m.conv("decoder.conv_out", 3, rc[-1], gain=0.5)
    return m.sd


# ----------------------------------------------------------------------------------------------------------
# checkpoint files (SURVEY.md §8(f) rank 4)
def load_state_dict(path: str, device="cpu") -> Dict[str, torch.Tensor]:
    """Checkpoint file -> state dict with the reference key layout (``load_quantized_state_dict``,
    ``src/core/model_loader.py:84-153``): ``.safetensors`` in fp16 / bf16 / fp32 or fp8_e4m3fn storage (the CLI default
    model is ``*_fp8_e4m3fn.safetensors``, ``model_registry.py:56``) and ``.pth`` / ``.pt``.  The engines cast every
    tensor to their bf16 / fp32 layouts on the GPU, so fp8 and fp16 storage need no separate path.  A GGUF
    (block-quantised) checkpoint is not a dense state dict: read it with ``load_gguf``, or pass the path to
    ``pipeline.build_engine``."""
    low = path.lower()
    if low.endswith(".safetensors"):
        from safetensors.torch import load_file
        sd = load_file(path, device=str(device))
    elif low.endswith((".pth", ".pt")):
        sd = torch.load(path, map_location=device, weights_only=True)
        if isinstance(sd, dict) and "state_dict" in sd and all(not torch.is_tensor(v) for v in sd.values()):
            sd = sd["state_dict"]
    elif low.endswith(".gguf"):
        raise NotImplementedError("a GGUF checkpoint is block-quantised, not a dense state dict: read it with "
                                  "weights.load_gguf(path) or pass the path to pipeline.build_engine")
    else:
        raise ValueError(f"unknown checkpoint format: {path}")
    prefix = "model.diffusion_model."          # ComfyUI-style exports (model_loader.py:143-147)
    if any(k.startswith(prefix) for k in sd):
        sd = {(k[len(prefix):] if k.startswith(prefix) else k): v for k, v in sd.items()}
    return sd


def detect_dit_variant(sd: Dict[str, torch.Tensor]) -> str:
    """3B (dim 2560, 32 layers) or 7B (dim 3072, 36 layers) from the checkpoint itself."""
    dim = sd["vid_in.proj.weight"].shape[0]
    if dim == 2560:
        return "3b"
    if dim == 3072:
        return "7b"
    raise ValueError(f"unrecognised NaDiT width {dim}")


# ----------------------------------------------------------------------------------------------------------
# GGUF checkpoints (model_loader.py:156-239): read without the `gguf` package, dequantised on the device at load
GGML_F32, GGML_F16 = 0, 1
_GGUF_MAGIC = b"GGUF"
_DIT_PREFIX = "model.diffusion_model."
# GGUF metadata value types -> struct format of one scalar (8 STRING and 9 ARRAY are variable-length)
_GGUF_SCALAR = {0: "B", 1: "b", 2: "H", 3: "h", 4: "I", 5: "i", 6: "f", 7: "?", 10: "Q", 11: "q", 12: "d"}
_GGUF_INT32, _GGUF_STRING, _GGUF_ARRAY = 5, 8, 9


def gguf_type_size(ggml_type: int) -> Tuple[int, int]:
    """(elements, bytes) per block of a GGML type the engine dequantises; raises (naming the type) for any other."""
    import ctypes
    from . import lib
    e, b = ctypes.c_int(), ctypes.c_int()
    lib._check(lib.load().svr2_gguf_type_size(int(ggml_type), ctypes.byref(e), ctypes.byref(b)), "svr2_gguf_type_size")
    return e.value, b.value


def _known_block(ggml_type: int) -> Optional[Tuple[int, int]]:
    from . import lib
    try:
        return gguf_type_size(ggml_type)
    except lib.Svr2Error:
        return None


class GGUFQuantized:
    """One block-quantised tensor of a GGUF file: ``tensor_type`` (GGML id), ``tensor_shape`` (logical) and ``data``,
    the raw blocks (a read-only uint8 view of the file).  The attribute names are those of the reference's
    ``GGUFTensor``, so ``dequantizing`` takes either."""

    __slots__ = ("name", "tensor_type", "tensor_shape", "offset", "nbytes", "_mm", "_path")

    def __init__(self, name, tensor_type, tensor_shape, offset, nbytes, mm, path):
        self.name, self.tensor_type, self.tensor_shape = name, tensor_type, tensor_shape
        self.offset, self.nbytes, self._mm, self._path = offset, nbytes, mm, path

    @property
    def shape(self) -> torch.Size:
        return self.tensor_shape

    @property
    def data(self) -> np.ndarray:
        if self.nbytes is None:
            raise NotImplementedError(f"{self._path}: tensor {self.name!r} has GGML type {self.tensor_type}, "
                                      "which the engine does not dequantize")
        return self._mm[self.offset:self.offset + self.nbytes]

    def __repr__(self):
        return f"GGUFQuantized({self.name!r}, type={self.tensor_type}, shape={tuple(self.tensor_shape)})"


class GGUFCheckpoint(Mapping):
    """Read-only ``Mapping[str, tensor | GGUFQuantized]`` over a ``numpy.memmap`` of a GGUF file.  F32 / F16 tensors
    come back as CPU tensors of their logical shape (copied out of the file on access), every other type as a
    ``GGUFQuantized`` record.  ``infos`` maps each key to (GGUF tensor name, GGML type, logical shape, absolute byte
    offset, byte length or None for a type the engine does not dequantize)."""

    def __init__(self, path: str):
        self.path = path
        self._mm = np.memmap(path, dtype=np.uint8, mode="r")
        self.infos = self._parse()

    def _parse(self):
        mm, path = self._mm, self.path
        size = mm.shape[0]
        pos = 0

        def take(n, what):
            nonlocal pos
            if pos + n > size:
                raise ValueError(f"{path}: GGUF file truncated in {what}")
            b = mm[pos:pos + n].tobytes()
            pos += n
            return b

        def scalar(fmt, what):
            return struct.unpack("<" + fmt, take(struct.calcsize(fmt), what))[0]

        def string(what):
            return take(scalar("Q", what), what).decode("utf-8")

        def value(vtype, what):
            if vtype == _GGUF_STRING:
                return string(what)
            if vtype == _GGUF_ARRAY:
                etype, n = scalar("I", what), scalar("Q", what)
                if etype in _GGUF_SCALAR:          # read the whole array at once
                    fmt = _GGUF_SCALAR[etype]
                    return (etype, list(struct.unpack(f"<{n}{fmt}", take(n * struct.calcsize(fmt), what))))
                return (etype, [value(etype, what) for _ in range(n)])
            if vtype not in _GGUF_SCALAR:
                raise ValueError(f"{path}: unknown GGUF value type {vtype} in {what}")
            return scalar(_GGUF_SCALAR[vtype], what)

        if take(4, "the header") != _GGUF_MAGIC:
            raise ValueError(f"{path}: not a GGUF file (bad magic)")
        version = scalar("I", "the header")
        if version not in (2, 3):
            raise ValueError(f"{path}: GGUF version {version} is not supported (versions 2 and 3 are)")
        n_tensors, n_kv = scalar("Q", "the header"), scalar("Q", "the header")
        alignment, orig_shapes = 32, {}
        for _ in range(n_kv):
            key = string("the metadata")
            vtype = scalar("I", f"metadata {key!r}")
            v = value(vtype, f"metadata {key!r}")
            if key == "general.alignment":
                alignment = int(v)
            elif key.startswith("comfy.gguf.orig_shape."):
                if vtype != _GGUF_ARRAY or v[0] != _GGUF_INT32:
                    raise TypeError(f"{path}: bad original shape metadata for {key}: expected an ARRAY of INT32")
                orig_shapes[key[len("comfy.gguf.orig_shape."):]] = torch.Size(v[1])
        raw = []
        for _ in range(n_tensors):
            name = string("the tensor infos")
            n_dims = scalar("I", f"tensor {name!r}")
            dims = [scalar("Q", f"tensor {name!r}") for _ in range(n_dims)]
            raw.append((name, dims, scalar("I", f"tensor {name!r}"), scalar("Q", f"tensor {name!r}")))
        data0 = (pos + alignment - 1) // alignment * alignment

        names = [r[0] for r in raw]
        prefixed = any(n.startswith(_DIT_PREFIX) for n in names)
        infos = {}
        for name, dims, ttype, off in raw:
            if prefixed and not name.startswith(_DIT_PREFIX):
                continue
            key = name[len(_DIT_PREFIX):] if prefixed else name
            shape = orig_shapes.get(name, torch.Size(tuple(reversed(dims))))
            n_el = math.prod(dims)
            if ttype in (GGML_F32, GGML_F16):
                nbytes = n_el * (4 if ttype == GGML_F32 else 2)
            else:
                blk = _known_block(ttype)
                nbytes = None
                if blk is not None:
                    if dims and dims[0] % blk[0]:
                        raise ValueError(f"{path}: tensor {name!r}: row length {dims[0]} is not a multiple of the "
                                         f"GGML type {ttype} block size {blk[0]}")
                    nbytes = n_el // blk[0] * blk[1]
            start = data0 + off
            if start + (nbytes or 0) > size:
                raise ValueError(f"{path}: GGUF file truncated before the end of tensor {name!r}")
            infos[key] = (name, ttype, shape, start, nbytes)
        return infos

    def __getitem__(self, key):
        name, ttype, shape, start, nbytes = self.infos[key]
        if ttype in (GGML_F32, GGML_F16):
            a = np.array(self._mm[start:start + nbytes]).view(np.float32 if ttype == GGML_F32 else np.float16)
            return torch.from_numpy(a).reshape(shape)
        return GGUFQuantized(name, ttype, shape, start, nbytes, self._mm, self.path)

    def __iter__(self):
        return iter(self.infos)

    def __len__(self):
        return len(self.infos)


def load_gguf(path: str) -> GGUFCheckpoint:
    """GGUF DiT checkpoint (``seedvr2_ema_{3b,7b}-Q4_K_M.gguf`` …) -> read-only mapping with the reference key layout:
    when any tensor name carries the ComfyUI prefix ``model.diffusion_model.``, only those tensors, prefix stripped
    (``_load_gguf_state``); logical shapes from ``comfy.gguf.orig_shape.<name>`` or the reversed GGUF dimensions."""
    return GGUFCheckpoint(path)


def _is_quantized(v) -> bool:
    return hasattr(v, "tensor_type") and hasattr(v, "tensor_shape")


def _raw_blocks(v) -> torch.Tensor:
    """The raw block bytes of a quantized entry as a 1-D uint8 tensor.  A reference ``GGUFTensor`` reports its logical
    shape through ``shape`` / ``size()`` / ``numel()``; its storage is reached through a plain-tensor view."""
    if isinstance(v, torch.Tensor):
        with torch._C.DisableTorchFunctionSubclass():
            t = v.as_subclass(torch.Tensor)
        return t.contiguous().view(torch.uint8).reshape(-1)
    a = np.asarray(v.data)
    out = torch.empty(a.nbytes, dtype=torch.uint8, pin_memory=torch.cuda.is_available())
    out.numpy()[:] = a.reshape(-1).view(np.uint8)
    return out


def dequantize_entry(v, device, key: str = "?") -> torch.Tensor:
    """A quantized entry (``GGUFQuantized`` or the reference's ``GGUFTensor``) -> dense fp16 tensor of its logical shape
    on ``device`` (CUDA): the tensor ``dequantize_tensor(v, torch.float16)`` yields in the reference."""
    from . import lib
    ttype = int(v.tensor_type)
    shape = torch.Size(int(s) for s in v.tensor_shape)
    try:
        be, bb = gguf_type_size(ttype)
    except lib.Svr2Error as e:
        raise NotImplementedError(f"GGUF tensor {key!r}: {e}") from None
    n = math.prod(shape)
    raw = _raw_blocks(v)
    if n % be or raw.numel() != n // be * bb:
        raise ValueError(f"GGUF tensor {key!r}: {raw.numel()} bytes do not hold {tuple(shape)} elements of GGML type "
                         f"{ttype} ({be} elements in {bb} bytes per block)")
    src = raw.to(device, non_blocking=True)
    if src.data_ptr() % 4:
        src = src.clone()
    out = torch.empty(shape, dtype=torch.float16, device=device)
    with torch.cuda.device(out.device) if out.is_cuda else contextlib.nullcontext():
        lib.call("svr2_gguf_dequant_f16", ttype, lib.ptr(src), n, lib.ptr(out), lib.stream(),
                 nbytes=float(src.numel() + 2 * n))
    return out


class _Dequantizing(Mapping):
    def __init__(self, sd, device):
        self._sd, self.device = sd, device

    def __getitem__(self, key):
        v = self._sd[key]
        return dequantize_entry(v, self.device, key) if _is_quantized(v) else v

    def __iter__(self):
        return iter(self._sd)

    def __len__(self):
        return len(self._sd)


def dequantizing(sd, device) -> Mapping:
    """Lazy view of a DiT state dict in which every quantized entry (a ``load_gguf`` record or the reference's
    ``GGUFTensor``) reads as a dense fp16 tensor on ``device``, dequantised by ``svr2_gguf_dequant_f16`` on access;
    other entries are returned as they are.  Nothing is converted ahead of time, so a loader that casts each key as it
    reads it holds at most one fp16 temporary."""
    return _Dequantizing(sd, device)
