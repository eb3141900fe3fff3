"""Host side of the alpha channel of RGBA clips.

Mirrors ``src/core/alpha_upscaling.py`` of the reference for the functions its pipeline uses:

  ``edge_guided_alpha_upscale(input_alpha, input_rgb, upscaled_rgb, method, debug)``   (``:289-438``)
  ``detect_edges_batch(images, method)``                                              (``:125-188``, Sobel)

plus ``upscale_into_image``, the engine's phase-4 step (``generation_phases.py:1142-1217``): the alpha of the input
frames refined against the decoded sample and written as channel 3 of the RGBA image.  Every op is a libsvr2.so kernel
(``csrc/alpha.cu``); the binary-mask / normalisation decisions stay on the device, so nothing here synchronises.
"""
from __future__ import annotations

import struct

import torch

from . import lib

_DTYPES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2, torch.uint8: 3}    # uint8: as preprocess reads it
OUT_F32, OUT_RGBA, OUT_RESIZE = 0, 1, 2


def _guide(rgb: torch.Tensor, name: str) -> torch.Tensor:
    if rgb.ndim != 4 or rgb.shape[1] != 3:
        raise ValueError(f"{name}: expected [T, 3, H, W], got {tuple(rgb.shape)}")
    if not rgb.is_cuda:
        raise lib.Svr2Error("the alpha path runs on the GPU only (no CPU fallback)")
    if rgb.dtype != torch.bfloat16:
        raise TypeError(f"{name}: the guide is the decoded sample in the compute dtype (bfloat16), got {rgb.dtype}")
    return rgb.contiguous()


def _scratch(frames: int, h: int, w: int, H: int, W: int, device) -> torch.Tensor:
    need = lib.load().svr2_alpha_upscale_scratch_bytes(frames, h, w, H, W)
    return torch.empty(need, device=device, dtype=torch.uint8)


def _run(src: torch.Tensor, channels: int, rgb: torch.Tensor, out: torch.Tensor, kind: int,
         scratch: torch.Tensor = None) -> torch.Tensor:
    """src [T,h,w,channels] (the alpha is the last channel), rgb [T,3,H,W] bf16 contiguous."""
    if src.dtype not in _DTYPES:
        src = src.float()
    src = src.contiguous()
    T, h, w = src.shape[0], src.shape[1], src.shape[2]
    H, W = rgb.shape[2], rgb.shape[3]
    if rgb.shape[0] != T:
        raise ValueError(f"alpha has {T} frames, the guide {rgb.shape[0]}")
    if scratch is None:
        scratch = _scratch(T, h, w, H, W, rgb.device)
    lib.call("svr2_alpha_upscale", lib.ptr(src), _DTYPES[src.dtype], channels, T, h, w, lib.ptr(rgb), H, W, lib.ptr(out),
             kind, lib.ptr(scratch), scratch.numel(), lib.stream(), nbytes=60.0 * T * H * W)
    return out


def read_flags(scratch: torch.Tensor) -> dict:
    """The branch decisions a call left in its scratch header (include/svr2.h).  Synchronises: diagnostics only."""
    raw = bytes(scratch[:24].cpu().numpy())
    binary, norm, twice, radius, ratio, gmin = struct.unpack("<4i2f", raw)
    return dict(binary=bool(binary), normalise=bool(norm), normalise_twice=bool(twice), radius=radius,
                binary_ratio=ratio, guide_min=gmin)


def edge_guided_alpha_upscale(input_alpha: torch.Tensor, input_rgb: torch.Tensor, upscaled_rgb: torch.Tensor,
                              method: str = "guided", debug=None) -> torch.Tensor:
    """input_alpha (T,1,h,w) in [0,1] (fp32 / bf16 / fp16, taken at bf16 precision like the reference's compute-dtype
    clip), upscaled_rgb (T,3,H,W) bf16 in [-1,1] or [0,1] -> (T,1,H,W) fp32 in [0,1] on the device.  ``input_rgb`` is
    accepted for interface parity and unused, as in the reference."""
    if method != "guided":
        raise NotImplementedError(f"method={method!r}: the reference's pipeline uses 'guided' only")
    if input_alpha.ndim != 4 or input_alpha.shape[1] != 1:
        raise ValueError(f"input_alpha: expected [T, 1, h, w], got {tuple(input_alpha.shape)}")
    rgb = _guide(upscaled_rgb, "upscaled_rgb")
    T, _, H, W = rgb.shape
    src = input_alpha.to(rgb.device).reshape(T, input_alpha.shape[2], input_alpha.shape[3], 1)
    out = torch.empty(T, 1, H, W, device=rgb.device, dtype=torch.float32)
    scratch = _scratch(T, src.shape[1], src.shape[2], H, W, rgb.device)
    _run(src, 1, rgb, out, OUT_F32, scratch)
    if debug is not None:
        f = read_flags(scratch)
        debug.log(f"Alpha type: {'binary mask' if f['binary'] else 'gradient alpha'}", category="alpha", indent_level=1)
        debug.log(f"Binary ratio: {f['binary_ratio']:.2%}", category="alpha", indent_level=1)
    return out


def detect_edges_batch(images: torch.Tensor, method: str = "sobel", debug=None) -> torch.Tensor:
    """images (T,3,H,W) bf16 in [-1,1] or [0,1] -> Sobel edge map (T,1,H,W) fp32 in [0,1], bit-exact with the
    reference's OpenCV path."""
    if method != "sobel":
        raise NotImplementedError(f"method={method!r}: the alpha path uses 'sobel' only")
    rgb = _guide(images, "images")
    T, _, H, W = rgb.shape
    out = torch.empty(T, 1, H, W, device=rgb.device, dtype=torch.float32)
    scratch = _scratch(T, 1, 1, H, W, rgb.device)
    lib.call("svr2_sobel_edges_f32", lib.ptr(rgb), T, H, W, lib.ptr(out), lib.ptr(scratch), scratch.numel(),
             lib.stream(), nbytes=14.0 * T * H * W)
    return out


def upscale_into_image(frames: torch.Tensor, sample: torch.Tensor, image: torch.Tensor) -> torch.Tensor:
    """Phase 4 of an RGBA clip: frames (T,h,w,4) on the device (the input clip, alpha in channel 3), sample (T,3,H,W)
    bf16 contiguous (decoded, before colour correction) -> channel 3 of image (T,H,W,4) bf16."""
    if frames.ndim != 4 or frames.shape[-1] != 4:
        raise ValueError(f"frames: expected [T, h, w, 4], got {tuple(frames.shape)}")
    return _run(frames, 4, _guide(sample, "sample"), image, OUT_RGBA)
