"""Host side of the post-decode colour correction and image formatting (SURVEY.md §8(f) rank 2).

Mirrors the reference operator interface of ``src/utils/color_fix.py`` — same function names, argument
meaning and value ranges — for the methods the engine ships:

  ``wavelet_reconstruction(content_feat, style_feat, debug=None)``          (``color_fix.py:187-246``)
  ``adaptive_instance_normalization(content_feat, style_feat)``             (``color_fix.py:94-119``)
  ``lab_color_transfer(content_feat, style_feat, debug, luminance_weight)`` (``color_fix.py:249-365``; CLI default)
  ``hsv_saturation_histogram_match(content_feat, style_feat, debug=None)``  (``color_fix.py:524-769``)
  ``wavelet_adaptive_color_correction(content_feat, style_feat, debug=None)`` (``color_fix.py:772-872``)

plus ``sample_to_image`` = ``optimized_sample_to_image_format`` + ``clamp(-1,1)*0.5+0.5``
(``generation_phases.py:1322-1345``), ``sample_to_image_u8`` (the same, then the CLI's 8-bit frames) and
``apply_color_correction`` = the method switch of
``generation_phases.py:1299-1317``.  Tensors are ``[T, 3, H, W]`` in ``[-1, 1]`` on the GPU; results are bf16 (the
pipeline's compute dtype).  Every op is a libsvr2.so kernel (``csrc/post.cu``, ``csrc/hsv.cu``); there is no torch
fallback.  The switch accepts "none", "lab", "wavelet", "adain" and "wavelet_adaptive"; "hsv" still raises there and
is reached through ``hsv_saturation_histogram_match``.
"""
from __future__ import annotations

import torch

from . import lib

WAVELET_LEVELS = 5      # wavelet_decomposition(levels=5), color_fix.py:160


def _as_planes(x: torch.Tensor) -> torch.Tensor:
    if x.ndim != 4 or x.shape[1] != 3:
        raise ValueError(f"expected [T, 3, H, W], got {tuple(x.shape)}")
    if not x.is_cuda:
        raise lib.Svr2Error("colour correction runs on the GPU only (no CPU fallback)")
    return x.to(torch.bfloat16).contiguous()


def _check_pair(content: torch.Tensor, style: torch.Tensor):
    if content.shape != style.shape:
        # the reference bilinearly resizes the style here (color_fix.py:207-221); the pipeline never needs it
        raise NotImplementedError(f"content {tuple(content.shape)} and style {tuple(style.shape)} must match")


def _wavelet(content: torch.Tensor, style: torch.Tensor, fp32: bool = False) -> torch.Tensor:
    """bf16 planes in; the reconstruction in bf16 (the reference's compute-dtype pass) or, with ``fp32``, the same
    pass on fp32 copies of the inputs without intermediate rounding (as wavelet_adaptive runs it), returned fp32."""
    T, _, H, W = content.shape
    planes = T * 3
    st = lib.stream()
    dt = torch.float32 if fp32 else torch.bfloat16
    high = torch.empty_like(content, dtype=dt)
    ping, pong = torch.empty_like(content, dtype=dt), torch.empty_like(content, dtype=dt)
    out = torch.empty_like(content, dtype=dt)
    nb = (4.0 if fp32 else 2.0) * content.numel()

    def level(src, *args, nbytes):
        if fp32:   # the first level of each pass reads the bf16 clip itself
            lib.call("svr2_wavelet_level_f32", lib.ptr(src), int(src.dtype == torch.bfloat16), *args, st, nbytes=nbytes)
        else:
            lib.call("svr2_wavelet_level_bf16", lib.ptr(src), *args, st, nbytes=nbytes)

    # content pass: keep the accumulated high frequencies (color_fix.py:224-225)
    src = content
    for i in range(WAVELET_LEVELS):
        dst = ping if (i % 2 == 0) else pong
        level(src, lib.ptr(dst), lib.ptr(high), None, None, planes, H, W, 2 ** i, int(i == 0), nbytes=4 * nb)
        src = dst
    # style pass: keep the last low-pass (color_fix.py:227-228); its last level also does high + low, clamp (:242-246)
    src = style
    for i in range(WAVELET_LEVELS):
        last = i == WAVELET_LEVELS - 1
        dst = ping if (i % 2 == 0) else pong
        level(src, None if last else lib.ptr(dst), None, lib.ptr(high) if last else None,
              lib.ptr(out) if last else None, planes, H, W, 2 ** i, 0, nbytes=(3 if last else 2) * nb)
        src = dst
    return out


def wavelet_reconstruction(content_feat: torch.Tensor, style_feat: torch.Tensor, debug=None) -> torch.Tensor:
    """Content high frequencies + style low frequencies (``color_fix.py:187-246``)."""
    _check_pair(content_feat, style_feat)
    return _wavelet(_as_planes(content_feat), _as_planes(style_feat))


def adaptive_instance_normalization(content_feat: torch.Tensor, style_feat: torch.Tensor) -> torch.Tensor:
    """Per-(frame, channel) mean/std transfer (``color_fix.py:94-119``)."""
    _check_pair(content_feat, style_feat)
    c, s = _as_planes(content_feat), _as_planes(style_feat)
    T, _, H, W = c.shape
    out = torch.empty_like(c)
    stats = torch.empty(T * 3 * 4, device=c.device, dtype=torch.float32)
    lib.call("svr2_adain_bf16", lib.ptr(c), lib.ptr(s), lib.ptr(out), T * 3, H * W, lib.ptr(stats), lib.stream(),
             nbytes=8.0 * c.numel())
    return out


def lab_color_transfer(content_feat: torch.Tensor, style_feat: torch.Tensor, debug=None,
                       luminance_weight: float = 0.8) -> torch.Tensor:
    """Wavelet base, then CIELAB histogram matching of a*, b* and a weighted L* (``color_fix.py:249-365``)."""
    _check_pair(content_feat, style_feat)
    c, s = _as_planes(content_feat), _as_planes(style_feat)
    base = _wavelet(c, s)
    T, _, H, W = c.shape
    hw, n = H * W, T * H * W
    st = lib.stream()
    c_lab = torch.empty(3, n, device=c.device, dtype=torch.float32)
    s_lab = torch.empty(3, n, device=c.device, dtype=torch.float32)
    lib.call("svr2_rgb_to_lab_f32", lib.ptr(base), lib.ptr(c_lab), T, hw, st, nbytes=18.0 * n)
    lib.call("svr2_rgb_to_lab_f32", lib.ptr(s), lib.ptr(s_lab), T, hw, st, nbytes=18.0 * n)
    need = lib.load().svr2_histogram_match_scratch_bytes(n)
    scratch = torch.empty(need, device=c.device, dtype=torch.uint8)
    matched = torch.empty(3, n, device=c.device, dtype=torch.float32)
    channels = (1, 2) if luminance_weight >= 1.0 else (0, 1, 2)
    for ch in channels:
        lib.call("svr2_histogram_match_f32", lib.ptr(c_lab[ch]), lib.ptr(s_lab[ch]), lib.ptr(matched[ch]), n,
                 lib.ptr(scratch), need, st, nbytes=80.0 * n)
    out = torch.empty_like(c)
    lib.call("svr2_lab_to_rgb_bf16", lib.ptr(c_lab[0]), lib.ptr(matched[0]) if luminance_weight < 1.0 else None,
             lib.ptr(matched[1]), lib.ptr(matched[2]), float(luminance_weight), lib.ptr(out), T, hw, st,
             nbytes=22.0 * n)
    return out


def _hsv_match(c: torch.Tensor, s: torch.Tensor, wavelet=None) -> torch.Tensor:
    T, _, H, W = c.shape
    n = T * H * W
    need = lib.load().svr2_hsv_scratch_bytes(n)
    if need <= 0:
        raise lib.Svr2Error(f"HSV colour correction takes fewer than 2^31 pixels per batch, got {n}")
    scratch = torch.empty(need, device=c.device, dtype=torch.uint8)
    out = torch.empty_like(c)
    # bytes per pixel: bins 12 + 44 | sorts of 2 entries (12 B content pairs, 8 B style keys): a histogram read and
    # 5 read + write passes over 34 key bits, 256 + 176 | match 32 + 8 + 4 | compose 16 (+ 18 for the blend)
    lib.call("svr2_hsv_saturation_match_bf16", lib.ptr(c), lib.ptr(s), lib.ptr(wavelet), lib.ptr(out), T, H * W,
             lib.ptr(scratch), need, lib.stream(), nbytes=(566.0 if wavelet is not None else 548.0) * n)
    return out


def hsv_saturation_histogram_match(content_feat: torch.Tensor, style_feat: torch.Tensor, debug=None) -> torch.Tensor:
    """Hue-conditional saturation histogram matching in HSV (``color_fix.py:524-769``): per 30-degree hue bin with more
    than 100 pixels on both sides, the content saturations take the style's distribution; hue and value are kept."""
    _check_pair(content_feat, style_feat)
    return _hsv_match(_as_planes(content_feat), _as_planes(style_feat))


def wavelet_adaptive_color_correction(content_feat: torch.Tensor, style_feat: torch.Tensor, debug=None) -> torch.Tensor:
    """fp32 wavelet reconstruction with the HSV saturation match blended in where the content is over-saturated
    against the style and the wavelet result still is (``color_fix.py:772-872``)."""
    _check_pair(content_feat, style_feat)
    c, s = _as_planes(content_feat), _as_planes(style_feat)
    return _hsv_match(c, s, _wavelet(c, s, fp32=True))


def sample_to_image(sample: torch.Tensor) -> torch.Tensor:
    """``[T, 3, H, W]`` in [-1, 1] -> ``[T, H, W, 3]`` in [0, 1] (``generation_phases.py:1322-1345``)."""
    x = _as_planes(sample)
    T, _, H, W = x.shape
    out = torch.empty(T, H, W, 3, device=x.device, dtype=torch.bfloat16)
    lib.call("svr2_sample_to_image_bf16", lib.ptr(x), lib.ptr(out), T, H * W, lib.stream(), nbytes=4.0 * x.numel())
    return out


def sample_to_image_rgba(sample: torch.Tensor, image: torch.Tensor) -> torch.Tensor:
    """``sample_to_image`` into channels 0..2 of an RGBA image ``[T, H, W, 4]`` bf16 whose channel 3 already holds the
    alpha (``generation_phases.py:1325-1345``: only the RGB is normalised, the alpha is kept as computed)."""
    x = _as_planes(sample)
    T, _, H, W = x.shape
    assert image.shape == (T, H, W, 4) and image.dtype == torch.bfloat16 and image.is_contiguous()
    lib.call("svr2_sample_to_image_rgba_bf16", lib.ptr(x), lib.ptr(image), T, H * W, lib.stream(),
             nbytes=4.0 * x.numel())
    return image


def sample_to_image_u8(sample: torch.Tensor, image_rgba: torch.Tensor = None) -> torch.Tensor:
    """``sample_to_image`` followed by the reference CLI's ``(frames.float() * 255.0).astype(np.uint8)``
    (``inference_cli.py:590, 763, 809``) in one pass: ``[T, 3, H, W]`` -> ``[T, H, W, 3]`` uint8.  With ``image_rgba``
    (``[T, H, W, 4]`` bf16 whose channel 3 holds the alpha, as for ``sample_to_image_rgba``) -> ``[T, H, W, 4]`` uint8,
    the alpha scaled by 255 and truncated without normalisation."""
    x = _as_planes(sample)
    T, _, H, W = x.shape
    C = 3 if image_rgba is None else 4
    if image_rgba is not None:
        assert image_rgba.shape == (T, H, W, 4) and image_rgba.dtype == torch.bfloat16 and image_rgba.is_contiguous()
    out = torch.empty(T, H, W, C, device=x.device, dtype=torch.uint8)
    lib.call("svr2_sample_to_image_u8", lib.ptr(x), lib.ptr(image_rgba), lib.ptr(out), T, H * W, lib.stream(),
             nbytes=3.0 * x.numel() + (3.0 * T * H * W if C == 4 else 0.0))
    return out


def apply_color_correction(sample: torch.Tensor, input_video: torch.Tensor, color_correction: str = "lab",
                           debug=None) -> torch.Tensor:
    """The method switch of ``generation_phases.py:1299-1317``."""
    if color_correction == "none":
        return _as_planes(sample)
    if color_correction == "lab":
        return lab_color_transfer(sample, input_video, debug, luminance_weight=0.8)
    if color_correction == "wavelet":
        return wavelet_reconstruction(sample, input_video, debug)
    if color_correction == "adain":
        return adaptive_instance_normalization(sample, input_video)
    if color_correction == "wavelet_adaptive":
        return wavelet_adaptive_color_correction(sample, input_video, debug)
    if color_correction == "hsv":
        # the kernel ships as hsv_saturation_histogram_match; the switch does not route to it yet
        raise NotImplementedError("color_correction='hsv': call hsv_saturation_histogram_match directly")
    raise ValueError(f"unknown color_correction {color_correction!r}")
