"""Host side of the clip pre-processing (SURVEY.md §8(f) rank 3).

Mirrors ``prepare_video_transforms(resolution, max_resolution)`` (reference
``src/core/generation_utils.py:47-84``): the returned object is called on a ``[T, C, H, W]`` clip in [0, 1] and
returns ``[C, T, Hp, Wp]`` in [-1, 1] — side resize with antialiased bicubic interpolation (``NaResize`` mode "side",
``side_resize.py:40-75``), ``clamp(0,1)``, ``DivisiblePad((16,16))``, ``Normalize(0.5,0.5)``, ``t c h w -> c t h w`` —
as ONE kernel (``csrc/pre.cu``), no intermediate tensors.  ``preprocess_frames`` takes the ComfyUI / CLI frame layout
``[T, H, W, C]`` directly (the reference permutes first, ``generation_phases.py:380-413``).
"""
from __future__ import annotations

import torch

from . import lib

_DTYPES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2,
           torch.uint8: 3}      # 8-bit RGB frames, read as the reference CLI reads them: fp16(u / 255)


def resized_size(h: int, w: int, resolution: int, max_resolution: int = 0):
    """Output (H, W) of SideResize (side_resize.py:40-75, torchvision _compute_resized_output_size) and whether the
    max_resolution cap triggers the reference's second resize."""
    short, long = (w, h) if w <= h else (h, w)
    new_short, new_long = resolution, int(resolution * long / short)
    nh, nw = (new_long, new_short) if w <= h else (new_short, new_long)
    if max_resolution > 0 and max(nh, nw) > max_resolution:
        scale = max_resolution / max(nh, nw)
        return (round(nh * scale), round(nw * scale)), True
    return (nh, nw), False


def _resize(x: torch.Tensor, channels_last: bool, H: int, W: int, finish: bool) -> torch.Tensor:
    if not x.is_cuda:
        raise lib.Svr2Error("pre-processing runs on the GPU only (no CPU fallback)")
    if x.dtype not in _DTYPES:
        x = x.float()
    x = x.contiguous()
    if channels_last:
        T, h, w, cin = x.shape
    else:
        T, cin, h, w = x.shape
        if cin != 3:
            x, cin = x[:, :3].contiguous(), 3
    Hp, Wp = ((H + 15) // 16 * 16, (W + 15) // 16 * 16) if finish else (H, W)
    out = torch.empty((3, T, Hp, Wp) if finish else (T, 3, H, W), device=x.device, dtype=torch.bfloat16)
    need = lib.load().svr2_resize_scratch_bytes(h, w, H, W)
    scratch = torch.empty(need, device=x.device, dtype=torch.uint8)
    lib.call("svr2_resize_bicubic_aa_bf16", lib.ptr(x), _DTYPES[x.dtype], int(channels_last), cin, T, h, w, lib.ptr(out),
             H, W, int(finish), lib.ptr(scratch), need, lib.stream(), nbytes=2.0 * out.numel() + x.numel() * x.element_size())
    return out


class VideoTransform:
    """What ``prepare_video_transforms`` returns (a torchvision ``Compose`` in the reference)."""

    def __init__(self, resolution: int, max_resolution: int = 0):
        self.resolution, self.max_resolution = int(resolution), int(max_resolution)

    def run(self, x: torch.Tensor, channels_last: bool) -> torch.Tensor:
        h, w = (x.shape[1], x.shape[2]) if channels_last else (x.shape[2], x.shape[3])
        (H, W), twice = resized_size(h, w, self.resolution, self.max_resolution)
        if twice:   # the reference resizes to the un-capped size first, then to the capped one (side_resize.py:62-73)
            (H1, W1), _ = resized_size(h, w, self.resolution, 0)
            x, channels_last = _resize(x, channels_last, H1, W1, finish=False), False
        return _resize(x, channels_last, H, W, finish=True)

    def __call__(self, video_tchw: torch.Tensor) -> torch.Tensor:
        return self.run(video_tchw, channels_last=False)

    def true_size(self, h: int, w: int):
        return resized_size(h, w, self.resolution, self.max_resolution)[0]


def prepare_video_transforms(resolution: int, max_resolution: int = 0, debug=None) -> VideoTransform:
    return VideoTransform(resolution, max_resolution)


def preprocess_frames(frames_thwc: torch.Tensor, resolution: int, max_resolution: int = 0) -> torch.Tensor:
    """[T, h, w, C>=3] in [0,1] (or uint8 RGB, read as the CLI reads it) -> [3, T, Hp, Wp] bf16 in [-1,1]."""
    return VideoTransform(resolution, max_resolution).run(frames_thwc, channels_last=True)
