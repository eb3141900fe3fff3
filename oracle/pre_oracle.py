"""TEST INFRASTRUCTURE ONLY — never imported by the product path.

CPU restatement of the reference's clip pre-processing (``prepare_video_transforms``,
``src/core/generation_utils.py:72-84``): side resize with antialiased bicubic interpolation
(``NaResize`` mode "side" -> ``SideResize`` -> ``torchvision.transforms.functional.resize``,
``src/data/image/transforms/side_resize.py:40-75``), ``clamp(0,1)``, ``DivisiblePad((16,16))``
(zeros at the bottom / right, ``divisible_crop.py:43-80``), ``Normalize(0.5, 0.5)`` and
``t c h w -> c t h w``.

Third-party algorithm restated: torchvision 0.26 ``resize`` on a bf16 tensor casts to fp32, calls
``torch.nn.functional.interpolate(mode="bicubic", align_corners=False, antialias=True)`` and casts the
result back (``_functional_tensor.resize``); torch 2.11 ``_upsample_bicubic2d_aa`` = separable
Keys cubic (a = -0.5) whose support widens by the down-scale factor, weights normalised to sum 1.
``aa_weights`` restates torch's CPU kernel, which made the goldens: ``oracle/make_golden.py`` runs the
reference's own transform classes on the CPU and checks this restatement against them
(``tests/golden/pre_*.npz``).  The reference runs its transform on the GPU, i.e. torch's CUDA kernel, whose
fp32 tap arithmetic differs from the CPU kernel's in the last bits (csrc/aa_resize.cuh); the device kernel
follows the CUDA one, and ``preprocess_torch`` below is the reference's op chain on any device, the bit-exact
yardstick of tests/test_resize_elementwise_gpu.py.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def resized_size(h: int, w: int, resolution: int, max_resolution: int = 0):
    """SideResize.__call__ (side_resize.py:40-75) with torchvision's _compute_resized_output_size."""
    short, long = (w, h) if w <= h else (h, w)
    new_short, new_long = resolution, int(resolution * long / short)
    nh, nw = (new_long, new_short) if w <= h else (new_short, new_long)
    if max_resolution > 0 and max(nh, nw) > max_resolution:
        scale = max_resolution / max(nh, nw)
        nh, nw = round(nh * scale), round(nw * scale)
        return (nh, nw), True           # the reference resizes a second time (side_resize.py:66-73)
    return (nh, nw), False


def _cubic(x: np.ndarray) -> np.ndarray:
    a = -0.5
    x = np.abs(x)
    return np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0,
                    np.where(x < 2.0, (((x - 5.0) * x + 8.0) * x - 4.0) * a, 0.0))


def aa_weights(in_size: int, out_size: int):
    """Per output index: first input tap, tap count and normalised fp32 weights (torch UpSample.h /
    UpSampleBilinear2d.cu, _compute_weights_span + _compute_weights)."""
    scale = np.float32(in_size) / np.float32(out_size)
    support = np.float32(2.0) * scale if scale >= 1.0 else np.float32(2.0)
    invscale = np.float32(1.0) / scale if scale >= 1.0 else np.float32(1.0)
    K = int(np.ceil(support)) * 2 + 1
    xmin = np.zeros(out_size, np.int64)
    xsize = np.zeros(out_size, np.int64)
    wts = np.zeros((out_size, K), np.float32)
    for i in range(out_size):
        center = np.float32(np.float64(scale) * (i + 0.5))
        lo = max(int(np.float32(np.float64(center) - np.float64(support) + 0.5)), 0)
        hi = min(int(np.float32(np.float64(center) + np.float64(support) + 0.5)), in_size)
        n = hi - lo
        j = np.arange(n)
        arg = np.float32((j + np.float64(np.float32(lo - np.float64(center))) + 0.5) * np.float64(invscale))
        w = _cubic(arg.astype(np.float64)).astype(np.float32)
        tot = np.float32(0.0)
        for v in w:
            tot = np.float32(tot + v)
        if tot != 0:
            w = (w / tot).astype(np.float32)
        xmin[i], xsize[i] = lo, n
        wts[i, :n] = w
    return xmin, xsize, wts


def resize_bicubic_aa(x: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """x [..., h, w] fp32 -> [..., H, W] fp32: horizontal taps first, then vertical, fp32 accumulation."""
    h, w = x.shape[-2:]
    if (h, w) == (H, W):
        return x.clone()
    xm, xs, xw = aa_weights(w, W)
    ym, ys, yw = aa_weights(h, H)
    K = xw.shape[1]
    idx = torch.from_numpy(np.minimum(xm[:, None] + np.arange(K)[None], w - 1))           # [W, K]
    tmp = (x[..., idx] * torch.from_numpy(xw)).sum(-1)                                       # [..., h, W]
    K = yw.shape[1]
    idy = torch.from_numpy(np.minimum(ym[:, None] + np.arange(K)[None], h - 1))           # [H, K]
    t2 = tmp.transpose(-1, -2)[..., idy] * torch.from_numpy(yw)                              # [..., W, H, K]
    return t2.sum(-1).transpose(-1, -2).contiguous()


def preprocess(frames: torch.Tensor, resolution: int, max_resolution: int = 0) -> torch.Tensor:
    """frames [T, h, w, C>=3] in [0,1] (any float dtype; rounded to the bf16 compute dtype first,
    generation_phases.py:380-388) -> [3, T, Hp, Wp] fp32 holding bf16 values in [-1,1]; Hp, Wp = H, W rounded
    up to multiples of 16, the padding holds (0 - 0.5) / 0.5 = -1."""
    x = frames[..., :3].to(torch.bfloat16).float().permute(0, 3, 1, 2)                       # t c h w
    h, w = x.shape[-2:]
    (H, W), twice = resized_size(h, w, resolution, max_resolution)
    if twice:   # first to the un-capped size, then to the capped one, each rounded to bf16 (side_resize.py:62-73)
        (H1, W1), _ = resized_size(h, w, resolution, 0)
        x = resize_bicubic_aa(x, H1, W1).to(torch.bfloat16).float()
    y = resize_bicubic_aa(x, H, W).to(torch.bfloat16).float().clamp(0.0, 1.0)
    ph, pw = (16 - H % 16) % 16, (16 - W % 16) % 16
    y = torch.nn.functional.pad(y, (0, pw, 0, ph))
    y = ((y - 0.5).to(torch.bfloat16).float() / 0.5).to(torch.bfloat16).float()
    return y.permute(1, 0, 2, 3).contiguous()


# ---- the reference's op chain as torch ops, on the clip's own device
def compute_dtype(x: torch.Tensor) -> torch.Tensor:
    """A clip in the pipeline's bf16 compute dtype (generation_phases.py:380-388); 8-bit frames as the reference CLI
    reads them, fp16(fp32(u) / 255) (inference_cli.py:613, 336-339), then bf16."""
    if x.dtype == torch.uint8:
        x = (x.float() / 255.0).half()
    return x.to(torch.bfloat16)


def resize_bf16(x: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """torchvision's resize of a bf16 [..., h, w] tensor: nothing at the same size, otherwise fp32,
    interpolate(bicubic, align_corners=False, antialias=True), back to bf16."""
    if tuple(x.shape[-2:]) == (H, W):
        return x
    return F.interpolate(x.float(), size=(H, W), mode="bicubic", align_corners=False, antialias=True).to(torch.bfloat16)


def finish_bf16(y: torch.Tensor) -> torch.Tensor:
    """[T, 3, H, W] bf16 -> [3, T, Hp, Wp]: clamp(0, 1), DivisiblePad((16, 16)) (zeros at the bottom / right),
    Normalize(0.5, 0.5) in place in bf16, t c h w -> c t h w (a view, as the reference's Lambda returns it)."""
    y = y.clamp(0.0, 1.0)
    H, W = y.shape[-2:]
    y = F.pad(y, (0, (16 - W % 16) % 16, 0, (16 - H % 16) % 16), mode="constant", value=0.0)
    return y.sub_(0.5).div_(0.5).permute(1, 0, 2, 3)


def preprocess_torch(clip_tchw: torch.Tensor, resolution: int, max_resolution: int = 0) -> torch.Tensor:
    """prepare_video_transforms(resolution, max_resolution) on a [T, 3, h, w] clip in the compute dtype, as torch ops
    on the clip's device: on a GPU tensor this is the reference's Compose exactly (torch's CUDA resize)."""
    h, w = clip_tchw.shape[-2:]
    (H, W), twice = resized_size(h, w, resolution, max_resolution)
    x = clip_tchw
    if twice:
        (H1, W1), _ = resized_size(h, w, resolution, 0)
        x = resize_bf16(x, H1, W1)
    return finish_bf16(resize_bf16(x, H, W))
