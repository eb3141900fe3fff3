"""Generation noise: the reference's ``input_noise_scale`` and ``latent_noise_scale`` (generation_phases.py:415-431,
679-704) on the engine's kernels (``csrc/noise.cu``).

Draws come from torch's CUDA generator, in the reference's order and memory layout:

* input noise: one generator seeded ``seed + 1_000_000`` (:329-330) feeds every batch in turn.  The reference calls
  ``randn_like`` on the transformed clip, whose memory order depends on the batch (``input_noise_layout``), and the
  draw fills memory in that order; ``draw_input_noise`` returns a view with the same strides.
* latent noise: ``r`` is drawn right after the DiT noise from the generator seeded ``seed`` (:663, 680-683), with the
  strides of the reference's latent, a channels-last view of (16, T', h, w) memory (infer.py:187); ``draw_latent_noise``
  returns that view.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

from . import lib

INPUT_NOISE_SEED_OFFSET = 1_000_000      # seed_vae = seed + 1000000, generation_phases.py:329
SCHEDULE_T = 1000.0                      # configs_{3b,7b}/main.yaml: diffusion.schedule.T
VAE_TEMPORAL, VAE_SPATIAL = 4, 8         # infer.py:282-283 (temporal / spatial_downsample_factor defaults)


def check_scale(name: str, value: float) -> float:
    """A noise scale as the reference takes it: finite and >= 0 (values above 1 are computed as given)."""
    v = float(value)
    if not math.isfinite(v) or v < 0:
        raise ValueError(f"{name} must be finite and >= 0, got {value!r}")
    return v


def input_generator(seed: int, device) -> torch.Generator:
    return torch.Generator(device=device).manual_seed(seed + INPUT_NOISE_SEED_OFFSET)


# memory orders of the reference's transformed clip (3, T, Hp, Wp): the kernel's noise_layout codes
TCHW, CTHW, THWC = 0, 1, 2
_MEMORY_PERM = {TCHW: (1, 0, 2, 3), CTHW: (0, 1, 2, 3), THWC: (1, 2, 3, 0)}    # memory dims in logical c t h w terms


def input_noise_layout(frames: int, size: Tuple[int, int], resized: Tuple[int, int], resized_twice: bool,
                       padded: Tuple[int, int]) -> int:
    """Memory order of the reference's transformed clip for a batch of ``frames`` frames (after the uniform padding)
    of ``size`` (h, w), resized to ``resized`` (in two steps when ``resized_twice``) and zero-padded to ``padded``.

    The batch reaches the transform as a (t c h w) view of the frames' (t h w c) memory (generation_phases.py:95-104),
    and every step of the transform keeps a channels-last input channels-last.  A batch that needs the 4n+1 padding is
    concatenated along frames as c t h w (:109-124), which gives contiguous (c t h w) memory; the bicubic resize and the
    zero pad then write contiguous (t c h w) memory, and a batch they both leave alone (torchvision returns the input
    when the size does not change) keeps (c t h w)."""
    if frames % 4 == 1:
        return THWC
    if resized == tuple(size) and not resized_twice and tuple(padded) == tuple(size):
        return CTHW
    return TCHW


def input_noise_buffer(clip_shape, device, layout: int = TCHW, generator: Optional[torch.Generator] = None):
    """A (3, T, Hp, Wp) bf16 view of contiguous memory in the order ``layout``: zeros, or with ``generator`` the
    reference's ``randn_like(transformed_video)`` (:419) for a clip laid out that way."""
    perm = _MEMORY_PERM[layout]
    mem_shape = tuple(clip_shape[d] for d in perm)
    if generator is None:
        mem = torch.zeros(mem_shape, device=device, dtype=torch.bfloat16)
    else:
        mem = torch.randn(mem_shape, generator=generator, device=device, dtype=torch.bfloat16)
    return mem.permute(*[perm.index(d) for d in range(4)])


def draw_input_noise(clip_shape, generator: torch.Generator, device, layout: int = TCHW) -> torch.Tensor:
    """The next input-noise draw of ``generator`` for a clip of shape (3, T, Hp, Wp) whose reference memory order is
    ``layout``."""
    return input_noise_buffer(clip_shape, device, layout, generator)


def _layout_of(noise: torch.Tensor) -> Optional[int]:
    for layout, perm in _MEMORY_PERM.items():
        if noise.permute(*perm).is_contiguous():
            return layout
    return None


def draw_latent_noise(latent_shape, generator: torch.Generator, device) -> torch.Tensor:
    """``randn_like(base_noise)`` (:683) for a latent of shape (T', h, w, c): a (T', h, w, c) view of contiguous
    (c, T', h, w) bf16 memory."""
    T, h, w, c = latent_shape
    return torch.randn((c, T, h, w), generator=generator, device=device, dtype=torch.bfloat16).permute(1, 2, 3, 0)


def add_input_noise(x: torch.Tensor, noise: torch.Tensor, scale: float) -> torch.Tensor:
    """:416-429 out of place: x (3, T, Hp, Wp) bf16 contiguous, noise of the same shape (the raw standard-normal draw,
    read in place when its memory is in one of the three orders of ``input_noise_layout``) -> x * (1 - b) +
    (x + noise * 0.05) * b with b = scale * 0.5, rounded as the reference's bf16 ops."""
    if tuple(noise.shape) != tuple(x.shape):
        raise ValueError(f"input_noise must have the clip's shape {tuple(x.shape)}, got {tuple(noise.shape)}")
    assert x.dtype == torch.bfloat16 and x.is_cuda and x.is_contiguous()
    n = noise.to(x.device, torch.bfloat16)
    layout = _layout_of(n)
    if layout is None:
        n, layout = n.contiguous(), CTHW
    b = scale * 0.5                                                              # a Python double, as in :425
    out = torch.empty_like(x)
    C, T, Hp, Wp = x.shape
    lib.call("svr2_input_noise_bf16", lib.ptr(x), lib.ptr(n), layout, lib.ptr(out), T, Hp * Wp, 1 - b, b,
             lib.stream(), nbytes=6.0 * x.numel())
    return out


def latent_noise_coefficients(scale: float, latent_shape, device) -> Tuple[torch.Tensor, torch.Tensor]:
    """(A(t), B(t)) of the lerp schedule at the shifted augmentation timestep, one fp32 each on the device, by the
    reference's own op sequence so that every rounding (and on CUDA ATen's reciprocal multiply for a division by a
    Python scalar) is the one the reference's GPU run makes.  No host copy, so it captures into a CUDA graph.

    ``_add_noise`` (generation_phases.py:686-693) passes ``x.shape[1:]`` of the (T', h, w, c) latent, so
    ``timestep_transform`` (infer.py:277-311) sees frames = (h - 1) * 4 + 1, height = 8 * w and width = 8 * c."""
    T, h, w, c = latent_shape
    t = torch.full((1,), SCHEDULE_T, device=device, dtype=torch.bfloat16) * scale          # :688, rounded to bf16
    dims = [torch.full((1,), v, device=device, dtype=torch.int64) for v in (h, w, c)]      # :689, int64 like torch.tensor
    frames = (dims[0] - 1) * VAE_TEMPORAL + 1                                              # infer.py:284-286
    heights = dims[1] * VAE_SPATIAL
    widths = dims[2] * VAE_SPATIAL

    def lin(x1, y1, x2, y2):                                                               # infer.py:289-292
        m = (y2 - y1) / (x2 - x1)
        b = y1 - m * x1
        return lambda x: m * x + b

    img_shift_fn = lin(256 * 256, 1.0, 1024 * 1024, 3.2)                                   # infer.py:294-300
    vid_shift_fn = lin(256 * 256 * 37, 1.0, 1280 * 720 * 145, 5.0)
    shift = torch.where(frames > 1, vid_shift_fn(heights * widths * frames), img_shift_fn(heights * widths))
    t = t / SCHEDULE_T                                                                     # infer.py:303-305
    t = shift * t / (1 + (shift - 1) * t)
    t = t * SCHEDULE_T
    return 1 - (t / SCHEDULE_T), t / SCHEDULE_T                                            # lerp.py A(t), B(t)


def sr_condition(noise: torch.Tensor, latent: torch.Tensor, latent_noise: Optional[torch.Tensor] = None,
                 coefficients: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> torch.Tensor:
    """DiT input (T'*h*w, 2c+1) bf16 = [noise | cond | 1] of task "sr" (infer.py:54-78).  cond = latent, or with
    ``latent_noise`` r (T', h, w, c) and the ``coefficients`` (A, B): A * latent + B * (noise * 0.1 + r * 0.05)
    (generation_phases.py:681-697)."""
    T, h, w, c = latent.shape
    noise = noise.to(latent.device, torch.bfloat16).contiguous()
    latent = latent.to(torch.bfloat16).contiguous()
    assert latent.is_cuda and tuple(noise.shape) == tuple(latent.shape)
    rows = T * h * w
    out = torch.empty(rows, 2 * c + 1, device=latent.device, dtype=torch.bfloat16)
    r = a = b = None
    if latent_noise is not None:
        if tuple(latent_noise.shape) != tuple(latent.shape):
            raise ValueError(f"latent_noise must have the latent's shape {tuple(latent.shape)}, "
                             f"got {tuple(latent_noise.shape)}")
        r = latent_noise.to(latent.device, torch.bfloat16).permute(3, 0, 1, 2).contiguous()   # channel-major memory
        a, b = (v.to(torch.float32).contiguous() for v in coefficients)
    lib.call("svr2_sr_condition_bf16", lib.ptr(noise), lib.ptr(latent), lib.ptr(r), lib.ptr(a), lib.ptr(b),
             lib.ptr(out), rows, c, lib.stream(), nbytes=2.0 * rows * (2 * c + 1) + 2.0 * noise.numel() * (2 if r is None else 3))
    return out
