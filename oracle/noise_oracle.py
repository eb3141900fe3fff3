"""TEST INFRASTRUCTURE ONLY — never imported by the product path.

Torch restatement of the reference's two generation-noise blends, run on the device its inputs live on (as
``hsv_oracle.py``): on the CPU it computes what the reference computes, on the GPU it follows the reference's own GPU
arithmetic (ATen's bf16 ops with fp32 opmath, a division by a Python scalar as a reciprocal multiply), which is what
``csrc/noise.cu`` and ``noise.latent_noise_coefficients`` are held to bit for bit.

  * ``input_noise``:   generation_phases.py:416-429
  * ``coefficients``:  the timestep of :688-691 through ``timestep_transform`` (infer.py:277-311) into the lerp
                       schedule's A(t), B(t) (schedules/lerp.py, base.py:82-87)
  * ``sr_condition``:  :680-697 and ``get_condition`` (infer.py:54-78), flattened to the DiT's (L, 2c+1) rows
  * ``draws``:         the draw order and memory layout of :329-330, 419, 663, 680-683, with the clip's memory
                       order from ``clip_layout``
"""
from __future__ import annotations

import torch

SCHEDULE_T = 1000.0


def input_noise(tv: torch.Tensor, noise: torch.Tensor, scale: float) -> torch.Tensor:
    """tv (3,T,Hp,Wp) bf16, noise the raw standard-normal draw of the same shape."""
    noise = noise * 0.05                                                     # :422
    blend_factor = scale * 0.5                                               # :425
    return tv * (1 - blend_factor) + (tv + noise) * blend_factor            # :428


def timestep_transform(timesteps: torch.Tensor, latents_shapes: torch.Tensor) -> torch.Tensor:
    """infer.py:277-311 with transform = True, vt = 4, vs = 8."""
    frames = (latents_shapes[:, 0] - 1) * 4 + 1
    heights = latents_shapes[:, 1] * 8
    widths = latents_shapes[:, 2] * 8

    def get_lin_function(x1, y1, x2, y2):
        m = (y2 - y1) / (x2 - x1)
        b = y1 - m * x1
        return lambda x: m * x + b

    img_shift_fn = get_lin_function(x1=256 * 256, y1=1.0, x2=1024 * 1024, y2=3.2)
    vid_shift_fn = get_lin_function(x1=256 * 256 * 37, y1=1.0, x2=1280 * 720 * 145, y2=5.0)
    shift = torch.where(frames > 1, vid_shift_fn(heights * widths * frames), img_shift_fn(heights * widths))
    timesteps = timesteps / SCHEDULE_T
    timesteps = shift * timesteps / (1 + (shift - 1) * timesteps)
    return timesteps * SCHEDULE_T


def coefficients(scale: float, latent_shape, device):
    """(A(t), B(t)) fp32 (1,) of ``_add_noise`` for a latent of shape (T', h, w, c): note ``x.shape[1:]``."""
    t = torch.tensor([1000.0], device=device, dtype=torch.bfloat16) * scale          # :688
    shape = torch.tensor(tuple(latent_shape)[1:], device=device)[None]               # :689
    t = timestep_transform(t, shape)                                                  # :690
    return 1 - (t / SCHEDULE_T), t / SCHEDULE_T                                       # lerp.py A, B


def sr_condition(noise: torch.Tensor, latent: torch.Tensor, r: torch.Tensor = None, scale: float = 0.0):
    """(T'*h*w, 2c+1) bf16 DiT input rows [noise | cond | 1]."""
    T, h, w, c = latent.shape
    blur = latent
    if scale > 0:
        aug = noise * 0.1 + r * 0.05                                                  # :683
        a, b = coefficients(scale, latent.shape, latent.device)
        blur = a.reshape(1, 1, 1, 1) * latent + b.reshape(1, 1, 1, 1) * aug           # base.py:86-87
    cond = torch.zeros([T, h, w, c + 1], device=latent.device, dtype=latent.dtype)    # infer.py:55-76
    cond[..., :-1] = blur
    cond[..., -1:] = 1.0
    return torch.cat([noise, cond], -1).reshape(T * h * w, 2 * c + 1)


# memory order of the reference's transformed clip (3, T, Hp, Wp), as a permutation of its logical c t h w dims
TCHW, CTHW, THWC = (1, 0, 2, 3), (0, 1, 2, 3), (1, 2, 3, 0)


def clip_layout(frames: int, size, resized, resized_twice: bool, padded):
    """The memory order the reference's transform leaves (generation_phases.py:95-124, generation_utils.py:72-84): a
    batch of 4n+1 frames keeps the (t h w c) order of its frames; a 4n+1-padded batch is contiguous (c t h w) after the
    padding and contiguous (t c h w) after a bicubic resize or a zero pad (neither runs when the size is unchanged)."""
    if frames % 4 == 1:
        return THWC
    if tuple(resized) == tuple(size) and not resized_twice and tuple(padded) == tuple(size):
        return CTHW
    return TCHW


def laid_out(shape, perm, device):
    """An empty bf16 tensor of logical ``shape`` whose memory runs in the order ``perm``."""
    mem = torch.empty(tuple(shape[d] for d in perm), device=device, dtype=torch.bfloat16)
    return mem.permute(*[perm.index(d) for d in range(len(perm))])


def draws(seed: int, clips, latent_shape, device, latent_noise: bool = True):
    """The draws of a run, in the reference's order and memory layout: one input-noise draw per batch clip from one
    generator seeded seed + 1_000_000, as randn_like on the clip ``(shape (3, T, Hp, Wp), memory order)``; then the DiT
    noise (T', h, w, c) and r (randn_like on a channels-last view of c T' h w memory) from a generator seeded
    ``seed``.  Returns ([input draws], noise, r)."""
    g = torch.Generator(device=device).manual_seed(seed + 1_000_000)
    ins = [laid_out(shape, perm, device).normal_(generator=g) for shape, perm in clips]   # randn_like, :419
    g = torch.Generator(device=device).manual_seed(seed)
    lat = laid_out(latent_shape, (3, 0, 1, 2), device)
    base = torch.empty_like(lat).normal_(generator=g)
    r = torch.empty_like(base).normal_(generator=g) if latent_noise else None
    return ins, base, r
