"""TEST INFRASTRUCTURE ONLY — never imported by the product path.

The hsv / wavelet_adaptive restatement of ``color_oracle.py`` (``color_fix.py:524-872``), run on the device its inputs
live on.  On the CPU it computes exactly what ``color_oracle`` computes (its colour-space conversions and saturation
map are reused as they are); on the GPU it follows the reference's own GPU arithmetic, which is what the CUDA kernels
are held to bit for bit:

  * ``histogram_match_1d`` builds its ``linspace`` on the source's device (the reference passes ``device=``,
    ``color_fix.py:755``): torch's CUDA linspace counts the second half back from the end, the CPU one does not;
  * ``wavelet_blur`` indexes with device tensors (same taps, same order as ``color_oracle.wavelet_blur``);
  * ``h / 6.0`` on a CUDA tensor is a multiplication by the fp32 reciprocal (ATen's scalar-divisor fast path).

``bin_counts`` returns the per-hue-bin mask sizes the reference's loop sees, for coverage checks.
"""
from __future__ import annotations

import torch

from oracle import color_oracle as co

NUM_BINS, MIN_PIXELS = 12, 100


def wavelet_blur(image: torch.Tensor, radius: int) -> torch.Tensor:
    """color_oracle.wavelet_blur with the index tensors on the image's device."""
    H, W = image.shape[-2:]
    radius = min(radius, max(1, min(H, W) // 8))
    ys = torch.arange(H, device=image.device)
    xs = torch.arange(W, device=image.device)
    out = torch.zeros_like(image)
    for dy in (-1, 0, 1):
        row = image.index_select(-2, (ys + dy * radius).clamp(0, H - 1))
        for dx in (-1, 0, 1):
            out = out + row.index_select(-1, (xs + dx * radius).clamp(0, W - 1)) * (co._K1[dy + 1] * co._K1[dx + 1])
    return out


def wavelet_reconstruction_fp32(content: torch.Tensor, style: torch.Tensor) -> torch.Tensor:
    """color_oracle.wavelet_reconstruction(mode="fp32") on the inputs' device."""
    def decompose(image, levels=5):
        high = torch.zeros_like(image)
        low = image
        for i in range(levels):
            low = wavelet_blur(image, 2 ** i)
            high = (high + image) - low
            image = low
        return high, low
    high, _ = decompose(content.float())
    _, low = decompose(style.float())
    return (high + low).clamp(-1.0, 1.0)


def histogram_match_1d(source: torch.Tensor, reference: torch.Tensor) -> torch.Tensor:
    """color_oracle.histogram_match_1d with the linspace on the source's device (color_fix.py:744-769)."""
    order = torch.sort(source, stable=True).indices
    ref_sorted = torch.sort(reference).values
    n_s, n_r = source.numel(), reference.numel()
    if n_s != n_r:
        idx = (torch.linspace(0, 1, n_s, device=source.device) * (n_r - 1)).long().clamp_(0, n_r - 1)
        ref_sorted = ref_sorted[idx]
    out = torch.empty_like(source)
    out[order] = ref_sorted
    return out


def bin_masks(h: torch.Tensor):
    """The reference's 12 hue masks in loop order (color_fix.py:717-727)."""
    bw = 1.0 / NUM_BINS
    for b in range(NUM_BINS):
        if b == 0:
            yield b, ((h >= 0) & (h < bw)) | (h >= (1.0 - bw))
        else:
            yield b, (h >= b * bw) & (h < (b + 1) * bw)


def hue_conditional_saturation_match(c_h, c_s, s_h, s_s) -> torch.Tensor:
    out = c_s.clone()
    for (b, cm), (_, sm) in zip(bin_masks(c_h), bin_masks(s_h)):
        cs, ss = c_s[cm], s_s[sm]
        if cs.numel() > MIN_PIXELS and ss.numel() > MIN_PIXELS:
            out[cm] = histogram_match_1d(cs, ss)
    return out


def _hsv(x: torch.Tensor) -> torch.Tensor:
    return co.rgb_to_hsv(((x.float() + 1.0) * 0.5).clamp(0.0, 1.0))


def hsv_saturation_histogram_match(content: torch.Tensor, style: torch.Tensor, out_bf16: bool = True) -> torch.Tensor:
    c_hsv, s_hsv = _hsv(content), _hsv(style)
    m_s = hue_conditional_saturation_match(c_hsv[:, 0], c_hsv[:, 1], s_hsv[:, 0], s_hsv[:, 1])
    rgb = co.hsv_to_rgb(torch.stack([c_hsv[:, 0], m_s, c_hsv[:, 2]], 1)).clamp(0.0, 1.0)
    res = rgb * 2.0 - 1.0
    return res.to(torch.bfloat16).float() if out_bf16 else res


def adaptive_blend(content: torch.Tensor, style: torch.Tensor, wav: torch.Tensor, hsv: torch.Tensor):
    """color_fix.py:817-851: (blended result in fp32, w_sat - s_sat)."""
    c_sat, s_sat, w_sat = co.saturation_map(content.float()), co.saturation_map(style.float()), co.saturation_map(wav)
    weight = torch.sigmoid(5.0 * ((c_sat - s_sat) - 0.15))
    weight = (weight * ((w_sat - s_sat) > (0.15 * 0.5)).float()).clamp(0.0, 1.0)
    return wav * (1.0 - weight) + hsv * weight, w_sat - s_sat


def wavelet_adaptive_color_correction(content: torch.Tensor, style: torch.Tensor) -> torch.Tensor:
    c, s = content.float(), style.float()
    wav = wavelet_reconstruction_fp32(c, s)
    res, _ = adaptive_blend(c, s, wav, hsv_saturation_histogram_match(c, s, out_bf16=False))
    return res.to(torch.bfloat16).float()


def bin_counts(content: torch.Tensor, style: torch.Tensor):
    """(content counts, style counts) per hue bin, as lists of 12 ints."""
    c_h, s_h = _hsv(content)[:, 0], _hsv(style)[:, 0]
    return ([int(m.sum()) for _, m in bin_masks(c_h)], [int(m.sum()) for _, m in bin_masks(s_h)])
