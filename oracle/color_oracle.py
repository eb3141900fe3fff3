"""TEST INFRASTRUCTURE ONLY — never imported by the product path.

CPU restatement (plain torch) of the reference's post-decode colour correction
(``src/utils/color_fix.py``) for the three methods the engine ships:

  * ``wavelet``  — ``wavelet_reconstruction``            (``color_fix.py:122-246``)
  * ``adain``    — ``adaptive_instance_normalization``   (``color_fix.py:72-119``)
  * ``lab``      — ``lab_color_transfer`` (CLI default)  (``color_fix.py:249-521``)

and of the final image formatting of phase 4 (``generation_phases.py:1322-1345``:
``t c h w -> t h w c``, ``clamp(-1,1) * 0.5 + 0.5``).

Pinned: ``oracle/make_golden.py`` imports the reference module itself, checks these
functions against it on the same inputs and writes ``tests/golden/color_*.npz``.

Rounding points.  The reference runs wavelet / AdaIN in the pipeline's compute dtype
(bf16): every torch op rounds its result to bf16 (convolutions accumulate in fp32).
``mode="ref_bf16"`` reproduces exactly those rounding points; ``mode="fp32"`` is the
same math without intermediate rounding.  LAB runs in fp32 in the reference
(``ensure_float32_precision``, ``color_fix.py:299-301``) after a bf16 wavelet pass.
"""
from __future__ import annotations

import torch

_K1 = (0.25, 0.5, 0.25)   # the 3x3 kernel of color_fix.py:142-146 is the outer product of (1,2,1)/4


def _r(x: torch.Tensor, mode: str) -> torch.Tensor:
    """One reference rounding point."""
    return x.to(torch.bfloat16).float() if mode == "ref_bf16" else x


def wavelet_blur(image: torch.Tensor, radius: int) -> torch.Tensor:
    """color_fix.py:122-157: 3x3 (1,2,1)x(1,2,1)/16 blur, dilation = radius (capped at min(H,W)//8),
    replicate padding.  fp32 in, fp32 out (the caller rounds)."""
    H, W = image.shape[-2:]
    radius = min(radius, max(1, min(H, W) // 8))
    ys = torch.arange(H)
    xs = torch.arange(W)
    out = torch.zeros_like(image)
    for dy in (-1, 0, 1):
        yy = (ys + dy * radius).clamp(0, H - 1)
        row = image.index_select(-2, yy)
        for dx in (-1, 0, 1):
            xx = (xs + dx * radius).clamp(0, W - 1)
            out = out + row.index_select(-1, xx) * (_K1[dy + 1] * _K1[dx + 1])
    return out


def wavelet_decomposition(image: torch.Tensor, levels: int = 5, mode: str = "ref_bf16"):
    """color_fix.py:160-184.  Returns (high, low)."""
    image = _r(image.float(), mode)
    high = torch.zeros_like(image)
    low = image
    for i in range(levels):
        low = _r(wavelet_blur(image, 2 ** i), mode)
        high = _r(_r(high + image, mode) - low, mode)      # high_freq.add_(image).sub_(low_freq)
        image = low
    return high, low


def wavelet_reconstruction(content: torch.Tensor, style: torch.Tensor, mode: str = "ref_bf16") -> torch.Tensor:
    """color_fix.py:187-246 for equal shapes: content high frequencies + style low frequencies, clamp."""
    assert content.shape == style.shape
    high, _ = wavelet_decomposition(content, mode=mode)
    _, low = wavelet_decomposition(style, mode=mode)
    return _r(high + low, mode).clamp(-1.0, 1.0)


def calc_mean_std(feat: torch.Tensor, eps: float = 1e-5, mode: str = "ref_bf16"):
    """color_fix.py:72-91 (unbiased variance over H*W per (b, c))."""
    b, c = feat.shape[:2]
    f = feat.float().reshape(b, c, -1)
    var = _r(_r(f.var(dim=2), mode) + eps, mode)
    std = _r(var.sqrt(), mode).reshape(b, c, 1, 1)
    mean = _r(f.mean(dim=2), mode).reshape(b, c, 1, 1)
    return mean, std


def adaptive_instance_normalization(content: torch.Tensor, style: torch.Tensor, mode: str = "ref_bf16") -> torch.Tensor:
    """color_fix.py:94-119."""
    content, style = _r(content.float(), mode), _r(style.float(), mode)
    s_mean, s_std = calc_mean_std(style, mode=mode)
    c_mean, c_std = calc_mean_std(content, mode=mode)
    normalized = _r(_r(content - c_mean, mode) / c_std, mode)
    return _r(_r(normalized * s_std, mode) + s_mean, mode)


# ---------------------------------------------------------------- CIELAB (fp32)
_RGB2XYZ = torch.tensor([[0.4124564, 0.3575761, 0.1804375],
                         [0.2126729, 0.7151522, 0.0721750],
                         [0.0193339, 0.1191920, 0.9503041]], dtype=torch.float32)
_XYZ2RGB = torch.tensor([[3.2404542, -1.5371385, -0.4985314],
                         [-0.9692660, 1.8760108, 0.0415560],
                         [0.0556434, -0.2040259, 1.0572252]], dtype=torch.float32)
_EPS = 6.0 / 29.0
_KAPPA = (29.0 / 3.0) ** 3


def rgb_to_lab(rgb01: torch.Tensor) -> torch.Tensor:
    """color_fix.py:368-413.  rgb01 [B,3,H,W] fp32 in [0,1] -> LAB [B,3,H,W] (D65)."""
    lin = torch.where(rgb01 > 0.04045, torch.pow((rgb01 + 0.055) / 1.055, 2.4), rgb01 / 12.92)
    B, _, H, W = lin.shape
    xyz = torch.matmul(lin.permute(0, 2, 3, 1).reshape(-1, 3), _RGB2XYZ.T).reshape(B, H, W, 3).permute(0, 3, 1, 2)
    xyz = torch.stack([xyz[:, 0] / 0.95047, xyz[:, 1], xyz[:, 2] / 1.08883], 1)
    f = torch.where(xyz > _EPS ** 3, torch.pow(xyz, 1.0 / 3.0), (xyz * _KAPPA + 16.0) / 116.0)
    L = f[:, 1] * 116.0 - 16.0
    a = (f[:, 0] - f[:, 1]) * 500.0
    b = (f[:, 1] - f[:, 2]) * 200.0
    return torch.stack([L, a, b], 1)


def lab_to_rgb(lab: torch.Tensor) -> torch.Tensor:
    """color_fix.py:416-474.  LAB -> rgb in [0,1]."""
    L, a, b = lab[:, 0], lab[:, 1], lab[:, 2]
    fy = (L + 16.0) / 116.0
    fx = a / 500.0 + fy
    fz = fy - b / 200.0

    def inv(f):
        return torch.where(f > _EPS, torch.pow(f, 3.0), (f * 116.0 - 16.0) / _KAPPA)

    xyz = torch.stack([inv(fx) * 0.95047, inv(fy), inv(fz) * 1.08883], 1)
    B, _, H, W = xyz.shape
    lin = torch.matmul(xyz.permute(0, 2, 3, 1).reshape(-1, 3), _XYZ2RGB.T).reshape(B, H, W, 3).permute(0, 3, 1, 2)
    rgb = torch.where(lin > 0.0031308, torch.pow(lin.clamp(min=0.0), 1.0 / 2.4) * 1.055 - 0.055, lin * 12.92)
    return rgb.clamp(0.0, 1.0)


def histogram_match(source: torch.Tensor, reference: torch.Tensor) -> torch.Tensor:
    """color_fix.py:477-521 for equally sized inputs: the r-th smallest source value is replaced by the
    r-th smallest reference value (ties broken by a stable sort here; the reference's sort is unstable, so
    elements with exactly equal source values may swap their — adjacent — reference values)."""
    assert source.numel() == reference.numel()
    flat = source.flatten()
    order = torch.sort(flat, stable=True).indices
    ref_sorted = torch.sort(reference.flatten()).values
    out = torch.empty_like(flat)
    out[order] = ref_sorted
    return out.reshape(source.shape)


def lab_color_transfer(content: torch.Tensor, style: torch.Tensor, luminance_weight: float = 0.8) -> torch.Tensor:
    """color_fix.py:249-365: bf16 wavelet pass, then fp32 LAB histogram matching.  Returns fp32 values that
    are bf16-representable (the reference casts back to the compute dtype)."""
    base = wavelet_reconstruction(content, style, mode="ref_bf16")
    c01 = ((base + 1.0) * 0.5).clamp(0.0, 1.0)
    s01 = ((style.to(torch.bfloat16).float() + 1.0) * 0.5).clamp(0.0, 1.0)
    c_lab, s_lab = rgb_to_lab(c01), rgb_to_lab(s01)
    m_a = histogram_match(c_lab[:, 1], s_lab[:, 1])
    m_b = histogram_match(c_lab[:, 2], s_lab[:, 2])
    if luminance_weight < 1.0:
        m_L = histogram_match(c_lab[:, 0], s_lab[:, 0])
        res_L = c_lab[:, 0] * luminance_weight + m_L * (1.0 - luminance_weight)
    else:
        res_L = c_lab[:, 0]
    rgb = lab_to_rgb(torch.stack([res_L, m_a, m_b], 1))
    return (rgb * 2.0 - 1.0).to(torch.bfloat16).float()


def sample_to_image(sample: torch.Tensor, mode: str = "ref_bf16") -> torch.Tensor:
    """generation_phases.py:1322-1345: [T,C,H,W] in [-1,1] -> [T,H,W,C] in [0,1]."""
    x = _r(sample.float(), mode).permute(0, 2, 3, 1)
    return _r(_r(x.clamp(-1.0, 1.0) * 0.5, mode) + 0.5, mode).contiguous()


def blend_overlapping_frames(prev_tail: torch.Tensor, cur_head: torch.Tensor, overlap: int) -> torch.Tensor:
    """generation_utils.py:284-312 on frames [overlap, H, W, C]: Hann cross-fade over the middle third for
    overlap >= 3, linear below; weights and products carry the frames' dtype (bf16 inside the pipeline: every op
    rounds to bf16; fp32 in the multi-GPU merge of inference_cli.py:1241-1270).  Returns fp32 values."""
    dt = prev_tail.dtype
    if overlap >= 3:
        t = torch.linspace(0.0, 1.0, steps=overlap, dtype=dt)
        u = ((t - 1.0 / 3.0) / (2.0 / 3.0 - 1.0 / 3.0)).clamp(0.0, 1.0)
        w_prev = 0.5 + 0.5 * torch.cos(torch.pi * u)
    else:
        w_prev = torch.linspace(1.0, 0.0, steps=overlap, dtype=dt)
    w_prev = w_prev.view(overlap, 1, 1, 1)
    w_cur = 1.0 - w_prev
    return (prev_tail * w_prev + cur_head.to(dt) * w_cur).float()


def merge_shards(chunks, overlap: int) -> torch.Tensor:
    """inference_cli.py:1241-1274: concatenate per-GPU results (fp32), cross-fading the `overlap` frames that a
    chunk shares with the accumulated result; chunks not longer than the overlap contribute nothing."""
    chunks = [c.float() for c in chunks]
    if overlap <= 0 or len(chunks) == 1:
        return torch.cat(chunks, 0)
    result = chunks[0]
    for c in chunks[1:]:
        if c.shape[0] > overlap and result.shape[0] >= overlap:
            blended = blend_overlapping_frames(result[-overlap:], c[:overlap], overlap)
            result = torch.cat([result[:-overlap], blended, c[overlap:]], 0)
        elif c.shape[0] > overlap:
            result = torch.cat([result, c[overlap:]], 0)
    return result


# ---------------------------------------------------------------- HSV / wavelet-adaptive (round-2 groundwork)
# The engine does not ship these two modes yet (color_fix.apply_color_correction raises for them); the
# restatements below are pinned to the reference so that the kernels can be built against them next.
def rgb_to_hsv(rgb01: torch.Tensor) -> torch.Tensor:
    """color_fix.py:614-649.  rgb [B,3,H,W] in [0,1] -> (h, s, v) in [0,1]; on channel ties the later of the
    reference's three masked assignments wins (blue over green over red)."""
    r, g, b = rgb01[:, 0], rgb01[:, 1], rgb01[:, 2]
    maxc, minc = rgb01.max(1).values, rgb01.min(1).values
    rng = maxc - minc
    ok = rng > 1e-10
    rnz = torch.where(ok, rng, torch.ones_like(rng))
    h = torch.zeros_like(maxc)
    h = torch.where((maxc == r) & ok, torch.remainder((g - b) / rnz, 6.0), h)
    h = torch.where((maxc == g) & ok, (b - r) / rnz + 2.0, h)
    h = torch.where((maxc == b) & ok, (r - g) / rnz + 4.0, h)
    h = h / 6.0
    s = torch.where(maxc > 1e-10, rng / maxc.clamp(min=1e-10), torch.zeros_like(maxc))
    return torch.stack([h, s, maxc], 1)


def hsv_to_rgb(hsv: torch.Tensor) -> torch.Tensor:
    """color_fix.py:652-695."""
    h, s, v = hsv[:, 0] * 6.0, hsv[:, 1], hsv[:, 2]
    i = torch.floor(h).long() % 6
    f = h - torch.floor(h)
    p, q, t = v * (1.0 - s), v * (1.0 - s * f), v * (1.0 - s * (1.0 - f))
    table = ((v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q))
    out = [torch.zeros_like(v) for _ in range(3)]
    for k, sel in enumerate(table):
        m = i == k
        for c in range(3):
            out[c] = torch.where(m, sel[c], out[c])
    return torch.stack(out, 1)


def histogram_match_1d(source: torch.Tensor, reference: torch.Tensor) -> torch.Tensor:
    """color_fix.py:744-769: rank mapping with the quantile index (linspace * (n_ref - 1)).long() when the two
    populations differ in size."""
    order = torch.sort(source, stable=True).indices
    ref_sorted = torch.sort(reference).values
    n_s, n_r = source.numel(), reference.numel()
    if n_s != n_r:
        idx = (torch.linspace(0, 1, n_s) * (n_r - 1)).long().clamp_(0, n_r - 1)
        ref_sorted = ref_sorted[idx]
    out = torch.empty_like(source)
    out[order] = ref_sorted
    return out


def hue_conditional_saturation_match(c_h, c_s, s_h, s_s, num_bins: int = 12, min_pixels: int = 100) -> torch.Tensor:
    """color_fix.py:698-741: per 30-degree hue bin; bin 0 also takes hue >= 11/12 (red wrap-around), and bin 11 then
    re-matches those same pixels from the ORIGINAL saturations (the reference's loop overwrites them)."""
    bw = 1.0 / num_bins
    out = c_s.clone()
    for b in range(num_bins):
        lo, hi = b * bw, (b + 1) * bw
        if b == 0:
            cm = ((c_h >= 0) & (c_h < hi)) | (c_h >= (1.0 - bw))
            sm = ((s_h >= 0) & (s_h < hi)) | (s_h >= (1.0 - bw))
        else:
            cm, sm = (c_h >= lo) & (c_h < hi), (s_h >= lo) & (s_h < hi)
        cs, ss = c_s[cm], s_s[sm]
        if cs.numel() > min_pixels and ss.numel() > min_pixels:
            out[cm] = histogram_match_1d(cs, ss)
    return out


def hsv_saturation_histogram_match(content: torch.Tensor, style: torch.Tensor, out_bf16: bool = True) -> torch.Tensor:
    """color_fix.py:524-611 for equal shapes (fp32 inside; result cast to the input dtype)."""
    c01 = ((content.float() + 1.0) * 0.5).clamp(0.0, 1.0)
    s01 = ((style.float() + 1.0) * 0.5).clamp(0.0, 1.0)
    c_hsv, s_hsv = rgb_to_hsv(c01), rgb_to_hsv(s01)
    m_s = hue_conditional_saturation_match(c_hsv[:, 0], c_hsv[:, 1], s_hsv[:, 0], s_hsv[:, 1])
    rgb = hsv_to_rgb(torch.stack([c_hsv[:, 0], m_s, c_hsv[:, 2]], 1)).clamp(0.0, 1.0)
    res = rgb * 2.0 - 1.0
    return res.to(torch.bfloat16).float() if out_bf16 else res


def saturation_map(x: torch.Tensor) -> torch.Tensor:
    """color_fix.py:858-872."""
    rgb = ((x + 1.0) * 0.5).clamp(0.0, 1.0)
    maxc, minc = rgb.max(1, keepdim=True).values, rgb.min(1, keepdim=True).values
    return torch.where(maxc > 1e-10, (maxc - minc) / maxc.clamp(min=1e-10), torch.zeros_like(maxc))


def wavelet_adaptive_color_correction(content: torch.Tensor, style: torch.Tensor) -> torch.Tensor:
    """color_fix.py:772-855: everything in fp32 (inputs are cast first, so the wavelet pass does NOT round to bf16
    here), HSV result blended into the wavelet result where the content is over-saturated."""
    c, s = content.float(), style.float()
    wav = wavelet_reconstruction(c, s, mode="fp32")
    hsv = hsv_saturation_histogram_match(c, s, out_bf16=False)
    c_sat, s_sat, w_sat = saturation_map(c), saturation_map(s), saturation_map(wav)
    weight = torch.sigmoid(5.0 * ((c_sat - s_sat) - 0.15))
    weight = (weight * ((w_sat - s_sat) > (0.15 * 0.5)).float()).clamp(0.0, 1.0)
    return (wav * (1.0 - weight) + hsv * weight).to(content.dtype).float()
