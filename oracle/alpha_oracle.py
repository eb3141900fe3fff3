"""TEST INFRASTRUCTURE ONLY — fp32 torch restatement of the reference's alpha path
(``src/core/alpha_upscaling.py:125-438``: ``detect_edges_batch`` + ``edge_guided_alpha_upscale``).

It runs on the CPU or on the GPU and needs no OpenCV: the uint8 RGB->gray conversion and the 3x3 Sobel are restated in
integer arithmetic (``oracle/make_alpha_golden.py`` checks them against cv2 and the whole restatement against the
reference's own function).  ``taps`` exposes the intermediates the GPU tests need: the flags, the edges, the guided
filter output ``q`` and the values each binary-mask threshold is applied to.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

EPS = 0.002


def binary_ratio(alpha: torch.Tensor):
    """(near_zero.float() + near_one.float()) / numel and ratio > 0.95 (:319-324), the reference's ops literally: a
    true division on the CPU, a multiply by fl(1 / fl(numel)) on the GPU."""
    flat = alpha.float().flatten()
    near_zero = (flat < 0.1).sum().float()
    near_one = (flat > 0.9).sum().float()
    ratio = (near_zero + near_one) / flat.numel()
    return ratio, bool(ratio > 0.95)


def gray_u8(u8: torch.Tensor) -> torch.Tensor:
    """cv2.cvtColor(RGB2GRAY) on uint8 (T,3,H,W) -> (T,H,W) int32: OpenCV's 15-bit fixed-point weights."""
    u = u8.to(torch.int32)
    return (9798 * u[:, 0] + 19235 * u[:, 1] + 3735 * u[:, 2] + (1 << 14)) >> 15


def reflect101(n: int, device) -> torch.Tensor:
    """Indices -1..n of an axis of length n under OpenCV's BORDER_REFLECT_101 (a one-pixel axis reflects onto itself)."""
    i = torch.arange(-1, n + 1, device=device).abs()
    return torch.where(i >= n, 2 * n - 2 - i, i).clamp(0, n - 1)


def sobel_sq(gray: torch.Tensor) -> torch.Tensor:
    """gx^2 + gy^2 of cv2.Sobel(gray, CV_64F, 1,0 / 0,1, ksize=3), BORDER_REFLECT_101, fp64 (exact integers).  gray
    (T,H,W), any H, W >= 1 (torch's 'reflect' pad needs 2)."""
    H, W = gray.shape[1:]
    p = gray.to(torch.float64)[:, reflect101(H, gray.device)][:, :, reflect101(W, gray.device)]
    gx = (p[:, :-2, 2:] - p[:, :-2, :-2]) + 2 * (p[:, 1:-1, 2:] - p[:, 1:-1, :-2]) + (p[:, 2:, 2:] - p[:, 2:, :-2])
    gy = (p[:, 2:, :-2] - p[:, :-2, :-2]) + 2 * (p[:, 2:, 1:-1] - p[:, :-2, 1:-1]) + (p[:, 2:, 2:] - p[:, :-2, 2:])
    return gx * gx + gy * gy


def detect_edges_batch(images: torch.Tensor) -> torch.Tensor:
    """(T,3,H,W) in [-1,1] or [0,1] -> Sobel edges (T,1,H,W) fp32 (:125-188)."""
    x = images.float()
    if x.min() < 0:
        x = (x + 1) / 2
    u8 = (x * 255).clamp(0, 255).to(torch.uint8)
    mag = torch.sqrt(sobel_sq(gray_u8(u8)))
    mx = mag.amax(dim=(1, 2), keepdim=True)
    e = torch.where(mx > 0, mag / mx * 255, torch.zeros_like(mag)).to(torch.uint8)     # numpy: a flat frame -> 0
    e = e.float()
    return (e / torch.full_like(e, 255.0))[:, None]       # a true division on every device (torch's CUDA
                                                          # tensor / scalar multiplies by the rounded reciprocal)


def box(x: torch.Tensor, r: int) -> torch.Tensor:
    return F.avg_pool2d(x, kernel_size=2 * r + 1, stride=1, padding=r)


def guided_filter(I: torch.Tensor, p: torch.Tensor, r: int, eps: float = EPS, taps: dict = None) -> torch.Tensor:
    """_apply_guided_filter (:234-286); taps receives the coefficients a and b."""
    mI, mp = box(I, r), box(p, r)
    var = box(I * I, r) - mI * mI
    cov = box(I * p, r) - mI * mp
    a = cov / (var + eps)
    b = mp - a * mI
    if taps is not None:
        taps.update(a=a, b=b)
    return box(a, r) * I + box(b, r)


def refine_binary(q: torch.Tensor, edges: torch.Tensor, taps: dict) -> torch.Tensor:
    """Steps 3-8 of the binary-mask branch (:370-408) on the guided filter's output q."""
    zone = F.max_pool2d(edges, kernel_size=3, stride=1, padding=1)
    in_edges = q * (1 - torch.clamp(edges / 0.25, 0, 1)) + torch.sigmoid((q - 0.5) * 12.0) * torch.clamp(edges / 0.25, 0, 1)
    combined = torch.where(zone < 0.05, (q > 0.5).float(), in_edges)
    pre = torch.where(zone < 0.03, (combined > 0.5).float(), combined)
    out = torch.where((pre > 0.3) & (pre < 0.7) & ~(edges > 0.15), (pre > 0.5).float(), pre)
    taps.update(q=q, zone=zone, combined=combined, pre_cleanup=pre)
    return out


def edge_guided_alpha_upscale(input_alpha: torch.Tensor, upscaled_rgb: torch.Tensor, taps: dict = None) -> torch.Tensor:
    """input_alpha (T,1,h,w) (bf16 values), upscaled_rgb (T,3,H,W) -> (T,1,H,W) fp32 (:289-438)."""
    taps = {} if taps is None else taps
    alpha = input_alpha.float()
    rgb = upscaled_rgb.float()
    H, W = rgb.shape[2], rgb.shape[3]
    ratio, is_binary = binary_ratio(alpha)
    taps.update(ratio=ratio, binary=is_binary, normalise=bool(rgb.min() < 0))
    rgb_n = (rgb + 1) / 2 if taps["normalise"] else rgb
    taps["normalise_twice"] = bool(rgb_n.min() < 0)
    edges = detect_edges_batch(rgb_n)
    base = F.interpolate(alpha, size=(H, W), mode="bicubic", align_corners=False, antialias=True).clamp(0, 1)
    # guide.mean(dim=1) (:212): on the CPU the channel sum over 3; on the GPU the sum times ATen's fp32 mean factor
    I = rgb_n.mean(dim=1, keepdim=True)
    taps.update(edges=edges, base=base, guide=I)
    if is_binary:
        q = guided_filter(I, base, 2, taps=taps)
        out = refine_binary(q, edges, taps)
    else:
        q = guided_filter(I, base, 3, taps=taps)
        out = q
        taps.update(q=q)
    return out.clamp(0, 1)


def threshold_distance(taps: dict) -> torch.Tensor:
    """Per pixel, how close the binary-mask branch came to flipping a decision: the distance of q to 0.5, of the
    combined value to 0.5 and of the value before the mid-gray cleanup to 0.3 / 0.5 / 0.7 (the edge-zone thresholds act
    on the bit-exact edges and cannot flip)."""
    q, c, p = taps["q"], taps["combined"], taps["pre_cleanup"]
    d = torch.minimum((q - 0.5).abs(), (c - 0.5).abs())
    for t in (0.3, 0.5, 0.7):
        d = torch.minimum(d, (p - t).abs())
    return d


# ---- golden cases: name -> geometry, alpha kind, seed, guide range
CASES = {
    "alpha_bin_img": dict(T=1, h=40, w=56, H=100, W=140, kind="binary", seed=1),
    "alpha_grad_img": dict(T=1, h=40, w=56, H=100, W=140, kind="gradient", seed=2),
    "alpha_bin_t5": dict(T=5, h=37, w=53, H=90, W=128, kind="binary", seed=3, lo=-1.1, hi=1.05),  # min < -1: twice
    "alpha_flat": dict(T=1, h=24, w=32, H=60, W=80, kind="binary", seed=4, flat=True, sharp=1.0),  # edge max 0
    "alpha_nonneg": dict(T=1, h=40, w=56, H=100, W=140, kind="binary", seed=5, lo=0.0, hi=1.0),    # no normalisation
    "alpha_ratio95": dict(T=1, h=20, w=40, H=50, W=100, kind="ratio95", seed=6),                   # ratio == 0.95
}


def _ellipse(T, hh, ww, cy, cx, ry, rx, sharp):
    y = ((torch.arange(hh) + 0.5) / hh).view(1, hh, 1)
    x = ((torch.arange(ww) + 0.5) / ww).view(1, 1, ww)
    d = torch.sqrt(((y - cy.view(T, 1, 1)) / ry) ** 2 + ((x - cx.view(T, 1, 1)) / rx) ** 2)
    return ((1 - d) * sharp + 0.5).clamp(0, 1)


def make_inputs(T, h, w, H, W, kind, seed, lo=-1.0, hi=1.0, flat=False, sharp=0.35):
    """(input_alpha (T,1,h,w) bf16, upscaled_rgb (T,3,H,W) bf16): an object (an ellipse that drifts from frame to frame)
    over a smooth background; the alpha is its antialiased mask (binary) or a smooth ramp inside it (gradient)."""
    g = torch.Generator().manual_seed(seed)
    cy = 0.5 + 0.1 * (torch.rand(T, generator=g) - 0.5)
    cx = 0.5 + 0.1 * (torch.rand(T, generator=g) - 0.5)
    ry, rx = 0.3, 0.35
    if kind == "ratio95":
        alpha = (torch.arange(w) >= w // 2).float().view(1, 1, w).expand(T, h, w).clone()
        n = alpha.numel()
        assert n % 20 == 0
        alpha.view(-1)[torch.randperm(n, generator=g)[: n // 20]] = 0.5          # exactly 5 % mid-gray
        mask = (torch.arange(W) >= W // 2).float().view(1, 1, W).expand(T, H, W)
    else:
        alpha = _ellipse(T, h, w, cy, cx, ry, rx, sharp * min(h, w))
        if kind == "gradient":
            y = ((torch.arange(h) + 0.5) / h).view(1, h, 1)
            x = ((torch.arange(w) + 0.5) / w).view(1, 1, w)
            ramp = 0.5 + 0.4 * torch.sin(6.0 * x + 4.0 * y + torch.rand(T, 1, 1, generator=g) * 6.28)
            alpha = (_ellipse(T, h, w, cy, cx, ry, rx, 2.0) * ramp).clamp(0, 1)
        mask = _ellipse(T, H, W, cy, cx, ry, rx, 0.35 * min(H, W))
    bg = F.interpolate(torch.rand(T, 3, H // 10 + 2, W // 10 + 2, generator=g), size=(H, W), mode="bilinear",
                       align_corners=False)
    fg = torch.rand(T, 3, 1, 1, generator=g)
    img = bg * (1 - mask[:, None]) + fg * mask[:, None] + 0.03 * torch.randn(T, 3, H, W, generator=g)
    rgb = lo + (hi - lo) * img
    if lo >= 0:
        rgb = rgb.clamp(min=0)
    if flat:
        rgb = torch.full((T, 3, H, W), -0.2)
    return alpha[:, None].to(torch.bfloat16), rgb.to(torch.bfloat16)
