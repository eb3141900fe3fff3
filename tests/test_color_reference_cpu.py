"""The fp64 references of tests/test_color_elementwise_gpu.py pinned on the CPU against oracle/color_oracle.py (itself
pinned to the reference's goldens): the oracle's fp32 result must lie within the bound the GPU test grants a correct
fp32 kernel, so a bug in the fp64 restatement shows up here and not first on a GPU."""
import torch

import test_color_elementwise_gpu as ref
from oracle import color_oracle


def bf16_rgb(n, seed, lo=-1.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(3, n, generator=g) * (hi - lo) + lo).to(torch.bfloat16)


def dark_and_grey_pixels():
    """dark pixels on both sides of the sRGB and LAB thresholds, every grey in [-1, 1], random and out-of-range rgb"""
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float()
    v = v[torch.isfinite(v)]
    dark = v[(v >= -1) & (v <= -0.7)].unique()
    r, g, b = torch.meshgrid(dark, dark, dark, indexing="ij")
    greys = v[v.abs() <= 2].expand(3, -1)
    x = torch.cat([torch.stack([r.flatten(), g.flatten(), b.flatten()])[:, ::7], greys,
                   bf16_rgb(20000, 1).float(), bf16_rgb(5000, 2, -1.5, 1.5).float()], 1)
    return x.to(torch.bfloat16)


def test_rgb_to_lab_reference_pinned_to_oracle():
    x = dark_and_grey_pixels()
    n = x.shape[1]
    want = ref.rgb_to_lab_ref(x.double())
    rgb01 = ((x.float() + 1.0) * 0.5).clamp(0.0, 1.0).T.reshape(1, n, 1, 3).permute(0, 3, 1, 2)
    lab = color_oracle.rgb_to_lab(rgb01).reshape(3, n).double()
    for c, (v, e) in enumerate(want):
        err = (lab[c] - v).abs()
        assert (err <= e).all(), (c, err.max().item(), (err / e).max().item())
        # the oracle and the restatement agree far inside the bound: fp32 noise, not a different formula
        assert (err / e).mean() < 0.1, (c, (err / e).mean().item())


def test_lab_to_rgb_reference_pinned_to_oracle():
    g = torch.Generator().manual_seed(3)
    n = 30000
    L = torch.cat([torch.rand(n, generator=g) * 140 - 20, torch.linspace(0, 20, 4001)])
    a = torch.cat([torch.rand(n, generator=g) * 300 - 150, torch.zeros(4001)])
    b = torch.cat([torch.rand(n, generator=g) * 300 - 150, torch.linspace(-2, 2, 4001)])
    Lm = L.flip(0)
    for lw in (0.0, 0.5, 0.8, 1.0):
        got = ref.lab_to_rgb_ref(L.double(), None if lw == 1.0 else Lm.double(), a.double(), b.double(), lw)
        Lmix = L if lw == 1.0 else L * lw + Lm * (1.0 - lw)
        lab = torch.stack([Lmix, a, b]).reshape(1, 3, -1, 1)
        want = color_oracle.lab_to_rgb(lab).reshape(3, -1).double()
        for c, (v, e) in enumerate(got):
            err = (want[c] - v.clamp(0, 1)).abs()
            assert (err <= e).all(), (lw, c, err.max().item())


def test_wavelet_blur_reference_pinned_to_oracle():
    g = torch.Generator().manual_seed(4)
    for P, H, W, radius in ((3, 37, 53, 16), (1, 1, 9, 4), (2, 23, 5, 16), (1, 270, 480, 16), (1, 300, 300, 2)):
        img = torch.rand(P, H, W, generator=g) * 2 - 1
        z, a = ref.blur_ref(img, ref.capped_radius(H, W, radius), 0, H)
        want = color_oracle.wavelet_blur(img, radius).double()
        assert ((want - z).abs() <= 8 * ref.U * a).all(), (P, H, W, radius)


def test_adain_statistics_reference():
    """the plane statistics against torch's own fp64 mean / unbiased var; hw = 1 gives variance 0"""
    x = bf16_rgb(1961, 5)
    m, v, ea, e2 = ref.plane_stats(x)
    xd = x.double()
    assert torch.allclose(m, xd.mean(1), rtol=1e-12, atol=0) and torch.allclose(v, xd.var(1), rtol=1e-12, atol=0)
    assert torch.allclose(e2, (xd * xd).mean(1), rtol=1e-12) and torch.allclose(ea, xd.abs().mean(1), rtol=1e-12)
    assert (ref.plane_stats(x[:, :1])[1] == 0).all()
