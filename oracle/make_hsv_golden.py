"""TEST INFRASTRUCTURE ONLY — generates tests/golden/color_hsv_*.npz from the REFERENCE.

Run in the build container (needs /root/reference):

    python -m oracle.make_hsv_golden

For every case it runs the reference's own ``hsv_saturation_histogram_match`` and
``wavelet_adaptive_color_correction`` (``src/utils/color_fix.py:524-872``) on CPU bf16 inputs, checks the restatement
in ``oracle/hsv_oracle.py`` against them — bit for bit for the colour-space conversions, as a distribution and
>= 35 dB for the results (a third of the saturations are tied and the reference's sort is unstable, so the tie order
is unspecified) — prints the per-hue-bin counts, and stores inputs and reference outputs.
"""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import color_oracle as co  # noqa: E402
from oracle import hsv_oracle as ho  # noqa: E402
from oracle import ref_import  # noqa: E402
from oracle.make_golden import color_inputs  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")

HSV_CASES = {
    # name: (T, H, W, style kind)
    "color_hsv_t3_48x64": (3, 48, 64, "shifted"),    # T > 1, wrap-band and h == 1 pixels, every bin matched
    "color_hsv_t2_24x24": (2, 24, 24, "shifted"),    # sparse bins: some hold <= 100 pixels on one side
    "color_hsv_t2_40x56_desat": (2, 40, 56, "desat"),  # style = content with its range about the max halved: every
                                                       # bin has equal counts, the saturations differ (s_style = s / 2)
}


def edge_pixels() -> torch.Tensor:
    """[3, k] rgb values in [-1, 1] (bf16-exact) at the corners of RGB -> HSV: h == 1 (a tiny negative (g-b)/range),
    the wrap band just below it, grays, black, channel ties r=g, g=b, r=b and the primaries."""
    e = 2.0 ** -24
    px = [(1.0, -e, 0.0), (1.0, -e, 0.0), (1.0, -0.2, -0.1), (0.9, -0.5, -0.3), (0.7, 0.1, 0.2),
          (0.3, 0.3, 0.3), (-1.0, -1.0, -1.0), (0.5, 0.5, -0.5), (-0.5, 0.5, 0.5), (0.5, -0.5, 0.5),
          (1.0, -1.0, -1.0), (-1.0, 1.0, -1.0), (-1.0, -1.0, 1.0)]
    return torch.tensor(px).T.contiguous()


def hsv_inputs(T, H, W, kind, seed=17):
    """(content, style) bf16 [T,3,H,W] in [-1,1]."""
    content, style = color_inputs(T, H, W, seed=seed)
    if kind == "desat":
        c01 = torch.round((content.float() + 1.0) * 64.0) / 128.0          # on a 1/128 grid: every step below exact
        mx = c01.max(1, keepdim=True).values
        s01 = mx - (mx - c01) * 0.5
        content, style = (c01 * 2.0 - 1.0).to(torch.bfloat16), (s01 * 2.0 - 1.0).to(torch.bfloat16)
        assert torch.equal(((style.float() + 1.0) * 0.5), s01) and torch.equal(((content.float() + 1.0) * 0.5), c01)
        return content, style
    # a warm tint pushes many pixels into the red bins (wrap band), and the style is a desaturated, shifted version
    tint = torch.tensor([1.0, 0.7, 0.45]).view(1, 3, 1, 1)
    content = (content.float() * tint + 0.1).clamp(-1, 1).to(torch.bfloat16)
    style = (style.float() * tint * 0.85).clamp(-1, 1).to(torch.bfloat16)
    e = edge_pixels().to(torch.bfloat16)
    content[0, :, 0, :e.shape[1]] = e
    style[-1, :, -1, :e.shape[1]] = e
    return content, style


def main():
    if ref_import.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_import.REFERENCE_ROOT)
    ref = importlib.import_module("src.utils.color_fix")

    class _Dbg:
        def log(self, *a, **k):
            pass

    sat = lambda x: co.saturation_map(x.float()).flatten().sort().values
    for name, (T, H, W, kind) in HSV_CASES.items():
        content, style = hsv_inputs(T, H, W, kind)
        c01 = ((content.float() + 1.0) * 0.5).clamp(0.0, 1.0)
        hsv = co.rgb_to_hsv(c01)
        assert torch.equal(ref._rgb_to_hsv_batch(c01.clone()), hsv), name
        assert torch.equal(ref._hsv_to_rgb_batch(hsv.clone()), co.hsv_to_rgb(hsv)), name
        cc, sc = ho.bin_counts(content, style)
        h = hsv[:, 0]
        print(f"{name}: {T}x{H}x{W}, {int((h == 1.0).sum())} pixels at h == 1, "
              f"{int(((h >= 1.0 - 1.0 / 12) & (h < 1.0)).sum())} in the wrap band")
        print("   content per bin:", cc)
        print("   style per bin:  ", sc)
        print("   matched bins:   ", [int(a > 100 and b > 100) for a, b in zip(cc, sc)],
              " equal counts:", [b for b in range(12) if cc[b] == sc[b]])
        outs = {"hsv": ref.hsv_saturation_histogram_match(content.clone(), style.clone(), _Dbg()),
                "wavelet_adaptive": ref.wavelet_adaptive_color_correction(content.clone(), style.clone(), _Dbg())}
        for key, fn in (("hsv", ho.hsv_saturation_histogram_match), ("wavelet_adaptive", ho.wavelet_adaptive_color_correction)):
            assert outs[key].dtype == torch.bfloat16
            o = fn(content, style)
            pinned = co.hsv_saturation_histogram_match if key == "hsv" else co.wavelet_adaptive_color_correction
            assert torch.equal(o, pinned(content, style)), (name, key)     # on the CPU: the pinned restatement
            dsat = (sat(o) - sat(outs[key])).abs()
            mse = ((o - outs[key].float()) ** 2).mean().item()
            db = 99.0 if mse == 0 else 10 * np.log10(4.0 / mse)
            print(f"   {key}: sorted-saturation diff max {dsat.max().item():.4f} mean {dsat.mean().item():.5f}, {db:.1f} dB")
            assert dsat.mean() < 2e-3 and db > 35.0, (name, key)
        np.savez_compressed(os.path.join(GOLD, name + ".npz"), content=content.float().numpy(),
                            style=style.float().numpy(), counts=np.array([cc, sc], dtype=np.int64),
                            **{k: v.float().numpy().astype(np.float32) for k, v in outs.items()})


if __name__ == "__main__":
    main()
