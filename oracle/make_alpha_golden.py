"""TEST INFRASTRUCTURE ONLY — generates tests/golden/alpha_*.npz from the REFERENCE's alpha path.

Run in the build container (needs the reference tree and OpenCV):

    python oracle/make_alpha_golden.py

It (1) checks ``alpha_oracle.gray_u8`` against ``cv2.cvtColor(RGB2GRAY)`` on all 256^3 RGB triples, (2) runs the
reference's own ``detect_edges_batch`` and ``edge_guided_alpha_upscale`` (``src/core/alpha_upscaling.py``, CPU fp32)
on the seeded inputs of ``alpha_oracle.CASES``, (3) asserts that the oracle reproduces the edges bit for bit and the
output to 1e-6, and (4) stores the reference outputs with the case parameters.
"""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import alpha_oracle as ao  # noqa: E402
from oracle import ref_import  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def check_gray(cv2):
    v = np.arange(256, dtype=np.uint8)
    rgb = np.stack(np.meshgrid(v, v, v, indexing="ij"), -1).reshape(4096, 4096, 3)
    ref = cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY)
    ora = ao.gray_u8(torch.from_numpy(rgb).permute(2, 0, 1)[None])[0].numpy()
    assert np.array_equal(ref.astype(np.int32), ora), "gray formula differs from cv2.cvtColor"
    print("gray: oracle == cv2.cvtColor(RGB2GRAY) on all 256^3 triples")


def main():
    import cv2
    if ref_import.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_import.REFERENCE_ROOT)
    ref = importlib.import_module("src.core.alpha_upscaling")
    check_gray(cv2)
    for name, case in ao.CASES.items():
        alpha, rgb = ao.make_inputs(**case)
        T, h, w = alpha.shape[0], alpha.shape[2], alpha.shape[3]
        with torch.no_grad():
            rgb_n = rgb.float()
            if rgb_n.min() < 0:
                rgb_n = (rgb_n + 1) / 2
            ref_edges = ref.detect_edges_batch(images=rgb_n.clone(), method="sobel")
            out = ref.edge_guided_alpha_upscale(input_alpha=alpha.clone(), input_rgb=torch.zeros(T, 3, h, w),
                                                upscaled_rgb=rgb.clone(), method="guided", debug=None)
        taps = {}
        ora = ao.edge_guided_alpha_upscale(alpha, rgb, taps)
        assert out.dtype == torch.float32 and out.shape == ora.shape
        assert torch.equal(ao.detect_edges_batch(rgb_n), ref_edges), f"{name}: edges differ"
        err = (ora - out).abs().max().item()
        assert err <= 1e-6, f"{name}: oracle deviates from the reference ({err})"
        print(f"{name}: {tuple(out.shape)} binary={taps['binary']} ratio={taps['ratio'].item():.4f} "
              f"normalise={taps['normalise']}/{taps['normalise_twice']} edge max={ref_edges.max().item():.3f} "
              f"oracle-vs-reference edges bit-exact, max|d|={err:.1e}")
        meta = np.array([case["T"], case["h"], case["w"], case["H"], case["W"], case["seed"], int(taps["binary"])])
        np.savez_compressed(os.path.join(GOLD, name + ".npz"), out=out.numpy(), edges=ref_edges.numpy(), meta=meta)


if __name__ == "__main__":
    main()
