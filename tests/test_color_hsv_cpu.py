"""CPU: the hsv / wavelet_adaptive restatement against the goldens made by the reference's own color_fix.py
(oracle/make_hsv_golden.py), the coverage of those goldens, and the C-ABI entry points of the CUDA path."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import color_oracle as co
from oracle import hsv_oracle as ho
from oracle.make_hsv_golden import HSV_CASES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
HSV_ENTRY_POINTS = {"svr2_hsv_scratch_bytes": 1, "svr2_hsv_saturation_match_bf16": 9, "svr2_wavelet_level_f32": 12}


def load(name):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    return g, torch.from_numpy(g["content"]).to(torch.bfloat16), torch.from_numpy(g["style"]).to(torch.bfloat16)


@pytest.mark.parametrize("name", list(HSV_CASES))
def test_hsv_oracle_matches_reference_goldens(name):
    """Same saturation distribution and >= 35 dB (the reference's sort is unstable: the tie order is unspecified)."""
    g, content, style = load(name)                  # the stored inputs: regenerating them depends on the host's CPU kernels
    assert tuple(content.shape) == (HSV_CASES[name][0], 3) + HSV_CASES[name][1:3] == tuple(style.shape)
    sat = lambda x: co.saturation_map(x.float()).flatten().sort().values
    for key, fn in (("hsv", ho.hsv_saturation_histogram_match), ("wavelet_adaptive", ho.wavelet_adaptive_color_correction)):
        out, ref = fn(content, style), torch.from_numpy(g[key])
        assert (sat(out) - sat(ref)).abs().mean() < 2e-3, key
        assert 10 * torch.log10(4.0 / ((out - ref) ** 2).mean()) > 35.0, key
    assert g["counts"].tolist() == list(ho.bin_counts(content, style))


def test_device_restatement_equals_pinned_one_on_cpu():
    """On the CPU the device-following restatement is the pinned color_oracle one, bit for bit."""
    _, content, style = load("color_hsv_t3_48x64")
    assert torch.equal(ho.hsv_saturation_histogram_match(content, style), co.hsv_saturation_histogram_match(content, style))
    assert torch.equal(ho.wavelet_adaptive_color_correction(content, style),
                       co.wavelet_adaptive_color_correction(content, style))
    assert torch.equal(ho.wavelet_reconstruction_fp32(content, style),
                       co.wavelet_reconstruction(content, style, mode="fp32"))


def test_hsv_goldens_cover_the_corner_cases():
    counts, frames, wrap, at_one = {}, 0, 0, 0
    for name, (T, H, W, kind) in HSV_CASES.items():
        g, content, style = load(name)
        counts[name] = g["counts"]
        frames = max(frames, T)
        h = ho._hsv(content)[:, 0]
        wrap += int(((h >= 1.0 - 1.0 / 12) & (h < 1.0)).sum())
        at_one += int((h == 1.0).sum())
    cc = np.concatenate([c[0] for c in counts.values()])
    sc = np.concatenate([c[1] for c in counts.values()])
    assert frames > 1 and wrap > 0 and at_one > 0
    assert ((cc <= 100) | (sc <= 100)).any()                             # a bin left unmatched
    assert ((cc == sc) & (cc > 100)).any()                               # a matched bin with equal counts
    assert ((cc != sc) & (cc > 100) & (sc > 100)).any()                  # a matched bin through the quantile index


def test_hsv_entry_points_declared_and_bound(svr2lib):
    import __graft_entry__
    __graft_entry__.build()
    hdr = open(os.path.join(ROOT, "include", "svr2.h")).read()
    lib = svr2lib.load()
    for name, nargs in HSV_ENTRY_POINTS.items():
        assert re.search(rf"\b{name}\s*\(", hdr), name
        assert len(svr2lib.SIGNATURES[name]) == nargs and hasattr(lib, name)


def test_hsv_refuses_bad_arguments_without_touching_memory(svr2lib):
    """Argument checks run before any launch: each refusal is an error status with a message, not a fault."""
    lib = svr2lib.load()
    n = 5 * 2160 * 3840
    need = lib.svr2_hsv_scratch_bytes(n)
    assert need >= 68 * n and need < 80 * n                               # header, msat, 3 key + 2 value buffers, CUB
    assert lib.svr2_hsv_scratch_bytes(0) == 0 and lib.svr2_hsv_scratch_bytes(1 << 31) == 0
    fake = ctypes.c_void_p(1 << 20)
    rc = lib.svr2_hsv_saturation_match_bf16(fake, fake, None, fake, 5, 2160 * 3840, fake, need - 1, None)
    assert rc == -1 and b"scratch too small" in lib.svr2_last_error()
    assert lib.svr2_hsv_saturation_match_bf16(fake, fake, None, fake, 0, 2160 * 3840, fake, need, None) == -1
    assert b"empty" in lib.svr2_last_error()
    assert lib.svr2_hsv_saturation_match_bf16(fake, fake, fake, fake, 1 << 10, 1 << 21, fake, need, None) == -1
    assert b"2^31" in lib.svr2_last_error()
    assert lib.svr2_wavelet_level_f32(fake, 1, None, None, None, None, 3, 8, 8, 1, 1, None) == -1
    assert b"low is required" in lib.svr2_last_error()
    assert lib.svr2_wavelet_level_f32(fake, 1, fake, None, fake, None, 3, 8, 8, 1, 1, None) == -1
    assert lib.svr2_wavelet_level_f32(fake, 0, fake, None, None, None, 0, 8, 8, 1, 1, None) == -1
    assert b"empty image" in lib.svr2_last_error()
