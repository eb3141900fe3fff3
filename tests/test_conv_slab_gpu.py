"""The slab mainloop of the implicit-GEMM conv (include/svr2.h svr2_conv_mainloop), element by element (-m gpu).

Stride-1 3x3 convs on the swap-AB tiles and on the 256-column tiles load one activation box of bh + 2 rows per
(kt, kw, 64-channel block), the slab, and read its three vertical taps kh from rows kh .. kh + bh - 1 of it.  Each case
below runs through run_conv_case of test_conv_elementwise_gpu.py: every output element against its fp64 bound, a sentinel
in every byte of the allocation the conv must not write, and every GroupNorm partial sum.  The cases are chosen where the
slab addressing can go wrong: the first and last image rows (the slab's halo rows lie outside the tensor), ragged last
tile rows (H = 270, 135) and right edges, each tile shape, 1, 2, 4 and 8 channel blocks per tap, band seams, the fused
1x1x1 shortcut's one-use slabs, ldc > Cout and output halo frames.  Folded head frames on this path are the stride-1
cases of test_vae_head_fold_gpu.py, asserted here to take it."""
import pytest

from test_conv_elementwise_gpu import ConvCase, run_conv_case
from test_vae_head_fold_gpu import CASES as FOLD_CASES

K3 = (3, 3, 3)
SLAB_CASES = {
    # swap-AB (Cout = 128): 32 x 8, 16 x 16 and 8 x 32 tiles
    "swap_32x8_cin64_h270_stats": (ConvCase(64, 128, K3, 270, 40, 2, stats=True),
                                   dict(swap=True, bw=32, bh=8, tiles_h=34, tiles_w=2)),
    "swap_32x8_cin512_h135_band_seams": (ConvCase(512, 128, K3, 135, 384, 2, stats=True),
                                         dict(swap=True, bw=32, bh=8, tiles_h=17, band_h=4)),
    "swap_16x16_cin256_h270_ldc_dup": (ConvCase(256, 128, K3, 270, 13, 2, ldc=136, out_pad=2, dup=1),
                                       dict(swap=True, bw=16, bh=16, tiles_h=17)),
    "swap_8x32_cin128_h135_stats": (ConvCase(128, 128, K3, 135, 7, 3, stats=True),
                                    dict(swap=True, bw=8, bh=32, tiles_h=5)),
    "swap_shortcut_c2_128": (ConvCase(128, 128, K3, 45, 70, 2, C2=128, out_pad=2, dup=1),
                             dict(swap=True, bw=32, bh=8, tiles_h=6, tiles_w=3)),
    # 256-column tiles (Cout >= 256): 16 x 8 and 8 x 16
    "n256_16x8_cin512_h135_band_seams": (ConvCase(512, 256, K3, 135, 200, 2, stats=True),
                                         dict(swap=False, bw=16, bh=8, tiles_h=17, tiles_w=13, band_h=7)),
    "n256_8x16_cin256_h270_residual_ldc": (ConvCase(256, 256, K3, 270, 6, 2, residual=True, ldc=264, out_pad=2),
                                           dict(swap=False, bw=8, bh=16, tiles_h=17)),
    "n512_16x8_cin128_stats_dup": (ConvCase(128, 512, K3, 33, 50, 2, stats=True, out_pad=2, dup=1),
                                   dict(swap=False, bw=16, bh=8, tiles_h=5)),
    "n256_16x8_cin64": (ConvCase(64, 256, K3, 37, 23, 3), dict(swap=False, bw=16, bh=8, tiles_h=5)),
    "n256_shortcut_c2_512": (ConvCase(256, 256, K3, 20, 40, 2, C2=512, out_pad=2), dict(swap=False, bw=16, bh=8)),
}

# one geometry of each kind that stays on the one-ring mainloop
RING_CASES = {
    "row_tiles_128x1": (512, 256, K3, 1, 5, 4000),
    "stride2_pair_view": (256, 256, K3, 2, 26, 86),
    "stride2_pair_view_swap": (128, 128, K3, 2, 38, 140),
    "kt1_3x3": (256, 256, (1, 3, 3), 1, 20, 40),
    "kt1_1x1x1_swap": (256, 128, (1, 1, 1), 1, 19, 45),
    "cout32": (512, 32, K3, 1, 17, 30),
    "cout192_128_column_tiles": (256, 192, K3, 1, 20, 40),
    "swap_too_small_128_column_tiles": (128, 128, K3, 1, 8, 8),
}


def mainloop(lib, Cin, Cout, k, stride_hw, H, W):
    return lib.load().svr2_conv_mainloop(Cin, Cout, *k, stride_hw, H, W)


@pytest.mark.parametrize("name", list(SLAB_CASES))
def test_case_takes_the_slab_path(svr2lib, name):
    c, _ = SLAB_CASES[name]
    assert mainloop(svr2lib, c.Cin, c.Cout, c.k, c.stride_hw, c.H, c.W) == 1


@pytest.mark.parametrize("name", list(RING_CASES))
def test_excluded_geometry_takes_the_ring(svr2lib, name):
    Cin, Cout, k, s, H, W = RING_CASES[name]
    assert mainloop(svr2lib, Cin, Cout, k, s, H, W) == 0


def test_folded_head_cases_take_the_slab_path(svr2lib):
    names = [n for n, c in FOLD_CASES.items() if c.stride_hw == 1 and c.Cout >= 128]
    assert {"swap_128_T5_stats", "generic_256_T5_residual"} <= set(names)
    for n in names:
        c = FOLD_CASES[n]
        assert mainloop(svr2lib, c.Cin, c.Cout, K3, 1, c.H, c.W) == 1, n


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SLAB_CASES))
def test_slab_conv_elementwise(svr2lib, name):
    case, expect = SLAB_CASES[name]
    run_conv_case(svr2lib, case, seed=sum(map(ord, name)), expect=expect)
