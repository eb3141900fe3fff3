"""-m gpu: every convolution path of the VAE element by element, at the tile, band and halo edges of its raster.

A fault in the implicit-GEMM conv's addressing is local (one tile, one edge row, one band seam, one halo frame) and
moves a relative-L2 error over a whole 4K output by less than its tolerance.  Here every output element is held to its
own bound against an fp64 reference on the same bf16 operands, every byte of the output allocation outside the body
must keep a sentinel bit pattern, and the GroupNorm partial sums are compared per frame and channel octet:
  a. the implicit-GEMM conv (svr2_conv3d_bf16 / _stats / _shortcut_stats) on geometries chosen per raster feature
     (band seams and ragged last bands, 128 x 1 row tiles, the swap-AB 16 x 16 and 8 x 32 tiles, the stride-2 pair view,
     frame-major kt = 1, temporal stride 2 incl. the later-slice form, ldc > Cout, halo frames with and without
     duplication, the fused 1x1x1 shortcut, the residual);
  b. the Upsample3D pixel-shuffle GEMM (svr2_upsample_shuffle_bf16);
  c. the two convs that run as GEMMs: the encoder's conv_in (svr2_im2col3_bf16 + linear) and the decoder's conv_out
     (EPI_F32 linear + svr2_conv_tap_gather);
  d. every distinct conv launch of a 1088 x 1920 encode + decode and of a 712 x 400 portrait clip, as recorded from
     the VAE module's own launch sequence, once at T_out = 1.

Per-element bound: |y - r| <= ulp_bf16(r) per bf16 rounding point + c * 2^-24 * S, S = sum |x| |w| (+ |bias|, |res|).
Products of bf16 operands are exact in fp32.  The tensor core adds a k-slice of products to the fp32 accumulator with
one alignment truncation of at most 2^-23 of the largest magnitude it handles (<= S); assuming the hardware normalises
at least every 8 products, K products take <= K/8 such steps: c = K/4.  Every fp32 add after that (bias, residual, the
27 tap partials of conv_out) rounds once more: +1 each.  The fp64 reference's own error (<= K * 2^-53 * S) is
negligible.  With unit-variance operands S ~ 0.64 sqrt(K), so at the largest K the VAE uses (14 336) the bound is
~1.6e-2 against outputs of standard deviation ~1, while one dropped 64-channel tap block moves an element by
~ sqrt(64 / K) ~ 6.7e-2 of it: a local fault lands most of its elements outside the bound."""
import ctypes
import importlib
from typing import NamedTuple

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
# a NaN payload no kernel writes (a kernel's NaN would be the canonical 0x7FC0 / 0x7FFF; random operands give none)
SENTINEL = 0x7FA5
MAX_STRIP = 1 << 25                 # output elements per reference strip (fp64 temporaries of ~256 MB each)


def bits(t):
    return t.view(torch.int16)


def sentinel_fill(t):
    bits(t).fill_(SENTINEL)
    return t


def rnd(shape, seed, std=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=DEV, dtype=torch.float32) * std).to(torch.bfloat16)


def ulp_bf16(r):
    """ulp of bf16 at |r| (fp64): 2^(floor(log2 |r|) - 7), the subnormal ulp 2^-133 below 2^-126"""
    _, e = torch.frexp(r)
    u = torch.exp2((e - 8).to(r.dtype))
    return torch.where(r.abs() < 2.0 ** -126, torch.full_like(r, 2.0 ** -133), u)


# ====================================================================== raster geometry (conv_tile_shape, conv3d_impl)
class Raster(NamedTuple):
    swap: bool
    bw: int
    bh: int
    band_h: int
    tiles_w: int
    tiles_h: int


def raster(Cin, Cout, k, stride_hw, H, W):
    """The tile shape and band of tile rows the conv picks (csrc/gemm.cu: conv_tile_shape and the band rule)."""
    Ho, Wo = (H, W) if stride_hw == 1 else (H // 2, W // 2)
    swap = 64 < Cout <= 128 and Ho * Wo >= 256
    bw, bh = 16, 8
    if swap:
        bw, bh = (8, 32) if Wo <= 8 else (16, 16) if Wo <= 16 else (32, 8)
    elif Wo >= 128 and Ho < 8:
        bw, bh = 128, 1
    elif Wo <= 8:
        bw, bh = 8, 16
    tiles_w, tiles_h = -(-Wo // bw), -(-Ho // bh)
    row_bytes = bh * stride_hw * W * Cin * 2
    band = min(max(1, (12 << 20) // row_bytes), tiles_h)
    if bh == 1 and bw in (128, 256) and k[1] == 3:        # one-row tiles: 8 MiB of input rows, at least 2
        band = min(max(2, (8 << 20) // row_bytes), Ho)
    return Raster(swap, bw, bh, band if k[0] > 1 else tiles_h, tiles_w, tiles_h)


def where(rs, t, h, w):
    th, tw = h // rs.bh, w // rs.bw
    band, row = divmod(th, rs.band_h)
    last = -(-rs.tiles_h // rs.band_h) - 1
    return (f"tile (th {th}, tw {tw}) of {rs.tiles_h} x {rs.tiles_w} ({rs.bh} x {rs.bw} px{', swap-AB' if rs.swap else ''}), "
            f"band {band} of {last + 1} (band_h {rs.band_h}), tile row {row} in the band")


def check_elements(y, r, bound, what, loc):
    """y, r, bound: (T, h, W, C) of one strip; loc(t, h, w) names the raster position of a pixel."""
    err = (y.double() - r).abs()
    bad = ~(err <= bound)                                 # NaN (e.g. an unwritten sentinel) counts as bad
    n = int(bad.sum())
    if n:
        t, h, w, c = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {n} elements outside the bound; first (t {t}, h {h}, w {w}, c {c}) in {loc(t, h, w)}: "
                             f"got {y[t, h, w, c].item():.6g}, want {r[t, h, w, c].item():.6g}, "
                             f"|err| {err[t, h, w, c].item():.3g} > {bound[t, h, w, c].item():.3g}")


def check_untouched(region, what):
    bad = bits(region) != SENTINEL
    n = int(bad.sum())
    assert n == 0, f"{what}: {n} elements written, first at {bad.nonzero()[0].tolist()}"


# ====================================================================== fp64 reference of the implicit-GEMM conv
def conv_ref_rows(x, w, kt, kh, kw, stride_t, stride_hw, pad, T_out, Wo, h0, h1):
    """(r, S) over output rows [h0, h1): r = conv(x, w) and S = conv(|x|, |w|) in fp64, (T_out, h1 - h0, Wo, Cout).
    x (T_in_total, H, W, Cin) bf16 exactly as the kernel reads it (frame 0 = the first frame of its tensor map),
    w (Cout, kt, kh, kw, Cin) bf16.  Spatial zero padding: `pad` on every side for stride 1; for stride 2 the
    input's one missing column / row past the right / bottom edge (the pair view's out-of-bounds fill)."""
    _, H, W, _ = x.shape
    lo, hi = h0 * stride_hw - pad, (h1 - 1) * stride_hw - pad + kh
    right = (Wo - 1) * stride_hw - pad + kw - W
    xs = x[:, max(lo, 0):min(hi, H)].permute(3, 0, 1, 2)[None].double()
    xs = F.pad(xs, (pad, max(right, 0), max(-lo, 0), max(hi - H, 0)))
    wd = w.permute(0, 4, 1, 2, 3).double()
    out = []
    for xi, wi in ((xs, wd), (xs.abs(), wd.abs())):
        o = F.conv3d(xi, wi, stride=(stride_t, stride_hw, stride_hw))[0, :, :T_out, :, :Wo]
        out.append(o.permute(1, 2, 3, 0))
    return out


class ConvCase(NamedTuple):
    Cin: int
    Cout: int
    k: tuple
    H: int
    W: int
    T: int                  # input frames after the halo (kt - 1 frames) -> T_out = (T - 1) // stride_t + 1
    stride_t: int = 1
    stride_hw: int = 1
    ldc: int = 0            # 0: Cout
    out_pad: int = 0
    dup: int = 0
    residual: bool = False
    stats: bool = False
    C2: int = 0             # fused 1x1x1 shortcut over a second tensor of C2 channels
    later_slice: bool = False   # stride_t = 2 after the first temporal slice: pointer one frame on, T_out = T / 2
    cin_real: int = 0       # weights zero past this input channel (the decoder's conv_in: 16 of 64)


def run_conv_case(lib, c: ConvCase, seed=0, expect=None):
    """Launches one conv on sentinel-filled output (and NaN-filled statistics) and checks every element of the
    allocation; `expect`: the Raster fields the case is named after."""
    kt, kh, kw = c.k
    pad_t = kt - 1
    pad_hw = 1 if (c.stride_hw == 1 and kh == 3) else 0
    Ho, Wo = (c.H, c.W) if c.stride_hw == 1 else (c.H // 2, c.W // 2)
    ldc = c.ldc or c.Cout
    rs = raster(c.Cin, c.Cout, c.k, c.stride_hw, c.H, c.W)
    if expect:
        got = {f: getattr(rs, f) for f in expect}
        assert got == expect, f"case does not reach its raster feature: {got} != {expect}"
    if c.later_slice:
        assert c.stride_t == 2 and c.T % 2 == 0
        T_out, first, T_in = c.T // 2, 1, pad_t - 1 + c.T
    else:
        T_out, first, T_in = (c.T - 1) // c.stride_t + 1, 0, pad_t + c.T
    xbuf = rnd((first + T_in, c.H, c.W, c.Cin), seed)        # halo frames hold their own data (a previous slice's)
    x = xbuf[first:]
    K = kt * kh * kw * c.Cin
    w = rnd((c.Cout, kt, kh, kw, c.Cin), seed + 1, std=K ** -0.5)
    if c.cin_real:
        w[..., c.cin_real:] = 0
    bias = rnd((c.Cout,), seed + 2)
    # output: a guard frame, the halo frames, the body, a slack frame; ldc - Cout padding channels
    ybuf = sentinel_fill(torch.empty(1 + c.out_pad + T_out + 1, Ho, Wo, ldc, device=DEV, dtype=torch.bfloat16))
    y = ybuf[1:]
    res = None
    if c.residual:       # indexed with the output's offsets (halo frames included): NaN where it must not be read
        res = rnd((c.out_pad + T_out, Ho, Wo, ldc), seed + 3)
        res[:c.out_pad] = float("nan")
        res[..., c.Cout:] = float("nan")
    P = lib.ptr
    xp = ctypes.c_void_p(x.data_ptr())
    yp = ctypes.c_void_p(y.data_ptr())
    slots = ctypes.c_int(0)
    part = None
    if c.C2:
        x2 = rnd((T_out, c.H, c.W, c.C2), seed + 4)
        wsc = rnd((c.Cout, c.C2), seed + 5, std=c.C2 ** -0.5)
        wcat = torch.cat([w.reshape(c.Cout, K), wsc], 1).contiguous()
        args = (xp, T_in, c.H, c.W, c.Cin, P(wcat), c.Cout, kt, kh, kw, T_out, P(bias), P(x2), c.C2, yp, c.out_pad, c.dup)
        assert lib.load().svr2_conv3d_shortcut_stats_bf16(*args, None, 0, ctypes.byref(slots), lib.stream()) == 0
    else:
        wk = w.reshape(c.Cout, K).contiguous()
        epi = lib.EPI_BIAS | (lib.EPI_RESIDUAL if c.residual else 0)
        args = (xp, T_in, c.H, c.W, c.Cin, P(wk), c.Cout, kt, kh, kw, c.stride_t, c.stride_hw, pad_hw, T_out, epi,
                P(bias), P(res), yp, c.out_pad, c.dup, ldc)
        if c.stats:
            assert lib.load().svr2_conv3d_stats_bf16(*args, None, 0, ctypes.byref(slots), lib.stream()) == 0
    if c.C2 or c.stats:
        assert slots.value == lib.load().svr2_conv_stat_slots(c.Cout, Ho, Wo) == \
            rs.tiles_w * rs.tiles_h * (2 if rs.swap else 4)
        n_part = T_out * slots.value * (c.Cout // 8)
        part = torch.full((n_part + 64, 4), float("nan"), device=DEV)         # 64 guard slots
        extra = (P(part), n_part * 16, ctypes.byref(slots))
        lib.call("svr2_conv3d_shortcut_stats_bf16" if c.C2 else "svr2_conv3d_stats_bf16", *args, *extra, lib.stream())
    else:
        lib.call("svr2_conv3d_bf16", *args, lib.stream())
    torch.cuda.synchronize()

    name = f"conv {c.Cin}{'+' + str(c.C2) if c.C2 else ''}->{c.Cout} k{kt}{kh}{kw} s{c.stride_t}{c.stride_hw} " \
           f"{c.T}x{c.H}x{c.W}"
    # ---- outside the body: the guard and slack frames, the padding channels, the halo frames
    check_untouched(ybuf[0], name + ": guard frame before the output")
    check_untouched(ybuf[-1], name + ": slack frame after the output")
    check_untouched(y[..., c.Cout:], name + ": channels [Cout, ldc)")
    body = y[c.out_pad:c.out_pad + T_out, ..., :c.Cout]
    for f in range(c.out_pad):
        if c.dup:
            assert torch.equal(bits(y[f, ..., :c.Cout]), bits(body[0])), f"{name}: halo frame {f} != frame 0"
        else:
            check_untouched(y[f], f"{name}: halo frame {f} (out_dup_head = 0)")

    # ---- the body, element by element, in strips of output rows
    c_mul = K / 4 + 1 + (1 if c.residual else 0)              # see the module docstring; +1 bias add, +1 residual add
    if c.C2:
        c_mul += c.C2 / 4
    rows = max(1, MAX_STRIP // (T_out * Wo * c.Cout))
    loc = lambda t, h, w_: where(rs, t, h, w_)   # noqa: E731
    for h0 in range(0, Ho, rows):
        h1 = min(Ho, h0 + rows)
        r, S = conv_ref_rows(x, w, kt, kh, kw, c.stride_t, c.stride_hw, pad_hw, T_out, Wo, h0, h1)
        r += bias.double()
        S += bias.double().abs()
        if c.C2:
            x2s = x2[:, h0:h1].double()
            r += x2s @ wsc.double().T
            S += x2s.abs() @ wsc.double().abs().T
        bound = ulp_bf16(r)                                  # the rounding bf16(acc + bias)
        if c.residual:
            rres = res[c.out_pad:, h0:h1, :, :c.Cout].double()
            r, S = r + rres, S + rres.abs()
            bound = bound + ulp_bf16(r)                      # the second rounding bf16(t + res)
        bound = bound + c_mul * U * S
        check_elements(body[:, h0:h1], r, bound, name, lambda t, h, w_: loc(t, h + h0, w_))
        del r, S, bound

    # ---- GroupNorm partial sums: every slot written, per (frame, octet, channel half) sums over the slots
    if part is not None:
        assert torch.isfinite(part[:n_part]).all(), \
            f"{name}: {int((~torch.isfinite(part[:n_part])).any(1).sum())} statistics slots not written, first " \
            f"(frame, slot, octet) {divmod_slot(int((~torch.isfinite(part[:n_part])).any(1).nonzero()[0]), slots.value, c.Cout)}"
        assert torch.isnan(part[n_part:]).all(), f"{name}: statistics written past T_out * slots * Cout / 8"
        got = part[:n_part].double().view(T_out, slots.value, c.Cout // 8, 2, 2).sum(1)       # (.., half, [sum, sq])
        yb = body.double().reshape(T_out, Ho * Wo, c.Cout // 8, 2, 4)
        want = torch.stack([yb.sum((1, 4)), (yb * yb).sum((1, 4))], -1)
        mag = torch.stack([yb.abs().sum((1, 4)), (yb * yb).sum((1, 4))], -1)
        # one slot sums <= 256 pixels x 4 channels in fp32 (thread-local chains, then a shuffle tree): <= 1024 + 8
        # roundings of <= 2^-24 of the slot's magnitude sum; the slots are added here in fp64
        tol = 1032 * U * mag + 1e-30
        bad = ~((got - want).abs() <= tol)
        if bad.any():
            t, o, half, kind = bad.nonzero()[0].tolist()
            raise AssertionError(f"{name}: GroupNorm {'sum' if kind == 0 else 'sum of squares'} of frame {t}, channels "
                                 f"{8 * o + 4 * half}..{8 * o + 4 * half + 3}: {got[t, o, half, kind].item():.8g} vs "
                                 f"{want[t, o, half, kind].item():.8g} ({int(bad.sum())} bad)")


def divmod_slot(i, slots, Cout):
    f, rem = divmod(i, slots * (Cout // 8))
    return f, *divmod(rem, Cout // 8)


# ====================================================================== a. raster features
CASES = {
    # several full bands of one tile row plus ragged last rows / columns: 512 ch x 1030 px rows = 8.4 MB per tile row
    "bands_of_one_row": (ConvCase(512, 256, (3, 3, 3), 36, 1030, 2), dict(band_h=1, tiles_h=5, tiles_w=65)),
    # bands of 2 tile rows, the last one short (5 = 2 + 2 + 1), statistics over the seams
    "bands_ragged_last_stats": (ConvCase(512, 256, (3, 3, 3), 37, 600, 3, stats=True),
                                dict(swap=False, band_h=2, tiles_h=5, tiles_w=38)),
    # 128 x 1 row tiles under the 8 MiB band rule: H_out 5 = 2 + 2 + 1, ragged last tile column
    "row_tiles_8mib_band": (ConvCase(512, 256, (3, 3, 3), 5, 4000, 2), dict(bw=128, bh=1, band_h=2, tiles_w=32)),
    "row_tiles_8mib_band_stats": (ConvCase(512, 512, (3, 3, 3), 5, 4000, 1, stats=True),
                                  dict(bw=128, bh=1, band_h=2, tiles_w=32)),
    # swap-AB narrow tiles, stride 1 and through the stride-2 pair view, ragged in both directions
    "swap_16x16": (ConvCase(256, 128, (3, 3, 3), 40, 13, 2), dict(swap=True, bw=16, bh=16, tiles_h=3)),
    "swap_8x32_stats": (ConvCase(128, 128, (3, 3, 3), 70, 7, 2, stats=True), dict(swap=True, bw=8, bh=32, tiles_h=3)),
    "swap_16x16_pair": (ConvCase(128, 128, (3, 3, 3), 44, 30, 3, stride_t=2, stride_hw=2),
                        dict(swap=True, bw=16, bh=16, tiles_h=2)),
    "swap_8x32_pair_stats": (ConvCase(128, 128, (1, 3, 3), 90, 14, 2, stride_hw=2, stats=True),
                             dict(swap=True, bw=8, bh=32, tiles_h=2)),
    # pair view, odd tiles_w, ragged H_out: plain (256 ch) and swap-AB tiles
    "pair_odd_tiles_w": (ConvCase(256, 256, (3, 3, 3), 26, 86, 2, stride_hw=2, ldc=264),
                         dict(swap=False, bw=16, bh=8, tiles_w=3, tiles_h=2)),
    "pair_odd_tiles_w_swap_stats": (ConvCase(128, 128, (3, 3, 3), 38, 140, 2, stride_hw=2, stats=True),
                                    dict(swap=True, bw=32, bh=8, tiles_w=3, tiles_h=3)),
    # kt = 1: frame-major order (the band is the whole frame)
    "kt1_frame_major": (ConvCase(256, 256, (1, 3, 3), 20, 40, 3, stride_hw=2), dict(band_h=2, tiles_h=2)),
    "kt1_swap_1x1x1": (ConvCase(256, 128, (1, 1, 1), 19, 45, 3, ldc=136), dict(swap=True, band_h=3)),
    # temporal stride 2: odd T, even T (one unread trailing frame), and a later temporal slice
    "stride_t2_odd_T": (ConvCase(256, 256, (3, 3, 3), 12, 20, 5, stride_t=2, stride_hw=2), dict(swap=False)),
    "stride_t2_even_T": (ConvCase(256, 256, (3, 3, 3), 12, 20, 4, stride_t=2, stride_hw=2), dict(swap=False)),
    "stride_t2_later_slice": (ConvCase(256, 256, (3, 3, 3), 12, 20, 4, stride_t=2, stride_hw=2, later_slice=True),
                              dict(swap=False)),
    "stride_t2_later_slice_swap": (ConvCase(128, 128, (3, 3, 3), 36, 44, 4, stride_t=2, stride_hw=2, later_slice=True),
                                   dict(swap=True)),
    # production odd shapes: encoder conv_out (512 -> 32, 32-column tiles), decoder conv_in (16 of 64 channels -> 512)
    "encoder_conv_out": (ConvCase(512, 32, (3, 3, 3), 17, 30, 2, out_pad=0), dict(swap=False, bw=16, bh=8)),
    "decoder_conv_in_stats": (ConvCase(64, 512, (3, 3, 3), 13, 23, 2, stats=True, cin_real=16), dict(swap=False)),
    # fused 1x1x1 shortcut, C2 != Cin, ragged edges, halo frames duplicated or not
    "shortcut_swap_stats": (ConvCase(128, 128, (3, 3, 3), 30, 44, 2, C2=256, out_pad=2, dup=1),
                            dict(swap=True, bw=32, bh=8)),
    "shortcut_256_stats": (ConvCase(256, 256, (3, 3, 3), 17, 33, 2, C2=128, out_pad=2, dup=0),
                           dict(swap=False, bw=16, bh=8)),
    "shortcut_512_stats": (ConvCase(512, 512, (3, 3, 3), 9, 19, 1, C2=256), dict(swap=False)),
    # residual into an output with 2 halo frames: duplicated (first slice) and not (later slices), with ldc > Cout
    "residual_halo_dup_stats": (ConvCase(128, 128, (3, 3, 3), 21, 50, 2, out_pad=2, dup=1, residual=True, stats=True),
                                dict(swap=True)),
    "residual_halo_nodup": (ConvCase(256, 256, (3, 3, 3), 11, 37, 2, out_pad=2, dup=0, residual=True, ldc=272),
                            dict(swap=False)),
    "residual_halo_swap_ldc": (ConvCase(128, 128, (3, 3, 3), 21, 50, 2, out_pad=2, dup=1, residual=True, ldc=144),
                               dict(swap=True)),
    "residual_512_row_tiles": (ConvCase(512, 512, (3, 3, 3), 3, 300, 2, out_pad=2, dup=1, residual=True),
                               dict(bw=128, bh=1)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_conv_raster_feature(svr2lib, name):
    case, expect = CASES[name]
    run_conv_case(svr2lib, case, seed=sum(map(ord, name)), expect=expect)


# ====================================================================== b. Upsample3D pixel shuffle
@pytest.mark.parametrize("C,temporal,drop,dup,F_,H,W", [
    (256, 0, 0, 1, 2, 5, 32),        # spatial, W % 32 == 0, ragged last m-tile (320 rows)
    (256, 0, 0, 0, 2, 7, 20),        # spatial, W % 32 != 0, halo frames left alone
    (512, 1, 1, 1, 3, 3, 64),        # temporal, first slice: (f = 0, z = 1) dropped
    (512, 1, 1, 1, 2, 5, 12),        # temporal, dropped head, W % 32 != 0
    (256, 1, 0, 0, 2, 3, 96),        # temporal, later slice: nothing dropped, halo untouched
])
def test_upsample_shuffle_elementwise(svr2lib, C, temporal, drop, dup, F_, H, W):
    z = 2 if temporal else 1
    T_out = F_ * z - (1 if temporal and drop else 0)
    x = rnd((F_, H, W, C), 1)
    w = rnd((4 * z * C, C), 2, std=C ** -0.5)
    b = rnd((4 * z * C,), 3)
    ybuf = sentinel_fill(torch.empty(1 + 2 + T_out + 1, 2 * H, 2 * W, C, device=DEV, dtype=torch.bfloat16))
    y = ybuf[1:]
    svr2lib.call("svr2_upsample_shuffle_bf16", svr2lib.ptr(x), F_, H, W, C, svr2lib.ptr(w), svr2lib.ptr(b), temporal, drop,
                 svr2lib.ptr(y), 2, dup, svr2lib.stream())
    torch.cuda.synchronize()
    check_untouched(ybuf[0], "shuffle: guard frame")
    check_untouched(ybuf[-1], "shuffle: slack frame")
    for f in range(2):
        if dup:
            assert torch.equal(bits(y[f]), bits(y[2])), f"shuffle: halo frame {f} != frame 0"
        else:
            check_untouched(y[f], f"shuffle: halo frame {f}")
    # channel n = ((x * 2 + y) * Z + z) * C + c  ->  output pixel (2h + x, 2w + y), frame f * Z + z
    xd = x.double().reshape(-1, C)
    r = (xd @ w.double().T + b.double()).view(F_, H, W, 2, 2, z, C)
    S = (xd.abs() @ w.double().abs().T + b.double().abs()).view(F_, H, W, 2, 2, z, C)
    r, S = (t.permute(0, 5, 1, 3, 2, 4, 6).reshape(F_ * z, 2 * H, 2 * W, C) for t in (r, S))
    if temporal and drop:
        r, S = torch.cat([r[:1], r[2:]]), torch.cat([S[:1], S[2:]])
    bound = ulp_bf16(r) + (C / 4 + 1) * U * S           # one k-loop of K = C, the bias add, one bf16 rounding

    def loc(t, h, w_):
        f, zz = divmod(t + (1 if temporal and drop and t else 0), z)
        m = (f * H + h // 2) * W + w_ // 2
        return f"GEMM row {m} (m-tile {m // 128}), column group (x {h % 2}, y {w_ % 2}, z {zz})"
    check_elements(y[2:2 + T_out], r, bound, f"shuffle C{C} t{temporal} drop{drop} {F_}x{H}x{W}", loc)


# ====================================================================== c. the two convs that run as GEMMs
def causal_conv_ref(xbuf, w):
    """fp64 (r, S) of the causal 3x3x3 conv, zero spatial padding 1: xbuf (2 + T, H, W, Cin) incl. the halo frames,
    w (Cout, 3, 3, 3, Cin) -> (T, H, W, Cout)"""
    T = xbuf.shape[0] - 2
    return conv_ref_rows(xbuf, w, 3, 3, 3, 1, 1, 1, T, xbuf.shape[2], 0, xbuf.shape[1])


@pytest.mark.parametrize("T,H,W", [(1, 37, 53), (3, 18, 29), (2, 8, 130)])
def test_encoder_conv_in_im2col_linear(svr2lib, T, H, W):
    """encoder.conv_in: 3 channels stored in 8 (channels 3..7 hold NaN: never read), im2col3 into 128 columns (81 taps,
    47 zero columns), one biased linear 128 -> 128."""
    x8 = rnd((2 + T, H, W, 8), 1)
    x8[..., 3:] = float("nan")
    col = sentinel_fill(torch.empty(T * H * W + 1, 128, device=DEV, dtype=torch.bfloat16))
    svr2lib.call("svr2_im2col3_bf16", svr2lib.ptr(x8), T, H, W, 3, 8, svr2lib.ptr(col), 128, svr2lib.stream())
    w = rnd((128, 3, 3, 3, 3), 2, std=81 ** -0.5)
    wk = F.pad(w.reshape(128, 81), (0, 128 - 81)).contiguous()
    b = rnd((128,), 3)
    out = sentinel_fill(torch.empty(T * H * W + 1, 128, device=DEV, dtype=torch.bfloat16))
    svr2lib.linear(col[:-1], wk, bias=b, out=out[:-1])
    torch.cuda.synchronize()
    check_untouched(col[-1], "im2col3: row past T*H*W")
    check_untouched(out[-1], "conv_in: row past T*H*W")
    xp = F.pad(x8[..., :3].permute(3, 0, 1, 2), (1, 1, 1, 1))                    # (3, 2 + T, H + 2, W + 2)
    want = xp.unfold(1, 3, 1).unfold(2, 3, 1).unfold(3, 3, 1).permute(1, 2, 3, 4, 5, 6, 0).reshape(T * H * W, 81)
    bad = bits(col[:-1, :81]) != bits(want.contiguous())
    assert not bad.any(), f"im2col3: {int(bad.sum())} columns differ, first (row, col) {bad.nonzero()[0].tolist()}"
    assert (bits(col[:-1, 81:]) == 0).all(), "im2col3: columns 81..127 must be +0"
    r, S = causal_conv_ref(x8[..., :3], w)
    r, S = r + b.double(), S + b.double().abs()
    bound = ulp_bf16(r) + (128 / 4 + 1) * U * S
    check_elements(out[:-1].view(T, H, W, 128), r, bound, f"encoder conv_in {T}x{H}x{W}", lambda t, h, w_: "the frame")


@pytest.mark.parametrize("T,H,W", [(1, 37, 45), (3, 20, 33), (2, 9, 264)])
def test_decoder_conv_out_tap_gather(svr2lib, T, H, W):
    """decoder.conv_out (128 -> 3): z[tap * 3 + co][pixel] = EPI_F32 GEMM over every pixel incl. the 2 halo frames, then
    svr2_conv_tap_gather sums the 27 taps (zero outside the frame), adds the bias, rounds once and writes NCDHW."""
    npix = (2 + T) * H * W
    n4 = (npix + 3) // 4 * 4       # the fp32 GEMM output needs N % 4 == 0: spare pixel rows the gather never reads
    xflat = rnd((n4, 128), 1)
    xbuf = xflat[:npix].view(2 + T, H, W, 128)
    w = rnd((3, 3, 3, 3, 128), 2, std=(27 * 128) ** -0.5)
    b = rnd((3,), 3)
    wt = w.permute(1, 2, 3, 0, 4).reshape(81, 128).contiguous()                # row = tap * 3 + co
    ldz = n4 + 4
    z = torch.full((81, ldz), float("nan"), device=DEV)
    svr2lib.linear(wt, xflat, epi=svr2lib.EPI_F32, out=z[:, :n4])
    obuf = sentinel_fill(torch.empty(3 * T * H * W + 16, device=DEV, dtype=torch.bfloat16))
    out = obuf[8:8 + 3 * T * H * W]
    svr2lib.call("svr2_conv_tap_gather", svr2lib.ptr(z), ldz, 3, svr2lib.ptr(b), T, H, W, svr2lib.ptr(out), 1,
                 svr2lib.stream())
    torch.cuda.synchronize()
    assert torch.isnan(z[:, n4:]).all(), "EPI_F32: columns past N written"
    check_untouched(obuf[:8], "conv_out: before the output")
    check_untouched(obuf[-8:], "conv_out: after the output")
    r, S = causal_conv_ref(xbuf, w)
    r, S = r + b.double(), S + b.double().abs()
    # per tap a K = 128 GEMM (c = 32), then 27 fp32 tap adds and the bias add, one bf16 rounding
    bound = ulp_bf16(r) + (128 / 4 + 28) * U * S
    border = lambda t, h, w_: "border" if h in (0, H - 1) or w_ in (0, W - 1) else "interior"   # noqa: E731
    check_elements(out.view(3, T, H, W).permute(1, 2, 3, 0), r, bound, f"decoder conv_out {T}x{H}x{W}", border)


# ====================================================================== d. every conv launch of the VAE at production sizes
@pytest.fixture(scope="module")
def production_launches(pkg):
    """Distinct conv launches of B200VideoVAE at 1088 x 1920 (encode + decode) and 712 x 400 (a portrait clip whose
    sizes are no tile multiples), recorded from the module's launch sequence on the CPU (kernel layer replaced by a
    recorder, as in tests/test_native_vae_cpu.py)."""
    lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    mp = pytest.MonkeyPatch()
    launches = {}

    def record(name, *a, flops=0.0, nbytes=0.0, tag=""):
        if name in ("svr2_conv3d_bf16", "svr2_conv3d_stats_bf16"):
            key = ConvCase(Cin=a[4], Cout=a[6], k=tuple(a[7:10]), H=a[2], W=a[3], T=1, stride_t=a[10], stride_hw=a[11],
                           out_pad=a[18], dup=a[19], residual=a[16] is not None, stats=name.endswith("stats_bf16"))
        elif name == "svr2_conv3d_shortcut_stats_bf16":
            key = ConvCase(Cin=a[4], Cout=a[6], k=tuple(a[7:10]), H=a[2], W=a[3], T=1, C2=a[13], out_pad=a[15], dup=a[16])
        else:
            return
        launches.setdefault(key, name)

    try:
        mp.setattr(lib, "device_check", lambda: (132, 9, 0))
        eng = vae.B200VideoVAE(pkg.weights.synth_vae_state_dict(seed=1, dtype=torch.float16), device="cpu")
        eng.native = False
        mp.setattr(lib, "call", record)
        mp.setattr(lib, "stream", lambda: None)
        mp.setattr(lib, "_bf16c", lambda t, name: t)
        mp.setattr(type(eng), "_require_cuda", lambda self, what: None)
        mp.setattr(type(eng), "_frames_that_fit", lambda self, H, W, state_bytes_per_pixel=0: 10 ** 6)
        mp.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
        for H, W in ((1088, 1920), (712, 400)):
            eng.encode(torch.zeros(1, 3, 1, H, W, dtype=torch.bfloat16))
            eng.decode(torch.zeros(1, 16, 1, H // 8, W // 8, dtype=torch.bfloat16))
    finally:
        mp.undo()
    return list(launches)


def test_production_conv_launches_stats(svr2lib, production_launches):
    """Each distinct launch once at T_out = 1 (residual / statistics / halo as recorded), element by element."""
    cases = production_launches
    assert len(cases) >= 30 and any(c.C2 for c in cases) and any(c.stride_t == 2 for c in cases)
    kinds = {raster(c.Cin, c.Cout, c.k, c.stride_hw, c.H, c.W)[:3] for c in cases}
    assert {(True, 32, 8), (False, 16, 8)} <= kinds, kinds
    failures = []
    for i, c in enumerate(cases):
        try:
            run_conv_case(svr2lib, c, seed=100 + i)
        except AssertionError as e:
            failures.append(str(e).split("\n")[0])
        torch.cuda.empty_cache()
    assert not failures, f"{len(failures)} of {len(cases)} launches:\n" + "\n".join(failures)
