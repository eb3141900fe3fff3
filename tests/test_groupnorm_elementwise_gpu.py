"""-m gpu: every VAE GroupNorm(32)(+SiLU) launch element by element against fp64, including offset and near-flat groups.

Both paths are checked through the C ABI: the stand-alone svr2_groupnorm_bf16 (statistics pass, finalize, apply) and
svr2_groupnorm_from_stats_bf16 (finalize from a conv epilogue's per-slot partial sums, apply).  Outputs start as a
sentinel bit pattern with a guard frame before and after; the halo frames must equal frame 0 bit for bit when
duplicated and keep the sentinel otherwise; a second launch must be bit-identical; and the per-channel coefficients
(a, b) the finalize leaves in its scratch are checked on their own, so a statistics fault is reported as one.
  a. the stand-alone path at every channel count, below / at / past its pixel stride, 4x-unroll tails, the one -> two
     block step at hw = 4096 / 4097, a 1088 x 1920 frame, 1 and 3 frames, with and without SiLU and each halo form;
  b. the fused path fed with synthetic partials (1 .. 64 800 slots, the 4K shard's count) and with partials from real
     svr2_conv3d_stats_bf16 / _shortcut_stats_bf16 launches;
  c. offset groups (mean / std up to 256, the offset shared by a group's channels or spread across them), constant
     groups, a constant frame with a one-pixel border ring (a conv over a black frame) and half-flat frames;
  d. every distinct GroupNorm launch of the VAE at 1088 x 1920 and 712 x 400, on random and on near-flat frames.

Reference, per (frame, group) of the bf16 input as the kernel reads it, in fp64: mean m, variance v (centred),
rstd = (v + eps)^-1/2, a = rstd gamma, b = beta - m a, t = a x + b, one bf16 rounding, then for SiLU the exact silu
and a second bf16 rounding.  Rounding points are followed as intervals (tests/test_dit_block_elementwise_gpu.py): a
value the kernel computes in fp32 is t +- e; at a bf16 rounding point the kernel's result lies between rne(t - e) and
rne(t + e), so the check is bit-exact wherever e cannot cross a rounding boundary.

Kernel error budget (U = 2^-24), that of a correct fp32 / fp64 implementation:
  - statistics: sums in fp32 chains of at most c terms, the rest in fp64, give |dm| <= c U E|x| and
    |dv| <= 3 c U min(E[x^2], 18 v) + N 2^-53 E[x^2] (N = hw * channels per group: any fp64 chain).  The raw moments
    E[x^2] - m^2 cancel by E[x^2] / v = 1 + (m / std)^2; an implementation may take v from them while that loses
    less than about four bits (E[x^2] <= 18 v) and must not beyond: the bound never grows with (m / std)^2 past 18.
    c per path: the stand-alone statistics chains, 4 ceil(pixels per block / pixel stride); a conv epilogue slot,
    1032 (<= 256 pixels x 4 channels per lane chain, then a shuffle tree: tests/test_conv_elementwise_gpu.py);
    synthetic partials (fp64 slot sums rounded once to fp32, shifted re-sums of 4 values), 8.
  - rstd: the interval [(v + dv + eps)^-1/2, (max(v - dv, 0) + eps)^-1/2], plus 7 U (the fp32 casts of v and m, the
    eps add, rsqrtf's 2 ulp, the product with gamma): relative ra on a.
  - b = beta - m~ a~ and t~ = fma(x, a~, b~): t~ - t = (a~ - a)(x - m) - a~ dm + the roundings of m~ a~, of b~ and of
    the fma, so e_t = |a| ra |x - m| + |a| (1 + ra) |dm| + 1.01 U (|m a| (1 + ra) + |b| + |t|).
  - silu_fast: relative 2^-19 (1 + |x| + |x|^3 / 20), |silu'| <= 1.1.
Every random-operand case asserts that its median bound is at most 1/20 of the output's standard deviation."""
import ctypes
import importlib
import math
from typing import NamedTuple

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
EPS = 1e-6
SENTINEL = 0x7FA5          # a NaN payload no kernel writes
MAX_STRIP = 1 << 25        # elements per fp64 reference strip
C_CONV = 1032              # fp32 chain length of a conv epilogue statistics slot
C_SYNTH = 8                # synthetic partials: one fp32 rounding per slot sum; shifted re-sums of 4 values


# ====================================================================== helpers (as in the conv / DiT element tests)
def bits(t):
    return t.view(torch.int16)


def sentinel_fill(t):
    bits(t).fill_(SENTINEL)
    return t


def check_untouched(region, what):
    bad = bits(region) != SENTINEL
    n = int(bad.sum())
    assert n == 0, f"{what}: {n} elements written, first at {bad.nonzero()[0].tolist()}"


def rne_bf16(z):
    """fp64 -> the nearest bf16 value (ties to even), exactly"""
    m, e = torch.frexp(z)
    return torch.round(m * 256.0) * torch.exp2((e - 8).to(z.dtype))


def round_iv(z, e):
    """(r, B): the reference value and the bound of a bf16 rounding point whose fp32 input is z +- e"""
    r = rne_bf16(z)
    return r, torch.maximum(rne_bf16(z + e) - r, r - rne_bf16(z - e))


def fast_rel(x):
    a = x.abs()
    return 2.0 ** -19 * (1 + a + a * a * a / 20)


class Sensitivity:
    """Samples of a check's bound and of the output it protects; the median bound must stay below std / 20."""

    def __init__(self, what):
        self.what, self.b, self.s = what, [], []

    def add(self, B, signal):
        step = max(1, B.numel() // 200000)
        self.b.append(B.flatten()[::step].float().cpu())
        self.s.append(signal.flatten()[::step].float().cpu())

    def assert_sensitive(self):
        b, s = torch.cat(self.b), torch.cat(self.s)
        med, sd = b.median().item(), s.std().item()
        assert med <= sd / 20, f"{self.what}: median bound {med:.3g} is not small against the output's std {sd:.3g}"


def rnd(shape, seed, std=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV, dtype=torch.float32) * std


def affine(C, seed):
    return (rnd((C,), seed) * 0.1 + 1).to(torch.bfloat16), (rnd((C,), seed + 1) * 0.1).to(torch.bfloat16)


# ====================================================================== the fp64 reference
class Stats(NamedTuple):
    mean: torch.Tensor      # (F, 32) fp64
    var: torch.Tensor
    eabs: torch.Tensor      # E|x|
    e2: torch.Tensor        # E[x^2]


def group_stats(x):
    """x (F, hw, C) bf16 -> fp64 per (frame, group) statistics, two passes over pixel strips"""
    Fr, hw, C = x.shape
    cpg = C // 32
    rows = max(1, MAX_STRIP // C)
    s = torch.zeros(Fr, 32, device=DEV, dtype=torch.float64)
    sa, s2, sc = s.clone(), s.clone(), s.clone()
    for p0 in range(0, hw, rows):
        xd = x[:, p0:p0 + rows].double().view(Fr, -1, 32, cpg)
        s += xd.sum((1, 3))
        sa += xd.abs().sum((1, 3))
        s2 += (xd * xd).sum((1, 3))
    n = hw * cpg
    mean = s / n
    for p0 in range(0, hw, rows):
        xd = x[:, p0:p0 + rows].double().view(Fr, -1, 32, cpg) - mean[:, None, :, None]
        sc += (xd * xd).sum((1, 3))
    return Stats(mean, sc / n, sa / n, s2 / n)


class Coef(NamedTuple):
    a: torch.Tensor         # (F, C) fp64 reference
    b: torch.Tensor
    ra: torch.Tensor        # relative bound on a
    dm: torch.Tensor        # bound on the mean
    m: torch.Tensor         # (F, C) mean of the channel's group


def coef_ref(st, gamma, beta, c, n):
    """(a, b) and their error budget (module docstring), expanded to channels"""
    v = st.var
    dv = 3 * c * U * torch.minimum(st.e2, 18 * v) + n * 2.0 ** -53 * st.e2
    rstd = (v + EPS).rsqrt()
    lo, hi = (v + dv + EPS).rsqrt(), ((v - dv).clamp_min(0) + EPS).rsqrt()
    ra = torch.maximum(hi / rstd - 1, 1 - lo / rstd) + 7 * U
    dm = c * U * st.eabs + U * st.mean.abs()
    C = gamma.numel()
    ex = lambda t: t.repeat_interleave(C // 32, dim=1)          # noqa: E731
    a = ex(rstd) * gamma.double()
    m = ex(st.mean)
    return Coef(a, beta.double() - m * a, ex(ra), ex(dm), m)


def check_coef(got, cr, what):
    """got (F, C, 2) fp32 (a, b) from the finalize's scratch"""
    ga, gb = got[..., 0].double(), got[..., 1].double()
    Ba = cr.ra * cr.a.abs() + 2.0 ** -140
    ma = (cr.m * cr.a).abs()
    Bb = ma * cr.ra + cr.a.abs() * (1 + cr.ra) * cr.dm + 1.01 * 2 * U * (ma * (1 + cr.ra) + cr.b.abs()) + 2.0 ** -140
    for name, g, r, B in (("a = rstd gamma", ga, cr.a, Ba), ("b = beta - mean a", gb, cr.b, Bb)):
        err = (g - r).abs()
        bad = ~(err <= B)
        if bad.any():
            f, ch = bad.nonzero()[0].tolist()
            raise AssertionError(f"{what}: coefficient {name}: {int(bad.sum())} channels outside the bound; first frame "
                                 f"{f}, channel {ch} (group {ch // (r.shape[1] // 32)}): got {g[f, ch].item():.9g}, "
                                 f"want {r[f, ch].item():.9g}, |err| {err[f, ch].item():.3g} > {B[f, ch].item():.3g}")


def check_body(y, x, cr, silu, what, sens=None):
    """y, x (F, hw, C): every element within its bound, in pixel strips"""
    Fr, hw, C = x.shape
    rows = max(1, MAX_STRIP // (Fr * C))
    a, b, ra, dm, m = (t[:, None, :] for t in cr)
    for p0 in range(0, hw, rows):
        xd = x[:, p0:p0 + rows].double()
        t = a * xd + b
        e = a.abs() * ra * (xd - m).abs() + a.abs() * (1 + ra) * dm + 1.01 * U * ((m * a).abs() * (1 + ra) + b.abs() + t.abs())
        r, B = round_iv(t, e)
        if silu:
            z = r * torch.sigmoid(r)
            r, B = round_iv(z, 1.1 * B + fast_rel(r) * z.abs() + 2.0 ** -120)
        got = y[:, p0:p0 + rows].double()
        err = (got - r).abs()
        bad = ~(err <= B)
        n = int(bad.sum())
        if n:
            f, p, ch = bad.nonzero()[0].tolist()
            raise AssertionError(f"{what}: {n} elements outside the bound; first frame {f}, pixel {p + p0}, channel "
                                 f"{ch} (group {ch // (C // 32)}): got {got[f, p, ch].item():.6g}, want "
                                 f"{r[f, p, ch].item():.6g}, |err| {err[f, p, ch].item():.3g} > {B[f, p, ch].item():.3g}")
        if sens is not None:
            sens.add(B, r)
        del xd, t, e, r, B, got, err


# ====================================================================== launching both paths
def standalone_chain(hw, C):
    """longest fp32 chain of the statistics pass: 4 values per pixel, pixels per block / pixel stride per thread"""
    blocks = max(1, -(-hw // 4096))
    ppb = -(-hw // blocks)
    return 4 * -(-ppb // (256 * 8 // C)), blocks


def launch_standalone(lib, x, y, gamma, beta, silu, pad, dup):
    Fr, hw, C = x.shape
    need = lib.load().svr2_groupnorm_scratch_bytes(Fr, hw, C)
    scratch = torch.full(((need + 7) // 8,), float("nan"), device=DEV, dtype=torch.float64)
    lib.call("svr2_groupnorm_bf16", lib.ptr(x), lib.ptr(y), Fr, hw, C, lib.ptr(gamma), lib.ptr(beta), EPS, silu, pad,
             dup, lib.ptr(scratch), scratch.numel() * 8, lib.stream())
    _, blocks = standalone_chain(hw, C)
    off = 64 * blocks * Fr                       # doubles of block partials before the coefficients
    return scratch[off:off + Fr * C].view(torch.float32).view(Fr, C, 2)


def launch_fused(lib, x, y, gamma, beta, silu, pad, dup, part, slots):
    Fr, hw, C = x.shape
    coef = torch.full((Fr * C * 2 + 64,), float("nan"), device=DEV)
    lib.call("svr2_groupnorm_from_stats_bf16", lib.ptr(x), lib.ptr(y), Fr, hw, C, lib.ptr(gamma), lib.ptr(beta), EPS,
             silu, pad, dup, lib.ptr(part), slots, lib.ptr(coef), lib.stream())
    torch.cuda.synchronize()
    assert torch.isnan(coef[Fr * C * 2:]).all(), "fused finalize wrote past frames * C coefficients"
    return coef[:Fr * C * 2].view(Fr, C, 2)


def synth_partials(x, slots, seed):
    """[frames][slots][C/8] float4 (sum, sumsq of channels 0-3, sum, sumsq of 4-7) over a random split of the pixels
    into `slots` runs (some empty when slots > hw), summed in fp64 and rounded once to fp32; 64 NaN guard slots"""
    Fr, hw, C = x.shape
    g = torch.Generator(device="cpu").manual_seed(seed)
    cuts = torch.sort(torch.randint(0, hw + 1, (slots - 1,), generator=g)).values
    slot_of = torch.bucketize(torch.arange(hw), cuts, right=True).to(DEV)
    out = torch.zeros(Fr, slots, C // 8, 2, 2, device=DEV, dtype=torch.float64)
    rows = max(1, MAX_STRIP // C)
    for p0 in range(0, hw, rows):
        xd = x[:, p0:p0 + rows].double().view(Fr, -1, C // 8, 2, 4)
        sq = torch.stack([xd.sum(-1), (xd * xd).sum(-1)], -1)
        out.index_add_(1, slot_of[p0:p0 + rows], sq)
    part = torch.full((Fr * slots * (C // 8) + 64, 4), float("nan"), device=DEV)
    part[:Fr * slots * (C // 8)] = out.view(-1, 4).float()
    return part


def run_gn(lib, x, silu, pad, dup, *, fused=None, seed=0, what="", sensitive=True):
    """Launches one GroupNorm on sentinel-filled output and checks all of it.  fused: None for the stand-alone path,
    else (part, slots, c)."""
    Fr, hw, C = x.shape
    gamma, beta = affine(C, seed + 7)
    ybuf = sentinel_fill(torch.empty(1 + pad + Fr + 1, hw, C, device=DEV, dtype=torch.bfloat16))
    y = ybuf[1:]
    if fused is None:
        c, _ = standalone_chain(hw, C)
        go = lambda: launch_standalone(lib, x, y, gamma, beta, silu, pad, dup)     # noqa: E731
        path = "stand-alone"
    else:
        part, slots, c = fused
        go = lambda: launch_fused(lib, x, y, gamma, beta, silu, pad, dup, part, slots)    # noqa: E731
        path = f"fused ({slots} slots)"
    what = f"groupnorm {path} {Fr}x{hw}x{C} silu{silu} pad{pad} dup{dup}{' ' + what if what else ''}"
    coef = go().clone()
    torch.cuda.synchronize()
    first = ybuf.clone()
    coef2 = go()
    torch.cuda.synchronize()
    assert torch.equal(bits(ybuf), bits(first)), f"{what}: a second launch is not bit-identical"
    assert torch.equal(coef.view(torch.int32), coef2.view(torch.int32)), f"{what}: coefficients not bit-reproducible"
    del first
    check_untouched(ybuf[0], what + ": guard frame before the output")
    check_untouched(ybuf[-1], what + ": guard frame after the output")
    for f in range(pad):
        if dup:
            assert torch.equal(bits(y[f]), bits(y[pad])), f"{what}: halo frame {f} != frame 0"
        else:
            check_untouched(y[f], f"{what}: halo frame {f} (out_dup_head = 0)")
    st = group_stats(x)
    cr = coef_ref(st, gamma, beta, c, hw * (C // 32))
    check_coef(coef, cr, what)
    sens = Sensitivity(what) if sensitive else None
    check_body(y[pad:pad + Fr], x, cr, silu, what, sens)
    if sens is not None:
        sens.assert_sensitive()
    return st


def ordinary(shape, seed):
    return (rnd(shape, seed) * 2 + 0.5).to(torch.bfloat16)


# ====================================================================== a. the stand-alone path
class GnCase(NamedTuple):
    T: int
    hw: int
    C: int
    silu: int
    pad: int
    dup: int
    fused: bool = False


STANDALONE = {
    "c128_hw1": GnCase(1, 1, 128, 1, 2, 1),                       # hw below the pixel stride (16, 8, 4)
    "c256_hw3_nodup": GnCase(3, 3, 256, 0, 2, 0),
    "c512_hw3": GnCase(1, 3, 512, 1, 0, 0),
    "c128_unroll_tail": GnCase(3, 16 * 4 * 3 + 16 * 2 + 5, 128, 1, 2, 1),
    "c256_unroll_tail": GnCase(1, 8 * 4 * 7 + 13, 256, 0, 2, 0),
    "c512_unroll_tail": GnCase(3, 4 * 4 * 9 + 3, 512, 1, 0, 0),
    "c128_hw4096": GnCase(1, 4096, 128, 1, 2, 1),                 # one full block
    "c512_hw4096": GnCase(3, 4096, 512, 0, 2, 0),
    "c256_hw4097": GnCase(3, 4097, 256, 1, 2, 1),                 # two blocks, the last one ragged
    "c512_hw4097": GnCase(1, 4097, 512, 1, 0, 0),
    "c128_hw4097_nodup": GnCase(1, 4097, 128, 0, 2, 0),
    "c512_hw20000": GnCase(1, 20000, 512, 1, 2, 1),
    "c128_1088x1920": GnCase(1, 1088 * 1920, 128, 1, 2, 1),       # 511 blocks, checked in strips
}


@pytest.mark.parametrize("name", list(STANDALONE))
def test_groupnorm_standalone(svr2lib, name):
    c = STANDALONE[name]
    x = ordinary((c.T, c.hw, c.C), seed=sum(map(ord, name)))
    run_gn(svr2lib, x, c.silu, c.pad, c.dup, seed=3)


def test_groupnorm_halo_argument_checks(svr2lib):
    """frame 0 is always copied into exactly two halo frames: out_dup_head with any other out_t_pad is refused"""
    lib = svr2lib
    x = ordinary((1, 64, 128), 1)
    y = sentinel_fill(torch.empty(1 + 2, 64, 128, device=DEV, dtype=torch.bfloat16))
    gamma, beta = affine(128, 2)
    need = lib.load().svr2_groupnorm_scratch_bytes(1, 64, 128)
    scratch = torch.empty((need + 7) // 8, device=DEV, dtype=torch.float64)
    coef = torch.empty(2 * 128, device=DEV)
    part = synth_partials(x, 3, 1)
    for pad in (0, 1, 3):
        with pytest.raises(lib.Svr2Error, match="out_dup_head"):
            lib.call("svr2_groupnorm_bf16", lib.ptr(x), lib.ptr(y[1:]), 1, 64, 128, lib.ptr(gamma), lib.ptr(beta), EPS,
                     1, pad, 1, lib.ptr(scratch), scratch.numel() * 8, lib.stream())
        with pytest.raises(lib.Svr2Error, match="out_dup_head"):
            lib.call("svr2_groupnorm_from_stats_bf16", lib.ptr(x), lib.ptr(y[1:]), 1, 64, 128, lib.ptr(gamma),
                     lib.ptr(beta), EPS, 1, pad, 1, lib.ptr(part), 3, lib.ptr(coef), lib.stream())
        # the conv epilogue and the upsample's shuffle store copy frame 0 the same way
        w = torch.zeros(128, 27 * 128, device=DEV, dtype=torch.bfloat16)
        with pytest.raises(lib.Svr2Error, match="out_dup_head"):
            lib.call("svr2_conv3d_bf16", lib.ptr(x), 3, 8, 8, 128, lib.ptr(w), 128, 3, 3, 3, 1, 1, 1, 1, lib.EPI_BIAS,
                     lib.ptr(gamma), None, lib.ptr(y[1:]), pad, 1, 128, lib.stream())
        with pytest.raises(lib.Svr2Error, match="out_dup_head"):
            lib.call("svr2_upsample_shuffle_bf16", lib.ptr(x), 1, 4, 4, 128, lib.ptr(w), lib.ptr(gamma), 0, 0,
                     lib.ptr(y[1:]), pad, 1, lib.stream())
    torch.cuda.synchronize()
    check_untouched(y, "refused launches")


# ====================================================================== b. the fused path
@pytest.mark.parametrize("slots,T,hw,C,silu,pad,dup", [
    (1, 1, 300, 128, 1, 2, 1),
    (7, 3, 1000, 256, 0, 0, 0),
    (255, 1, 3000, 512, 1, 2, 0),
    (257, 3, 129, 128, 1, 2, 1),             # more slots than pixels: empty slots
    (4099, 1, 40000, 256, 1, 2, 1),
    (64800, 1, 129600, 128, 1, 2, 1),        # the 4K shard's slot count at Cout = 128
])
def test_groupnorm_fused_synthetic_partials(svr2lib, slots, T, hw, C, silu, pad, dup):
    x = ordinary((T, hw, C), seed=slots)
    part = synth_partials(x, slots, seed=slots)
    run_gn(svr2lib, x, silu, pad, dup, fused=(part, slots, C_SYNTH), seed=5)


def conv_stats(lib, x, Cout, seed, C2=0, bias_offset=0.0, group_tied=False):
    """svr2_conv3d_stats_bf16 (or _shortcut_stats_bf16 with C2 > 0): causal 3x3x3 conv of x (2 + T, H, W, Cin) ->
    (y (T, H*W, Cout) bf16, partials, slots).  group_tied: the channels of a GroupNorm group share weights and bias."""
    Tp, H, W, Cin = x.shape
    T = Tp - 2
    K = 27 * Cin
    w = rnd((Cout, K), seed, std=K ** -0.5)
    bias = rnd((Cout,), seed + 1) + bias_offset
    if group_tied:
        w, bias = (t[::Cout // 32].repeat_interleave(Cout // 32, 0) for t in (w, bias))
    w, bias = w.to(torch.bfloat16).contiguous(), bias.to(torch.bfloat16)
    y = torch.empty(T, H, W, Cout, device=DEV, dtype=torch.bfloat16)
    slots = ctypes.c_int(0)
    P = lib.ptr
    if C2:
        x2 = rnd((T, H, W, C2), seed + 2).to(torch.bfloat16)
        wsc = rnd((Cout, C2), seed + 3, std=C2 ** -0.5).to(torch.bfloat16)
        wcat = torch.cat([w, wsc], 1).contiguous()
        args = (P(x), Tp, H, W, Cin, P(wcat), Cout, 3, 3, 3, T, P(bias), P(x2), C2, P(y), 0, 0)
        name = "svr2_conv3d_shortcut_stats_bf16"
    else:
        args = (P(x), Tp, H, W, Cin, P(w), Cout, 3, 3, 3, 1, 1, 1, T, lib.EPI_BIAS, P(bias), None, P(y), 0, 0, Cout)
        name = "svr2_conv3d_stats_bf16"
    assert getattr(lib.load(), name)(*args, None, 0, ctypes.byref(slots), lib.stream()) == 0
    n = T * slots.value * (Cout // 8)
    part = torch.full((n + 64, 4), float("nan"), device=DEV)
    lib.call(name, *args, P(part), n * 16, ctypes.byref(slots), lib.stream())
    torch.cuda.synchronize()
    assert torch.isfinite(part[:n]).all(), "every statistics slot must be written"
    return y.view(T, H * W, Cout), part, slots.value


@pytest.mark.parametrize("Cin,Cout,T,H,W,C2,silu,pad,dup", [
    (64, 128, 2, 20, 36, 0, 1, 2, 1),
    (128, 256, 3, 19, 30, 0, 1, 2, 0),
    (256, 512, 1, 12, 20, 0, 0, 0, 0),
    (128, 128, 1, 45, 130, 0, 1, 2, 1),
    (128, 128, 2, 30, 44, 256, 1, 2, 1),
    (256, 256, 1, 17, 33, 128, 0, 2, 0),
])
def test_groupnorm_fused_conv_partials(svr2lib, Cin, Cout, T, H, W, C2, silu, pad, dup):
    """conv + statistics epilogue + GroupNorm from its partials, end to end"""
    x = rnd((2 + T, H, W, Cin), 11).to(torch.bfloat16)
    y, part, slots = conv_stats(svr2lib, x, Cout, 12, C2=C2)
    run_gn(svr2lib, y, silu, pad, dup, fused=(part, slots, C_CONV), seed=13)


# ====================================================================== c. offset and near-flat groups
def offset_input(T, hw, C, ratio, spread, seed):
    """groups of std 0.25 whose mean is `ratio` std (alternating in sign from group to group): the offset shared by the
    group's channels, or spread across them (each channel's own offset, ratio +- 0.5 std)"""
    x = rnd((T, hw, C), seed)
    off = torch.full((C,), float(ratio), device=DEV)
    if spread:
        off = off + 0.5 * rnd((C,), seed + 1)
    sign = torch.where(torch.arange(C, device=DEV) // (C // 32) % 2 == 0, 1.0, -1.0)
    x = x * 0.25 + off * sign * 0.25          # std 0.25 like a SiLU'd activation, mean ratio * 0.25
    return x.to(torch.bfloat16)


def ring_frame(T, H, W, C, seed, base=1.7, ring=0.05):
    """a constant frame with a one-pixel border ring, as a conv over a black frame leaves it; one value per group"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    b = (base * (1 + 0.1 * torch.randn(32, generator=g, device=DEV))).repeat_interleave(C // 32)
    x = b.expand(T, H, W, C).clone()
    x[:, 0] += ring
    x[:, -1] += ring
    x[:, :, 0] += ring
    x[:, :, -1] += ring
    return x.to(torch.bfloat16).view(T, H * W, C)


def both_paths(lib, x, silu, pad, dup, what, sensitive=True, seed=0):
    """the stand-alone path, then the fused one on partials of 128-pixel slots (a conv epilogue's); both are run and
    reported"""
    failures = []
    slots = max(1, x.shape[1] // 128)
    for fused in (None, (synth_partials(x, slots, seed + 1), slots, C_SYNTH)):
        try:
            run_gn(lib, x, silu, pad, dup, fused=fused, seed=seed, what=what, sensitive=sensitive)
        except AssertionError as e:
            failures.append(str(e).split("\n")[0])
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("ratio", [0, 4, 16, 64, 256])
@pytest.mark.parametrize("spread", [0, 1])
@pytest.mark.parametrize("C,hw", [(128, 4096), (512, 1024)])
def test_groupnorm_offset_groups(svr2lib, ratio, spread, C, hw):
    """stand-alone chains of 1024 values at both channel counts, so that the fp32 mean's budget c U E|x| stays
    below 1/20 of the output's spread even at mean / std = 256"""
    x = offset_input(1, hw, C, ratio, spread, seed=ratio + 10 * spread + C)
    both_paths(svr2lib, x, 1, 2, 1, f"mean/std {ratio}{' spread' if spread else ''}", seed=ratio)


@pytest.mark.parametrize("C", [128, 256, 512])
def test_groupnorm_constant_groups(svr2lib, C):
    """variance 0 (one value per group): the output is beta (through SiLU) up to the fp32 evaluation of a x + b"""
    x = (1.7 * (1 + 0.1 * rnd((32,), C))).repeat_interleave(C // 32).expand(2, 3000, C).contiguous().to(torch.bfloat16)
    both_paths(svr2lib, x, 1, 2, 1, "constant groups", sensitive=False)


@pytest.mark.parametrize("C,H,W", [(128, 64, 64), (256, 45, 80), (512, 17, 30), (128, 136, 240)])
def test_groupnorm_flat_frame_border_ring(svr2lib, C, H, W):
    x = ring_frame(1, H, W, C, seed=H)
    both_paths(svr2lib, x, 1, 2, 1, f"flat {H}x{W} frame with a border ring", sensitive=False)
    both_paths(svr2lib, x, 0, 0, 0, f"flat {H}x{W} frame with a border ring", sensitive=False)


@pytest.mark.parametrize("C", [128, 512])
def test_groupnorm_half_flat_frame(svr2lib, C):
    """even groups flat (ring frame), odd groups ordinary data in the same frame"""
    H, W = 40, 60
    flat = ring_frame(2, H, W, C, seed=3)
    x = ordinary((2, H * W, C), 4)
    grp = torch.arange(C, device=DEV) // (C // 32)
    x = torch.where((grp % 2 == 0)[None, None], flat, x)
    both_paths(svr2lib, x, 1, 2, 1, "half-flat frame", sensitive=False)


def test_groupnorm_flat_conv_output_end_to_end(svr2lib):
    """a conv over a constant frame (zero padding makes the border ring) feeding the fused path with its own partials"""
    x = torch.full((3, 48, 80, 128), 0.5, device=DEV).to(torch.bfloat16)
    y, part, slots = conv_stats(svr2lib, x, 128, 21, bias_offset=1.0, group_tied=True)
    run_gn(svr2lib, y, 1, 2, 1, fused=(part, slots, C_CONV), seed=22, what="conv over a flat frame", sensitive=False)


# ====================================================================== d. every GroupNorm launch of the VAE
@pytest.fixture(scope="module")
def production_launches(pkg):
    """Distinct GroupNorm launches of B200VideoVAE at 1088 x 1920 (encode + decode) and 712 x 400, recorded from the
    module's launch sequence on the CPU (kernel layer replaced by a recorder)"""
    lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    mp = pytest.MonkeyPatch()
    launches = []

    def record(name, *a, flops=0.0, nbytes=0.0, tag=""):
        if name in ("svr2_groupnorm_bf16", "svr2_groupnorm_from_stats_bf16"):
            c = GnCase(T=a[2], hw=a[3], C=a[4], silu=a[8], pad=a[9], dup=a[10], fused=name.endswith("stats_bf16"))
            if c not in launches:
                launches.append(c)

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
        # a decode in temporal slices of one latent frame: the later slices keep their halo frames (dup = 0); the
        # capture flag skips the sliced pass's device-memory housekeeping
        mp.setattr(type(eng), "_frames_that_fit", lambda self, H, W, state_bytes_per_pixel=0: 4)
        mp.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
        eng.decode(torch.zeros(1, 16, 3, 712 // 8, 400 // 8, dtype=torch.bfloat16))
    finally:
        mp.undo()
    return launches


def test_production_groupnorm_launches(svr2lib, production_launches):
    """Each distinct launch on random data and on a near-flat frame (constant + border ring), on its own path"""
    cases = production_launches
    assert {c.fused for c in cases} == {False, True}, cases
    assert {(0, 0), (2, 0), (2, 1)} <= {(c.pad, c.dup) for c in cases}, cases
    failures = []
    for i, c in enumerate(cases):
        for kind in ("random", "near-flat"):
            if kind == "random":
                x = ordinary((c.T, c.hw, c.C), 100 + i)
            else:
                H = int(math.isqrt(c.hw))
                while c.hw % H:
                    H -= 1
                x = ring_frame(c.T, H, c.hw // H, c.C, seed=200 + i)
            fused = None
            if c.fused:
                slots = max(1, c.hw // 128)
                fused = (synth_partials(x, slots, 300 + i), slots, C_SYNTH)
            try:
                run_gn(svr2lib, x, c.silu, c.pad, c.dup, fused=fused, seed=i, what=kind, sensitive=kind == "random")
            except AssertionError as e:
                failures.append(str(e).split("\n")[0])
            del x, fused
            torch.cuda.empty_cache()
    assert not failures, f"{len(failures)} of {2 * len(cases)} launches:\n" + "\n".join(failures)
