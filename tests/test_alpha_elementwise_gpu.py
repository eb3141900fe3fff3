"""-m gpu: the alpha path of RGBA clips (csrc/alpha.cu, svr2_alpha_upscale and svr2_sobel_edges_f32 through the C ABI)
element by element: the branch flags and statistics, guided-filter passes A and B, the binary-mask edge-zone refinement
and the bf16 RGBA write.  The base resize (out_kind 2) has its own module, tests/test_resize_elementwise_gpu.py.

The reference runs this path on its GPU tensors, so torch's CUDA rounding is the target.  Each call is checked three ways:
  a. the flags and statistics left in the scratch (layout in include/svr2.h): binary_ratio and binary bit-equal to the
     reference's expression evaluated by torch on the same device tensor, the guide's minimum and both normalisation
     flags, the gx^2 + gy^2 plane and each frame's own maximum of it, exactly;
  b. p (the clamped base), A and B from the scratch, and the output, bit for bit (torch.equal) against torch's CUDA op
     chain of alpha_upscaling.py:212-286 and :358-426 (oracle/alpha_oracle.py): pass A on the kernel's own p, pass B
     and the refinement on the kernel's own A and B, and the whole chain from the alpha;
  c. A, B and the output against fp64 intervals that assume nothing of torch (below).

Error budgets of part c, U = 2^-24.  Every fp32 operation rounds once: a value known within z +- e rounds to within
z +- (e + U (|z| + e)).  Products, quotients and sums propagate their operands' bounds to first order plus the cross
terms.  The inputs are exact: the guide channels g (bf16, or (x + 1) / 2 of them as fp32 ops), p, A and B (read back).
  - guide: I = fl(fl(g0 + g1) + g2) * factor, with torch's fp32 mean factor (fl(1/3) or one ulp off it), read out of
    torch by averaging a one-hot channel tensor of the same shape;
  - box sums of (2R+1)^2 <= 49 terms, added row-major over the window from 0 (ATen's avg_pool2d order, zeros outside
    the image): the terms' own bounds plus one rounding of each exact partial sum; the divisor is (2R+1)^2 everywhere,
    zero padding included (count_include_pad), so a window wider than the image is still / 25 or 49;
  - var = cii - mi^2 cancels: its bound is that of cii plus that of mi^2, not relative to var;
  - a = cov / (var + eps): var + eps >= 0.002 - e_var, so the quotient's bound stays finite; b = mp - a mi;
  - q = box(a) I + box(b); the gradient branch is clamp(q, 0, 1);
  - the binary branch as intervals [lo, hi]: sigmoid((q - 0.5) 12) with expf within 2 ulp (4 U relative) and the
    correctly rounded 1 / (1 + e); the edge strength min(e / 0.25, 1) and the edge-zone tests on the Sobel edges and
    their 3x3 max-pool are exact (those decisions must match), while the thresholds on q, on the combined value (0.5)
    and on the value before the mid-gray cleanup (0.3, 0.5, 0.7) accept either outcome only where the interval
    straddles the threshold (the hull of both outcomes).
bf16 outputs (out_kind 1) lie in [rne(lo), rne(hi)].  Non-vacuity: the median bound of A, B and q is at most 1/20 of the
spread (std) of the values it protects, and at least 99 % of the bf16 output intervals hold a single value.

Every output sits between sentinel guard regions that must keep their bits; with out_kind 1 channels 0..2 of the RGBA
image keep their sentinel and channel 3 of every pixel loses it.  Every failure names the frame, row and column, the
32 x 32 tile and whether the pixel's window is clipped by the image border."""
from typing import NamedTuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import alpha_oracle as ao
from oracle import pre_oracle
from test_conv_elementwise_gpu import SENTINEL, U, bits, check_untouched, sentinel_fill
from test_dit_block_elementwise_gpu import Sensitivity, check, rne_bf16
from test_resize_elementwise_gpu import align256, taps_for

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16
GUARD = 64                      # sentinel elements before and after every output (bytes after the scratch)
TILE = 32                       # output tile edge of the stencil kernels
HDR_BYTES = 48                  # the scratch header before the per-frame Sobel maxima
MAX_CHUNK = 1 << 23             # pixels per fp64 reference chunk
UB = U * (1 + 2.0 ** -20)       # U plus room for the fp64 arithmetic of the bounds themselves
DTYPES = {"f32": (torch.float32, 0), "bf16": (BF16, 1), "f16": (torch.float16, 2), "u8": (torch.uint8, 3)}
OUT_F32, OUT_RGBA, OUT_RESIZE = 0, 1, 2
f32 = lambda v: float(np.float32(v))                                         # noqa: E731
EPS, T03, T05, T15, T3, T7 = f32(ao.EPS), f32(0.03), f32(0.05), f32(0.15), f32(0.3), f32(0.7)


# ====================================================================== calling the kernel, reading its scratch
class Scratch(NamedTuple):
    flags: dict
    fmax: torch.Tensor      # [T] int64, per-frame max of gx^2 + gy^2
    sq: torch.Tensor        # [T, H, W] int64
    p: torch.Tensor         # [T, H, W] fp32, the clamped base resize
    A: torch.Tensor
    B: torch.Tensor


def read_scratch(scratch, T, h, w, H, W, flags_only=False):
    """The intermediates a call left in its scratch (include/svr2.h)"""
    i32, f = scratch[:16].view(torch.int32).tolist(), scratch[16:24].view(torch.float32).tolist()
    flags = dict(binary=i32[0], normalise=i32[1], normalise_twice=i32[2], radius=i32[3], binary_ratio=f[0],
                 guide_min=f[1])
    n = T * H * W
    fmax = scratch[HDR_BYTES:HDR_BYTES + 4 * T].view(torch.int32).long()
    if flags_only:
        return Scratch(flags, fmax, None, None, None, None)
    hdr = align256(HDR_BYTES + 4 * T)
    sq = scratch[hdr:hdr + 4 * n].view(torch.int32).long().view(T, H, W)
    K, L = max(taps_for(h, H), taps_for(w, W)), max(H, W)
    o = hdr + align256(4 * n) + 2 * align256(8 * L) + 2 * align256(4 * L * K)
    planes = []
    for _ in range(3):
        planes.append(scratch[o:o + 4 * n].view(torch.float32).view(T, H, W))
        o += align256(4 * n)
    return Scratch(flags, fmax, sq, *planes)


def call(lib, src, code, channels, rgb, out_kind):
    """svr2_alpha_upscale on src [T, h, w, channels] (the alpha is the last channel) and rgb [T, 3, H, W] bf16, every
    buffer sentinel-guarded.  Returns (out, scratch): out [T, H, W] fp32 or [T, H, W, 4] bf16 (channels 0..2 checked
    untouched here, channel 3 checked written)."""
    T, h, w = src.shape[:3]
    H, W = rgb.shape[2:]
    rgba = out_kind == OUT_RGBA
    n = T * H * W * (4 if rgba else 1)
    buf = sentinel_fill(torch.empty(n + 2 * GUARD, device=DEV, dtype=BF16 if rgba else torch.float32))
    out = buf[GUARD:GUARD + n]
    need = lib.load().svr2_alpha_upscale_scratch_bytes(T, h, w, H, W)
    sbuf = sentinel_fill(torch.empty(need + 2 * GUARD, device=DEV, dtype=torch.uint8).view(torch.int16)).view(torch.uint8)
    rc = lib.load().svr2_alpha_upscale(lib.ptr(src), code, channels, T, h, w, lib.ptr(rgb), H, W, lib.ptr(out), out_kind,
                                       lib.ptr(sbuf), need, lib.stream())
    assert rc == 0, lib.load().svr2_last_error()
    what = f"{T}x{h}x{w}x{channels} -> {H}x{W}, out_kind {out_kind}"
    check_untouched(buf[:GUARD], what + ": guard before the output")
    check_untouched(buf[GUARD + n:], what + ": guard after the output")
    check_untouched(sbuf[need:].view(torch.int16), what + ": bytes after the scratch")
    if rgba:
        img = out.view(T, H, W, 4)
        check_untouched(img[..., :3], what + ": RGBA channels 0..2")
        unwritten = bits(img[..., 3]) == SENTINEL
        assert not unwritten.any(), (f"{what}: {int(unwritten.sum())} alpha values not written, first at "
                                     f"{unwritten.nonzero()[0].tolist()}")
        return img, sbuf[:need]
    return out.view(T, H, W), sbuf[:need]


def where_fn(what, H, W, R):
    def loc(t, y, x):
        clipped = y < R or x < R or y >= H - R or x >= W - R
        return (f"{what}: frame {t}, row {y}, col {x}, tile ({y // TILE}, {x // TILE}), "
                f"{'window clipped by the border' if clipped else 'window inside the image'}")
    return loc


def equal(got, want, what, loc):
    """bit for bit (a NaN, e.g. an unwritten sentinel, fails)"""
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    check(got, want.double(), torch.zeros((), device=got.device, dtype=torch.float64).expand(got.shape), what, loc)


def check_iv(got, lo, hi, what, loc):
    """lo <= got <= hi element by element (a NaN fails)"""
    g = got.double()
    bad = ~((g >= lo) & (g <= hi))
    n = int(bad.sum())
    if n:
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {n} of {bad.numel()} elements outside the interval; first at {loc(*i)}: "
                             f"got {got[i].item():.9g}, want [{lo[i].item():.9g}, {hi[i].item():.9g}]")


# ====================================================================== torch's CUDA op chain
def guide_of(rgb):
    """rgb_normalized (:327-329) in fp32 and whether it was normalised"""
    g = rgb.float()
    norm = bool(g.min() < 0)
    return ((g + 1) / 2 if norm else g), norm


def mean_factor(T, H, W):
    """the fp32 factor of torch's CUDA guide.mean(dim=1) at this shape: the mean of a one-hot channel tensor"""
    one_hot = torch.zeros(T, 3, H, W, device=DEV)
    one_hot[:, 0] = 1
    f = one_hot.mean(dim=1)
    assert (f == f.view(-1)[0]).all()
    return f.view(-1)[0].item()


# ====================================================================== fp64 intervals (module docstring)
def rb(z, e):
    """bound after one fp32 rounding of a value within z +- e"""
    return e + UB * (z.abs() + e)


def iv_add(x, ex, y, ey):
    z = x + y
    return z, rb(z, ex + ey)


def iv_sub(x, ex, y, ey):
    return iv_add(x, ex, -y, ey)


def iv_mul(x, ex, y, ey):
    z = x * y
    return z, rb(z, x.abs() * ey + y.abs() * ex + ex * ey)


def iv_div(x, ex, y, ey):
    assert bool((y.abs() > ey).all()), "divisor interval contains 0"
    z = x / y
    return z, rb(z, (ex + z.abs() * ey) / (y.abs() - ey))


def iv_box(x, ex, r):
    """box mean (avg_pool2d, count_include_pad) of values within x +- ex [T, H, W]: the window summed row-major from
    0 as ATen's kernel does, zeros outside the image; each partial sum rounds once"""
    k, (H, W) = 2 * r + 1, x.shape[1:]
    xp = F.pad(x, (r, r, r, r))
    ep = F.pad(ex, (r, r, r, r)) if torch.is_tensor(ex) else None
    s, e = torch.zeros_like(x), torch.zeros_like(x)
    for j in range(k * k):
        t = xp[:, j // k:j // k + H, j % k:j % k + W]
        et = ep[:, j // k:j // k + H, j % k:j % k + W] if ep is not None else 0.0
        s = s + t
        e = e + et if j == 0 else rb(s, e + et)
    return s / (k * k), rb(s / (k * k), e / (k * k))


def iv_guide(g, factor):
    """I = fl(fl(g0 + g1) + g2) * factor, g [T, 3, H, W] exact fp32 channel values, factor torch's (exact)"""
    g = g.double()
    s1 = g[:, 0] + g[:, 1]
    s, es = iv_add(s1, UB * s1.abs(), g[:, 2], 0.0)
    return iv_mul(s, es, torch.full_like(s, factor), 0.0)


def iv_pass_a(I, eI, p, r):
    mi, emi = iv_box(I, eI, r)
    mp, emp = iv_box(p, 0.0, r)
    cii, ecii = iv_box(*iv_mul(I, eI, I, eI), r)
    cip, ecip = iv_box(*iv_mul(I, eI, p, 0.0), r)
    var, evar = iv_sub(cii, ecii, *iv_mul(mi, emi, mi, emi))
    cov, ecov = iv_sub(cip, ecip, *iv_mul(mi, emi, mp, emp))
    den, eden = iv_add(var, evar, torch.full_like(var, EPS), 0.0)
    a, ea = iv_div(cov, ecov, den, eden)
    b, eb = iv_sub(mp, emp, *iv_mul(a, ea, mi, emi))
    return a, ea, b, eb


def iv_q(I, eI, A, B, r):
    ma, ema = iv_box(A.double(), 0.0, r)
    mb, emb = iv_box(B.double(), 0.0, r)
    return iv_add(*iv_mul(ma, ema, I, eI), mb, emb)


def rd(x):
    return x - UB * x.abs()


def ru(x):
    return x + UB * x.abs()


def step(lo, hi, t):
    """(v > t) as 0 / 1 for v in [lo, hi]: the least and the greatest outcome"""
    return (lo > t).double(), (hi > t).double()


def iv_refine(ql, qh, edges):
    """[lo, hi] of steps 3-8 of the binary branch (:370-408) for q in [ql, qh]; edges exact"""
    e = edges.double()
    zone = F.max_pool2d(e[:, None], 3, 1, 1)[:, 0]
    tl, th = rd(ql - 0.5), ru(qh - 0.5)
    t12l, t12h = rd(12 * tl), ru(12 * th)
    El, Eh = torch.exp(-t12h) * (1 - 4 * U), torch.exp(-t12l) * (1 + 4 * U)
    Dl, Dh = rd(1 + El), ru(1 + Eh)
    sl, sh = rd(1 / Dh), ru(1 / Dl)
    es = (e * 4).clamp(0, 1)
    ol, oh = rd(1 - es), ru(1 - es)
    prods = torch.stack([ql * ol, ql * oh, qh * ol, qh * oh])
    m1l, m1h = rd(prods.amin(0)), ru(prods.amax(0))
    iel, ieh = rd(m1l + rd(sl * es)), ru(m1h + ru(sh * es))
    bl, bh = step(ql, qh, 0.5)
    solid, very, tight = zone < T05, zone < T03, e > T15
    cl, ch = torch.where(solid, bl, iel), torch.where(solid, bh, ieh)
    fbl, fbh = step(cl, ch, 0.5)
    pl, ph = torch.where(very, fbl, cl), torch.where(very, fbh, ch)
    certain = ~tight & (pl > T3) & (ph < T7)
    possible = ~tight & (ph > T3) & (pl < T7)
    sbl, sbh = step(pl, ph, 0.5)
    lo = torch.where(certain, sbl, torch.where(possible, torch.minimum(pl, sbl), pl))
    hi = torch.where(certain, sbh, torch.where(possible, torch.maximum(ph, sbh), ph))
    return lo, hi


# ====================================================================== one call, every check
class Case(NamedTuple):
    T: int
    h: int
    w: int
    H: int
    W: int
    kind: str = "binary"        # binary | gradient (ao.make_inputs) | noise-binary | noise-gradient (any size)
    dtype: str = "bf16"
    channels: int = 1
    seed: int = 0
    lo: float = -1.0
    hi: float = 1.0


def make_case(c: Case):
    """(src [T, h, w, channels] in c.dtype, rgb [T, 3, H, W] bf16) on the device"""
    if c.kind in ("binary", "gradient"):
        alpha, rgb = ao.make_inputs(c.T, c.h, c.w, c.H, c.W, c.kind, c.seed, c.lo, c.hi)
        alpha, rgb = alpha[:, 0].float().to(DEV), rgb.to(DEV)
    else:       # any size, down to one pixel: a noisy guide, a 0/1 or a mid-gray alpha
        g = torch.Generator(device=DEV).manual_seed(c.seed)
        rgb = (torch.rand(c.T, 3, c.H, c.W, generator=g, device=DEV) * (c.hi - c.lo) + c.lo).to(BF16)
        alpha = torch.rand(c.T, c.h, c.w, generator=g, device=DEV)
        alpha = (alpha > 0.5).float() if c.kind == "noise-binary" else alpha * 0.6 + 0.2
    if c.dtype == "u8":
        a = (alpha * 255).round().to(torch.uint8)
    else:
        a = alpha.to(DTYPES[c.dtype][0])
    src = torch.rand(c.T, c.h, c.w, c.channels, device=DEV).to(a.dtype)
    src[..., -1] = a
    return src, rgb


class Sens:
    def __init__(self, what):
        self.a, self.b, self.q = Sensitivity(what + ": A"), Sensitivity(what + ": B"), Sensitivity(what + ": q")
        self.single, self.total = 0, 0

    def assert_sensitive(self):
        for s in (self.a, self.b, self.q):
            s.assert_sensitive()
        if self.total:
            frac = self.single / self.total
            assert frac >= 0.99, f"only {100 * frac:.2f} % of {self.total} bf16 output intervals hold a single value"


def run_case(lib, c: Case, out_kinds=(OUT_F32, OUT_RGBA), sens=None, expect_binary=None, inputs=None):
    src, rgb = make_case(c) if inputs is None else inputs
    T, H, W = c.T, c.H, c.W
    code = DTYPES[c.dtype][1]
    X = pre_oracle.compute_dtype(src[..., -1])[:, None]          # the alpha as the kernel loads it, [T, 1, h, w]
    taps = {}
    want = ao.edge_guided_alpha_upscale(X, rgb, taps)[:, 0]
    if expect_binary is not None:
        assert taps["binary"] == expect_binary, (c, taps["ratio"].item())
    g, norm = guide_of(rgb)
    factor = mean_factor(T, H, W)
    # the guide as torch's CUDA mean computes it: the channel sum in order, times the factor
    assert torch.equal(taps["guide"][:, 0], ((g[:, 0] + g[:, 1]) + g[:, 2]) * factor), "torch's mean is not sum * factor"
    outs = {}
    for kind in out_kinds:
        out, scratch = call(lib, src, code, c.channels, rgb, kind)
        outs[kind] = (out, read_scratch(scratch, T, c.h, c.w, H, W))
    out, s = outs[out_kinds[0]]
    what = f"{c}"
    R = 2 if taps["binary"] else 3
    loc = where_fn(what, H, W, R)
    # a. flags and statistics
    fl = s.flags
    ratio = taps["ratio"].item()
    assert np.float32(fl["binary_ratio"]).view(np.int32) == np.float32(ratio).view(np.int32), (what, fl, ratio)
    assert (fl["binary"], fl["radius"]) == (int(taps["binary"]), R), (what, fl)
    assert (fl["normalise"], fl["normalise_twice"]) == (int(taps["normalise"]), int(taps["normalise_twice"])), (what, fl)
    assert fl["guide_min"] == rgb.min().item(), (what, fl)
    g8 = ao.gray_u8(((g + 1) / 2 if taps["normalise_twice"] else g).mul(255).clamp(0, 255).to(torch.uint8))
    sq = ao.sobel_sq(g8).long()
    equal(s.sq, sq, what + ": gx^2 + gy^2", loc)
    assert torch.equal(s.fmax, sq.amax(dim=(1, 2))), (what, s.fmax.tolist(), sq.amax(dim=(1, 2)).tolist())
    # b. bit for bit against torch's chain: p; pass A on the kernel's p; pass B on the kernel's A, B; the whole chain
    equal(s.p, taps["base"][:, 0], what + ": p vs torch", loc)
    I = taps["guide"]
    ta = {}
    ao.guided_filter(I, s.p[:, None], R, taps=ta)
    equal(s.A, ta["a"][:, 0], what + ": pass A, a vs torch", loc)
    equal(s.B, ta["b"][:, 0], what + ": pass A, b vs torch", loc)
    q = ao.box(s.A[:, None], R) * I + ao.box(s.B[:, None], R)
    tb = {}
    after_b = (ao.refine_binary(q, taps["edges"], tb) if taps["binary"] else q).clamp(0, 1)[:, 0]
    # c. fp64 intervals, a chunk of frames at a time
    step_t = max(1, MAX_CHUNK // (H * W))
    for t0 in range(0, T, step_t):
        t1 = min(T, t0 + step_t)
        floc = lambda f, y, x, t0=t0: loc(t0 + f, y, x)                       # noqa: E731
        I64, eI = iv_guide(g[t0:t1], factor)
        a, ea, b, eb = iv_pass_a(I64, eI, s.p[t0:t1].double(), R)
        check(s.A[t0:t1], a, ea, what + ": pass A, a vs fp64", floc)
        check(s.B[t0:t1], b, eb, what + ": pass A, b vs fp64", floc)
        qz, eq = iv_q(I64, eI, s.A[t0:t1], s.B[t0:t1], R)
        if taps["binary"]:
            lo, hi = iv_refine(qz - eq, qz + eq, taps["edges"][t0:t1, 0])
        else:
            lo, hi = qz - eq, qz + eq
        lo, hi = lo.clamp(0, 1), hi.clamp(0, 1)
        if sens is not None:
            sens.a.add(ea, a)
            sens.b.add(eb, b)
            sens.q.add(eq, qz)
        for kind, (o, _) in outs.items():
            if kind == OUT_RGBA:
                o = o[t0:t1, ..., 3]
                lo_b, hi_b = rne_bf16(lo), rne_bf16(hi)
                check_iv(o, lo_b, hi_b, what + ": bf16 alpha vs fp64", floc)
                if sens is not None:
                    sens.single += int((lo_b == hi_b).sum())
                    sens.total += lo_b.numel()
            else:
                check_iv(o[t0:t1], lo, hi, what + ": alpha vs fp64", floc)
    for kind, (o, sk) in outs.items():
        for name in ("p", "A", "B", "sq", "fmax"):
            assert torch.equal(getattr(sk, name), getattr(s, name)), (what, kind, name)
        got = o[..., 3] if kind == OUT_RGBA else o
        cast = (lambda v: v.to(BF16)) if kind == OUT_RGBA else (lambda v: v)
        equal(got, cast(after_b), f"{what}: out_kind {kind}: pass B on the kernel's a, b vs torch", loc)
        equal(got, cast(want), f"{what}: out_kind {kind}: the whole chain vs torch", loc)
    return taps


# ====================================================================== a. flags and statistics
def ratio_alpha(T, h, w, dtype, channels, seed, extra_mid=0):
    """An alpha with exactly 5 % (+ extra_mid) mid-gray values, the rest split between 0 and 1: ratio 0.95 exactly in
    real arithmetic"""
    n = T * h * w
    assert n % 20 == 0
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = (torch.rand(n, generator=g, device=DEV) > 0.4).float()
    a[torch.randperm(n, generator=g, device=DEV)[:n // 20 + extra_mid]] = 0.5
    a = a.view(T, h, w)
    a = (a * 255).round().to(torch.uint8) if dtype == "u8" else a.to(DTYPES[dtype][0])
    src = torch.zeros(T, h, w, channels, device=DEV, dtype=a.dtype)
    src[..., -1] = a
    return src


def roundings_disagree(n):
    """whether (0.95 n) / n > 0.95 differs between a true division and a multiply by fl(1 / fl(n)), in fp32"""
    c, nf = np.float32(n * 19 // 20), np.float32(n)
    return bool((c / nf > np.float32(0.95)) != (c * (np.float32(1) / nf) > np.float32(0.95)))


def check_flags(lib, src, code, rgb, what):
    _, scratch = call(lib, src, code, src.shape[-1], rgb, OUT_RESIZE)
    fl = read_scratch(scratch, *src.shape[:3], *rgb.shape[2:], flags_only=True).flags
    ratio, binary = ao.binary_ratio(pre_oracle.compute_dtype(src[..., -1]))
    got, want = np.float32(fl["binary_ratio"]), np.float32(ratio.item())
    assert got.view(np.int32) == want.view(np.int32), f"{what}: binary_ratio {got!r}, torch {want!r}"
    assert (fl["binary"], fl["radius"]) == (int(binary), 2 if binary else 3), (what, fl)
    return fl


RATIO_SIZES = [(1, 40, 60), (1, 20, 40), (2, 11, 30), (21, 720, 1280)]


@pytest.mark.parametrize("channels", [1, 4])
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_binary_ratio_bits(svr2lib, dtype, channels):
    """binary_ratio and binary equal torch's CUDA expression on the same device tensor, at a ratio of exactly 0.95
    where a true division and the reciprocal multiply disagree on > 0.95 (1x40x60, 21x720x1280) and where they agree
    (1x20x40, 2x11x30), one value above and below, and on random values around the 0.1 / 0.9 thresholds."""
    code = DTYPES[dtype][1]
    assert [roundings_disagree(T * h * w) for T, h, w in RATIO_SIZES] == [True, False, False, True]
    for T, h, w in RATIO_SIZES:
        if T > 1 and h > 100 and (dtype, channels) != ("u8", 1):
            continue            # the 19 M alpha once, as bytes
        rgb = torch.full((T, 3, h // 4, w // 4), 0.25, device=DEV, dtype=BF16)
        for extra in (0, -1, 1):
            check_flags(svr2lib, ratio_alpha(T, h, w, dtype, channels, T * h + extra, extra), code, rgb,
                        f"{T}x{h}x{w} {dtype} x{channels}, mid-gray n/20 {extra:+d}")
    # values at the thresholds, in every dtype's rounding to bf16
    g = torch.Generator(device=DEV).manual_seed(channels)
    near = torch.tensor([0.0, 0.0996, 0.0999999, 0.1, 0.1001, 0.5, 0.8984, 0.8999999, 0.9, 0.9004, 1.0], device=DEV)
    vals = near[torch.randint(0, len(near), (3 * 17 * 23,), generator=g, device=DEV)]
    if dtype == "u8":
        vals = torch.randint(0, 256, (3 * 17 * 23,), generator=g, device=DEV).float() / 255
    src = torch.zeros(3, 17, 23, channels, device=DEV)
    src[..., -1] = vals.view(3, 17, 23)
    src = (src * 255).round().to(torch.uint8) if dtype == "u8" else src.to(DTYPES[dtype][0])
    check_flags(svr2lib, src, code, torch.zeros(3, 3, 4, 4, device=DEV, dtype=BF16), f"threshold values {dtype}")


@pytest.mark.parametrize("T", [3, 5])
def test_binary_ratio_bits_above_2_24(svr2lib, T):
    """n > 2^24 alpha values (T x 2160 x 3840): the two counts and n are rounded to fp32 before the ratio"""
    rgb = torch.zeros(T, 3, 288, 512, device=DEV, dtype=BF16)
    assert T * 2160 * 3840 > 1 << 24
    for extra in (0, 1, -1, 7):
        check_flags(svr2lib, ratio_alpha(T, 2160, 3840, "u8", 1, extra + 10, extra), 3, rgb, f"{T}x2160x3840 {extra:+d}")


def test_guide_min_and_normalisation_flags(svr2lib):
    """guide minimum +0 (no normalisation), -0.0 (not below 0), -1e-7 (once), -1 ((x + 1) / 2 = 0: once), below -1
    (the edge detector normalises again)"""
    a = torch.ones(1, 20, 30, 1, device=DEV)
    for low, norm, twice in ((0.0, 0, 0), (-0.0, 0, 0), (-1e-7, 1, 0), (-1.0, 1, 0), (-1.5, 1, 1)):
        rgb = torch.full((1, 3, 40, 60), 0.25, device=DEV, dtype=BF16)
        rgb[0, 1, 7, 11] = low
        _, scratch = call(svr2lib, a, 0, 1, rgb, OUT_RESIZE)
        fl = read_scratch(scratch, 1, 20, 30, 40, 60, flags_only=True).flags
        assert (fl["normalise"], fl["normalise_twice"]) == (norm, twice), (low, fl)
        assert fl["guide_min"] == torch.tensor(low).to(BF16).item(), (low, fl)
    for low in (0.0, -1e-7, -1.5):
        c = Case(1, 20, 30, 40, 60, "noise-binary", seed=3, lo=low, hi=1.0)
        run_case(svr2lib, c)


def test_per_frame_sobel_maxima(svr2lib):
    """A flat frame between two textured ones, and textures of different contrast: every frame's edges are normalised
    by its own maximum (the flat frame's edges are 0), in svr2_sobel_edges_f32 and in the binary branch"""
    c = Case(3, 40, 56, 100, 140, "binary", seed=9)
    src, rgb = make_case(c)
    rgb[1] = 0.3
    rgb[2] = (rgb[2].float() * 0.3).to(BF16)
    lib = svr2lib.load()
    edges = sentinel_fill(torch.empty(3 * 100 * 140 + 2 * GUARD, device=DEV))
    scratch = torch.empty(lib.svr2_alpha_upscale_scratch_bytes(3, 1, 1, 100, 140), device=DEV, dtype=torch.uint8)
    rc = lib.svr2_sobel_edges_f32(svr2lib.ptr(rgb), 3, 100, 140, svr2lib.ptr(edges[GUARD:]), svr2lib.ptr(scratch),
                                  scratch.numel(), svr2lib.stream())
    assert rc == 0, lib.svr2_last_error()
    check_untouched(edges[:GUARD], "guard before the edges")
    check_untouched(edges[-GUARD:], "guard after the edges")
    want = ao.detect_edges_batch(rgb)[:, 0]
    equal(edges[GUARD:-GUARD].view(3, 100, 140), want, "edges", where_fn("edges", 100, 140, 1))
    assert want[1].abs().max().item() == 0 and want[0].max().item() == 1 and want[2].max().item() == 1
    fmax = read_scratch(scratch, 3, 1, 1, 100, 140, flags_only=True).fmax
    assert fmax[1].item() == 0 and fmax[0].item() > fmax[2].item() > 0, fmax.tolist()
    # the same frames through the binary branch, every check of run_case
    run_case(svr2lib, c, inputs=(src, rgb), expect_binary=True)


# ====================================================================== b, c. passes A and B, both branches
BRANCH_CASES = [Case(2, 40, 56, 100, 140, "binary", "bf16", 1, seed=1),
                Case(2, 40, 56, 100, 140, "gradient", "f32", 4, seed=2),
                Case(5, 37, 53, 90, 128, "binary", "f16", 4, seed=3, lo=-1.1, hi=1.05),
                Case(1, 100, 140, 40, 56, "binary", "u8", 4, seed=5, lo=0.0, hi=1.0),
                Case(2, 100, 140, 40, 56, "gradient", "bf16", 1, seed=6),
                Case(1, 90, 120, 2049, 3333, "gradient", "u8", 1, seed=7),
                Case(1, 90, 120, 2049, 3333, "binary", "f32", 1, seed=8)]


@pytest.mark.parametrize("c", BRANCH_CASES, ids=lambda c: f"{c.kind}-{c.dtype}x{c.channels}-{c.T}x{c.h}x{c.w}-{c.H}x{c.W}")
def test_passes_and_refinement(svr2lib, c):
    """Both branches, both float outputs, up- and down-scaled alphas from every source dtype with 1 and 4 channels, a
    guide below -1, a guide that needs no normalisation, and 1 x 2049 x 3333, where torch's mean factor is
    fl(N) / fl(3 N) != fl(1/3)"""
    sens = Sens(f"{c}")
    taps = run_case(svr2lib, c, sens=sens, expect_binary=c.kind == "binary")
    if c.H == 2049:
        assert mean_factor(c.T, c.H, c.W) != f32(1 / 3)
    sens.assert_sensitive()
    assert taps["binary"] == (c.kind == "binary")


@pytest.mark.parametrize("kind", ["binary", "gradient"])
def test_4k_shard(svr2lib, kind):
    """The 4K shard shape: 5 frames, 720p alpha -> 2160 x 3840"""
    sens = Sens(kind)
    run_case(svr2lib, Case(5, 720, 1280, 2160, 3840, kind, "bf16", 4, seed=11), out_kinds=(OUT_RGBA, OUT_F32), sens=sens,
             expect_binary=kind == "binary")
    sens.assert_sensitive()


# ====================================================================== d. raster edges
SIZES = [1, 2, 3, 4, 6, 7, 8, 31, 32, 33, 63, 64, 65]


@pytest.mark.parametrize("W", SIZES)
def test_raster_edges(svr2lib, W):
    """Every output size H, W in SIZES crossed, radius 2 and 3: windows wider than the image (still / 25 or 49),
    one-pixel Sobel axes (reflect-101 onto itself), the 32 x 32 tile edges"""
    for H in SIZES:
        for kind in ("noise-binary", "noise-gradient"):
            c = Case(2, max(1, (H + 1) // 2), max(1, (W + 2) // 3), H, W, kind, "bf16", 4, seed=H * 100 + W)
            run_case(svr2lib, c, expect_binary=kind == "noise-binary")


def test_frame_counts(svr2lib):
    """65535 tiny frames (the grid's z limit), both branches; 65536 is refused by both entry points"""
    for kind in ("noise-binary", "noise-gradient"):
        run_case(svr2lib, Case(65535, 1, 2, 2, 3, kind, "bf16", 1, seed=4), expect_binary=kind == "noise-binary")
    lib = svr2lib.load()
    x = torch.zeros(65536 * 4, device=DEV)
    s = torch.empty(1 << 20, device=DEV, dtype=torch.uint8)
    rc = lib.svr2_alpha_upscale(svr2lib.ptr(x), 0, 1, 65536, 1, 1, svr2lib.ptr(x), 1, 1, svr2lib.ptr(x), 0,
                                svr2lib.ptr(s), s.numel(), svr2lib.stream())
    assert rc != 0 and b"65535" in lib.svr2_last_error()
    rc = lib.svr2_sobel_edges_f32(svr2lib.ptr(x), 65536, 1, 1, svr2lib.ptr(x), svr2lib.ptr(s), s.numel(), svr2lib.stream())
    assert rc != 0 and b"65535" in lib.svr2_last_error()


# ====================================================================== e. memory contract of the base resize
def test_resize_only_writes_its_plane(svr2lib):
    """out_kind 2 writes the T x H x W plane and nothing past it, at sizes that are not multiples of the thread tile"""
    for T, h, w, H, W in ((1, 7, 7, 1, 1), (2, 5, 3, 33, 65), (3, 40, 60, 31, 63)):
        src, rgb = make_case(Case(T, h, w, H, W, "noise-gradient", seed=T))
        out, scratch = call(svr2lib, src, 1, 1, rgb, OUT_RESIZE)
        X = src[..., -1].float()[:, None]
        want = F.interpolate(X, size=(H, W), mode="bicubic", align_corners=False, antialias=True).clamp(0, 1)[:, 0]
        equal(out, want, f"{T}x{h}x{w} -> {H}x{W} base", where_fn("base", H, W, 0))
