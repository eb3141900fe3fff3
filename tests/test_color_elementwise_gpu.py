"""-m gpu: every post-decode colour-correction launch (csrc/post.cu) element by element against fp64.

Each launch is checked through the C ABI on its own operands, which for a chained stage are the previous launch's
actual output, so every stage is exact or bounded per element; one bit-exact wiring check (e) ties the stages to the
host code of color_fix.py.  Outputs start as a sentinel NaN pattern with a guard region before and after: every element
a launch owns must lose the sentinel, every guard element must keep it.  fp64 references are built in strips.
  a. one wavelet level (svr2_wavelet_level_bf16 / _f32, the fp32 one with bf16 and with fp32 input): widths 1, 2, odd,
     255 / 256 / 257, 511 / 513 (the two-pixels-per-thread layout and its grid edge), every H, W in 1..23 with an
     uncapped radius (the kernel's max(1, min(H, W) // 8) cap against the reference's wavelet_blur rule), H = 1 where
     y - r and y + r both clamp, 37 x 53, 270 x 480, 1080 x 1920 and 2160 x 3840 with 1, 3, 6 and 15 planes, in its
     three launch forms; and the refusals.
  b. AdaIN (svr2_adain_bf16): the (mean, std) it leaves in its scratch on their own, then the apply step from them.
  c. RGB -> LAB (svr2_rgb_to_lab_f32) and LAB -> RGB (svr2_lab_to_rgb_bf16) against an fp64 restatement of the
     reference's _rgb_to_lab_batch / _lab_to_rgb_batch with its fp32 constants, plus a bias check.
  d. histogram matching (svr2_histogram_match_f32): exact.
  e. wiring: color_fix's wavelet_reconstruction, lab_color_transfer and adaptive_instance_normalization equal chains
     of the launches checked above, bit for bit.
  f. svr2_sample_to_image_bf16 / _rgba_bf16: bit-exact.

Error budgets (U = 2^-24, u = 2^-53; a value the kernel computes in fp32 is z +- e; at a bf16 rounding point the
kernel's result must lie between rne(z - e) and rne(z + e), so the check is bit-exact wherever e cannot cross a
rounding boundary):
  a. low: the fp32 sum of the nine exact terms k_i k_j img, |error| <= 8 U sum |terms|; bf16 low then rounds once.
     high = rne(rne(h_prev + img) - low) from the kernel's own low, exact (fp32 emulation); the fp32 planes drop the
     rne.  out = clamp(rne(add_to + low), -1, 1): the low interval carried through that monotone map.
  b. statistics: the kernel sums in fp64 chains of c = ceil(hw / 1024) + 37 terms (strided per thread, a 5-level
     shuffle tree, 32 warp sums), so |dmean| <= c u E|x| + u |m| and
     |dvar| <= hw / (hw - 1) (c u (E[x^2] + 2 |m| E|x|) + 3 u m^2) + (hw + 2) u var; mean and std are those intervals
     carried through rn(fp32(mean)) and rn(sqrt(rn(rn(fp32(var)) + eps))).  hw = 1 has var 0 (include/svr2.h).
     apply: rne(rne(rne(rne(x - m_c) / s_c) s_s) + m_s) from the kernel's own stats, exact (fp32 emulation).
  c. forward error propagation per element, op by op: an fp32 rounding adds U (|z| + e); a product or quotient by an
     exact fp32 constant scales e; a three-term dot product adds 3 U sum |m_i| (|l_i| + e_i) (with or without FMA
     contraction); powf adds POWF_MAX_ULP ulps of its result (ulp(y) <= 2^-23 |y|) to the exact image of its input
     interval.  Where a value lies within its bound of a branch threshold (0.04045, epsilon^3, 6/29, 0.0031308) both
     branches are accepted.  lab_to_rgb's clamp and final bf16 rounding take the interval's ends.
     Bias (rgb -> lab; lab -> rgb ends in a bf16 rounding that hides any fp32-level bias): per case and channel,
     |mean(kernel - z)| / mean(e) <= BIAS_MAX = 0.01 on random frames (measured on an H100: 0.0038 at most) and on
     the dark pixels whose sRGB and LAB both stay on their linear segments (0.0016), where only fp32 roundings enter.
     Lattices of crafted or clamped pixels that go through powf measure up to 0.036 (the dark cube's L*; powf's
     error is not zero-mean over such a lattice) and take BIAS_MAX_LATTICE = 0.05.  One ulp too high in kappa
     (903.2964 for 903.2963) measures 0.023 on the linear dark pixels' L*, and one unit in the 7th digit of green's
     rgb -> Y coefficient 0.042 on a random frame's L* and 0.089 on the dark cube's.
  d. exact: the reference's sort may order ties either way, so within every group of equal source values
     (-0.0 == +0.0) the multiset of outputs must equal that group's slice of the sorted reference values.
  e, f. exact.
Every random-operand case with a bounded (not exact) check asserts that its median bound is at most 1/20 of the
output's standard deviation."""
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
U64 = 2.0 ** -53
TINY = 2.0 ** -140          # absolute slack for fp32 subnormal results
GUARD = 64                  # sentinel elements before and after every output
SENTINEL = {2: 0x7FA5, 4: 0x7FA5A5A5}     # NaN payloads no kernel writes
MAX_STRIP = 1 << 22         # elements per fp64 reference strip
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
# CUDA C++ Programming Guide 12.9, "Mathematical Functions" appendix, table of single-precision functions with their
# maximum ulp error: powf(x, y), 4 ulp (full range; the build does not use -use_fast_math).
POWF_MAX_ULP = 4
BIAS_MAX = 0.01             # rgb -> lab on random frames and on dark pixels that take no powf
BIAS_MAX_LATTICE = 0.05     # on lattices of crafted or clamped pixels that go through powf
WAVELET_LEVELS = 5


# ====================================================================== helpers (as in the GroupNorm element test)
def bits(t):
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def sentinel_fill(t):
    bits(t).fill_(SENTINEL[t.element_size()])
    return t


def check_untouched(region, what):
    bad = bits(region) != SENTINEL[region.element_size()]
    n = int(bad.sum())
    assert n == 0, f"{what}: {n} elements written, first at {bad.nonzero()[0].tolist()}"


def check_all_written(region, what):
    bad = bits(region) == SENTINEL[region.element_size()]
    n = int(bad.sum())
    assert n == 0, f"{what}: {n} elements never written, first at {bad.nonzero()[0].tolist()}"


class Guarded:
    """n elements of `dtype` between two guard regions, all sentinel; `offset` extra elements before the view shift
    its address off 16-byte alignment"""

    def __init__(self, n, dtype, offset=0):
        self.n, self.lead = n, GUARD + offset
        self.buf = sentinel_fill(torch.empty(n + 2 * GUARD + offset, device=DEV, dtype=dtype))
        self.v = self.buf[self.lead:self.lead + n]

    def check(self, what, written=True):
        check_untouched(self.buf[:self.lead], what + ": guard before the output")
        check_untouched(self.buf[self.lead + self.n:], what + ": guard after the output")
        (check_all_written if written else check_untouched)(self.v, what)


def rne_bf16(z):
    """fp64 -> the nearest bf16 value (ties to even), exactly"""
    m, e = torch.frexp(z)
    return torch.round(m * 256.0) * torch.exp2((e - 8).to(z.dtype))


def round_iv(z, e):
    """(r, B): the reference value and the bound of a bf16 rounding point whose fp32 input is z +- e"""
    r = rne_bf16(z)
    return r, torch.maximum(rne_bf16(z + e) - r, r - rne_bf16(z - e))


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


def fail_at(bad, got, want, B, what):
    n = int(bad.sum())
    if n:
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {n} elements outside the bound; first at {list(i)}: got {got[i].item():.9g}, "
                             f"want {want[i].item():.9g}, |err| {abs(got[i].item() - want[i].item()):.3g} > "
                             f"{B[i].item():.3g}")


def check_bound(got, want, B, what):
    got = got.double()
    fail_at(~((got - want).abs() <= B), got, want, B, what)


def check_between(got, lo, hi, what):
    got = got.double()
    bad = ~((got >= lo) & (got <= hi))
    fail_at(bad, got, (lo + hi) / 2, (hi - lo) / 2, what)


def check_equal(got, want, what):
    bad = ~(got.float() == want.float())
    fail_at(bad, got.double(), want.double(), torch.zeros_like(got, dtype=F64), what)


def uniform(shape, seed, lo=-1.0, hi=1.0, dtype=BF16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.rand(shape, generator=g, device=DEV) * (hi - lo) + lo).to(dtype)


def f32c(x):
    """the fp32 cast of a reference double constant"""
    return torch.tensor(x, dtype=F32).item()


@pytest.fixture(scope="module")
def cf(pkg):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.color_fix")


# ====================================================================== a. one wavelet level
K1 = (0.25, 0.5, 0.25)


def capped_radius(H, W, r):
    """wavelet_blur's rule (color_fix.py:136-140)"""
    return min(r, max(1, min(H, W) // 8))


def blur_ref(img, r, y0, y1):
    """rows [y0, y1) of the (1,2,1) x (1,2,1) / 16 blur of img (P, H, W) at dilation r, replicate borders:
    (fp64 nine-term sum, sum of |terms|)"""
    P, H, W = img.shape
    ys = torch.arange(y0, y1, device=img.device)
    xs = torch.arange(W, device=img.device)
    z = torch.zeros(P, y1 - y0, W, device=img.device, dtype=F64)
    a = torch.zeros_like(z)
    for i, dy in enumerate((-1, 0, 1)):
        rows = img.index_select(1, (ys + dy * r).clamp(0, H - 1)).double()
        for j, dx in enumerate((-1, 0, 1)):
            t = rows.index_select(2, (xs + dx * r).clamp(0, W - 1)) * (K1[i] * K1[j])
            z += t
            a += t.abs()
    return z, a


WAVELET_KINDS = ("bf16", "f32 from bf16", "f32")


def wavelet_level(lib, kind, img, low, high, add_to, out, radius, first):
    P, H, W = img.shape
    if kind == "bf16":
        lib.call("svr2_wavelet_level_bf16", lib.ptr(img), lib.ptr(low), lib.ptr(high), lib.ptr(add_to), lib.ptr(out),
                 P, H, W, radius, first, lib.stream())
    else:
        lib.call("svr2_wavelet_level_f32", lib.ptr(img), int(img.dtype == BF16), lib.ptr(low), lib.ptr(high),
                 lib.ptr(add_to), lib.ptr(out), P, H, W, radius, first, lib.stream())


def wavelet_case(lib, kind, P, H, W, radius, seed, sens=None):
    """One image through the level's three launch forms: content level 0 (first: high from 0), a later content level
    (high accumulates), and the style pass's last level (out = clamp(add_to + low), low untouched)."""
    T = BF16 if kind == "bf16" else F32
    n = P * H * W
    img = uniform((P, H, W), seed, dtype=BF16 if kind != "f32" else F32)
    hprev = uniform((P, H, W), seed + 1, -2, 2, T)
    add_to = uniform((P, H, W), seed + 2, -1.5, 1.5, T)
    what = f"wavelet {kind} {P}x{H}x{W} radius {radius}"
    low1, high1, low2, high2, low3, out3 = (Guarded(n, T) for _ in range(6))
    high2.v.copy_(hprev.flatten())
    shape = lambda g: g.v.view(P, H, W)          # noqa: E731
    wavelet_level(lib, kind, img, shape(low1), shape(high1), None, None, radius, 1)
    wavelet_level(lib, kind, img, shape(low2), shape(high2), None, None, radius, 0)
    wavelet_level(lib, kind, img, shape(low3), None, add_to, shape(out3), radius, 0)
    torch.cuda.synchronize()
    for g, name in ((low1, "low"), (high1, "high (first)"), (low2, "low"), (high2, "high"), (out3, "out")):
        g.check(f"{what}: {name}")
    low3.check(f"{what}: low of the last level (add_to set)", written=False)
    assert torch.equal(bits(low1.v), bits(low2.v)), f"{what}: low differs between two launches"
    r = capped_radius(H, W, radius)
    rows = max(1, MAX_STRIP // (P * W))
    lo_g, h1_g, h2_g, o_g = shape(low1), shape(high1), shape(high2), shape(out3)
    for y0 in range(0, H, rows):
        y1 = min(H, y0 + rows)
        s = (slice(None), slice(y0, y1))
        z, a = blur_ref(img, r, y0, y1)
        e = 8 * U * a
        if T == BF16:
            want, B = round_iv(z, e)
            lo_lo, lo_hi = rne_bf16(z - e), rne_bf16(z + e)
        else:
            want, B = z, e + TINY
            lo_lo, lo_hi = (z - e).float(), (z + e).float()
        check_bound(lo_g[s], want, B, f"{what}: low (dilation {r})")
        if sens is not None:
            sens.add(B, want)
        # high = rne(rne(h_prev + img) - low), from the kernel's own low
        lo = lo_g[s].float()
        for hp, got, name in ((torch.zeros_like(lo), h1_g[s], "high (first)"), (hprev[s].float(), h2_g[s], "high")):
            t = hp + img[s].float()
            t = (t.to(BF16).float() if T == BF16 else t) - lo
            check_equal(got, t.to(BF16) if T == BF16 else t, f"{what}: {name}")
        # out = clamp(rne(add_to + low), -1, 1): the low interval through a monotone map
        ends = []
        for lo_end in (lo_lo, lo_hi):
            v = add_to[s].float() + lo_end.float()
            ends.append((v.to(BF16).float() if T == BF16 else v).clamp(-1, 1).double())
        check_between(o_g[s], ends[0], ends[1], f"{what}: out")
        del z, a, e, want, B


WAVELET_GEOMS = [  # planes, H, W, radius
    (3, 5, 1, 4), (1, 7, 2, 1), (3, 9, 3, 2), (1, 4, 255, 16), (3, 3, 256, 4), (1, 6, 257, 8), (3, 2, 511, 2),
    (1, 5, 513, 16), (3, 1, 300, 16), (1, 1, 2, 16), (1, 64, 64, 8), (3, 37, 53, 16), (15, 37, 53, 4),
    (6, 270, 480, 16), (1, 1080, 1920, 16), (3, 2160, 3840, 16), (1, 2160, 3840, 1),
]


@pytest.mark.parametrize("kind", WAVELET_KINDS)
@pytest.mark.parametrize("P,H,W,radius", WAVELET_GEOMS)
def test_wavelet_level(svr2lib, kind, P, H, W, radius):
    sens = Sensitivity(f"wavelet {kind} {P}x{H}x{W}") if P * H * W >= 64 else None
    wavelet_case(svr2lib, kind, P, H, W, radius, seed=P * 7 + H * 131 + W, sens=sens)
    if sens is not None:
        sens.assert_sensitive()


@pytest.mark.parametrize("kind", ("bf16", "f32"))
def test_wavelet_level_small_sizes_radius_cap(svr2lib, kind):
    """every H, W in 1..23 with an uncapped radius: the kernel applies wavelet_blur's cap itself"""
    for H in range(1, 24):
        for W in range(1, 24):
            wavelet_case(svr2lib, kind, 1, H, W, 16, seed=H * 100 + W)


def test_wavelet_level_refusals(svr2lib):
    lib = svr2lib
    x = uniform((1, 4, 4), 1)
    low, out = Guarded(16, BF16), Guarded(16, BF16)
    lowf = Guarded(16, F32)
    P = lib.ptr
    for name, args in (("svr2_wavelet_level_bf16", (P(x), P(low.v), None, None, None)),
                       ("svr2_wavelet_level_f32", (P(x), 1, P(lowf.v), None, None, None))):
        with pytest.raises(lib.Svr2Error, match="65535"):
            lib.call(name, *args, 1, 65536, 1, 1, 1, lib.stream())
        with pytest.raises(lib.Svr2Error, match="65535"):
            lib.call(name, *args, 65536, 1, 1, 1, 1, lib.stream())
    for name, head, lo, o in (("svr2_wavelet_level_bf16", (P(x),), low, out),
                              ("svr2_wavelet_level_f32", (P(x), 1), lowf, Guarded(16, F32))):
        with pytest.raises(lib.Svr2Error, match="add_to and out"):
            lib.call(name, *head, P(lo.v), None, P(x), None, 1, 4, 4, 1, 1, lib.stream())
        with pytest.raises(lib.Svr2Error, match="add_to and out"):
            lib.call(name, *head, P(lo.v), None, None, P(o.v), 1, 4, 4, 1, 1, lib.stream())
        with pytest.raises(lib.Svr2Error, match="low is required"):
            lib.call(name, *head, None, None, None, None, 1, 4, 4, 1, 1, lib.stream())
        torch.cuda.synchronize()
        lo.check(f"{name}: refused launches", written=False)
        o.check(f"{name}: refused launches", written=False)


# ====================================================================== b. AdaIN
ADAIN_EPS = f32c(1e-5)


def plane_stats(x):
    """x (P, hw) bf16 -> fp64 mean, unbiased variance (0 for hw = 1), E|x|, E[x^2]; two passes over strips"""
    P, hw = x.shape
    cols = max(1, MAX_STRIP // P)
    s = torch.zeros(P, device=x.device, dtype=F64)
    sa, s2, sc = s.clone(), s.clone(), s.clone()
    for p0 in range(0, hw, cols):
        xd = x[:, p0:p0 + cols].double()
        s += xd.sum(1)
        sa += xd.abs().sum(1)
        s2 += (xd * xd).sum(1)
    m = s / hw
    for p0 in range(0, hw, cols):
        sc += ((x[:, p0:p0 + cols].double() - m[:, None]) ** 2).sum(1)
    var = sc / (hw - 1) if hw > 1 else torch.zeros_like(m)
    return m, var, sa / hw, s2 / hw


def adain_mean_of(m):
    return m.float().to(BF16).float()


def adain_std_of(v):
    vb = v.cpu().float().to(BF16).float()
    return (vb + ADAIN_EPS).to(BF16).float().sqrt().to(BF16).float()


def check_adain_stats(x, got, what):
    """got (P, 2) fp32 (mean, std) from the kernel's scratch"""
    P, hw = x.shape
    m, v, ea, e2 = plane_stats(x)
    c = -(-hw // 1024) + 37
    dm = c * U64 * ea + U64 * m.abs()
    if hw > 1:
        dv = hw / (hw - 1) * (c * U64 * (e2 + 2 * m.abs() * ea) + 3 * U64 * m * m) + (hw + 2) * U64 * v
    else:
        dv = torch.zeros_like(v)
    got = got.cpu()
    check_between(got[:, 0], adain_mean_of(m - dm).cpu().double(), adain_mean_of(m + dm).cpu().double(),
                  f"{what}: plane mean")
    check_between(got[:, 1], adain_std_of(v - dv).double(), adain_std_of(v + dv).double(), f"{what}: plane std")


def adain_case(lib, content, style, what):
    P, hw = content.shape
    out, stats = Guarded(P * hw, BF16), Guarded(4 * P, F32)
    lib.call("svr2_adain_bf16", lib.ptr(content), lib.ptr(style), lib.ptr(out.v), P, hw, lib.ptr(stats.v),
             lib.stream())
    torch.cuda.synchronize()
    out.check(what + ": output")
    stats.check(what + ": statistics scratch")
    st = stats.v.view(2 * P, 2)
    check_adain_stats(content, st[:P], what + " content")
    check_adain_stats(style, st[P:], what + " style")
    mc, sc, ms, ss = st[:P, 0:1], st[:P, 1:2], st[P:, 0:1], st[P:, 1:2]
    y = out.v.view(P, hw)
    cols = max(1, MAX_STRIP // P)
    for p0 in range(0, hw, cols):
        x = content[:, p0:p0 + cols].float()
        nrm = ((x - mc).to(BF16).float() / sc).to(BF16).float()
        check_equal(y[:, p0:p0 + cols], ((nrm * ss).to(BF16).float() + ms).to(BF16), what + ": output")
    return st, y


def near_flat(P, hw, seed, spread):
    """planes of mean close to +-1 (alternating) with a spread of `spread`"""
    sign = torch.where(torch.arange(P, device=DEV) % 2 == 0, 1.0, -1.0)[:, None]
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (sign * (0.995 + spread * torch.randn(P, hw, generator=g, device=DEV))).to(BF16)


def half_black(P, hw, seed):
    x = uniform((P, hw), seed)
    x[:, : hw // 2] = -1.0
    return x


ADAIN_CASES = {   # name: (P, hw, content maker)
    "hw1961": (6, 37 * 53, lambda P, hw, s: uniform((P, hw), s)),
    "hw1000": (3, 1000, lambda P, hw, s: uniform((P, hw), s, -0.3, 0.7)),
    "hw1025": (3, 1025, lambda P, hw, s: uniform((P, hw), s)),
    "hw2": (3000, 2, lambda P, hw, s: uniform((P, hw), s)),             # n - 1 against n: a factor 2 in var
    "hw3": (600, 3, lambda P, hw, s: uniform((P, hw), s)),
    "hw5_many_planes": (65535, 5, lambda P, hw, s: uniform((P, hw), s)),  # one apply block per plane
    "hw300_many_planes": (3000, 300, lambda P, hw, s: uniform((P, hw), s)),
    "4k_plane": (3, 2160 * 3840, lambda P, hw, s: uniform((P, hw), s)),
    "constant": (6, 4097, lambda P, hw, s: uniform((P, 1), s).expand(P, hw).contiguous()),
    "near_flat_1e-3": (6, 20000, lambda P, hw, s: near_flat(P, hw, s, 1e-3)),
    "near_flat_1e-4": (6, 20000, lambda P, hw, s: near_flat(P, hw, s, 1e-4)),
    "near_flat_4k": (3, 2160 * 3840, lambda P, hw, s: near_flat(P, hw, s, 1e-3)),
    "half_black": (6, 270 * 480, lambda P, hw, s: half_black(P, hw, s)),
}


@pytest.mark.parametrize("name", list(ADAIN_CASES))
def test_adain(svr2lib, name):
    P, hw, make = ADAIN_CASES[name]
    seed = sum(map(ord, name))
    content = make(P, hw, seed)
    style = make(P, hw, seed + 1) if name in ("constant",) or name.startswith("near") else \
        uniform((P, hw), seed + 1, -0.8, 0.9)
    adain_case(svr2lib, content, style, f"adain {name} {P}x{hw}")


def test_adain_single_pixel_planes(svr2lib):
    """hw = 1: variance 0 (torch's var() gives NaN there), std = bf16(sqrt(bf16(eps))), every output = style mean"""
    content, style = uniform((9, 1), 1), uniform((9, 1), 2)
    st, out = adain_case(svr2lib, content, style, "adain hw 1")
    want_std = torch.tensor(ADAIN_EPS).to(BF16).float().sqrt().to(BF16).float().item()
    assert (st[:, 1] == want_std).all(), st[:, 1]
    assert torch.equal(out, style)


def test_adain_refusals(svr2lib):
    lib = svr2lib
    x = uniform((1, 4), 1)
    with pytest.raises(lib.Svr2Error, match="65535"):
        lib.call("svr2_adain_bf16", lib.ptr(x), lib.ptr(x), lib.ptr(x), 65536, 1, lib.ptr(x), lib.stream())
    with pytest.raises(lib.Svr2Error, match="scratch"):
        lib.call("svr2_adain_bf16", lib.ptr(x), lib.ptr(x), lib.ptr(x), 1, 4, None, lib.stream())


# ====================================================================== c. RGB <-> LAB
# the reference's constants as its fp32 tensors see them (color_fix.py:299-321, 368-474)
RGB2XYZ = [[f32c(v) for v in row] for row in ((0.4124564, 0.3575761, 0.1804375),
                                                (0.2126729, 0.7151522, 0.0721750),
                                                (0.0193339, 0.1191920, 0.9503041))]
XYZ2RGB = [[f32c(v) for v in row] for row in ((3.2404542, -1.5371385, -0.4985314),
                                                (-0.9692660, 1.8760108, 0.0415560),
                                                (0.0556434, -0.2040259, 1.0572252))]
WHITE_X, WHITE_Z = f32c(0.95047), f32c(1.08883)
LAB_EPS = f32c(6.0 / 29.0)
LAB_EPS3 = f32c((6.0 / 29.0) ** 3)
LAB_KAPPA = f32c((29.0 / 3.0) ** 3)
SRGB_T, SRGB_A, SRGB_S, SRGB_G, SRGB_LIN = f32c(0.04045), f32c(0.055), f32c(1.055), f32c(2.4), f32c(12.92)
SRGB_INV_T, SRGB_INV_G = f32c(0.0031308), f32c(1.0 / 2.4)
THIRD = f32c(1.0 / 3.0)


# (value, bound) pairs: the fp64 restatement is the value part alone
def rnd32(v, e):
    return v, e + U * (v.abs() + e) + TINY


def addc(x, c):
    return rnd32(x[0] + c, x[1])


def mulc(x, c):
    return rnd32(x[0] * c, x[1] * abs(c))


def divc(x, c):
    return rnd32(x[0] / c, x[1] / abs(c))


def add(x, y):
    return rnd32(x[0] + y[0], x[1] + y[1])


def sub(x, y):
    return rnd32(x[0] - y[0], x[1] + y[1])


def dot(xs, ms):
    v = sum(m * x[0] for m, x in zip(ms, xs))
    e = sum(abs(m) * x[1] for m, x in zip(ms, xs))
    return v, e + 3 * U * sum(abs(m) * (x[0].abs() + x[1]) for m, x in zip(ms, xs)) + TINY


def powf(x, p, floor0=True):
    """powf(x, p) over the interval x +- e: the exact image, plus POWF_MAX_ULP ulps of the result"""
    f = (lambda t: t.clamp_min(0) ** p) if floor0 else (lambda t: t ** p)
    v = f(x[0])
    e = torch.maximum((f(x[0] + x[1]) - v).abs(), (v - f(x[0] - x[1])).abs())
    return v, e + POWF_MAX_ULP * 2.0 ** -23 * (v.abs() + e) + TINY


def clamp_iv(x, scale):
    """* scale (exact), then clamp to [0, 1]: the interval's ends clamped"""
    v, e = x[0] * scale, x[1] * scale
    c = v.clamp(0.0, 1.0)
    return c, torch.maximum((v + e).clamp(0.0, 1.0) - c, c - (v - e).clamp(0.0, 1.0))


def branch(x, thr, above, below):
    """the kernel takes `above` where x > thr; within its bound of thr either branch is accepted"""
    a, b = above(x), below(x)
    up = x[0] > thr
    v, e = torch.where(up, a[0], b[0]), torch.where(up, a[1], b[1])
    ov, oe = torch.where(up, b[0], a[0]), torch.where(up, b[1], a[1])
    amb = (x[0] - thr).abs() <= x[1]
    return v, torch.where(amb, torch.maximum(e, (ov - v).abs() + oe), e)


def lab_f(t):
    return branch(t, LAB_EPS3, lambda t: powf(t, THIRD), lambda t: divc(addc(mulc(t, LAB_KAPPA), 16.0), 116.0))


def lab_finv(f):
    return branch(f, LAB_EPS, lambda f: powf(f, 3.0, floor0=False),
                  lambda f: divc(addc(mulc(f, 116.0), -16.0), LAB_KAPPA))


def rgb_to_lab_ref(x):
    """x (3, n) fp64: the bf16 rgb values in [-1, 1] -> [(value, bound)] for L*, a*, b*"""
    lin = []
    for c in range(3):
        t = clamp_iv(rnd32(x[c] + 1.0, torch.zeros_like(x[c])), 0.5)
        lin.append(branch(t, SRGB_T, lambda t: powf(divc(addc(t, SRGB_A), SRGB_S), SRGB_G),
                          lambda t: divc(t, SRGB_LIN)))
    X = divc(dot(lin, RGB2XYZ[0]), WHITE_X)
    Y = dot(lin, RGB2XYZ[1])
    Z = divc(dot(lin, RGB2XYZ[2]), WHITE_Z)
    fx, fy, fz = lab_f(X), lab_f(Y), lab_f(Z)
    return [addc(mulc(fy, 116.0), -16.0), mulc(sub(fx, fy), 500.0), mulc(sub(fy, fz), 200.0)]


def lab_to_rgb_ref(L_c, L_m, a, b, lw):
    """fp32 L_content, L_matched (or None), a*, b* -> the rgb value in [0, 1] and its bound, per channel, before the
    clamp and the final [-1, 1] bf16 rounding"""
    z = torch.zeros_like(L_c)
    if L_m is None:
        L = (L_c, z)
    else:
        L = add(mulc((L_c, z), f32c(lw)), mulc((L_m, z), f32c(1.0 - lw)))
    fy = divc(addc(L, 16.0), 116.0)
    fx = add(divc((a, z), 500.0), fy)
    fz = sub(fy, divc((b, z), 200.0))
    xyz = [mulc(lab_finv(fx), WHITE_X), lab_finv(fy), mulc(lab_finv(fz), WHITE_Z)]
    out = []
    for c in range(3):
        lin = dot(xyz, XYZ2RGB[c])
        out.append(branch(lin, SRGB_INV_T, lambda t: addc(mulc(powf(t, SRGB_INV_G), SRGB_S), -SRGB_A),
                          lambda t: mulc(t, SRGB_LIN)))
    return out


def lab_to_bf16_interval(v, e):
    """clamp(0, 1), * 2 - 1 (one fp32 rounding), bf16: (reference, low end, high end)"""
    ends = []
    for t in (v - e, v, v + e):
        zz = 2.0 * t.clamp(0.0, 1.0) - 1.0
        ends.append(zz)
    r = rne_bf16(ends[1])
    return r, rne_bf16(ends[0] - U * ends[0].abs()), rne_bf16(ends[2] + U * ends[2].abs())


class Bias:
    """mean signed error over mean bound, per channel"""

    def __init__(self, what, names, limit):
        self.what, self.names, self.limit = what, names, limit
        self.err, self.bound = [0.0] * len(names), [0.0] * len(names)

    def add(self, c, err, B):
        self.err[c] += err.sum().item()
        self.bound[c] += B.sum().item()

    def ratios(self):
        return [e / b if b > 0 else 0.0 for e, b in zip(self.err, self.bound)]

    def assert_unbiased(self):
        r = self.ratios()
        assert all(abs(x) <= self.limit for x in r), \
            f"{self.what}: mean signed error / mean bound " + ", ".join(f"{n} {x:+.4f}" for n, x in zip(self.names, r)) \
            + f" (limit {self.limit})"


def rgb_to_lab_case(lib, rgb, what, sensitive=True, bias_limit=BIAS_MAX):
    """rgb (T, 3, hw) bf16 -> the kernel's LAB [3][T*hw] fp32, every element checked"""
    T, _, hw = rgb.shape
    n = T * hw
    out = Guarded(3 * n, F32)
    lib.call("svr2_rgb_to_lab_f32", lib.ptr(rgb), lib.ptr(out.v), T, hw, lib.stream())
    torch.cuda.synchronize()
    out.check(what + ": lab")
    lab = out.v.view(3, n)
    x = rgb.permute(1, 0, 2).reshape(3, n)
    bias = Bias(what + ": rgb -> lab", ("L*", "a*", "b*"), bias_limit)
    sens = Sensitivity(what + ": rgb -> lab") if sensitive else None
    for p0 in range(0, n, MAX_STRIP // 4):
        p1 = min(n, p0 + MAX_STRIP // 4)
        ref = rgb_to_lab_ref(x[:, p0:p1].double())
        for c, (v, e) in enumerate(ref):
            got = lab[c, p0:p1]
            check_bound(got, v, e, f"{what}: rgb -> lab channel {'Lab'[c]}")
            bias.add(c, got.double() - v, e)
            if sens is not None:
                sens.add(e, v)
        del ref
    bias.assert_unbiased()
    if sens is not None:
        sens.assert_sensitive()
    return lab


def lab_to_rgb_case(lib, L_c, L_m, a, b, lw, T, hw, what, sensitive=True):
    n = T * hw
    out = Guarded(3 * n, BF16)
    lib.call("svr2_lab_to_rgb_bf16", lib.ptr(L_c), lib.ptr(L_m), lib.ptr(a), lib.ptr(b), lw, lib.ptr(out.v), T, hw,
             lib.stream())
    torch.cuda.synchronize()
    what = f"{what}: lab -> rgb (luminance weight {lw})"
    out.check(what)
    rgb = out.v.view(T, 3, hw).permute(1, 0, 2).reshape(3, n)
    sens = Sensitivity(what) if sensitive else None
    for p0 in range(0, n, MAX_STRIP // 4):
        p1 = min(n, p0 + MAX_STRIP // 4)
        s = slice(p0, p1)
        ref = lab_to_rgb_ref(L_c[s].double(), None if L_m is None else L_m[s].double(), a[s].double(),
                             b[s].double(), lw)
        for c, (v, e) in enumerate(ref):
            r, lo, hi = lab_to_bf16_interval(v, e)
            got = rgb[c, s]
            check_between(got, lo, hi, f"{what}: channel {'rgb'[c]}")
            if sens is not None:
                sens.add(torch.maximum(hi - r, r - lo), r)
        del ref
    if sens is not None:
        sens.assert_sensitive()
    return out.v.view(T, 3, hw)


def bf16_values(with_inf=False):
    """every finite bf16 value (and +-inf), as fp32"""
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF16).float()
    return v[~torch.isnan(v) if with_inf else torch.isfinite(v)].to(DEV)


def dark_cube(top=-0.7):
    """every combination of the bf16 values in [-1, top] per channel: sRGB 0 .. 0.15, across the linear-segment
    threshold 0.04045 and epsilon^3 in X, Y and Z; with top = -0.921875, sRGB <= 0.039: the linear segment and the
    kappa branch only, no powf"""
    v = bf16_values()
    v = v[(v >= -1) & (v <= top)].unique()
    r, g, b = torch.meshgrid(v, v, v, indexing="ij")
    return torch.stack([r.flatten(), g.flatten(), b.flatten()]).to(BF16)[None]


def rgb_corners():
    vals = torch.tensor([-1.0, 0.0, 1.0, -0.5, 0.5], device=DEV)
    r, g, b = torch.meshgrid(vals, vals, vals, indexing="ij")
    return torch.stack([r.flatten(), g.flatten(), b.flatten()]).to(BF16)[None]


RGB_CASES = {
    "dark_cube": dark_cube,
    "dark_linear": lambda: dark_cube(-0.921875),
    "all_bf16_greys": lambda: bf16_values().to(BF16).expand(3, -1).contiguous()[None],
    "black_white_grey": rgb_corners,
    "out_of_range_2x37x53": lambda: uniform((2, 3, 37 * 53), 5, -1.5, 1.5),
    "random_3x270x480": lambda: uniform((3, 3, 270 * 480), 6),
    "random_4k": lambda: uniform((1, 3, 2160 * 3840), 7),
}


@pytest.mark.parametrize("name", list(RGB_CASES))
def test_rgb_lab_round_trip(svr2lib, name):
    """rgb -> lab on crafted and random pixels, then lab -> rgb of the kernel's own LAB at every luminance weight (the
    matched L* a rolled copy of L*)"""
    rgb = RGB_CASES[name]().contiguous()
    T, _, hw = rgb.shape
    sensitive = name.startswith(("random", "out_of"))
    lattice = name in ("dark_cube", "all_bf16_greys", "black_white_grey", "out_of_range_2x37x53")
    lab = rgb_to_lab_case(svr2lib, rgb, f"{name} {T}x{hw}", sensitive, BIAS_MAX_LATTICE if lattice else BIAS_MAX)
    Lm = lab[0].roll(1).contiguous()
    for lw in (0.0, 0.5, 0.8, 1.0):
        lab_to_rgb_case(svr2lib, lab[0], None if lw == 1.0 else Lm, lab[1], lab[2], lw, T, hw, f"{name} {T}x{hw}",
                        sensitive)


def fp32_neighbours(x, k):
    """the 2k + 1 fp32 values around x"""
    b = torch.tensor([x], dtype=F32).view(torch.int32)
    return (b + torch.arange(-k, k + 1, dtype=torch.int32)).view(F32)


def lab_thresholds():
    """L* around 8 (f = 6/29) and around 2.83 (grey lin = 0.0031308), a* / b* 0 and small, by fp32 ulps and by steps"""
    L = torch.cat([fp32_neighbours(8.0, 64), fp32_neighbours(2.8278, 64), torch.linspace(0, 20, 4001),
                   torch.tensor([0.0, -0.0, 1e-30, -1e-30])])
    ab = torch.tensor([0.0, 1e-3, -1e-3, 0.5, -0.5, 3.0, -3.0])
    Lg, ag, bg = torch.meshgrid(L, ab, ab, indexing="ij")
    return Lg.flatten(), ag.flatten(), bg.flatten()


def lab_out_of_gamut():
    g = torch.Generator().manual_seed(17)
    n = 3 * 37 * 53
    return torch.rand(n, generator=g) * 140 - 20, torch.rand(n, generator=g) * 400 - 200, \
        torch.rand(n, generator=g) * 400 - 200


@pytest.mark.parametrize("name,make", [("thresholds", lab_thresholds), ("out_of_gamut", lab_out_of_gamut)])
def test_lab_to_rgb_crafted(svr2lib, name, make):
    L, a, b = (t.to(DEV, F32).contiguous() for t in make())
    n = L.numel()
    Lm = L.flip(0).contiguous()
    for lw in (0.0, 0.5, 0.8, 1.0):
        lab_to_rgb_case(svr2lib, L, None if lw == 1.0 else Lm, a, b, lw, 1, n, f"lab {name} {n}", sensitive=False)


# ====================================================================== d. histogram matching
def match_case(lib, src, ref, what):
    """src, ref fp32 (n,) -> the kernel's output, checked exactly; operands and output at 4-byte-only aligned views"""
    n = src.numel()
    s, r, out = Guarded(n, F32, 1), Guarded(n, F32, 3), Guarded(n, F32, 1)
    s.v.copy_(src)
    r.v.copy_(ref)
    need = lib.load().svr2_histogram_match_scratch_bytes(n)
    scratch = torch.empty(need, device=DEV, dtype=torch.uint8)
    lib.call("svr2_histogram_match_f32", lib.ptr(s.v), lib.ptr(r.v), lib.ptr(out.v), n, lib.ptr(scratch), need,
             lib.stream())
    torch.cuda.synchronize()
    out.check(what)
    assert torch.equal(bits(s.v), bits(src)) and torch.equal(bits(r.v), bits(ref)), f"{what}: operands changed"
    o = out.v
    idx = torch.sort(o + 0.0, stable=True).indices              # + 0.0: -0.0 and +0.0 in one tie group
    idx = idx[torch.sort(src[idx] + 0.0, stable=True).indices]
    S = torch.sort(ref + 0.0).values
    got = o[idx] + 0.0
    if not torch.equal(got, S):
        bad = (got != S).nonzero()[0].item()
        raise AssertionError(f"{what}: rank {bad} of the (source, output) order holds {got[bad].item()!r}, the sorted "
                             f"reference {S[bad].item()!r}; {int((got != S).sum())} ranks differ")
    assert torch.equal(torch.sort(bits(o)).values, torch.sort(bits(ref)).values), \
        f"{what}: the output is not a bitwise permutation of the reference values"
    return o


def quantised(n, levels, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(0, levels, (n,), generator=g, device=DEV).float() * 0.25 - 1


def signed_zeros(n, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.tensor([-0.0, 0.0, 1.0, -1.0], device=DEV)[torch.randint(0, 4, (n,), generator=g, device=DEV)]


MATCH_CASES = {
    "n1": lambda: (uniform((1,), 1, dtype=F32), uniform((1,), 2, dtype=F32)),
    "n2": lambda: (uniform((2,), 1, dtype=F32), uniform((2,), 2, dtype=F32)),
    "n255": lambda: (uniform((255,), 1, dtype=F32), uniform((255,), 2, -3, 5, F32)),
    "n256": lambda: (uniform((256,), 1, dtype=F32), uniform((256,), 2, -3, 5, F32)),
    "n257": lambda: (uniform((257,), 1, dtype=F32), uniform((257,), 2, -3, 5, F32)),
    "all_equal": lambda: (torch.full((4099,), 0.3, device=DEV), torch.full((4099,), -2.0, device=DEV)),
    "quantised": lambda: (quantised(100003, 7, 1), quantised(100003, 3, 2)),
    "signed_zeros": lambda: (signed_zeros(65537, 1), signed_zeros(65537, 2)),
    "past_2^24": lambda: (quantised((1 << 24) + 5, 1000, 3), uniform(((1 << 24) + 5,), 4, dtype=F32)),
    "4k_batch": lambda: (uniform((5 * 2160 * 3840,), 5, dtype=F32), quantised(5 * 2160 * 3840, 50000, 6)),
}


@pytest.mark.parametrize("name", list(MATCH_CASES))
def test_histogram_match(svr2lib, name):
    src, ref = MATCH_CASES[name]()
    match_case(svr2lib, src, ref, f"histogram match {name} n={src.numel()}")


def test_histogram_match_lab_channels(svr2lib):
    """the kernel's own L*, a*, b* of two random frames (one of them mostly black), as lab_color_transfer feeds it"""
    c = uniform((2, 3, 37 * 53), 8)
    s = uniform((2, 3, 37 * 53), 9)
    s[:, :, : 37 * 20] = -1.0
    lc = rgb_to_lab_case(svr2lib, c, "content 2x37x53")
    ls = rgb_to_lab_case(svr2lib, s, "style 2x37x53", sensitive=False)
    for ch in range(3):
        match_case(svr2lib, lc[ch], ls[ch], f"histogram match of LAB channel {ch}")


def test_histogram_match_refuses_2_to_the_32(svr2lib):
    x = torch.zeros(4, device=DEV)
    scratch = torch.empty(64, device=DEV, dtype=torch.uint8)
    with pytest.raises(svr2lib.Svr2Error, match="2\\^32"):
        svr2lib.call("svr2_histogram_match_f32", svr2lib.ptr(x), svr2lib.ptr(x), svr2lib.ptr(x), 1 << 32,
                     svr2lib.ptr(scratch), 64, svr2lib.stream())


# ====================================================================== e. wiring
def wavelet_chain(lib, c, s):
    """five levels at radii 1..16: content pass accumulating high (`first` on level 0), style pass whose last level
    writes out = clamp(high + low)"""
    T, _, H, W = c.shape
    P = T * 3
    high, out = torch.empty_like(c), torch.empty_like(c)
    tmp = (torch.empty_like(c), torch.empty_like(c))
    src = c
    for i in range(WAVELET_LEVELS):
        wavelet_level(lib, "bf16", src.view(P, H, W), tmp[i % 2], high, None, None, 2 ** i, int(i == 0))
        src = tmp[i % 2]
    src = s
    for i in range(WAVELET_LEVELS):
        last = i == WAVELET_LEVELS - 1
        wavelet_level(lib, "bf16", src.view(P, H, W), None if last else tmp[i % 2], None, high if last else None,
                      out if last else None, 2 ** i, 0)
        src = tmp[i % 2]
    return out


def lab_chain(lib, c, s, lw):
    T, _, H, W = c.shape
    n, hw = T * H * W, H * W
    base = wavelet_chain(lib, c, s)
    lab = []
    for x in (base, s):
        t = torch.empty(3, n, device=DEV)
        lib.call("svr2_rgb_to_lab_f32", lib.ptr(x), lib.ptr(t), T, hw, lib.stream())
        lab.append(t)
    need = lib.load().svr2_histogram_match_scratch_bytes(n)
    scratch = torch.empty(need, device=DEV, dtype=torch.uint8)
    m = torch.empty(3, n, device=DEV)
    for ch in ((1, 2) if lw >= 1.0 else (0, 1, 2)):
        lib.call("svr2_histogram_match_f32", lib.ptr(lab[0][ch]), lib.ptr(lab[1][ch]), lib.ptr(m[ch]), n,
                 lib.ptr(scratch), need, lib.stream())
    out = torch.empty_like(c)
    lib.call("svr2_lab_to_rgb_bf16", lib.ptr(lab[0][0]), lib.ptr(m[0]) if lw < 1.0 else None, lib.ptr(m[1]),
             lib.ptr(m[2]), lw, lib.ptr(out), T, hw, lib.stream())
    return out


@pytest.mark.parametrize("T,H,W", [(2, 37, 53), (2, 270, 480), (5, 2160, 3840)])
def test_color_fix_runs_the_checked_launches(cf, svr2lib, T, H, W):
    c = uniform((T, 3, H, W), T * H + W)
    s = uniform((T, 3, H, W), T * H + W + 1, -0.9, 0.8)
    what = f"{T}x{H}x{W}"
    assert torch.equal(bits(cf.wavelet_reconstruction(c, s)), bits(wavelet_chain(svr2lib, c, s))), what + " wavelet"
    for lw in (0.8, 1.0):
        assert torch.equal(bits(cf.lab_color_transfer(c, s, None, luminance_weight=lw)),
                           bits(lab_chain(svr2lib, c, s, lw))), f"{what} lab, luminance weight {lw}"
    out = torch.empty_like(c)
    svr2lib.call("svr2_adain_bf16", svr2lib.ptr(c), svr2lib.ptr(s), svr2lib.ptr(out), T * 3, H * W,
                 svr2lib.ptr(torch.empty(T * 12, device=DEV)), svr2lib.stream())
    assert torch.equal(bits(cf.adaptive_instance_normalization(c, s)), bits(out)), what + " adain"


# ====================================================================== f. sample -> image
def image_ref(x):
    """clamp(-1, 1) * 0.5 (exact), + 0.5 in fp32, bf16"""
    return (x.float().clamp(-1, 1) * 0.5 + 0.5).to(BF16)


@pytest.mark.parametrize("T,hw", [(1, 2160 * 3840), (3, 37 * 53), (1, 65279)])
def test_sample_to_image(svr2lib, T, hw):
    x = uniform((T, 3, hw), hw, -3, 3)
    if T * hw >= 65279:       # every bf16 value but NaN somewhere
        v = bf16_values(with_inf=True).to(BF16)
        x.view(-1)[: v.numel()] = v
    want = image_ref(x).permute(0, 2, 1)
    out = Guarded(T * hw * 3, BF16)
    svr2lib.call("svr2_sample_to_image_bf16", svr2lib.ptr(x), svr2lib.ptr(out.v), T, hw, svr2lib.stream())
    rgba = Guarded(T * hw * 4, BF16)
    svr2lib.call("svr2_sample_to_image_rgba_bf16", svr2lib.ptr(x), svr2lib.ptr(rgba.v), T, hw, svr2lib.stream())
    torch.cuda.synchronize()
    out.check(f"sample_to_image {T}x{hw}")
    check_equal(out.v.view(T, hw, 3), want, f"sample_to_image {T}x{hw}")
    check_untouched(rgba.buf[:GUARD], "rgba: guard before")
    check_untouched(rgba.buf[GUARD + rgba.n:], "rgba: guard after")
    img = rgba.v.view(T, hw, 4)
    check_untouched(img[..., 3], "rgba: alpha channel")
    check_equal(img[..., :3], want, f"sample_to_image_rgba {T}x{hw}")
