"""-m gpu: the antialiased bicubic resize (csrc/aa_resize.cuh) element by element, through both of its users: the clip
pre-processing svr2_resize_bicubic_aa_bf16 (csrc/pre.cu, the first kernel every clip goes through) and the base resize
of svr2_alpha_upscale (csrc/alpha.cu, out_kind 2).

A resize fault is local: one wrong border column of a 1920-wide output is 0.05 % of its elements, and a wrong load of
small values moves them by a few bf16 ulps, both inside a bulk "99.5 % equal, the rest within 2^-7" check.  Here every
element is held to its own bound, three ways:
  a. the tap tables.  The kernel's tables are read from the resize scratch (layout in include/svr2.h), expanded to
     dense [n_out, n_in] form and compared with == against torch's CUDA kernel's table, which can be read out exactly:
     interpolate(eye(n_in) as [1, n_in, 1, n_in], size (1, n_out)) is that table transposed, since the 1 -> 1 axis is a
     single unit tap and every other product is 1 w or 0 w (the vertical axis likewise from [1, n_in, n_in, 1]).  The
     padding taps count..K-1 must be 0 and every span must lie inside [0, n_in).
  b. the outputs against fp64, independent of torch (module docstring below).
  c. the outputs bit for bit (torch.equal) against torch's CUDA op chain, which is what the reference's Compose does on
     a GPU tensor (oracle/pre_oracle.py preprocess_torch, pinned to the reference's Compose on the CPU by
     tests/test_oracle_golden.py): the bf16 compute dtype (uint8 read as bf16(fp16(u / 255))), fp32 interpolate
     rounded to bf16, a second resize for the max_resolution cap, clamp, zero pad to 16, (x - 0.5) / 0.5 in bf16,
     c t h w; the alpha base resize as fp32 interpolate of the bf16 alpha, clamp(0, 1).

Error model of part b.  Per frame and channel, z = Wy X Wx^T and S = |Wy| |X| |Wx|^T in fp64 from the kernel's own
tables (the fp32 weights are exact in fp64), X the input as the kernel loads it (rounded to bf16).  The kernel forms
each row's horizontal sum as a product and nx - 1 fmas, each rounding once by at most U = 2^-24 of a partial bounded by
the row's sum of |x| |w|; the vertical sum over ny rows likewise, with S bounding every partial: its fp32 accumulator
lies within e = (nx + ny + 2) U S of z (the 2 covers the second-order terms).  Rounding is monotone, so
  - plain mode (bf16): the output lies in [rne(z - e), rne(z + e)];
  - finish mode: in [f(rne(z - e)), f(rne(z + e))], f(v) = bf16(bf16(clamp(v, 0, 1) - 0.5) / 0.5), and the padding
    rows and columns hold exactly -1;
  - alpha out_kind 2 (fp32): |y - clamp(z, 0, 1)| <= e (clamp is 1-Lipschitz).
Where the interval holds one bf16 value the check is bit-exact.  Non-vacuity: on random inputs at least 99.9 % of the
intervals hold a single bf16 value and the median e is below 1/1000 of a bf16 ulp of the output.  Part b checks
addressing, strides, loads, borders, padding and layout; it holds whatever fp32 formula the weights follow.

Every output allocation is surrounded by sentinel guard regions that must keep their bit pattern; every failure names
the frame, channel, output row and column, and whether the row / column is in a border span of its table (one that
touches input row / column 0 or the last one)."""
import importlib
from typing import NamedTuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import pre_oracle
from test_conv_elementwise_gpu import U, check_untouched, rnd, sentinel_fill, ulp_bf16
from test_dit_block_elementwise_gpu import check, rne_bf16

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16
GUARD = 64                  # sentinel elements before and after every output
MAX_PLANE_ELEMS = 1 << 25   # output elements per fp64 reference chunk
DTYPES = {"f32": (torch.float32, 0), "bf16": (BF16, 1), "f16": (torch.float16, 2), "u8": (torch.uint8, 3)}
MAX_TAPS = 31               # 2 ceil(2 * 7.5) + 1


@pytest.fixture(scope="module")
def pre(pkg):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.preprocess")


@pytest.fixture(scope="module")
def am(pkg):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.alpha")


# ====================================================================== tap tables
def taps_for(n_in, n_out):
    """taps per output index (aa_resize.cuh taps_for): 2 ceil(support) + 1, support = 2 max(scale, 1) in fp32"""
    scale = np.float32(n_in) / np.float32(n_out)
    support = scale + scale if scale >= 1 else np.float32(2)
    return int(np.ceil(support)) * 2 + 1


def align256(n):
    return (n + 255) // 256 * 256


class Axis(NamedTuple):
    first: torch.Tensor     # int64 [n_out]
    count: torch.Tensor     # int64 [n_out]
    w: torch.Tensor         # fp32 [n_out, K]
    n_in: int

    def dense(self):
        """[n_out, n_in] fp32, after checking the table's invariants"""
        n_out, K = self.w.shape
        j = torch.arange(K, device=DEV)
        live = j[None] < self.count[:, None]
        bad = (self.count < 1) | (self.count > K) | (self.first < 0) | (self.first + self.count > self.n_in)
        bad |= ((self.w != 0) & ~live).any(1)
        if bad.any():
            i = int(bad.nonzero()[0])
            raise AssertionError(f"{n_out} <- {self.n_in} table: {int(bad.sum())} bad spans, first at output {i}: first "
                                 f"{int(self.first[i])}, count {int(self.count[i])} (K {K}), weights {self.w[i].tolist()}")
        rows = torch.arange(n_out, device=DEV)[:, None].expand(n_out, K)
        D = torch.zeros(n_out, self.n_in, device=DEV, dtype=torch.float32)
        D[rows[live], (self.first[:, None] + j[None])[live]] = self.w[live]
        return D

    def border(self, i):
        if i >= self.w.shape[0]:
            return "padding"
        f, n = int(self.first[i]), int(self.count[i])
        return f"span {f}..{f + n - 1} of {self.n_in}" + (", border span" if f == 0 or f + n == self.n_in else "")


def read_tables(scratch, h, w, H, W):
    """(x axis, y axis) as the last call left them in the resize scratch (include/svr2.h)"""
    K, L = max(taps_for(h, H), taps_for(w, W)), max(H, W)
    seg_i, seg_w = align256(8 * L), align256(4 * L * K)
    ints = scratch[:2 * seg_i].view(torch.int32).long()
    wts = scratch[2 * seg_i:2 * seg_i + 2 * seg_w].view(torch.float32)
    o = seg_i // 4
    x = Axis(ints[:W], ints[L:L + W], wts[:W * K].view(W, K).clone(), w)
    y = Axis(ints[o:o + H], ints[o + L:o + L + H], wts[seg_w // 4:seg_w // 4 + H * K].view(H, K).clone(), h)
    return x, y


def torch_table(n_in, n_out, axis):
    """torch's CUDA antialiased bicubic table [n_out, n_in] along one axis, read out exactly through an identity"""
    eye = torch.eye(n_in, device=DEV)
    if axis == "x":
        t = F.interpolate(eye.view(1, n_in, 1, n_in), size=(1, n_out), mode="bicubic", align_corners=False, antialias=True)
    else:
        t = F.interpolate(eye.view(1, n_in, n_in, 1), size=(n_out, 1), mode="bicubic", align_corners=False, antialias=True)
    return t.reshape(n_in, n_out).t()


def resize_raw(lib, x, code, channels_last, cin, T, h, w, out, H, W, finish, scratch):
    return lib.load().svr2_resize_bicubic_aa_bf16(lib.ptr(x), code, int(channels_last), cin, T, h, w, lib.ptr(out), H, W,
                                                  int(finish), lib.ptr(scratch), scratch.numel(), lib.stream())


def kernel_tables(lib, h, w, H, W):
    """The tables the resize builds for (h, w) -> (H, W); the alpha resize builds its tables with the same kernel"""
    x = torch.zeros(1, 3, h, w, device=DEV, dtype=BF16)
    out = torch.empty(1, 3, H, W, device=DEV, dtype=BF16)
    scratch = torch.zeros(lib.load().svr2_resize_scratch_bytes(h, w, H, W), device=DEV, dtype=torch.uint8)
    assert resize_raw(lib, x, 1, False, 3, 1, h, w, out, H, W, False, scratch) == 0, lib.load().svr2_last_error()
    return read_tables(scratch, h, w, H, W)


def table_mismatch(got, n_in, n_out, axis):
    """(number of weights that differ from torch's, description of the first)"""
    D, R = got.dense(), torch_table(n_in, n_out, axis)
    bad = D != R
    n = int(bad.sum())
    if not n:
        return 0, ""
    i, j = bad.nonzero()[0].tolist()
    return n, (f"{axis} {n_in} -> {n_out}: output {i} ({got.border(i)}), input {j}: kernel {D[i, j].item()!r}, "
               f"torch {R[i, j].item()!r}")


SWEEP = [(a, b) for a in range(1, 97) for b in range(1, 97)]


def test_tables_every_small_pair(svr2lib):
    """Every (n_in, n_out) with both in 1..96: the tables equal torch's; the pairs beyond 7.5x down-scaling are refused."""
    lib = svr2lib
    x = torch.zeros(3 * 96 * 96, device=DEV, dtype=BF16)
    out = torch.empty(3 * 96 * 96, device=DEV, dtype=BF16)
    scratch = torch.empty(1 << 20, device=DEV, dtype=torch.uint8)
    n_bad, n_all, pairs, first, refusals = 0, 0, 0, "", []
    for n_in, n_out in SWEEP:
        if taps_for(n_in, n_out) > MAX_TAPS:
            assert n_in * 2 > 15 * n_out
            rc = resize_raw(lib, x, 1, False, 3, 1, n_in, n_in, out, n_out, n_out, False, scratch)
            if rc == 0 or b"7.5" not in lib.load().svr2_last_error():
                refusals.append((n_in, n_out, rc, lib.load().svr2_last_error()))
            continue
        assert n_in * 2 <= 15 * n_out
        assert lib.load().svr2_resize_scratch_bytes(n_in, n_in, n_out, n_out) <= scratch.numel()
        assert resize_raw(lib, x, 1, False, 3, 1, n_in, n_in, out, n_out, n_out, False, scratch) == 0
        tx, ty = read_tables(scratch, n_in, n_in, n_out, n_out)
        for got, axis in ((tx, "x"), (ty, "y")):
            n, msg = table_mismatch(got, n_in, n_out, axis)
            n_all += n_out * n_in
            if n:
                n_bad, pairs, first = n_bad + n, pairs + 1, first or msg
    assert n_bad == 0, f"{n_bad} of {n_all} dense weights differ from torch's in {pairs} axis tables; first: {first}"
    assert not refusals, f"{len(refusals)} pairs beyond 7.5x not refused with a message naming the limit: {refusals[:3]}"


def cap_pairs():
    """The two resizes of the max_resolution cap: (h, w) -> (H1, W1) -> (H, W)"""
    out = []
    for h, w, res, mx in ((540, 960, 1080, 1600), (1280, 720, 1080, 1440), (480, 854, 1080, 1280)):
        (H, W), twice = pre_oracle.resized_size(h, w, res, mx)
        (H1, W1), _ = pre_oracle.resized_size(h, w, res, 0)
        assert twice
        out += [(h, w, H1, W1), (H1, W1, H, W)]
    return out


REAL_AXES = [(480, 854, 1080, 1921), (720, 1280, 1080, 1920), (576, 720, 1080, 1350), (1080, 1920, 2160, 3840),
             (720, 1280, 2160, 3840), (2160, 3840, 1080, 1920), (997, 1000, 1000, 997), (75, 15, 10, 2)] + cap_pairs()


@pytest.mark.parametrize("h,w,H,W", REAL_AXES)
def test_tables_pipeline_axes(svr2lib, h, w, H, W):
    """The pipeline's real axes (a 480p clip at 1080, 720p / 576p / 1080p to 1080 and 4K, 4K down to 1080, 997 <-> 1000,
    the cap's two resizes) and the tap limit (75 -> 10 and 15 -> 2: exactly 7.5x, 31 taps)."""
    tx, ty = kernel_tables(svr2lib, h, w, H, W)
    K = max(taps_for(h, H), taps_for(w, W))
    assert tx.w.shape[1] == K <= MAX_TAPS
    msgs = []
    for got, n_in, n_out, axis in ((tx, w, W, "x"), (ty, h, H, "y")):
        n, msg = table_mismatch(got, n_in, n_out, axis)
        if n:
            msgs.append(f"{n} of {n_in * n_out} weights differ; first: {msg}")
    assert not msgs, "; ".join(msgs)


def test_tap_limit_refusals(svr2lib, am):
    """7.5x is the largest down-scale factor (31 taps): 751 -> 100 and 16 -> 2 are refused by both users, with a message
    that names the limit."""
    lib = svr2lib.load()
    assert taps_for(75, 10) == taps_for(15, 2) == 31 and taps_for(751, 100) == taps_for(16, 2) == 33
    x = torch.zeros(1, 3, 751, 751, device=DEV, dtype=BF16)
    out = torch.empty(3 * 100 * 100, device=DEV, dtype=BF16)
    scratch = torch.empty(1 << 22, device=DEV, dtype=torch.uint8)
    for h, w, H, W in ((751, 751, 100, 100), (751, 16, 100, 2), (16, 16, 2, 2), (100, 751, 100, 100)):
        assert resize_raw(svr2lib, x, 1, False, 3, 1, h, w, out, H, W, False, scratch) != 0
        assert b"7.5" in lib.svr2_last_error(), (h, w, H, W)
    rgb = torch.zeros(1, 3, 100, 100, device=DEV, dtype=BF16)
    a = torch.zeros(1, 751, 751, 1, device=DEV)
    s = am._scratch(1, 1, 1, 100, 100, DEV)         # the factor is checked before the scratch size
    rc = lib.svr2_alpha_upscale(svr2lib.ptr(a), 0, 1, 1, 751, 751, svr2lib.ptr(rgb), 100, 100, svr2lib.ptr(out), 2,
                                svr2lib.ptr(s), s.numel(), svr2lib.stream())
    assert rc != 0 and b"7.5" in lib.svr2_last_error()
    # 7.5x exactly is accepted
    assert resize_raw(svr2lib, x, 1, False, 3, 1, 750, 750, out, 100, 100, False, scratch) == 0


# ====================================================================== outputs: fp64 bounds and torch's op chain
class Stats:
    """Non-vacuity of the fp64 intervals over one or more calls (module docstring)."""

    def __init__(self):
        self.single, self.total, self.rel = 0, 0, []

    def add(self, z, e):
        lo, hi = rne_bf16(z - e), rne_bf16(z + e)
        self.single += int((lo == hi).sum())
        self.total += lo.numel()
        step = max(1, z.numel() // 100000)
        self.rel.append((e / ulp_bf16(rne_bf16(z))).flatten()[::step].float().cpu())

    def assert_sensitive(self, what):
        frac = self.single / max(1, self.total)
        med = torch.cat(self.rel).median().item()
        assert frac >= 0.999, f"{what}: only {100 * frac:.3f} % of {self.total} intervals hold a single bf16 value"
        assert med < 1e-3, f"{what}: median bound {med:.3g} bf16 ulps"


def loaded(x, dtype, layout, channel=None):
    """The input as the kernel loads it, [T, C, h, w] bf16 (the compute dtype; uint8 as the CLI reads it)"""
    v = pre_oracle.compute_dtype(x)
    if layout.startswith("cl"):
        v = v.permute(0, 3, 1, 2)
        v = v[:, :3] if channel is None else v[:, channel:channel + 1]
    return v


def make_input(shape, dtype, seed, nan_channel=None):
    """Random frames: around 0.5 with ~5 % of the values outside [0, 1]; fp32 values not representable in bf16; uint8
    with every byte value present; a NaN channel (channels-last) that no kernel may read."""
    if dtype == "u8":
        g = torch.Generator(device=DEV).manual_seed(seed)
        x = torch.randint(0, 256, shape, generator=g, device=DEV, dtype=torch.uint8)
        n = min(256, x.numel())
        x.view(-1)[torch.randperm(x.numel(), generator=g, device=DEV)[:n]] = torch.arange(n, device=DEV).to(torch.uint8)
        return x
    v = rnd(shape, seed).float() * 0.3 + 0.5
    if dtype == "f32":
        v = v * (1 + 2.0 ** -10 * rnd(shape, seed + 1).float())
    v = v.to(DTYPES[dtype][0])
    if nan_channel is not None:
        v[..., nan_channel] = float("nan")
    return v


def where_fn(what, t0, tx, ty):
    def loc(*i):
        f, c, y, x = (i if len(i) == 4 else (0, *i))
        return (f"{what}: frame {t0 + f}, channel {c}, row {y} ({ty.border(y)}), col {x} ({tx.border(x)})")
    return loc


def fp64_planes(X, tx, ty):
    """z, e and their tables' tap counts for planes X [P, h, w] (fp64)"""
    Dx, Dy = tx.dense().double(), ty.dense().double()
    z = Dy @ X @ Dx.t()
    S = Dy.abs() @ X.abs() @ Dx.abs().t()
    n = (tx.count[None, None, :] + ty.count[None, :, None] + 2).double()
    return z, n * U * S


def finish_map(b):
    """f(v) = bf16(bf16(clamp(v, 0, 1) - 0.5) / 0.5) of bf16 values b (fp64)"""
    return rne_bf16(b.clamp(0.0, 1.0) - 0.5) * 2.0


def check_resize_fp64(X, out, tx, ty, finish, what, stats=None):
    """X [T, 3, h, w] bf16 as loaded; out [T, 3, H, W] (plain) or [3, T, Hp, Wp] (finish)"""
    T = X.shape[0]
    H, W = ty.w.shape[0], tx.w.shape[0]
    step = max(1, MAX_PLANE_ELEMS // (3 * H * W))
    for t0 in range(0, T, step):
        t1 = min(T, t0 + step)
        z, e = fp64_planes(X[t0:t1].double().reshape(-1, X.shape[2], X.shape[3]), tx, ty)
        z, e = z.view(t1 - t0, 3, H, W), e.view(t1 - t0, 3, H, W)
        lo, hi = rne_bf16(z - e), rne_bf16(z + e)
        if finish:
            lo, hi = finish_map(lo), finish_map(hi)
            got = out[:, t0:t1, :H, :W].transpose(0, 1)
        else:
            got = out[t0:t1]
        check(got, (lo + hi) / 2, (hi - lo) / 2, what + " vs fp64", where_fn(what, t0, tx, ty))
        if stats is not None:
            stats.add(z, e)
    if finish:
        pad_rows, pad_cols = out[:, :, H:, :], out[:, :, :H, W:]
        for p, name in ((pad_rows, "padding rows"), (pad_cols, "padding columns")):
            bad = p != -1
            assert not bad.any(), f"{what}: {int(bad.sum())} {name} elements are not -1, first at {bad.nonzero()[0].tolist()}"


def check_equal(got, want, what, loc):
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    check(got, want.double(), torch.zeros((), device=got.device, dtype=torch.float64).expand(got.shape), what + " vs torch",
          loc)


class Case(NamedTuple):
    T: int
    h: int
    w: int
    H: int
    W: int
    dtype: str = "bf16"     # f32 | bf16 | f16 | u8
    layout: str = "cf3"     # cf3: [T, 3, h, w];  cl3 / cl4: [T, h, w, 3 | 4] (channel 3 holds NaN)
    finish: bool = False
    seed: int = 0


def run_case(lib, c: Case, stats=None, x=None):
    """One svr2_resize_bicubic_aa_bf16 call on random frames, checked against fp64 and against torch's op chain;
    returns the output (inside its guards)"""
    cl = c.layout.startswith("cl")
    cin = int(c.layout[2])
    shape = (c.T, c.h, c.w, cin) if cl else (c.T, 3, c.h, c.w)
    if x is None:
        x = make_input(shape, c.dtype, c.seed, 3 if c.layout == "cl4" and c.dtype != "u8" else None)
    Hp, Wp = ((c.H + 15) // 16 * 16, (c.W + 15) // 16 * 16) if c.finish else (c.H, c.W)
    n = 3 * c.T * Hp * Wp
    buf = sentinel_fill(torch.empty(n + 2 * GUARD, device=DEV, dtype=BF16))
    out = buf[GUARD:GUARD + n].view((3, c.T, Hp, Wp) if c.finish else (c.T, 3, c.H, c.W))
    scratch = torch.empty(lib.load().svr2_resize_scratch_bytes(c.h, c.w, c.H, c.W), device=DEV, dtype=torch.uint8)
    rc = resize_raw(lib, x, DTYPES[c.dtype][1], cl, cin, c.T, c.h, c.w, out, c.H, c.W, c.finish, scratch)
    assert rc == 0, lib.load().svr2_last_error()
    tx, ty = read_tables(scratch, c.h, c.w, c.H, c.W)
    what = f"{c}"
    check_untouched(buf[:GUARD], what + ": guard before the output")
    check_untouched(buf[GUARD + n:], what + ": guard after the output")
    X = loaded(x, c.dtype, c.layout)
    check_resize_fp64(X, out, tx, ty, c.finish, what, stats)
    y = pre_oracle.resize_bf16(X, c.H, c.W)
    want = pre_oracle.finish_bf16(y) if c.finish else y
    check_equal(out, want, what, lambda *i: where_fn(what, 0, tx, ty)(*((i[1], i[0], *i[2:]) if c.finish else i)))
    return out


DTYPE_CASES = [Case(2, 45, 150, 97, 120, dt, lay, fin, seed=s)
               for s, (dt, lay, fin) in enumerate((dt, lay, fin) for dt in DTYPES for lay in ("cl3", "cl4", "cf3")
                                                  for fin in (False, True))]


@pytest.mark.parametrize("c", DTYPE_CASES, ids=lambda c: f"{c.dtype}-{c.layout}-{'finish' if c.finish else 'plain'}")
def test_input_dtypes_and_layouts(svr2lib, c):
    """fp32 (outside [0, 1], not bf16-representable), bf16, fp16, uint8 (every byte value) in channels-last with 3 and
    4 channels and channels-first; up-scaling rows and down-scaling columns."""
    stats = Stats()
    run_case(svr2lib, c, stats)
    stats.assert_sensitive(f"{c}")


RASTER_W = {1: 7, 63: 40, 64: 150, 65: 65, 127: 300}     # output width -> input width (down 7x, up, down, same, down)
RASTER_H = {1: 5, 3: 1, 4: 29, 5: 2}                     # output height -> input height (down, one pixel, 7.25x, up)


@pytest.mark.parametrize("W", list(RASTER_W))
def test_output_raster_edges(svr2lib, W):
    """Output widths 1, 63, 64, 65, 127 and heights 1, 3, 4, 5 around the 64 x 4 thread tile, both modes."""
    for H in RASTER_H:
        run_case(svr2lib, Case(2, RASTER_H[H], RASTER_W[W], H, W, "bf16", "cf3", False, seed=H * W))
        run_case(svr2lib, Case(2, RASTER_H[H], RASTER_W[W], H, W, "f32", "cl4", True, seed=H * W + 1))


EDGE_CASES = [Case(1, 1, 50, 30, 100, "u8", "cl3", True), Case(1, 40, 1, 90, 3, "f16", "cf3", False),
              Case(2, 1, 1, 16, 16, "bf16", "cl4", True), Case(1, 1, 1, 1, 1, "f32", "cf3", False),
              Case(2, 200, 30, 50, 180, "bf16", "cf3", True), Case(2, 30, 200, 180, 50, "f32", "cl3", False),
              Case(1, 150, 20, 20, 150, "f16", "cl4", True), Case(1, 64, 48, 64, 48, "bf16", "cf3", True)]


@pytest.mark.parametrize("c", EDGE_CASES, ids=lambda c: f"{c.h}x{c.w}-to-{c.H}x{c.W}")
def test_input_edges_and_mixed_scaling(svr2lib, c):
    """Inputs of one pixel on either axis; up on one axis and down on the other, so that one axis's table is padded to
    the other's K (5 taps in a 17- or 31-tap table); the same size (one unit tap)."""
    run_case(svr2lib, c)


def test_finish_padding(svr2lib):
    """Pads of 0..15 rows and columns: the body against fp64 and torch, the padding exactly -1."""
    for p in range(16):
        run_case(svr2lib, Case(1, 23, 61, 32 - p, 48 - (15 - p), "bf16", "cf3", True, seed=p))


def test_frame_counts(svr2lib):
    """1, 5 and 65535 tiny frames (the grid's z limit); 65536 is refused."""
    for T in (1, 5):
        run_case(svr2lib, Case(T, 20, 30, 41, 25, "f16", "cl3", True, seed=T))
    run_case(svr2lib, Case(65535, 2, 3, 3, 4, "bf16", "cf3", False, seed=7))
    run_case(svr2lib, Case(65535, 3, 2, 4, 3, "u8", "cl4", True, seed=8))
    x = torch.zeros(3 * 4, device=DEV, dtype=BF16)
    out = torch.empty(3 * 4, device=DEV, dtype=BF16)
    scratch = torch.empty(1 << 16, device=DEV, dtype=torch.uint8)
    assert resize_raw(svr2lib, x, 1, False, 3, 65536, 1, 1, out, 1, 1, False, scratch) != 0
    assert b"65535" in svr2lib.load().svr2_last_error()


FULL_CASES = [Case(2, 480, 854, 1080, 1921, "u8", "cl3", True, seed=1),
              Case(5, 1080, 1920, 2160, 3840, "bf16", "cf3", True, seed=2),
              Case(1, 720, 1280, 2160, 3840, "f32", "cl4", False, seed=3)]


@pytest.mark.parametrize("c", FULL_CASES, ids=lambda c: f"{c.T}x{c.h}x{c.w}-to-{c.H}x{c.W}")
def test_full_size(svr2lib, c):
    """A 480p clip at resolution 1080, the 4K shard (5 x 1080p -> 2160 x 3840), 720p -> 4K."""
    stats = Stats()
    run_case(svr2lib, c, stats)
    stats.assert_sensitive(f"{c}")


@pytest.mark.parametrize("h,w,res,mx,dtype", [(540, 960, 1080, 1600, "bf16"), (96, 54, 160, 200, "u8"),
                                              (480, 854, 1080, 0, "f32")])
def test_pipeline_entry_points(svr2lib, pre, h, w, res, mx, dtype):
    """VideoTransform (t c h w) and preprocess_frames (t h w c) equal the reference's chain on the GPU bit for bit,
    including the two resizes of the max_resolution cap, each of which is also held to its fp64 bound."""
    (H, W), twice = pre.resized_size(h, w, res, mx)
    frames = make_input((2, h, w, 3), dtype, h + w)
    clip = loaded(frames, dtype, "cl3")
    want = pre_oracle.preprocess_torch(clip, res, mx)
    got = pre.preprocess_frames(frames, res, mx)
    loc = lambda *i: f"channel {i[0]}, frame {i[1]}, row {i[2]}, col {i[3]}"
    check_equal(got, want, f"preprocess_frames {h}x{w} res {res} max {mx} {dtype}", loc)
    got2 = pre.prepare_video_transforms(res, mx)(clip.contiguous())
    check_equal(got2, want, f"VideoTransform {h}x{w} res {res} max {mx}", loc)
    if twice:       # each resize of the chain against fp64, the second reading the first's bf16 output
        (H1, W1), _ = pre.resized_size(h, w, res, 0)
        mid = run_case(svr2lib, Case(2, h, w, H1, W1, dtype, "cl3", False), x=frames)
        last = run_case(svr2lib, Case(2, H1, W1, H, W, "bf16", "cf3", True), x=mid.contiguous())
        assert torch.equal(last, got)


# ====================================================================== the alpha base resize (out_kind 2)
def run_alpha_case(lib, am, T, h, w, H, W, dtype, channels, seed, stats=None):
    src = make_input((T, h, w, channels), dtype, seed)
    if channels == 4 and dtype != "u8":
        src[..., :3] = float("nan")          # only the alpha (the last channel) may be read
    rgb = torch.zeros(T, 3, H, W, device=DEV, dtype=BF16)
    n = T * H * W
    buf = sentinel_fill(torch.empty(n + 2 * GUARD, device=DEV, dtype=torch.float32))
    out = buf[GUARD:GUARD + n].view(T, H, W)
    am._run(src, channels, rgb, out, am.OUT_RESIZE)
    what = f"alpha {T}x{h}x{w}x{channels} {dtype} -> {H}x{W}"
    check_untouched(buf[:GUARD], what + ": guard before the output")
    check_untouched(buf[GUARD + n:], what + ": guard after the output")
    tx, ty = kernel_tables(lib, h, w, H, W)
    X = pre_oracle.compute_dtype(src[..., channels - 1])              # [T, h, w]
    step = max(1, MAX_PLANE_ELEMS // (H * W))
    for t0 in range(0, T, step):
        t1 = min(T, t0 + step)
        z, e = fp64_planes(X[t0:t1].double(), tx, ty)
        loc = lambda f, y, x, t0=t0: where_fn(what, t0, tx, ty)(f, 0, y, x)
        check(out[t0:t1], z.clamp(0.0, 1.0), e, what + " vs fp64", loc)
        if stats is not None:
            stats.add(z, e)
    want = F.interpolate(X.float()[:, None], size=(H, W), mode="bicubic", align_corners=False,
                         antialias=True).clamp(0.0, 1.0)[:, 0]
    check_equal(out, want, what, lambda f, y, x: where_fn(what, 0, tx, ty)(f, 0, y, x))


@pytest.mark.parametrize("channels", [1, 4])
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_alpha_resize_dtypes(svr2lib, am, dtype, channels):
    stats = Stats()
    run_alpha_case(svr2lib, am, 2, 45, 150, 97, 120, dtype, channels, seed=channels, stats=stats)
    stats.assert_sensitive(f"alpha {dtype} x{channels}")


def test_alpha_resize_raster_edges(svr2lib, am):
    for W in RASTER_W:
        for H in RASTER_H:
            run_alpha_case(svr2lib, am, 2, RASTER_H[H], RASTER_W[W], H, W, "bf16", 4, seed=H * W)


def test_alpha_resize_4k(svr2lib, am):
    stats = Stats()
    run_alpha_case(svr2lib, am, 1, 720, 1280, 2160, 3840, "f16", 4, seed=5, stats=stats)
    stats.assert_sensitive("alpha 720p -> 4K")
