"""-m gpu: every launch of a DiT block element by element against fp64, at the window, head and tile edges of its real
geometries (the 3B at 5 x 68 x 120 latents: 75 / 90 windows of 71..868 video tokens; the 7B at 2 x 135 x 240).

A fault in one window, one head, one kv tile or one tile column moves a relative-L2 error over the whole block by less
than its tolerance.  Here every element is held to its own bound, outputs start as a sentinel bit pattern (guard rows
and ldc padding must keep it, every row the kernel owns must lose it), and failures name the element's place in the
kernel's raster:
  a. window attention (svr2_attn_varlen_bf16): exact probes and random operands against an fp64 softmax;
  b. the QKV projection + q/k RMSNorm + RoPE + window scatter (svr2_linear_qkv_rope_bf16 + svr2_qk_norm_rope_rows_bf16,
     and the stand-alone svr2_qk_norm_rope_window_bf16);
  c. every distinct GEMM launch of a full-width 2-layer 3B and 7B forward, as recorded from B200NaDiT;
  d. svr2_rmsnorm_ada_bf16 and svr2_txt_window_mean_bf16.

Rounding points are followed as intervals.  A quantity the kernel computes in fp32 is z with |z_kernel - z| <= e, z the
fp64 value of the same formula on the same inputs.  At a bf16 rounding point the kernel's result lies between
rne(z - e) and rne(z + e) (rounding is monotone): the reference goes on with r = rne(z) and the bound
B = max(rne(z + e) - r, r - rne(z - e)), which is 0 unless a rounding boundary lies within e of z, one bf16 step then.
Between rounding points, B propagates through each operation (|f'| B plus the fp32 error of evaluating f).  The output
is checked as |y - r| <= B: where the interval holds one bf16 value the check is bit-exact, so a dropped or extra
rounding point shows up.

fp32 error terms (U = 2^-24):
  - a GEMM accumulator: <= (K / 4) U S, S = sum |a| |w|: the tensor core adds a k-slice of exact bf16 products with one
    alignment truncation of <= 2^-23 of the largest magnitude it handles (<= S), at least every 8 products (the same
    model as tests/test_conv_elementwise_gpu.py); + U (S + |b|) for the bias add;
  - an fp32 sum of n positive terms: relative (n + 5) U (lane-sequential chains, then a 5-level shuffle tree);
    1 / sqrt(x) of it: half that, + 4 U (sqrtf, the division, the scaling by 1/n and the eps add);
  - silu_fast / gelu_tanh_fast (ex2.approx behind __expf, __fdividef): relative 2^-19 (1 + |x| + |x|^3 / 20), covering
    ex2.approx's 2^-22 and the exponent argument's rounding, damped by e / (1 + e) <= 1 in x / (1 + e);
    |silu'| <= 1.1, |gelu_tanh'| <= 1.13;
  - every other fp32 add / multiply: U of its result; 2^-120 absolute where __fdividef flushes a tiny quotient to 0.

Window attention (part a).  O_i = sum_j pi_j v_j, pi = softmax(q k^T / sqrt(128)).  The kernel's probabilities
p_j = exp2(x_j - m) (x the scores in log2 units, m the running max) deviate from the exact ones by a relative
eps_p <= ln2 dx + 2^-21: dx covers the score accumulation at K = 128 (2 x 32 U S_qk sc for the score and the max,
S_qk = sum_d |q_d k_d| unscaled, sc = log2(e) / sqrt(128)) and the roundings of s sc, of m sc and of the fma that
forms x (U |s sc| + U |m sc| + U |x| <= 4 U M, M = max |s| sc; 6 U M budgeted), ex2.approx's 2^-21.  P enters the PV product
rounded to bf16 (relative <= 2^-8: half an ulp of 8 significant bits) while the row sum l adds the unrounded p, so
|O_kernel - O| <= A (2^-8 + 2 eps_p + (n / 4 + 2 n_kv + 4) U), A = sum_j pi_j |v_jc| (the PV accumulation over n keys
in 64-key tiles, the rescale by alpha once per tile, the final 1 / l and product).  The exact probes are constructed so
that P is exactly 0 or 1 and only the final division rounds.

q/k RMSNorm + RoPE (part b).  The projection's first rounding point p = bf16(x) may differ from the reference's by one
bf16 step where x sits near a rounding boundary (B_p above).  Through the norm y_d = p_d rr w_d, rr = (mean p^2 + eps)^-1/2,
a change dp moves rr by at most rr * rho, rho = sum_e |p_e| B_p,e / (sum_e p_e^2 + 128 eps), so
|dy_d| <= rr |w_d| (B_p,d + |p_d| rho) + 144 U |y_d| (the fp32 sum of 128 squares, rsqrt, two products).  The rotation
(y0, y1) -> (y0 c - y1 s, y1 c + y0 s) with the handle's own fp32 cos / sin gives |c| B_0 + |s| B_1 (and 4 U of the
products), then the output rounding.

Sensitivity: every random-operand check also asserts that its median bound is at most 1/20 of the standard deviation of
the signal it protects (the attention output, the normalised q / k, the epilogue's pre-residual value), so that neither
a loose bound nor a swamping residual can make a check vacuous."""
import importlib
import math
from typing import NamedTuple

import pytest
import torch
import torch.nn.functional as F

from oracle import dit_oracle
from test_conv_elementwise_gpu import MAX_STRIP, SENTINEL, U, bits, check_untouched, rnd, sentinel_fill
from test_native_geometry_cpu import rope_freqs
from test_ops_gpu import geometry_handle

pytestmark = pytest.mark.gpu
DEV = "cuda"
TXT = 58
EPS = 1e-5
GUARD = 3                                   # sentinel rows before and after every output
LOG2E = 1.4426950408889634
SC_LOG2 = LOG2E / math.sqrt(128.0)


# ====================================================================== interval rounding
def rne_bf16(z):
    """fp64 -> the nearest bf16 value (ties to even), exactly, without an fp32 intermediate"""
    m, e = torch.frexp(z)
    return torch.round(m * 256.0) * torch.exp2((e - 8).to(z.dtype))


def round_iv(z, e):
    """(r, B): the reference value and the bound of a bf16 rounding point whose fp32 input is z +- e"""
    r = rne_bf16(z)
    return r, torch.maximum(rne_bf16(z + e) - r, r - rne_bf16(z - e))


def fast_rel(x):
    """relative error of silu_fast / gelu_tanh_fast at x (module docstring)"""
    a = x.abs()
    return 2.0 ** -19 * (1 + a + a * a * a / 20)


def gelu_tanh(x):
    """0.5 x (1 + tanh u) as x sigmoid(2 u): the tanh form cancels to 0 in the negative tail, where the kernel's
    x / (1 + e^-2u) keeps its relative accuracy"""
    return x * torch.sigmoid(2 * 0.7978845608028654 * (x + 0.044715 * x ** 3))


def check(got, r, B, what, loc):
    """|got - r| <= B element by element (a NaN, e.g. an unwritten sentinel, fails); loc(*index) names the place"""
    err = (got.double() - r).abs()
    bad = ~(err <= B)
    n = int(bad.sum())
    if n:
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {n} of {bad.numel()} elements outside the bound; first at {loc(*i)}: "
                             f"got {got[i].item():.6g}, want {r[i].item():.6g}, |err| {err[i].item():.3g} > {B[i].item():.3g}")


class Sensitivity:
    """Samples of a check's bound and of the signal it protects; the median bound must stay below std / 20."""

    def __init__(self, what):
        self.what, self.b, self.s = what, [], []

    def add(self, B, signal):
        step = max(1, B.numel() // 200000)
        self.b.append(B.flatten()[::step].float().cpu())
        self.s.append(signal.flatten()[::step].float().cpu())

    def assert_sensitive(self):
        b, s = torch.cat(self.b), torch.cat(self.s)
        med, sd = b.median().item(), s.std().item()
        assert med <= sd / 20, f"{self.what}: median bound {med:.3g} is not small against the signal's std {sd:.3g}"


# ====================================================================== the real window layouts (svr2_dit_geometry)
class Layout(NamedTuple):
    name: str
    nfreq: int
    L: int
    n_win: int
    total: int
    max_len: int
    cu: torch.Tensor            # int32 on the device; cu_h: the same on the host (int64)
    cu_h: torch.Tensor
    row_src: torch.Tensor
    row_rope: torch.Tensor
    out_row_map: torch.Tensor
    tok_dst: torch.Tensor
    tok_rope: torch.Tensor
    txt_rows: torch.Tensor
    cos: torch.Tensor
    sin: torch.Tensor


_LAYOUTS = {}


def layout(lib, variant, geom, layer):
    """The window layout and RoPE tables of one layer (even: regular windows, odd: shifted), copied off the handle."""
    key = (variant, geom, layer)
    if key not in _LAYOUTS:
        T, Hp, Wp = geom
        with geometry_handle(lib, variant, 2, rope_freqs(variant, torch.float16), layers=2) as h:
            g = lib.dit_geometry(h, T, 2 * Hp, 2 * Wp, TXT, layer)
            L = T * Hp * Wp
            ints = dict(cu_seqlens=g.n_win + 1, row_src=g.total, row_rope=3 * g.total, out_row_map=g.total, tok_dst=L,
                        tok_rope=3 * L, txt_rows=g.n_txt_rows)
            t = {n: lib.host_copy(getattr(g, n), (sz,), torch.int32) for n, sz in ints.items()}
            tabs = {n: lib.host_copy(getattr(g, n), (g.rope_rows, g.nfreq), torch.float32) for n in ("rope_cos", "rope_sin")}
        cu_h = t["cu_seqlens"].long()
        _LAYOUTS[key] = Layout(f"{variant} {T}x{Hp}x{Wp} {'shifted' if layer & 1 else 'regular'}", g.nfreq, L, g.n_win,
                               g.total, g.max_len, t["cu_seqlens"].to(DEV), cu_h, t["row_src"].to(DEV),
                               t["row_rope"].to(DEV).view(g.total, 3), t["out_row_map"].to(DEV), t["tok_dst"].to(DEV),
                               t["tok_rope"].to(DEV).view(L, 3), t["txt_rows"].to(DEV), tabs["rope_cos"].to(DEV),
                               tabs["rope_sin"].to(DEV))
    return _LAYOUTS[key]


def window_of(cu_h, row):
    w = int(torch.searchsorted(cu_h, torch.tensor(row), right=True)) - 1
    return w, row - int(cu_h[w])


# ====================================================================== a. window attention
class AttnLayout(NamedTuple):
    name: str
    heads: int
    cu_h: torch.Tensor
    out_row_map: torch.Tensor


SYNTH_LENS = [65, 1, 193, 5, 62, 63, 64, 2083, 127, 128, 129, 191, 192, 256, 300, 400, 810, 868]
ATTN_LAYOUTS = ["synthetic", "3b-regular", "3b-shifted", "7b-regular", "7b-shifted"]
REAL = {"3b": ("3b", 20, (5, 68, 120)), "7b": ("7b", 24, (2, 135, 240))}


def attn_layout(lib, name):
    if name == "synthetic":          # every tile-edge length, 5 heads, a random scatter
        cu_h = torch.tensor([0] + SYNTH_LENS).cumsum(0)
        g = torch.Generator().manual_seed(3)
        return AttnLayout(name, 5, cu_h, torch.randperm(int(cu_h[-1]), generator=g).int().to(DEV))
    variant, kind = name.split("-")
    v, heads, geom = REAL[variant]
    lay = layout(lib, v, geom, int(kind == "shifted"))
    return AttnLayout(lay.name, heads, lay.cu_h, lay.out_row_map)


def length_groups(cu_h, heads, per_window):
    """windows of equal length, in chunks whose fp64 temporaries (per_window(n) elements per window) stay bounded"""
    lens = cu_h.diff().tolist()
    groups = {}
    for w, n in enumerate(lens):
        groups.setdefault(n, []).append(w)
    for n, ws in sorted(groups.items()):
        step = max(1, MAX_STRIP // (heads * per_window(n)))
        for i in range(0, len(ws), step):
            chunk = torch.tensor(ws[i:i + step])
            yield n, chunk, (cu_h[chunk][:, None] + torch.arange(n)).to(DEV)      # (windows, n) packed rows


def run_attn(lib, al, q, k, v):
    """svr2_attn_varlen_bf16 through out_row_map into a sentinel-filled o_all with guard rows; every row written, the
    guard rows untouched.  Returns the output in packed (window) row order."""
    total, heads = q.shape[:2]
    obuf = sentinel_fill(torch.empty(GUARD + total + GUARD, heads, 128, device=DEV, dtype=torch.bfloat16))
    o_all = obuf[GUARD:GUARD + total]
    cu = al.cu_h.int().to(DEV)
    lib.call("svr2_attn_varlen_bf16", lib.ptr(q), lib.ptr(k), lib.ptr(v), lib.ptr(o_all), lib.ptr(cu), len(cu) - 1,
             total, heads, int(al.cu_h.diff().max()), lib.ptr(al.out_row_map), lib.stream())
    torch.cuda.synchronize()
    check_untouched(obuf[:GUARD], f"attention {al.name}: guard rows before o_all")
    check_untouched(obuf[-GUARD:], f"attention {al.name}: guard rows after o_all")
    unwritten = (bits(o_all) == SENTINEL).all(-1).all(-1)
    if unwritten.any():
        r = int(unwritten.nonzero()[0])
        src = int((al.out_row_map.long() == r).nonzero()[0])
        w, i = window_of(al.cu_h, src)
        raise AssertionError(f"attention {al.name}: {int(unwritten.sum())} rows of o_all not written, first o_all row {r} "
                             f"(window {w}, q-tile {i // 128}, tile row {i % 128})")
    return o_all[al.out_row_map.long()]


def attn_loc(al, idx):
    """(chunk window, head, row, channel) -> the place in the kernel's raster"""
    def loc(cw, h, i, c, extra=""):
        w = window_of(al.cu_h, int(idx[cw, 0]))[0]
        n = int(al.cu_h[w + 1] - al.cu_h[w])
        t = i % 128
        return (f"window {w} (len {n}), head {h}, q-tile {i // 128} of {-(-n // 128)}, tile row {t} (warpgroup {t // 64}, "
                f"fragment row half {(t % 16) // 8}), channel {c}{extra}")
    return loc


@pytest.mark.parametrize("name", ATTN_LAYOUTS)
def test_attn_exact_probes(svr2lib, name):
    """(i) K = 0: every valid key has P = 1.  V holds indicator columns (channel c < 64: key index j with
    (j + 3 h) mod 64 == c), a window tag (channel 64) and a head tag (65): the output is the per-class key count / len,
    so a dropped, duplicated or leaked key moves a class by 1 / count (many ulps).  Only the final division rounds.
    (ii) One-hot codes: key j carries 32 at dims j mod 64 and 64 + j // 64, query i the codes of its target t(i, h), so
    the target scores 2048 / sqrt(128) and every other key at most half that: > 126 powers of two apart, P is 1 for the
    target and flushes to 0 for the rest.  Every row must then equal V[t] bit for bit.  Targets cycle over the first,
    a middle and the ragged last kv tile (rows 8 apart differ in their tile: the running max rises and stays put in
    both row halves), over every column mod 64, and differ per head."""
    al = attn_layout(svr2lib, name)
    heads, cu_h = al.heads, al.cu_h
    total = int(cu_h[-1])
    lens = cu_h.diff()
    pos = torch.cat([torch.arange(int(n)) for n in lens]).to(DEV)                      # index within the window
    win = torch.repeat_interleave(torch.arange(len(lens)), lens).to(DEV)
    n_row = lens.to(DEV)[win]
    hh = torch.arange(heads, device=DEV)

    # ---- (i) uniform scores
    q = rnd((total, heads, 128), 1)
    k = torch.zeros_like(q)
    v = torch.zeros_like(q)
    cls = (pos[:, None] + 3 * hh[None]) % 64                                          # (total, heads)
    v.scatter_(2, cls[..., None], 1.0)
    v[:, :, 64] = (win % 13 + 1).to(torch.bfloat16)[:, None]
    v[:, :, 65] = (hh + 1).to(torch.bfloat16)[None]
    got = run_attn(svr2lib, al, q, k, v)
    for n, chunk, idx in length_groups(cu_h, heads, lambda n: 4 * n * 128):
        vd = v[idx].double()                                                          # (cw, n, heads, 128)
        want = (vd.sum(1, keepdim=True) / n).expand_as(vd)
        r, B = round_iv(want, 2 * U * want.abs())        # fp32 1 / l and the product: 2 U; then the output rounding

        def loc_i(cw, i, h, c, chunk=chunk, n=n):
            t = i % 128
            what = f"key class {c} (kv columns {(c - 3 * h) % 64} mod 64)" if c < 64 else \
                ("window tag" if c == 64 else "head tag" if c == 65 else f"channel {c}")
            return (f"window {int(chunk[cw])} (len {n}), head {h}, q-tile {i // 128}, tile row {t} (warpgroup "
                    f"{t // 64}, fragment row half {(t % 16) // 8}), {what}")
        check(got[idx], r, B, f"attention {al.name}: uniform-score probe", loc_i)
        del vd, want, r, B

    # ---- (ii) dominant key
    n_kv = (n_row + 63) // 64
    last = n_row - 64 * (n_kv - 1)                                                    # valid keys of the last kv tile
    pick = (pos[:, None] + hh[None]) % 3                                              # 0 first, 1 middle, 2 last tile
    tile = torch.where(pick == 0, 0, torch.where(pick == 1, n_kv[:, None] // 2, n_kv[:, None] - 1))
    col = (5 * pos[:, None] + 7 * hh[None] + pos[:, None] // 64) % 64
    col = torch.where(tile == n_kv[:, None] - 1, col % last[:, None], col)
    tgt = 64 * tile + col                                                              # (total, heads), < len
    assert (tgt < n_row[:, None]).all()
    q = torch.zeros(total, heads, 128, device=DEV, dtype=torch.bfloat16)
    q.scatter_(2, (tgt % 64)[..., None], 32.0)
    q.scatter_(2, (64 + tgt // 64)[..., None], 32.0)
    k = torch.zeros_like(q)
    k.scatter_(2, (pos % 64)[:, None, None].expand(-1, heads, 1), 32.0)
    k.scatter_(2, (64 + pos // 64)[:, None, None].expand(-1, heads, 1), 32.0)
    v = rnd((total, heads, 128), 2)
    got = run_attn(svr2lib, al, q, k, v)
    start = cu_h.to(DEV)[win]
    want = v[start[:, None] + tgt, hh[None]]                                          # (total, heads, 128)
    bad = bits(got) != bits(want)
    if bad.any():
        row, h, c = bad.nonzero()[0].tolist()
        w, i = window_of(cu_h, row)
        t, ti = i % 128, int(tgt[row, h])
        raise AssertionError(
            f"attention {al.name}: dominant-key probe: {int(bad.sum())} elements differ; first window {w} "
            f"(len {int(lens[w])}), head {h}, q-tile {i // 128}, tile row {t} (warpgroup {t // 64}, fragment row half "
            f"{(t % 16) // 8}), channel {c}: target key {ti} (kv tile {ti // 64} of {int(n_kv[row])}, kv column "
            f"{ti % 64}): got {got[row, h, c].item():.6g}, want {want[row, h, c].item():.6g}")


@pytest.mark.parametrize("name", ATTN_LAYOUTS)
def test_attn_random_vs_fp64(svr2lib, name):
    """Random q / k / v; q rows scaled by 2^u, u uniform in [-1, 2] per row and head, so that the scores spread over
    several powers of two (log2-unit std 1..9) and later kv tiles raise the running max.  Bound: module docstring."""
    al = attn_layout(svr2lib, name)
    heads, cu_h = al.heads, al.cu_h
    total = int(cu_h[-1])
    g = torch.Generator(device=DEV).manual_seed(11)
    qs = torch.exp2(torch.rand(total, heads, 1, generator=g, device=DEV) * 3 - 1)
    q = (rnd((total, heads, 128), 21).float() * qs).to(torch.bfloat16)
    k = (rnd((total, heads, 128), 22).float() * 1.5).to(torch.bfloat16)
    v = rnd((total, heads, 128), 23)
    got = run_attn(svr2lib, al, q, k, v)
    sens = Sensitivity(f"attention {al.name}")
    for n, chunk, idx in length_groups(cu_h, heads, lambda n: n * n + 4 * n * 128):
        qd, kd, vd = (x[idx].double().permute(0, 2, 1, 3) for x in (q, k, v))          # (cw, heads, n, 128)
        s = qd @ kd.transpose(-1, -2) / math.sqrt(128.0)
        s_abs = (qd.abs() @ kd.abs().transpose(-1, -2)).amax(-1, keepdim=True)
        # s is already divided by sqrt(128): in log2 units the raw score's accumulation error is 32 U S_qk SC_LOG2
        # (twice: the score and the max) and M = max |s| log2(e) bounds |s sc|, |m sc| and |x| / 2
        dx = U * (64 * SC_LOG2 * s_abs + 6 * LOG2E * s.abs().amax(-1, keepdim=True))
        eps_p = math.log(2.0) * dx + 2.0 ** -21
        p = torch.softmax(s, -1)
        del s
        r = p @ vd
        A = p @ vd.abs()
        del p
        n_kv = -(-n // 64)
        E = A * (2.0 ** -8 + 2 * eps_p + (n / 4 + 2 * n_kv + 4) * U) + 2.0 ** -120
        rr, B = round_iv(r, E)
        sens.add(B, r)
        check(got[idx].permute(0, 2, 1, 3), rr, B, f"attention {al.name}: random operands vs fp64", attn_loc(al, idx))
        del qd, kd, vd, r, A, E, rr, B
    sens.assert_sensitive()


# ====================================================================== b. QKV projection + q/k RMSNorm + RoPE
def rope_rows(lay, ridx, nf):
    """cos / sin (rows, 6 nf) in apply_rope's layout, gathered from the handle's tables (row index -1: identity)"""
    cs, sn = [], []
    for a in range(3):
        i = ridx[:, a].long()
        ok = (i >= 0)[:, None]
        cs.append(torch.where(ok, lay.cos[i.clamp_min(0)].double(), 1.0).repeat_interleave(2, -1))
        sn.append(torch.where(ok, lay.sin[i.clamp_min(0)].double(), 0.0).repeat_interleave(2, -1))
    return torch.cat(cs, -1), torch.cat(sn, -1)


def pair_swap(t):
    return t.view(*t.shape[:-1], -1, 2).flip(-1).reshape(t.shape)


def norm_rope_ref(p, Bp, wrow, cos_r, sin_r):
    """(r, B) of the q or k output: p (rows, heads, 128) the projection's rounded values with bound Bp, wrow (rows, 128)
    the norm weight of each row, cos_r / sin_r (rows, 6 nf).  Propagation: module docstring."""
    ss = (p * p).sum(-1, keepdim=True)
    rr = 1.0 / torch.sqrt(ss / 128 + EPS)
    w = wrow[:, None, :]
    y = p * rr * w
    rho = (p.abs() * Bp).sum(-1, keepdim=True) / (ss + 128 * EPS)
    By = rr * w.abs() * (Bp + p.abs() * rho) + 144 * U * y.abs()
    yr = dit_oracle.apply_rope(y, cos_r, sin_r)
    nr = cos_r.shape[-1]
    c, s = cos_r.abs()[:, None], sin_r.abs()[:, None]
    Br = By.clone()
    Br[..., :nr] = By[..., :nr] * c + pair_swap(By)[..., :nr] * s + \
        4 * U * (y[..., :nr].abs() * c + pair_swap(y.abs())[..., :nr] * s)
    return round_iv(yr, Br)


def qkv_loc(lay, row_src, r0, nf):
    def loc(row, h, d):
        row += r0
        w, i = window_of(lay.cu_h, row)
        src = int(row_src[row])
        tok = f"video token {src} (m-tile {src // 128})" if src >= 0 else f"text token {-src - 1}"
        pair = d // 2
        ax = f"axis {pair // nf}, frequency {pair % nf}" if pair < 3 * nf else "not rotated"
        return f"{tok}, window {w} row {i}, head {h}, dim {d} (pair {pair}: {ax})"
    return loc


def check_qkv_rows(lay, heads, got, P, wq, wk, what, sens):
    """got: (q, k, v) in window order; P / Bp: a function of a row strip -> the rounded projection (n, 3, heads, 128)
    and its bound; wq / wk: (weights of video rows, of text rows)."""
    inner = heads * 128
    rows = max(1, MAX_STRIP // (3 * inner))
    src_all, src_h = lay.row_src, lay.row_src.cpu()
    for r0 in range(0, lay.total, rows):
        r1 = min(lay.total, r0 + rows)
        p, bp = P(r0, r1)
        vid = (src_all[r0:r1] >= 0)[:, None]
        cos_r, sin_r = rope_rows(lay, lay.row_rope[r0:r1], lay.nfreq)
        loc = qkv_loc(lay, src_h, r0, lay.nfreq)
        for which, (wv, wt) in enumerate((wq, wk)):
            r, B = norm_rope_ref(p[:, which], bp[:, which], torch.where(vid, wv.double(), wt.double()), cos_r, sin_r)
            sens.add(B, r)
            check(got[which][r0:r1], r, B, f"{what}: {'qk'[which]}", loc)
        check(got[2][r0:r1], p[:, 2], bp[:, 2], f"{what}: v", loc)


QKV_GEOMS = [("3b", 20, (5, 68, 120)), ("7b", 24, (2, 135, 240)), ("3b", 2, (3, 20, 36)), ("3b", 4, (5, 34, 60)),
             ("7b", 2, (2, 20, 36)), ("3b", 20, (1, 10, 14)), ("3b", 20, (2, 135, 240)), ("7b", 24, (5, 68, 120))]


@pytest.mark.parametrize("variant,heads,geom", QKV_GEOMS)
def test_qkv_rope_fused_vs_fp64(svr2lib, variant, heads, geom):
    """The production path: svr2_linear_qkv_rope_bf16 writes the video rows of q / k / v (RMSNorm + RoPE + window
    scatter in the QKV GEMM's epilogue), svr2_qk_norm_rope_rows_bf16 the text rows from the text stream's plain QKV GEMM.
    Regular and shifted layouts; M = L is no multiple of 128; the 3B's nfreq = 21 (text rows rotated at (j, j, j)) and
    the 7B's nfreq = 10 (pairs 30..63 and the text rows unrotated).  Every window row is written exactly once: the
    epilogue writes the video rows and no text row, the rows kernel the text rows and no video row."""
    T, Hp, Wp = geom
    d = inner = heads * 128
    L = T * Hp * Wp
    a_v, a_t = rnd((L, d), 1), rnd((TXT, d), 2)
    w_v, w_t = rnd((3 * inner, d), 3, std=d ** -0.5), rnd((3 * inner, d), 4, std=d ** -0.5)
    gn = torch.Generator(device=DEV).manual_seed(5)
    nq_v, nk_v, nq_t, nk_t = (torch.randn(128, generator=gn, device=DEV) * 0.5 + 1 for _ in range(4))
    nqk = torch.cat([nq_v, nk_v]).contiguous()
    P_ = svr2lib.ptr
    Xt = a_t.double() @ w_t.double().T
    St = a_t.double().abs() @ w_t.double().abs().T
    for layer in (0, 1):
        lay = layout(svr2lib, variant, geom, layer)
        what = f"QKV + RoPE {lay.name}, {heads} heads"
        rope = (P_(lay.cos), P_(lay.sin), lay.nfreq)
        bufs = [sentinel_fill(torch.empty(GUARD + lay.total + GUARD, heads, 128, device=DEV, dtype=torch.bfloat16))
                for _ in range(3)]
        q, k, v = (b[GUARD:GUARD + lay.total] for b in bufs)
        qkv_t = svr2lib.linear(a_t, w_t)
        svr2lib.call("svr2_linear_qkv_rope_bf16", P_(a_v), d, P_(w_v), d, L, heads, d, P_(lay.tok_dst), P_(lay.tok_rope),
                     *rope, P_(nqk), EPS, P_(q), P_(k), P_(v), svr2lib.stream())
        torch.cuda.synchronize()
        vid = lay.row_src >= 0
        for name, t in zip("qkv", (q, k, v)):
            written = (bits(t) != SENTINEL).any(-1).any(-1)
            assert torch.equal(written, vid), \
                f"{what}: QKV epilogue wrote {name} rows {int((written & ~vid).sum())} text rows / left " \
                f"{int((vid & ~written).sum())} video rows, first window row " \
                f"{int((written != vid).nonzero()[0])}"
            assert not (bits(t[vid]) == SENTINEL).any(), f"{what}: QKV epilogue left {name} elements of video rows unwritten"
        snap = [t[vid].clone() for t in (q, k, v)]
        svr2lib.call("svr2_qk_norm_rope_rows_bf16", None, P_(qkv_t), P_(lay.row_src), P_(lay.row_rope), *rope, P_(nq_v),
                     P_(nk_v), P_(nq_t), P_(nk_t), EPS, P_(lay.txt_rows), lay.n_win * TXT, heads, P_(q), P_(k), P_(v),
                     svr2lib.stream())
        torch.cuda.synchronize()
        for name, t, s, b in zip("qkv", (q, k, v), snap, bufs):
            check_untouched(b[:GUARD], f"{what}: guard rows before {name}")
            check_untouched(b[-GUARD:], f"{what}: guard rows after {name}")
            assert torch.equal(bits(t[vid]), bits(s)), f"{what}: the rows kernel rewrote video rows of {name}"
            miss = (bits(t) == SENTINEL).any(-1).any(-1)
            if miss.any():
                row = int(miss.nonzero()[0])
                w, i = window_of(lay.cu_h, row)
                raise AssertionError(f"{what}: {int(miss.sum())} {name} rows not written, first window {w} row {i} "
                                     f"(text token {i - int(lay.cu_h[w + 1] - lay.cu_h[w]) + TXT})")

        def proj(r0, r1):
            src = lay.row_src[r0:r1].long()
            m = src >= 0
            X = torch.empty(r1 - r0, 3 * inner, device=DEV, dtype=torch.float64)
            S = torch.empty_like(X)
            av = a_v[src[m]].double()
            X[m], S[m] = av @ w_v.double().T, av.abs() @ w_v.double().abs().T
            X[~m], S[~m] = Xt[-src[~m] - 1], St[-src[~m] - 1]
            p, bp = round_iv(X, d / 4 * U * S)           # the projection's accumulator, then its bf16 rounding point
            return p.view(-1, 3, heads, 128), bp.view(-1, 3, heads, 128)
        sens = Sensitivity(what)
        check_qkv_rows(lay, heads, (q, k, v), proj, (nq_v, nq_t), (nk_v, nk_t), what, sens)
        sens.assert_sensitive()
        del bufs, q, k, v, snap


@pytest.mark.parametrize("case", ["synthetic-3heads", "3b-regular-5heads", "3b-shifted-3heads", "7b-regular-3heads",
                                  "7b-shifted-5heads"])
def test_qk_norm_rope_window_vs_fp64(svr2lib, case):
    """The stand-alone kernel (svr2_qk_norm_rope_window_bf16, the path for head counts the fused epilogue does not
    take) on bf16 projections: odd head counts, the real layouts, and a synthetic table with random rows, text rows
    and -1 RoPE rows among the video rows.  v rows are copies, bit for bit."""
    name, heads = case.rsplit("-", 1)
    heads = int(heads[:-5])
    inner = heads * 128
    if name == "synthetic":
        L, nf, R, total = 50, 21, 40, 90
        g = torch.Generator().manual_seed(0)
        src = torch.randint(0, L, (total,), generator=g)
        is_txt = torch.rand(total, generator=g) < 0.3
        src = torch.where(is_txt, -(torch.randint(0, TXT, (total,), generator=g) + 1), src).int()
        rope = torch.randint(0, R, (total, 3), generator=g).int()
        rope[::5] = -1
        ang = torch.randn(R, nf, generator=g)
        lay = Layout("synthetic", nf, L, 1, total, total, None, torch.tensor([0, total]), src.to(DEV), rope.to(DEV),
                     None, None, None, None, ang.cos().to(DEV), ang.sin().to(DEV))
    else:
        variant, kind = name.split("-")
        lay = layout(svr2lib, variant, REAL[variant][2], int(kind == "shifted"))
        L = lay.L
    qkv_v, qkv_t = rnd((L, 3 * inner), 1), rnd((TXT, 3 * inner), 2)
    gn = torch.Generator(device=DEV).manual_seed(3)
    nq_v, nk_v, nq_t, nk_t = (torch.randn(128, generator=gn, device=DEV) * 0.5 + 1 for _ in range(4))
    P_ = svr2lib.ptr
    bufs = [sentinel_fill(torch.empty(GUARD + lay.total + GUARD, heads, 128, device=DEV, dtype=torch.bfloat16))
            for _ in range(3)]
    q, k, v = (b[GUARD:GUARD + lay.total] for b in bufs)
    svr2lib.call("svr2_qk_norm_rope_window_bf16", P_(qkv_v), P_(qkv_t), P_(lay.row_src), P_(lay.row_rope), P_(lay.cos),
                 P_(lay.sin), lay.nfreq, P_(nq_v), P_(nk_v), P_(nq_t), P_(nk_t), EPS, lay.total, heads, P_(q), P_(k),
                 P_(v), svr2lib.stream())
    torch.cuda.synchronize()
    what = f"q/k norm + RoPE (stand-alone) {lay.name}, {heads} heads"
    for name_, b in zip("qkv", bufs):
        check_untouched(b[:GUARD], f"{what}: guard rows before {name_}")
        check_untouched(b[-GUARD:], f"{what}: guard rows after {name_}")

    def rows(r0, r1):
        src = lay.row_src[r0:r1].long()
        x = torch.where((src >= 0)[:, None], qkv_v[src.clamp_min(0)], qkv_t[(-src - 1).clamp_min(0)]).double()
        return x.view(-1, 3, heads, 128), torch.zeros(r1 - r0, 3, heads, 128, device=DEV, dtype=torch.float64)
    sens = Sensitivity(what)
    check_qkv_rows(lay, heads, (q, k, v), rows, (nq_v, nq_t), (nk_v, nk_t), what, sens)
    sens.assert_sensitive()


# ====================================================================== c. the block's GEMM launches, from production
class Launch(NamedTuple):
    M: int
    N: int
    K: int
    epi: int
    lda: int
    ldc: int


def tile_width(M, N, epi, lib, sms):
    """pick_block_n and the few-row narrowing of linear_impl (csrc/gemm.cu), restated"""
    if epi & lib.EPI_SWIGLU:
        return 256
    bn = 256 if N >= 256 else 128 if N > 64 else 64 if N > 32 else 32 if N > 16 else 16
    m_tiles = -(-M // 128)
    while bn > 32 and 2 * m_tiles * -(-N // bn) <= sms:
        bn //= 2
    return bn


def epi_path(c, lib, bn):
    ct = {lib.EPI_BIAS | lib.EPI_GATE | lib.EPI_RESIDUAL, lib.EPI_GATE | lib.EPI_RESIDUAL, lib.EPI_BIAS, 0}
    if c.epi & lib.EPI_SWIGLU:
        return "SwiGLU"
    return "compile-time epilogue" if bn == 256 and c.epi in ct else "runtime-flag epilogue"


def flag_names(epi, lib):
    names = [n for n in ("BIAS", "GATE", "RESIDUAL", "SWIGLU", "GELU", "SILU") if epi & getattr(lib, "EPI_" + n)]
    return "|".join(names) or "none"


@pytest.fixture(scope="module")
def production(pkg):
    """B200NaDiT (native = False) at full width, 2 layers: the 3B with mm_layers = 1 at 5 x 136 x 240 (both separate
    and shared layers, the last layer's text stream without MLP and gate) and the 7B at 2 x 270 x 480.  Records every
    linear launch (shape, flags, lda, ldc), the rmsnorm_ada and txt_window_mean calls, and layer 0's video SwiGLU
    operands."""
    lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    rec = dict(linear={}, rmsnorm=set(), txt_mean=set(), swiglu=None, sd=None)
    for variant, over, (T, Hp, Wp) in (("3b", dict(layers=2, mm_layers=1), (5, 68, 120)),
                                       ("7b", dict(layers=2), (2, 135, 240))):
        cfg = dit.dit_config(variant, **over)
        sd = pkg.weights.synth_dit_state_dict(cfg, seed=17, dtype=torch.float16, device=DEV)
        eng = dit.B200NaDiT(cfg, sd)
        eng.native = False
        g = torch.Generator(device=DEV).manual_seed(1)
        vid = torch.randn(T * 2 * Hp * 2 * Wp, cfg["in_ch"], generator=g, device=DEV)
        txt = torch.randn(TXT, cfg["txt_in_dim"], generator=g, device=DEV)
        mp = pytest.MonkeyPatch()
        orig_call, orig_linear, orig_rms = lib.call, lib.linear, lib.rmsnorm_ada

        def call(name, *a, **kw):
            if name == "svr2_linear_bf16":
                c = Launch(M=a[4], N=a[5], K=a[6], epi=a[7], lda=a[1], ldc=a[12])
                rec["linear"].setdefault(c, f"{variant}")
            elif name == "svr2_txt_window_mean_bf16":
                rec["txt_mean"].add((a[2], a[3], a[4]))
            return orig_call(name, *a, **kw)

        def linear(a, w, **kw):
            out = orig_linear(a, w, **kw)
            if variant == "3b" and kw.get("epi", 0) & lib.EPI_SWIGLU and rec["swiglu"] is None and \
                    w.data_ptr() == eng.W["0.vid.mlp_in.w"].data_ptr():
                rec["swiglu"] = (a.clone(), out.clone())
            return out

        def rmsnorm_ada(x, scale, shift, **kw):
            rec["rmsnorm"].add((x.shape[0], x.shape[1], kw.get("mode", 0), kw.get("weight") is not None))
            return orig_rms(x, scale, shift, **kw)
        try:
            mp.setattr(lib, "call", call)
            mp.setattr(lib, "linear", linear)
            mp.setattr(lib, "rmsnorm_ada", rmsnorm_ada)
            eng(vid, txt, [[T, 2 * Hp, 2 * Wp]], [[TXT]])
            torch.cuda.synchronize()
        finally:
            mp.undo()
        if variant == "3b":
            rec["sd"] = {k: sd[k].to(torch.bfloat16) for k in ("blocks.0.mlp.vid.proj_in_gate.weight",
                                                              "blocks.0.mlp.vid.proj_in.weight")}
        del eng, sd
        torch.cuda.empty_cache()
    return rec


def epilogue_ref(lib, c, acc, S, bias, gate, res):
    """(r, B, pre) of one output strip: acc / S the fp64 accumulator and sum of |products| (SwiGLU: in the interleaved
    column order of the weight), at the rounding points of the EPI_* comments in csrc/gemm.cu; pre: the value before
    the residual add (the signal of the sensitivity check)."""
    e_acc = c.K / 4 * U * S
    if c.epi & lib.EPI_SWIGLU:
        # tile j of 256 weight rows = [128 gate rows ; 128 in rows] -> output columns 128 j .. 128 j + 127
        acc, e_acc = (t.view(t.shape[0], -1, 2, 128) for t in (acc, e_acc))
        rg, Bg = round_iv(acc[:, :, 0].flatten(1), e_acc[:, :, 0].flatten(1))         # bf16(acc[gate])
        ru, Bu = round_iv(acc[:, :, 1].flatten(1), e_acc[:, :, 1].flatten(1))         # bf16(acc[in])
        z = F.silu(rg)
        rs, Bs = round_iv(z, 1.1 * Bg + fast_rel(rg) * z.abs() + 2.0 ** -120)          # bf16(silu(.))
        z = rs * ru
        r, B = round_iv(z, rs.abs() * Bu + ru.abs() * Bs + Bs * Bu + U * z.abs())     # bf16(silu * in)
        return r, B, r
    z, e = acc, e_acc
    if bias is not None:
        b = bias.double()
        z, e = z + b, e + U * (S + b.abs())
    r, B = round_iv(z, e)                                                                 # bf16(acc + bias)
    if c.epi & lib.EPI_GELU:
        z = gelu_tanh(r)
        r, B = round_iv(z, 1.13 * B + fast_rel(r) * z.abs() + 2.0 ** -120)                # bf16(gelu_tanh(t))
    if c.epi & lib.EPI_GATE:
        g = gate.double()
        z = r * g
        r, B = round_iv(z, g.abs() * B + U * z.abs())                                      # bf16(t * gate)
    pre = r
    if c.epi & lib.EPI_RESIDUAL:
        z = r + res
        r, B = round_iv(z, B + U * z.abs())                                                # bf16(t + res)
    return r, B, pre


def run_linear_case(lib, c, seed, sms, what):
    """One launch with fresh random operands of the recorded shape and flags; output and residual with 16 columns of
    ldc padding beyond the recorded ldc and guard rows, all sentinel (padding: NaN in the residual)."""
    n_out = c.N // 2 if c.epi & lib.EPI_SWIGLU else c.N
    ldc = max(c.ldc, n_out) + 16
    a_buf = rnd((c.M, c.lda), seed)
    a_buf[:, c.K:] = float("nan")
    a = a_buf[:, :c.K]
    w = rnd((c.N, c.K), seed + 1, std=c.K ** -0.5)
    bias = rnd((c.N,), seed + 2) if c.epi & lib.EPI_BIAS else None
    gate = torch.randn(c.N, generator=torch.Generator(device=DEV).manual_seed(seed + 3), device=DEV) \
        if c.epi & lib.EPI_GATE else None
    res = None
    if c.epi & lib.EPI_RESIDUAL:
        res = rnd((c.M, ldc), seed + 4)
        res[:, n_out:] = float("nan")
    obuf = sentinel_fill(torch.empty(GUARD + c.M + GUARD, ldc, device=DEV, dtype=torch.bfloat16))
    out = obuf[GUARD:GUARD + c.M]
    P = lib.ptr
    lib.call("svr2_linear_bf16", P(a_buf), c.lda, P(w), c.K, c.M, c.N, c.K, c.epi, P(bias), P(gate), P(res), P(out), ldc,
             1.0, lib.stream())
    torch.cuda.synchronize()
    check_untouched(obuf[:GUARD], what + ": guard rows before the output")
    check_untouched(obuf[-GUARD:], what + ": guard rows after the output")
    check_untouched(out[:, n_out:], what + ": ldc padding columns")
    bn = tile_width(c.M, c.N, c.epi, lib, sms)
    cols_per_tile = bn // 2 if c.epi & lib.EPI_SWIGLU else bn
    path = epi_path(c, lib, bn)

    def loc(m, n):
        return (f"row {m} (m-tile {m // 128} of {-(-c.M // 128)}, tile row {m % 128}), column {n} (n-tile "
                f"{n // cols_per_tile} of {-(-n_out // cols_per_tile)}, tile column {n % cols_per_tile}), {bn}-column "
                f"tiles, {path}")
    sens = Sensitivity(what)
    rows = max(1, MAX_STRIP // c.N)
    for m0 in range(0, c.M, rows):
        m1 = min(c.M, m0 + rows)
        ad = a[m0:m1].double()
        acc, S = ad @ w.double().T, ad.abs() @ w.double().abs().T
        r, B, pre = epilogue_ref(lib, c, acc, S, bias, gate, None if res is None else res[m0:m1, :n_out].double())
        del acc, S
        sens.add(B, pre)
        check(out[m0:m1, :n_out], r, B, what, lambda m, n: loc(m + m0, n))
        del r, B, pre
    sens.assert_sensitive()
    return bn, path


def test_production_gemm_launches(svr2lib, production):
    """Every distinct svr2_linear_bf16 launch of the 3B and 7B forwards once, element by element, with the tile width
    the library picks for it (pick_block_n + the few-row narrowing, restated with this device's SM count)."""
    lib = svr2lib
    sms = lib.device_check()[0]
    cases = production["linear"]
    E = lib
    L3, L7 = 5 * 68 * 120, 2 * 135 * 240
    have = {(c.M, c.N, c.K, c.epi) for c in cases}
    need = {
        "3B stem vid_in (K = 192)": (L3, 2560, 192, E.EPI_BIAS),
        "3B stem txt_in (K = 5120, M = 58)": (TXT, 2560, 5120, E.EPI_BIAS),
        "3B text QKV": (TXT, 7680, 2560, 0),
        "3B video out projection": (L3, 2560, 2560, E.EPI_BIAS | E.EPI_GATE | E.EPI_RESIDUAL),
        "3B text out projection": (TXT, 2560, 2560, E.EPI_BIAS | E.EPI_GATE | E.EPI_RESIDUAL),
        "3B last text out projection (no gate)": (TXT, 2560, 2560, E.EPI_BIAS | E.EPI_RESIDUAL),
        "3B video SwiGLU": (L3, 13824, 2560, E.EPI_SWIGLU),
        "3B text SwiGLU": (TXT, 13824, 2560, E.EPI_SWIGLU),
        "3B video MLP out": (L3, 2560, 6912, E.EPI_GATE | E.EPI_RESIDUAL),
        "3B text MLP out": (TXT, 2560, 6912, E.EPI_GATE | E.EPI_RESIDUAL),
        "3B vid_out (N = 64)": (L3, 64, 2560, E.EPI_BIAS),
        "7B stem vid_in": (L7, 3072, 192, E.EPI_BIAS),
        "7B video GELU": (L7, 12288, 3072, E.EPI_BIAS | E.EPI_GELU),
        "7B text GELU": (TXT, 12288, 3072, E.EPI_BIAS | E.EPI_GELU),
        "7B video MLP out": (L7, 3072, 12288, E.EPI_BIAS | E.EPI_GATE | E.EPI_RESIDUAL),
        "7B text MLP out": (TXT, 3072, 12288, E.EPI_BIAS | E.EPI_GATE | E.EPI_RESIDUAL),
        "7B vid_out (N = 64)": (L7, 64, 3072, E.EPI_BIAS),
    }
    missing = [k for k, v in need.items() if v not in have]
    assert not missing, f"the forwards did not launch: {missing}"
    covered = {(rows, dim, mode, wt) for dim, rows, mode, wt in RMS_CASES}
    assert production["rmsnorm"] <= covered, \
        f"rmsnorm_ada launches (rows, dim, mode, weight) not covered by test_rmsnorm_ada_vs_fp64: {production['rmsnorm'] - covered}"
    kinds = {(tile_width(c.M, c.N, c.epi, lib, sms), epi_path(c, lib, tile_width(c.M, c.N, c.epi, lib, sms)))
             for c in cases}
    want_kinds = {(256, "compile-time epilogue"), (256, "SwiGLU"), (256, "runtime-flag epilogue"),
                  (64, "runtime-flag epilogue")}
    if sms >= 120:          # the 58 text rows narrow to 32-column (N <= 3072) and 128-column (7B GELU / QKV) tiles
        want_kinds |= {(32, "runtime-flag epilogue"), (128, "runtime-flag epilogue")}
    assert want_kinds <= kinds, f"tile widths / epilogue paths reached: {sorted(kinds)}"
    failures = []
    for i, (c, variant) in enumerate(cases.items()):
        what = f"{variant} linear M{c.M} N{c.N} K{c.K} epi {flag_names(c.epi, lib)}"
        try:
            run_linear_case(lib, c, 100 + 7 * i, sms, what)
        except AssertionError as e:
            failures.append(str(e).split("\n")[0])
        torch.cuda.empty_cache()
    assert not failures, f"{len(failures)} of {len(cases)} launches:\n" + "\n".join(failures)


def test_swiglu_weight_layout_matches_state_dict(svr2lib, production):
    """Layer 0's video SwiGLU as the module ran it (its interleaved mlp_in.w) against fp64 silu(a Wg^T) (a Wu^T) from
    the state dict's proj_in_gate / proj_in (the module's bf16 conversion of them)."""
    a, out = production["swiglu"]
    sd = production["sd"]
    wg, wu = sd["blocks.0.mlp.vid.proj_in_gate.weight"].double(), sd["blocks.0.mlp.vid.proj_in.weight"].double()
    hid, K = wg.shape
    c = Launch(a.shape[0], 2 * hid, K, svr2lib.EPI_SWIGLU, K, hid)
    # the same interleave the kernel expects (per 128 columns: gate block, in block), built from the state dict
    w_il = torch.stack([wg.view(hid // 128, 128, K), wu.view(hid // 128, 128, K)], 1).reshape(2 * hid, K)
    rows = max(1, MAX_STRIP // (2 * hid))
    sens = Sensitivity("SwiGLU of layer 0 vs the state dict")
    for m0 in range(0, c.M, rows):
        m1 = min(c.M, m0 + rows)
        ad = a[m0:m1].double()
        r, B, _ = epilogue_ref(svr2lib, c, ad @ w_il.T, ad.abs() @ w_il.abs().T, None, None, None)
        sens.add(B, r)
        check(out[m0:m1], r, B, "layer 0 video SwiGLU (module weights) vs silu(a Wg^T)(a Wu^T) of the state dict",
              lambda m, n: f"row {m + m0} (m-tile {(m + m0) // 128}), hidden unit {n} (n-tile {n // 128}, tile column "
                           f"{n % 128})")
    sens.assert_sensitive()


# ====================================================================== d. rmsnorm_ada, txt_window_mean
RMS_CASES = [(dim, rows, mode, wt) for dim, L in ((2560, 5 * 68 * 120), (3072, 2 * 135 * 240)) for rows in (TXT, L)
             for mode in (0, 1) for wt in (False, True)]


@pytest.mark.parametrize("dim,rows,mode,weighted", RMS_CASES)
def test_rmsnorm_ada_vs_fp64(svr2lib, dim, rows, mode, weighted):
    """mode 0: bf16(x rr [w] scale + shift); mode 1 (dit_oracle.mlp()): bf16(bf16(bf16(x rr [w]) scale) + shift), each
    rounding point followed as an interval (module docstring): rr in fp32 is relatively (dim / 64 + 8) U off
    (dim / 32 squares per lane, the shuffle tree, rsqrt)."""
    x = rnd((rows, dim), 1)
    g = torch.Generator(device=DEV).manual_seed(2)
    scale = torch.randn(dim, generator=g, device=DEV) * 0.3 + 1
    shift = torch.randn(dim, generator=g, device=DEV) * 0.3
    weight = torch.randn(dim, generator=g, device=DEV) * 0.3 + 1 if weighted else None
    ybuf = sentinel_fill(torch.empty(GUARD + rows + GUARD, dim, device=DEV, dtype=torch.bfloat16))
    y = ybuf[GUARD:GUARD + rows]
    svr2lib.call("svr2_rmsnorm_ada_bf16", svr2lib.ptr(x), svr2lib.ptr(y), rows, dim, EPS, svr2lib.ptr(weight),
                 svr2lib.ptr(scale), svr2lib.ptr(shift), mode, svr2lib.stream())
    torch.cuda.synchronize()
    what = f"rmsnorm_ada dim {dim}, {rows} rows, mode {mode}{', weight' if weighted else ''}"
    check_untouched(ybuf[:GUARD], what + ": guard rows before")
    check_untouched(ybuf[-GUARD:], what + ": guard rows after")
    rel_rr = (dim / 64 + 8) * U
    sc, sh = scale.double(), shift.double()
    sens = Sensitivity(what)
    step = max(1, MAX_STRIP // dim)
    for r0 in range(0, rows, step):
        xd = x[r0:r0 + step].double()
        t = xd * (1.0 / torch.sqrt((xd * xd).mean(-1, keepdim=True) + EPS))
        if weighted:
            t = t * weight.double()
        if mode == 0:
            z = t * sc + sh
            # products x rr [, w], scale: (2 + weighted) U; the shift add: U of the result
            r, B = round_iv(z, (rel_rr + (2 + weighted) * U) * (t * sc).abs() + U * z.abs())
        else:
            r1, B1 = round_iv(t, (rel_rr + (1 + weighted) * U) * t.abs())  # bf16(x rr [w])
            z = r1 * sc
            r2, B2 = round_iv(z, sc.abs() * B1 + U * z.abs())            # bf16(. * scale)
            z = r2 + sh
            r, B = round_iv(z, B2 + U * z.abs())                          # bf16(. + shift)
        sens.add(B, r)
        check(y[r0:r0 + step], r, B, what,
              lambda m, c: f"row {m + r0} (block row slot {(m + r0) % 8}), column {c} (16-byte vector {c // 8}, lane "
                           f"{(c // 8) % 32}, vector slot {c // 256})")
    sens.assert_sensitive()


@pytest.mark.parametrize("n_win,dim", [(75, 2560), (90, 2560), (162, 3072), (200, 3072), (1, 2560)])
def test_txt_window_mean_vs_fp64(svr2lib, production, n_win, dim):
    """The text rows' mean over the windows (na.py window_reverse of the text): the real window counts (3B 75 / 90,
    7B 162 / 200) with l = 58 rows of heads * 128 channels.  fp32 sum in window order, times fp32(1 / n_win)."""
    if n_win > 1:
        assert (n_win, TXT, dim) in production["txt_mean"], sorted(production["txt_mean"])
    x = rnd((n_win, TXT, dim), 1)
    obuf = sentinel_fill(torch.empty(GUARD + TXT + GUARD, dim, device=DEV, dtype=torch.bfloat16))
    o = obuf[GUARD:GUARD + TXT]
    svr2lib.call("svr2_txt_window_mean_bf16", svr2lib.ptr(x), svr2lib.ptr(o), n_win, TXT, dim, svr2lib.stream())
    torch.cuda.synchronize()
    what = f"txt_window_mean over {n_win} windows, dim {dim}"
    check_untouched(obuf[:GUARD], what + ": guard rows before")
    check_untouched(obuf[-GUARD:], what + ": guard rows after")
    xd = x.double()
    z = xd.mean(0)
    e = (n_win + 1) * U * xd.abs().sum(0) / n_win + 2 * U * z.abs()       # the window-order sum, 1 / n_win, the product
    r, B = round_iv(z, e)
    sens = Sensitivity(what)
    sens.add(B, r)
    check(o, r, B, what, lambda j, c: f"text row {j}, column {c} (16-byte vector {(j * dim + c) // 8})")
    sens.assert_sensitive()
