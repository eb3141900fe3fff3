"""-m gpu: the VAE mid-block attention's chunked launch sequence (vae._softmax_v; vae_engine.cu attention runs the same
launches, pinned by tests/test_native_vae_cpu.py) element by element, at the latents where its chunk, key-tile and
statistics-slot counts are largest: n = 129 600 (4K: 16 query chunks, the last a tail; 507 key tiles of 256, the last
64 wide; 1 014 row-sum slots, 64 sampled-key slots), n = 32 400 (1080p: 254 slots) and n = 4 450 (a 712 x 400 portrait:
n % 8 != 0, always the two-pass launches with N = ldn).  Every case runs T = 2 frames (the per-frame offsets f n) with
the single-pass branch and with the exact two-pass launches alone.

At these n a benign row spreads its weight over ~1e5 keys: one 256-key tile carries ~0.2 % of it, so a skipped tile, a
wrong chunk offset or a lost slot moves an output by ~1e-4, far inside any bound on random operands.  Hence exact probes:
  a. one-hot rows.  Query row m selects key pi(m), pi a permutation of its frame's keys, so every row and every key is
     checked.  Key j carries +-1 on 13 dimensions (the bits of j >> 4) and a one-hot of j & 15 on 16 more; the query
     carries A times its target's 13 signs and D on its target's one-hot dimension.  All scores are integers below 2^24,
     exact in the fp32 accumulator.  A key with other high bits scores >= 2 A S2 - D S2 ~ 140 powers of two below the
     target (2^-140: flushed, or clamped to 2^-125, per key; their sum over all keys stays below 2^-107 of the target);
     the target's 15 siblings (same high bits) score D S2 ~ 60 below it.
       - Sampled target (j % 16 == 0), or any target on the two-pass path: the target's exponent is the rounding error of
         its own fp32 score (< 2^-13), so P = bf16(exp2(x)) = 1 exactly, and the siblings' 2^-60 vanish from the fp32 sums:
         the output must equal V[pi(m)] bit for bit.
       - Unsampled target on the single-pass path: the sampled maximum is a sibling's, so the target's P~ = bf16(2^(~60))
         is rounded (relative <= 2^-8, half an ulp of 8 significant bits) while the fp32 row sum keeps the unrounded
         exponential; with the fp32 sums and products (< 2^-20) the pre-rounding output is V[pi(m)] (1 + e), |e| below
         one ulp of it, so the output is V[pi(m)] or a bf16 neighbour: one ulp.  The row sum is ~2^60 < 1e30, so the
         fallback flag must stay 0 in every chunk.
  b. uniform rows.  q = 0: every score is 0.  Column c of V is the indicator of key tile c (then, in a second V, of one
     64-key phase in every 128th tile).  Single-pass: P~ = exp2(0) = 1 exactly, the row sum is the integer n, rowscale =
     rn(1 / n): column c must be bf16(rn(count_c rn(1 / n))).  Two-pass: P = p for every key, p = bf16(exp2(-lse)) within
     2^-7 of 1 / n; count_c p is exact, so column c must be bf16(count_c p), and every column without keys +0.  A lost or
     doubled slot, tile or k-block, which (a) sees only as a normalisation error, changes whole columns here.
  c. the fallback at 4K: one row in a middle chunk and one in the tail chunk get a key ~150 powers of two above their
     sampled maximum.  Exactly those chunks raise the flag; they must equal the two-pass result bit for bit, and every
     other chunk (the next one included: the flag resets per chunk) its single-pass result without the crafted rows.
  d. (tests/test_attention_probs_gpu.py b) the combine kernels at the production slot and row counts.
  e. eng._attention end to end on the synthetic VAE weights at 1 x 270 x 480 x 512: every chunk's first and last rows and
     their m-tile neighbours plus 500 random rows against fp64, with the bound of tests/test_dit_block_elementwise_gpu.py
     part a carried through the output projection and the residual.

Every output sits between sentinel guard rows; the columns of V^T and P past n hold NaN (production leaves them
uninitialised), so any read of them shows.  Failures name the row's chunk and m-tile and the key's tile, slot and
64-column phase."""
import math
from typing import NamedTuple

import pytest
import torch

from test_conv_elementwise_gpu import U, bits, check_untouched, sentinel_fill, ulp_bf16
from test_dit_block_elementwise_gpu import Sensitivity, check, rne_bf16, round_iv

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 512
LOG2E = 1.4426950408889634
S2 = float(torch.tensor((1.0 / D ** 0.5) * LOG2E, dtype=torch.float32))   # vae._softmax_v's score scale, as the kernel gets it
GUARD = 3                                   # sentinel rows before and after every output
EXTRA = 64                                  # NaN columns past ldn in V^T and P
BF = torch.bfloat16
LATENTS = {129600: (270, 480), 32400: (135, 240), 4450: (89, 50)}


def bf(x):
    return float(torch.tensor(x).to(BF))


A_HI = bf(100 / S2)                         # 2 A S2 ~ 200: keys with other high bits vanish
D_LO = bf(60 / S2)                          # D S2 ~ 60: an unsampled target stays inside the single-pass range
D_FALL = bf(150 / S2)                       # ~150 powers of two above the sampled maximum: the row sum overflows


# ====================================================================== the sequence's geometry
class Geo(NamedTuple):
    n: int
    ldn: int
    cq: int
    chunks: int
    slots: int              # two-pass ROWSTAT slots
    slots_s: int            # sampled-key ROWSTAT slots
    slots_p: int            # single-pass row-sum slots
    tiles: int              # 256-key tiles
    single: bool


def geometry(lib, n, single_pass):
    """The formulas of vae._softmax_v / vae_engine.cu attention, restated."""
    ldn = (n + 7) // 8 * 8
    wave_rows = 66 * 128                    # one wave of 132 CTAs (66 m-tiles x 2 n-tiles of d = 512)
    cq = min(wave_rows * max(1, (1 << 32) // (wave_rows * ldn * 2)), (n + 127) // 128 * 128)
    L = lib.load()
    return Geo(n, ldn, cq, -(-n // cq), L.svr2_rowstat_slots(n), L.svr2_rowstat_slots(-(-n // 16)), 2 * -(-n // 256),
               -(-n // 256), single_pass and n >= 256 and n % 8 == 0)


def row_loc(g, r):
    f, m = divmod(r, g.n)
    return f"frame {f} row {m} (chunk {m // g.cq} of {g.chunks}, m-tile {(m % g.cq) // 128})"


def key_loc(g, j):
    return (f"key {j} (tile {j // 256} of {g.tiles}, slot {j // 128}, phase {(j % 256) // 64}"
            f"{', sampled' if j % 16 == 0 else ''})")


@pytest.fixture(scope="module")
def eng(pkg):
    import importlib
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    return vae.B200VideoVAE(pkg.weights.synth_vae_state_dict(seed=4321, dtype=torch.float16))


def run(eng, g, q, k_buf, v, T, single_pass):
    """eng._softmax_v with guarded buffers: o between sentinel rows; V^T and P with NaN columns past ldn (and past n in
    V^T).  Returns (o, per-chunk flags as each chunk's pexp_stat_combine left them, -1 where the branch did not run)."""
    n = g.n
    obuf = sentinel_fill(torch.empty(T * n + 2 * GUARD, D, device=DEV, dtype=BF))
    vt = torch.full((D, g.ldn + EXTRA), float("nan"), device=DEV, dtype=BF)
    P = torch.full((min(g.cq, n), g.ldn + EXTRA), float("nan"), device=DEV, dtype=BF)
    flag_log = torch.full((T * g.chunks,), -1, device=DEV, dtype=torch.int32)
    o = eng._softmax_v(q, k_buf, v, T, n, single_pass, o=obuf[GUARD:GUARD + T * n], vt=vt[:, :g.ldn], P=P[:, :g.ldn],
                       flag_log=flag_log)
    torch.cuda.synchronize()
    assert o.data_ptr() == obuf[GUARD].data_ptr()
    check_untouched(obuf[:GUARD], "guard rows before the output")
    check_untouched(obuf[GUARD + T * n:], "guard rows after the output")
    assert torch.isnan(vt[:, n:].float()).all(), "V^T written past n"
    assert torch.isnan(P[:, g.ldn:].float()).all(), "P written past ldn"
    return o, flag_log.tolist()


def frames(T, n, kf):
    """K for T frames of the same keys, with the 8 zero spare rows vae._attention allocates"""
    k_buf = torch.zeros(T * n + 8, D, device=DEV, dtype=BF)
    k_buf[:T * n] = kf.repeat(T, 1)
    return k_buf


def random_v(rows, seed):
    """random bf16 values of magnitude >= 1/4 (no zeros: a zero row would hide the siblings' 2^-60)"""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    v = torch.randn(rows, D, generator=gen, device=DEV)
    return torch.where(v.abs() < 0.25, torch.copysign(torch.full_like(v, 0.25), v) + v, v).to(BF)


# ====================================================================== a. one-hot probes
def probe_keys(n):
    j = torch.arange(n, device=DEV)
    hi = ((j[:, None] >> 4) >> torch.arange(13, device=DEV)) & 1
    kf = torch.zeros(n, D, device=DEV, dtype=BF)
    kf[:, :13] = (2 * hi - 1).to(BF)
    kf[j, 13 + (j & 15)] = 1
    return kf, (2 * hi - 1).float()


def probe_queries(code, targets, lo_scale):
    """q rows selecting `targets` (key indices): A on the target's 13 signs, lo_scale on its one-hot dimension"""
    q = torch.zeros(targets.numel(), D, device=DEV, dtype=BF)
    q[:, :13] = (A_HI * code[targets]).to(BF)
    q[torch.arange(targets.numel(), device=DEV), 13 + (targets & 15)] = lo_scale
    return q


def probe_operands(g, T, seed):
    assert g.n // 16 < 1 << 13 and 13 * A_HI + D_FALL < 2 ** 24        # 13 code bits; integer scores exact in fp32
    kf, code = probe_keys(g.n)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    pi = torch.stack([torch.randperm(g.n, generator=gen, device=DEV) for _ in range(T)])       # (T, n) targets
    q = torch.cat([probe_queries(code, pi[f], D_LO) for f in range(T)])
    v = random_v(T * g.n, seed + 1)
    return q, frames(T, g.n, kf), v, pi, code


def check_probes(g, o, v, pi, T, what):
    n = g.n
    src = (pi + torch.arange(T, device=DEV)[:, None] * n).flatten()         # global key row of every query row
    want = v[src]
    tgt = pi.flatten()
    exact = torch.ones_like(tgt, dtype=torch.bool) if not g.single else (tgt % 16 == 0)
    err = (o.double() - want.double()).abs()
    lim = torch.where(exact[:, None], torch.zeros_like(err), ulp_bf16(want.double()))
    bad_rows = (~(err <= lim)).any(1)                   # NaN (an unwritten sentinel) fails
    nb = int(bad_rows.sum())
    if nb:
        rows = bad_rows.nonzero()[:, 0]
        r = int(rows[0])
        chunks = sorted({(int(x) // n, (int(x) % n) // g.cq) for x in rows[:4096]})
        tiles = sorted({int(tgt[x]) // 256 for x in rows[:4096]})
        c = int((~(err[r] <= lim[r])).nonzero()[0])
        raise AssertionError(
            f"{what}: {nb} of {T * n} rows differ from V[pi(m)]; first {row_loc(g, r)} selecting {key_loc(g, int(tgt[r]))}: "
            f"column {c} got {o[r, c].item():.6g} (bits {int(bits(o[r:r + 1, c]))}), want {want[r, c].item():.6g}, "
            f"bound {lim[r, c].item():.3g}; (frame, chunk) of bad rows {chunks[:12]}, key tiles {tiles[:12]}"
            f"{' ...' if len(tiles) > 12 else ''}")


CASES = [(n, s) for n in LATENTS for s in (True, False)]


@pytest.mark.parametrize("n,single_pass", CASES, ids=[f"n{n}-{'single' if s else 'twopass'}" for n, s in CASES])
def test_one_hot_probes_every_row_every_key(eng, svr2lib, n, single_pass):
    g = geometry(svr2lib, n, single_pass)
    assert g.cq == eng._attention_chunk_rows(n)
    if n == 129600:                         # the 4K shape this module is about: 16 chunks of 8 448 rows, a 2 880-row tail
        assert (g.cq, g.chunks, n - (g.chunks - 1) * g.cq, g.slots, g.slots_s, g.slots_p) == (8448, 16, 2880, 1014, 64, 1014)
    T = 2
    q, k_buf, v, pi, _ = probe_operands(g, T, seed=n + single_pass)
    o, flags = run(eng, g, q, k_buf, v, T, single_pass)
    if g.single:
        up = [divmod(i, g.chunks) for i, fl in enumerate(flags) if fl]
        assert not up, f"the fallback flag went up for in-range rows in (frame, chunk) {up[:16]}"
    else:
        assert flags == [-1] * len(flags)
    check_probes(g, o, v, pi, T, f"one-hot probes n = {n}, {'single-pass' if g.single else 'two-pass'}")


# ====================================================================== b. uniform rows
def uniform_v(n, which):
    """V (n, D) in {0, 1}: column c marks key tile c ('tiles'), or phase c % 4 of the tiles t = c // 4 (mod 128)"""
    j = torch.arange(n, device=DEV)
    c = torch.arange(D, device=DEV)
    if which == "tiles":
        m = (j[:, None] // 256) == c[None, :]
    else:
        m = (((j % 256) // 64)[:, None] == (c % 4)[None, :]) & (((j // 256) % 128)[:, None] == (c // 4)[None, :])
    return m.to(BF)


@pytest.mark.parametrize("which", ["tiles", "phases"])
@pytest.mark.parametrize("n,single_pass", CASES, ids=[f"n{n}-{'single' if s else 'twopass'}" for n, s in CASES])
def test_uniform_rows_exact_column_sums(eng, svr2lib, n, single_pass, which):
    g = geometry(svr2lib, n, single_pass)
    T = 2
    vf = uniform_v(n, which)
    count = vf.double().sum(0)                                                  # keys per column, exact
    assert count.sum().item() == n and count[0].item() in (64.0, 256.0)
    gen = torch.Generator(device=DEV).manual_seed(n)
    kf = torch.randn(n, D, generator=gen, device=DEV).to(BF)                    # q = 0: K does not matter
    q = torch.zeros(T * n, D, device=DEV, dtype=BF)
    o, flags = run(eng, g, q, frames(T, n, kf), vf.repeat(T, 1), T, single_pass)
    what = f"uniform rows ({which}) n = {n}, {'single-pass' if g.single else 'two-pass'}"
    if g.single:
        assert flags == [0] * len(flags), f"{what}: flag raised: {flags}"
        rs = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(n), dtype=torch.float32)       # rn(1 / n)
        want = (count.float().cpu() * rs).to(BF).to(DEV)[None, :].expand(T * n, D)
    else:
        p = o[:, 0].double() / count[0]                                         # count_0 p is exact: p per row
        assert (p == p[0]).all(), f"{what}: the probability differs between rows"
        p0 = p[0].item()
        assert abs(p0 * n - 1) <= 2.0 ** -7, f"{what}: P = {p0:.6g} is not bf16(1 / n) = {1 / n:.6g}"
        want = rne_bf16(count * p0).to(BF)[None, :].expand(T * n, D)
    bad = bits(o) != bits(want.contiguous())
    nb = int(bad.sum())
    if nb:
        r, c = bad.nonzero()[0].tolist()
        cols = sorted(set(bad.nonzero()[:, 1].tolist()))
        what_c = (f"key tile {c}" if which == "tiles" else f"phase {c % 4} of tiles {c // 4} + 128 k") + \
            (" (no keys)" if count[c] == 0 else f" ({int(count[c])} keys)")
        raise AssertionError(f"{what}: {nb} elements differ; first {row_loc(g, r)}, column {c} = {what_c}: got "
                             f"{o[r, c].item():.6g}, want {want[r, c].item():.6g}; columns {cols[:16]}"
                             f"{' ...' if len(cols) > 16 else ''}")


# ====================================================================== c. the fallback at 4K
def test_fallback_flag_per_chunk_at_4k(eng, svr2lib):
    n, T = 129600, 2
    g = geometry(svr2lib, n, True)
    q, k_buf, v, pi, code = probe_operands(g, T, seed=7)
    base, flags = run(eng, g, q, k_buf, v, T, True)
    assert flags == [0] * len(flags)
    mid, tail = g.chunks // 2, g.chunks - 1
    crafted = {mid * g.cq + 77: 64 * 1000 + 37, tail * g.cq + 1000: n - 3}      # frame-0 row -> unsampled key
    qc = q.clone()
    for m, j in crafted.items():
        assert j % 16
        qc[m] = probe_queries(code, torch.tensor([j], device=DEV), D_FALL)[0]
    o1, flags = run(eng, g, qc, k_buf, v, T, True)
    o2, _ = run(eng, g, qc, k_buf, v, T, False)
    want_flags = [int(i in (mid, tail)) for i in range(T * g.chunks)]
    assert flags == want_flags, f"flags per (frame, chunk): got {flags}, want {want_flags}"
    for m, j in crafted.items():
        assert torch.equal(bits(o2[m]), bits(v[j])), f"two-pass: crafted {row_loc(g, m)} is not V[{j}]"
    for i in range(T * g.chunks):
        f, c = divmod(i, g.chunks)
        r0 = f * n + c * g.cq
        r1 = f * n + min(n, (c + 1) * g.cq)
        ref, name = (o2, "the two-pass result") if want_flags[i] else (base, "its single-pass result")
        assert torch.equal(bits(o1[r0:r1]), bits(ref[r0:r1])), f"frame {f} chunk {c}: not bit-equal to {name}"


# ====================================================================== e. eng._attention end to end
def test_attention_4k_rows_vs_fp64(eng, svr2lib, monkeypatch):
    import importlib
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    p = "decoder.mid_block.attentions.0."
    H, W = LATENTS[129600]
    n = H * W
    g = geometry(svr2lib, n, True)
    x = vae.Act(1, H, W, D, 0, DEV)
    gen = torch.Generator(device=DEV).manual_seed(6)
    x.buf.copy_(torch.randn(x.buf.shape, generator=gen, device=DEV, dtype=BF))
    seen = {}
    softmax_v = eng._softmax_v

    def spy(q, k_buf, v, T, n_, single_pass=True, **kw):
        o = softmax_v(q, k_buf, v, T, n_, single_pass, **kw)
        seen.update(q=q, k=k_buf[:T * n_], v=v, o=o)
        return o
    monkeypatch.setattr(eng, "_softmax_v", spy)
    out = eng._attention(x, p).buf.view(n, D)
    torch.cuda.synchronize()
    q, k, v, o = seen["q"], seen["k"], seen["v"], seen["o"]

    edge = set()
    for c in range(g.chunks):
        r0, r1 = c * g.cq, min(n, (c + 1) * g.cq) - 1
        edge |= {r for r in (r0, r0 + 1, r0 + 127, r0 + 128, r1 - 128, r1 - 127, r1 - 1, r1) if r0 <= r <= r1}
    rnd_rows = torch.randint(0, n, (500,), generator=torch.Generator().manual_seed(1)).tolist()
    rows = torch.tensor(sorted(edge | set(rnd_rows)), device=DEV)

    # attention output o, per element (module docstring of tests/test_dit_block_elementwise_gpu.py, part a)
    qd, kd, vd = q[rows].double(), k.double(), v.double()
    s = qd @ kd.T / math.sqrt(D)
    s_abs = (qd.abs() @ kd.abs().T).amax(-1, keepdim=True)
    M = s.abs().amax(-1, keepdim=True) * LOG2E
    # score: K = 512 accumulation (D / 4 U S_qk, for the score and the reference exponent), the fma forming x and the
    # scaled maximum (6 U M); exp2: the polynomial's 6e-5 (single-pass column pairs) or ex2.approx's 2^-21
    dx = U * (2 * (D / 4) * S2 * s_abs + 6 * M)
    eps_p = math.log(2.0) * dx + 6e-5
    prob = torch.softmax(s, -1)
    del s
    r = prob @ vd
    Aw = prob @ vd.abs()
    del prob
    # P~ rounded to bf16 (2^-8) against the row sum's unrounded terms; the P~ V accumulation over K = n (n / 4 U) and
    # the row sum's fp32 chains over 64 columns and `slots_p` slots; rowscale and its product (2 U)
    E = Aw * (2.0 ** -8 + 2 * eps_p + (n / 4 + g.slots_p + 64 + 2) * U) + 2.0 ** -120
    ro, Bo = round_iv(r, E)
    sens = Sensitivity("VAE attention at n = 129 600")
    sens.add(Bo, r)

    def loc(i, c):
        return f"{row_loc(g, int(rows[i]))}, column {c}"
    check(o[rows], ro, Bo, "attention output at n = 129 600 vs fp64", loc)
    sens.assert_sensitive()
    del qd, kd, vd, r, Aw, E, ro, Bo

    # the output projection (K = 512) + bias, one bf16 rounding, then + x with a second rounding (add_bf16x8)
    wo, bo = eng.W[p + "to_out.0.weight"].double(), eng.W[p + "to_out.0.bias"].double()
    od, xr = o[rows].double(), x.buf.view(n, D)[rows].double()
    z1 = od @ wo.T + bo
    S = od.abs() @ wo.abs().T + bo.abs()
    r1, B1 = round_iv(z1, (D / 4 + 1) * U * S)
    r2, B2 = round_iv(r1 + xr, B1 + U * (r1 + xr).abs())
    check(out[rows], r2, B2, "attention block output (projection + residual) at n = 129 600 vs fp64", loc)
