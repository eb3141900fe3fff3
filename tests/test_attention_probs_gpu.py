"""-m gpu: the single-pass probabilities of the VAE mid-block attention (vae._attention, vae_engine.cu) and the device
flag that sends a query chunk back to the exact two-pass launches, element by element against fp64 references on the
same bf16 operands:
  a. the exp2 of every column position of the PEXP epilogue (MUFU and polynomial column pairs) and its row sums;
  b. svr2_pexp_stat_combine / svr2_rowstat_max / svr2_rowstat_combine on hand-built partials;
  c. the whole single-pass launch sequence, with rows crafted so that the flag must (or must not) go up;
  d. the launch contract of svr2_linear_ex_bf16: run_if, EPI_ROWSCALE, ROWSTAT and the documented refusals."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
LOG2E = 1.4426950408889634
D = 512
S2 = D ** -0.5 * LOG2E          # vae._attention's score scale at d = 512 (exponents in log2 units)
INF, NAN = float("inf"), float("nan")


def rnd(*shape, std=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * std).to(DEV)


def halves(*shape, seed=0):
    """bf16 operands in {-1, -0.5, 0, 0.5, 1}: every product and every partial sum of K <= 256 of them is exact in
    fp32, so the GEMM accumulator equals the fp64 one whatever the summation order."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randint(-2, 3, shape, generator=g).double() * 0.5).to(DEV).to(torch.bfloat16)


def bits(t):
    return t.contiguous().view(torch.int16).int()


def samples(mask, x, val, k=6):
    idx = mask.nonzero()[:k].tolist()
    return ", ".join(f"(row {r}, col {c}: x={x[r, c].item():.4g} -> {val[r, c].item():.4g})" for r, c in idx)


# ====================================================================== a. exp2 sweep through the GEMM
FRACS = (0.0, 0.1, 0.25, 0.5, 0.6, 0.75, 0.9)      # x = integer - f: f = 0.5 gives 127.5, f = 0.6 gives 128.4
POINTS = (-126.0, -125.0, 127.0, 127.5, 128.0, 128.4, 128.5, 129.0, 150.0, 255.0, 256.0, 383.0, 384.0)


@pytest.mark.parametrize("N", [256, 264, 520, 776])
@pytest.mark.parametrize("with_stat", [False, True], ids=["pexp", "pexp_stat"])
def test_pexp_exp2_every_column_position(svr2lib, N, with_stat):
    """acc[m, n] = s_n = (n mod 256) - 255 exactly (a = e_0, w[n, 0] = s_n), gate = mhat[m] = j + f, out_scale = 1: element
    (m, n) sees x = s_n - mhat[m] (one fp32 rounding, reproduced below).  j runs over [-656, 200], so every x = k - f in
    [-200, 400] lands on every column position of a 256-wide tile, whichever column pairs take which exp2."""
    mhat = torch.cat([torch.arange(-656, 201, dtype=torch.float64) + f for f in FRACS]).float().to(DEV)
    M = mhat.numel()
    s = (torch.arange(N, device=DEV) % 256 - 255).float()
    a = torch.zeros(M, 64, device=DEV, dtype=torch.bfloat16)
    a[:, 0] = 1
    w = torch.zeros(N, 64, device=DEV, dtype=torch.bfloat16)
    w[:, 0] = s.to(torch.bfloat16)
    x = (s[None, :] - mhat[:, None]).double()          # the kernel's fmaf(acc, 1, -mhat), an fp32 operation
    for v in POINTS:
        assert ((x[:, :256] - v).abs() < 1e-3).any(0).all(), f"x = {v} does not reach every column position"

    Pbuf = torch.full((M, N + 8), -7.0, device=DEV, dtype=torch.bfloat16)     # 8 guard columns: ldc = N + 8
    slots = 2 * ((N + 255) // 256)
    stat = torch.full((M, 2 * (slots + 1)), NAN, device=DEV) if with_stat else None   # one guard slot per row
    svr2lib.linear(a, w, epi=svr2lib.EPI_PEXP, gate=mhat, out=Pbuf[:, :N], out_scale=1.0, stat_out=stat)
    torch.cuda.synchronize()
    P = Pbuf[:, :N]
    Pf = P.float()
    assert (Pbuf[:, N:] == -7.0).all(), "columns past N were written"
    bad = (x >= 128) & (Pf != INF)
    assert not bad.any(), f"{int(bad.sum())} elements with x >= 128 are not +inf, at column positions (mod 64) " \
        f"{sorted(set((bad.nonzero()[:, 1] % 64).tolist()))}: " + samples(bad, x, Pf)
    # x in [-125, 127]: the exp2 error (< 6e-5 polynomial, < 2^-22 MUFU) is far below half a bf16 ulp (>= 2^-9
    # relative), so only a rounding boundary between kernel and reference can separate them: at most 1 ulp.  Every
    # other x of the sweep differs by >= 0.1 (a factor >= 1.07, >= 9 ulps): a value from a wrong row or column, or a
    # wrong exponent, cannot pass.
    mid = (x >= -125) & (x <= 127)
    ref = torch.exp2(x).to(torch.bfloat16)
    bad = mid & ((bits(P) - bits(ref)).abs() > 1)
    assert not bad.any(), f"{int(bad.sum())} probabilities off by > 1 bf16 ulp: " + samples(bad, x, Pf)
    low = x < -125                                      # clamped (2^-125) or flushed (0): never more than 2^-124
    bad = low & (Pf > 2.0 ** -124)
    assert not bad.any(), "x < -125 gave more than 2^-124: " + samples(bad, x, Pf)
    bad = (x > 127) & (x < 128) & (Pf < 2.0 ** 127)
    assert not bad.any(), "x in (127, 128) gave less than 2^127: " + samples(bad, x, Pf)
    assert not torch.isnan(Pf).any(), "NaN probabilities: " + samples(torch.isnan(Pf), x, Pf)
    neg = bits(P) < 0                                   # sign bit: catches -0.0 as well
    assert not neg.any(), "negative probabilities: " + samples(neg, x, Pf)

    if with_stat:
        st = stat.view(M, slots + 1, 2)
        assert torch.isnan(st[:, slots]).all(), "stat_out written past 2 * ceil(N / 256) slots"
        got = st[:, :slots, 1].double().sum(1)
        want = torch.exp2(x).sum(1)                     # columns n < N only: a padded column (acc = 0, x = -mhat)
        xmax = x.max(1).values                          # would add 2^max, about half the row sum
        # rows with every x <= 99 (the sum stays finite) and some x >= -60 (terms below 2^-125 are clamped or flushed
        # by design; here they are < 2^-65 of the sum).  Per term < 6e-5 (polynomial), fp32 chains of <= 32 terms add
        # < 2e-6: 1e-4 relative.  A leaked padded column adds ~50 %, a dropped maximum column ~50 %.
        rows = (xmax <= 99) & (xmax >= -60)
        assert int(rows.sum()) > 500
        rel = ((got - want).abs() / want)[rows]
        assert torch.isfinite(rel).all() and rel.max().item() <= 1e-4, \
            f"row sums: max rel err {rel.max().item():.3e} (row {int(rows.nonzero()[rel.argmax()])})"
        over = xmax >= 128                              # a +inf element makes the row sum +inf (flag goes up)
        assert (got[over] == INF).all(), \
            f"{int((got[over] != INF).sum())} rows with x >= 128 have a finite row sum, e.g. x_max = " \
            f"{xmax[over][got[over] != INF][:4].tolist()} -> {got[over][got[over] != INF][:4].tolist()}"


# ====================================================================== b. combine kernels on hand-built partials
def _flag(v):
    return torch.full((1,), v, device=DEV, dtype=torch.int32)


def _combine(lib, part, slots, rows, flag):
    rscale = torch.full((rows,), NAN, device=DEV)
    mhat = torch.zeros(rows, device=DEV)                # not read
    lib.call("svr2_pexp_stat_combine", lib.ptr(part), slots, part.shape[1] // 2, lib.ptr(mhat), lib.ptr(rscale), rows,
             lib.ptr(flag), lib.stream())
    torch.cuda.synchronize()
    return rscale


def f32(v, toward=None):
    """v rounded to fp32, or its fp32 neighbour toward `toward`"""
    t = torch.tensor(v, dtype=torch.float32)
    return (t if toward is None else torch.nextafter(t, torch.tensor(toward, dtype=torch.float32))).item()


OK_EDGES = (f32(1e-30, INF), f32(1e30, 0.0), 1.0)      # the fp32 neighbours of the bounds inside the interval
BAD_SUMS = (0.0, -0.0, f32(1e-30), 1e-40, -1.0, f32(1e30), 3e38, INF, -INF, NAN)


# 254 / 1014: the row-sum slots of the 1080p and 4K latents (n = 32 400, 129 600), at a tail chunk's and a full chunk's rows
PEXP_ROWS = {254: 2880, 1014: 8448}


@pytest.mark.parametrize("slots", [1, 6, 33, 70, 254, 1014])
def test_pexp_stat_combine_rowscale_and_flag(svr2lib, slots):
    """rowscale = 1 / (sum of the slots' .y) when it lies in (1e-30, 1e30), else 0 and the flag goes up; the flag is
    raised for sums <= 1e-30, >= 1e30, +-inf and NaN, and for no other sum.  203 rows (not a multiple of the 8 rows per
    block), slots past the 32 lanes, ld = slots + 2 with NaN in the spare slots and NaN in every .x (neither is read)."""
    rows, ld = PEXP_ROWS.get(slots, 203), slots + 2
    g = torch.Generator(device="cpu").manual_seed(slots)
    part = torch.full((rows, ld, 2), NAN)
    scale = 10.0 ** (torch.rand(rows, 1, generator=g) * 50 - 25)          # row sums from ~1e-25 to ~1e25
    part[:, :slots, 1] = (0.5 + torch.rand(rows, slots, generator=g)) * scale
    for r, v in enumerate(OK_EDGES):                    # sums next to the bounds, held by one slot (exact sum)
        part[r, :slots, 1] = 0.0
        part[r, slots - 1, 1] = v
    part = part.to(DEV).view(rows, 2 * ld)
    want = 1.0 / part.view(rows, ld, 2)[:, :slots, 1].double().sum(1)

    flag = _flag(0)
    base = _combine(svr2lib, part, slots, rows, flag)
    assert flag.item() == 0, "flag raised for sums inside (1e-30, 1e30)"
    # fp32 sum of positive terms, <= 32 per lane (1014 slots) then a 5-level shuffle tree: < 37 * 2^-24 = 2.2e-6, plus
    # the rounding of 1 / s: 1e-5.  Every slot holds >= 1 / (3 * slots) of its row's sum (>= 3.3e-4 at 1014 slots), so a
    # dropped slot or a read spare slot (NaN) is far outside.
    rel = (base.double() - want).abs() / want
    assert torch.isfinite(rel).all() and rel.max().item() <= 1e-5, f"rowscale: max rel err {rel.max().item():.3e}"
    flag = _flag(1)
    _combine(svr2lib, part, slots, rows, flag)
    assert flag.item() == 1, "the combine must only raise the flag, never clear it"

    bad_rows = (0, 101, rows - 1)
    cases = [(v, (slots - 1,)) for v in BAD_SUMS]
    if slots > 1:
        cases.append((3e38, (0, slots - 1)))            # finite slots whose fp32 sum overflows
    for v, where in cases:
        for r in bad_rows:
            p = part.clone().view(rows, ld, 2)
            p[r, :slots, 1] = 0.0
            for i in where:
                p[r, i, 1] = v
            flag = _flag(0)
            rs = _combine(svr2lib, p.view(rows, 2 * ld), slots, rows, flag)
            assert flag.item() == 1, f"flag not raised for a row sum of {v} x {len(where)} (row {r})"
            assert rs[r].item() == 0.0, f"rowscale of a flagged row ({v}) must be 0, got {rs[r].item()}"
            others = torch.ones(rows, dtype=torch.bool, device=DEV)
            others[r] = False
            assert torch.equal(rs[others], base[others]), "a flagged row changed the other rows' rowscale"


@pytest.mark.parametrize("slots,rows", [(1, 1), (5, 3), (33, 203), (70, 203), (64, 8448), (64, 2880)])   # 64: 4K sampled keys
def test_rowstat_max_reference_exponent_and_flag_reset(svr2lib, slots, rows):
    """mhat[row] = max over the slots' .x (exact), -inf slots included; the spare slot past `slots` holds +1e9 and every
    .y is NaN (neither is read).  The flag is cleared for any row count, and a NULL flag_reset is accepted."""
    ld = slots + 1
    g = torch.Generator(device="cpu").manual_seed(slots)
    part = torch.full((rows, ld, 2), NAN)
    part[:, :slots, 0] = torch.rand(rows, slots, generator=g) * 100 - 50
    if slots > 1:
        part[:, :slots - 1:2, 0] = -INF
    part[:, slots, 0] = 1e9
    want = part[:, :slots, 0].max(1).values.to(DEV)
    part = part.to(DEV).view(rows, 2 * ld)
    for flag in (_flag(1), None):
        mhat = torch.full((rows,), NAN, device=DEV)
        svr2lib.call("svr2_rowstat_max", svr2lib.ptr(part), slots, ld, svr2lib.ptr(mhat), rows, svr2lib.ptr(flag),
                     svr2lib.stream())
        torch.cuda.synchronize()
        assert torch.equal(mhat, want), f"mhat: max abs diff {(mhat - want).abs().max().item()}"
        if flag is not None:
            assert flag.item() == 0, f"rowstat_max did not clear the flag (rows = {rows})"


@pytest.mark.parametrize("slots,rows", [(1, 5), (6, 203), (33, 203), (70, 203), (254, 2880), (254, 8448), (1014, 2880),
                                        (1014, 8448)])
def test_rowstat_combine_lse(svr2lib, slots, rows):
    """lse[row] = max + log2(sum_i l_i 2^(m_i - max)) against fp64, with -inf slots (the empty half-tiles of a ragged N;
    their .y is NaN and must not be read), a spare slot past `slots` that would dominate if read, and a row whose
    slots are all -inf (lse = -inf)."""
    ld = slots + 1
    g = torch.Generator(device="cpu").manual_seed(100 + slots)
    top = torch.rand(rows, 1, generator=g) * 80 - 40
    part = torch.empty(rows, ld, 2)
    part[:, :, 0] = top - torch.rand(rows, ld, generator=g) * 3          # every slot within 2^3 of the row max
    part[:, :, 1] = 1 + torch.rand(rows, ld, generator=g)
    if slots > 2:
        part[:, 1:slots:3, 0] = -INF
        part[:, 1:slots:3, 1] = NAN
    part[:, slots] = torch.tensor([1e3, 1.0])
    part[rows - 1, :slots, 0] = -INF
    m, l = part[:, :slots, 0].double(), part[:, :slots, 1].double()
    mx = m.max(1, keepdim=True).values
    want = (mx[:, 0] + torch.log2(torch.where(m > -INF, l * torch.exp2(m - mx), 0.0).sum(1))).to(DEV)
    part = part.to(DEV).view(rows, 2 * ld)
    lse = torch.full((rows,), NAN, device=DEV)
    svr2lib.call("svr2_rowstat_combine", svr2lib.ptr(part), slots, ld, svr2lib.ptr(lse), rows, svr2lib.stream())
    torch.cuda.synchronize()
    assert lse[rows - 1].item() == -INF, f"all -inf slots: lse = {lse[rows - 1].item()}"
    # |lse| < 48: fp32 ulp <= 3.8e-6, exp2f / log2f and the fp32 sum (<= 32 terms per lane, a 5-level tree) add < 8e-6:
    # 2e-5.  Every finite slot carries >= 2^-3 / (2 * slots) of its row's sum, so a dropped or extra slot moves lse by
    # > 1e-3 at 70 slots, > 8e-5 at 1014.
    err = (lse[:rows - 1].double() - want[:rows - 1]).abs()
    assert torch.isfinite(err).all() and err.max().item() <= 2e-5, f"lse: max abs err {err.max().item():.3e}"


# ====================================================================== c. the single-pass sequence
CQ, MQ = 256, 400                   # two query chunks: 256 + 144 rows


def attention(lib, q, k, vt, n, single):
    """The launches of vae._attention for one frame (q [MQ, D], k [n, D], vt = V^T [D, n]) in query chunks of CQ rows.
    single: the single-pass branch with its conditional two-pass fallback, wired to one device flag as in vae._attention;
    else the exact two-pass launches alone.  Returns the output and, per chunk, the flag as that chunk's
    svr2_pexp_stat_combine left it."""
    L = lib.load()
    slots = L.svr2_rowstat_slots(n)
    part = torch.empty(CQ, 2 * slots, device=DEV)
    lse = torch.empty(CQ, device=DEV)
    P = torch.empty(CQ, n, device=DEV, dtype=torch.bfloat16)
    o = torch.empty(MQ, D, device=DEV, dtype=torch.bfloat16)
    flags = []
    if single:
        slots_s, slots_p = L.svr2_rowstat_slots((n + 15) // 16), 2 * ((n + 255) // 256)
        part_s = torch.empty(CQ, 2 * slots_s, device=DEV)
        stat = torch.empty(CQ, 2 * slots_p, device=DEV)
        mhat = torch.empty(CQ, device=DEV)
        rscale = torch.empty(CQ, device=DEV)
        flag = torch.zeros(1, device=DEV, dtype=torch.int32)
    for r0 in range(0, MQ, CQ):
        rows = min(CQ, MQ - r0)
        qc, oc = q[r0:r0 + rows], o[r0:r0 + rows]
        run_if = None
        if single:
            lib.linear(qc, k[::16], epi=lib.EPI_ROWSTAT, out=part_s[:rows], out_scale=S2)
            lib.call("svr2_rowstat_max", lib.ptr(part_s), slots_s, slots_s, lib.ptr(mhat), rows, lib.ptr(flag), lib.stream())
            lib.linear(qc, k, epi=lib.EPI_PEXP, gate=mhat, out=P[:rows], out_scale=S2, stat_out=stat[:rows])
            lib.call("svr2_pexp_stat_combine", lib.ptr(stat), slots_p, slots_p, lib.ptr(mhat), lib.ptr(rscale), rows,
                     lib.ptr(flag), lib.stream())
            flags.append(flag.clone())
            lib.linear(P[:rows], vt, out=oc, rowscale=rscale)
            run_if = flag
        lib.linear(qc, k, epi=lib.EPI_ROWSTAT, out=part[:rows], out_scale=S2, run_if=run_if)
        lib.call("svr2_rowstat_combine", lib.ptr(part), slots, slots, lib.ptr(lse), rows, lib.stream())
        lib.linear(qc, k, epi=lib.EPI_PEXP, gate=lse, out=P[:rows], out_scale=S2, run_if=run_if)
        lib.linear(P[:rows], vt, out=oc, run_if=run_if)
    torch.cuda.synchronize()
    return o, [int(f.item()) for f in flags]


def softmax_v(q, k, v):
    S = (q.double() @ k.double().T) * D ** -0.5
    return torch.softmax(S, -1) @ v.double()


def qkv(n):
    """Random q (std 1.5: scores spread over ~+-7 powers of two), k, v; column 0 of q and k is zero so that one score
    can be set through it alone."""
    q, k, v = rnd(MQ, D, std=1.5, seed=n), rnd(n, D, seed=n + 1), rnd(n, D, seed=n + 2)
    q[:, 0] = 0
    k[:, 0] = 0
    return q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16)


def craft(q, k, m, j, x_target):
    """Copies of q, k in which key j scores ~x_target powers of two above row m's sampled reference exponent (the max
    over every 16th key); q[m, 0] * k[j, 0] is the only new product, so no other score changes."""
    q, k = q.clone(), k.clone()
    base = (q[m].double() @ k.double().T) * S2
    mhat = base[::16].max().item()
    a = 32.0
    b = torch.tensor((x_target + mhat - base[j].item()) / S2 / a).to(torch.bfloat16).item()
    q[m, 0], k[j, 0] = a, b
    return q, k, base[j].item() + a * b * S2 - mhat


def key_positions(n):
    """Unsampled keys (index % 16 != 0) at every column position modulo 64 (the epilogue's phase width, over which
    the MUFU / polynomial pattern of the column pairs repeats), spread over the four 64-column phases of one full
    256-column tile."""
    t = n // 256 - 1
    return [256 * t + 64 * (p % 4) + p for p in range(1, 64) if p % 16]


# Bound for benign rows: each probability is rounded to bf16 (<= 2^-8 relative), which moves sum_j p_j v_j by at most
# 2^-8 max|V|; the bf16 output adds <= 2^-8 max|V|; the fp32 accumulations are ~1e-6.  Any key carrying a few percent
# of a row's weight that went missing or was counted twice would exceed it.
def benign_bound(v):
    return 2.0 ** -7 * v.abs().max().item()


@pytest.mark.parametrize("n", [256, 264, 2040])
def test_single_pass_benign_rows(svr2lib, n):
    q, k, v = qkv(n)
    vt = v.T.contiguous()
    ref = softmax_v(q, k, v)
    o1, flags = attention(svr2lib, q, k, vt, n, True)
    o2, _ = attention(svr2lib, q, k, vt, n, False)
    assert flags == [0, 0], f"flag raised for benign rows: {flags}"
    for o, what in ((o1, "single-pass"), (o2, "two-pass")):
        err = (o.double() - ref).abs().max(1).values
        assert err.max().item() <= benign_bound(v), \
            f"{what}: max abs err {err.max().item():.4g} (row {int(err.argmax())}) > {benign_bound(v):.4g}"


@pytest.mark.parametrize("n", [256, 264, 2040])
def test_single_pass_key_far_above_reference_falls_back(svr2lib, n):
    """Row 77 gets one unsampled key ~150 powers of two above its sampled maximum, every other score stays benign.
    The key is tried at every column position (both the MUFU and the polynomial exp2 column pairs): the flag must go
    up and chunk 0 must be bit-equal to the exact two-pass launches; chunk 1 (benign) must keep its single-pass result,
    so the flag read after its pexp_stat_combine is 0 again."""
    q, k, v = qkv(n)
    vt = v.T.contiguous()
    o_benign, _ = attention(svr2lib, q, k, vt, n, True)
    no_flag, differs, chunk1 = [], [], []
    for j in key_positions(n):
        qc, kc, x = craft(q, k, 77, j, 150.0)
        assert 140 < x < 160, x
        o1, flags = attention(svr2lib, qc, kc, vt, n, True)
        o2, _ = attention(svr2lib, qc, kc, vt, n, False)
        if flags[0] != 1:
            no_flag.append(j % 64)
        elif not torch.equal(o1[:CQ], o2[:CQ]):
            differs.append(j % 64)
        if flags[1] != 0 or not torch.equal(o1[CQ:], o_benign[CQ:]):
            chunk1.append(j % 64)
    assert not no_flag, f"x ~ 150 did not raise the flag at key column positions (mod 64) {no_flag}"
    assert not differs, f"flagged chunk differs from the two-pass result at column positions {differs}"
    assert not chunk1, f"the benign chunk after a flagged one was not left single-pass at column positions {chunk1}"


@pytest.mark.parametrize("n", [264, 2040])
def test_single_pass_dominant_key_within_range(svr2lib, n):
    """A key ~90 powers of two above the sampled maximum (row sum ~2^90 < 1e30) needs no fallback: no flag, and the
    single-pass result meets the benign bound, at every column position."""
    q, k, v = qkv(n)
    vt = v.T.contiguous()
    ref = softmax_v(q, k, v)
    bad = []
    for j in key_positions(n):
        qc, kc, x = craft(q, k, 77, j, 90.0)
        assert 85 < x < 95, x
        o, flags = attention(svr2lib, qc, kc, vt, n, True)
        r = ref.clone()
        r[77] = softmax_v(qc[77:78], kc, v)[0]
        err = (o.double() - r).abs().max().item()
        if flags != [0, 0] or err > benign_bound(v):
            bad.append((j % 64, flags, round(err, 5)))
    assert not bad, f"(column position, flags, max abs err) with bound {benign_bound(v):.4g}: {bad}"


# ====================================================================== d. svr2_linear_ex_bf16 contract
def same_bits(a, b):
    it = torch.int16 if a.dtype == torch.bfloat16 else torch.int32
    return torch.equal(a.view(it), b.view(it))


def test_run_if_skips_or_runs_the_launch(svr2lib):
    """run_if -> 0: the output (and stat_out) keep their sentinel bit for bit; run_if -> 1: bit-equal to the launch
    without run_if.  The three launch kinds of the fallback (ROWSTAT, PEXP, plain P V) and PEXP with stat_out."""
    M, N, K = 300, 264, 128
    a, w = halves(M, K, seed=1), halves(N, K, seed=2)
    lse = torch.full((M,), 3.0, device=DEV)
    slots = svr2lib.load().svr2_rowstat_slots(N)
    kinds = (("rowstat", dict(epi=svr2lib.EPI_ROWSTAT, out_scale=0.25), (M, 2 * slots), torch.float32, False),
             ("pexp", dict(epi=svr2lib.EPI_PEXP, gate=lse, out_scale=0.25), (M, N), torch.bfloat16, False),
             ("pexp+stat", dict(epi=svr2lib.EPI_PEXP, gate=lse, out_scale=0.25), (M, N), torch.bfloat16, True),
             ("plain", dict(), (M, N), torch.bfloat16, False))
    for name, kw, shape, dt, with_stat in kinds:
        outs = []
        for flag in (None, _flag(0), _flag(1)):
            out = torch.full(shape, -5.0, device=DEV, dtype=dt)
            stat = torch.full((M, 2 * 2 * ((N + 255) // 256)), -5.0, device=DEV) if with_stat else None
            svr2lib.linear(a, w, out=out, stat_out=stat, run_if=flag, **kw)
            torch.cuda.synchronize()
            outs.append((out, stat))
        (o_ref, s_ref), (o0, s0), (o1, s1) = outs
        assert (o0 == -5.0).all() and (s0 is None or (s0 == -5.0).all()), f"{name}: run_if -> 0 wrote the output"
        assert not (o_ref == -5.0).all(), f"{name}: the reference launch wrote nothing"
        assert same_bits(o1, o_ref), f"{name}: run_if -> 1 differs from the launch without run_if"
        if with_stat:
            assert same_bits(s1, s_ref), f"{name}: stat_out differs under run_if -> 1"


# M = 300 gives 3 m-tiles, few enough that N = 120, 136 and 264 run 128-column tiles; M = 4300, N = 520 keeps the
# 256-column tiles (34 x 3 tiles fill the SMs).  Every M is ragged and every N ends in a partial tile.
@pytest.mark.parametrize("M,N,with_bias", [(300, 120, True), (300, 136, False), (300, 264, True), (4300, 520, True),
                                           (4300, 520, False)])
def test_rowscale_epilogue(svr2lib, M, N, with_bias):
    """EPI_ROWSCALE: out = bf16(acc * rowscale[m] (+ bias)) elementwise against fp64.  Operands in halves, rowscale in
    {0, 1/16, ..., 4} (0 is what the combine writes for a flagged row) and bias in eighths keep every intermediate exact
    in fp32, so kernel and reference round the same number: the comparison is bit for bit."""
    K = 256
    a, w = halves(M, K, seed=3), halves(N, K, seed=4)
    g = torch.Generator(device="cpu").manual_seed(M + N)
    rs = (torch.randint(0, 65, (M,), generator=g).float() / 16).to(DEV)
    bias = (torch.randint(-32, 33, (N,), generator=g).float() / 8).to(DEV).to(torch.bfloat16) if with_bias else None
    out = torch.full((M, N + 8), -5.0, device=DEV, dtype=torch.bfloat16)
    svr2lib.linear(a, w, bias=bias, out=out[:, :N], rowscale=rs)
    torch.cuda.synchronize()
    t = (a.double() @ w.double().T) * rs.double()[:, None]
    if with_bias:
        t = t + bias.double()[None, :]
    ref = t.to(torch.bfloat16)
    assert (out[:, N:] == -5.0).all(), "columns past N were written"
    diff = out[:, :N] != ref
    assert not diff.any(), f"{int(diff.sum())} elements differ: " + samples(diff, t, out[:, :N].float())


# N = 24 / 40 / 100 / 264 select 32 / 64 / 128 / 256-column tiles, each with a ragged last tile; out_scale < 0 takes the
# general branch (no scale folded into the exponent's FMA).  Scores spread over ~+-2 powers of two.
@pytest.mark.parametrize("N,out_scale", [(24, 0.1), (40, 0.1), (100, 0.1), (264, 0.1), (264, -0.1)])
def test_rowstat_lse(svr2lib, N, out_scale):
    M, K = 300, 128
    a, w = halves(M, K, seed=5), halves(N, K, seed=6)
    slots = svr2lib.load().svr2_rowstat_slots(N)
    part = torch.full((M, 2 * (slots + 1)), NAN, device=DEV)           # one guard slot per row
    svr2lib.linear(a, w, epi=svr2lib.EPI_ROWSTAT, out=part, out_scale=out_scale)
    lse = torch.full((M,), NAN, device=DEV)
    svr2lib.call("svr2_rowstat_combine", svr2lib.ptr(part), slots, slots + 1, svr2lib.ptr(lse), M, svr2lib.stream())
    torch.cuda.synchronize()
    assert torch.isnan(part.view(M, slots + 1, 2)[:, slots]).all(), "ROWSTAT wrote past svr2_rowstat_slots(N)"
    s = (a.double() @ w.double().T) * out_scale                        # exact accumulator, times the fp32 scale
    want = torch.logsumexp(s / LOG2E, 1) * LOG2E
    # ex2.approx (< 2^-22 relative), fp32 partial sums (<= 128 terms: < 8e-6), exp2f / log2f of the combine and the
    # fp32 ulp of |lse| < 16: 2e-5.  The smallest column of every row moves lse by more (checked), so no dropped,
    # doubled or padded column (a padded one would add 2^0) can hide under it.
    smallest = torch.log2(1 + torch.exp2(s.min(1).values - want)).min().item()
    assert smallest > 10 * 2e-5, smallest
    err = (lse.double() - want).abs()
    assert torch.isfinite(err).all() and err.max().item() <= 2e-5, \
        f"lse: max abs err {err.max().item():.3e} (row {int(err.argmax())})"


def test_linear_ex_refusals(svr2lib):
    """The documented refusals return non-zero with a message, before any launch (the output keeps its sentinel)."""
    L = svr2lib.load()
    K = 64
    a = halves(256, K, seed=7)

    def refused(N, epi, rowscale=None, stat=None, ld_stat=0, gate=None):
        w = halves(N, K, seed=8)
        out = torch.full((256, N), -5.0, device=DEV, dtype=torch.bfloat16)
        rc = L.svr2_linear_ex_bf16(svr2lib.ptr(a), K, svr2lib.ptr(w), K, 256, N, K, epi, None, svr2lib.ptr(gate), None,
                                   svr2lib.ptr(out), N, 1.0, svr2lib.ptr(rowscale), svr2lib.ptr(stat), ld_stat, None,
                                   svr2lib.stream())
        torch.cuda.synchronize()
        msg = L.svr2_last_error().decode()
        if rc != 0:
            assert (out == -5.0).all(), "a refused launch wrote the output"
        return rc != 0, msg

    rs = torch.ones(256, device=DEV)
    gate = torch.zeros(256, device=DEV)
    stat = torch.zeros(256, 2 * 8, device=DEV)
    for N in (16, 32, 64):                              # tiles narrower than 128 columns
        r, msg = refused(N, svr2lib.EPI_ROWSCALE, rowscale=rs)
        assert r and "ROWSCALE" in msg, (N, msg)
    r, msg = refused(128, svr2lib.EPI_ROWSCALE)         # no rowscale vector
    assert r and "ROWSCALE" in msg, msg
    for N in (8, 64, 128, 248):                         # stat_out needs 256-column tiles
        r, msg = refused(N, svr2lib.EPI_PEXP, stat=stat, ld_stat=8, gate=gate)
        assert r and "stat_out" in msg, (N, msg)
    r, msg = refused(520, svr2lib.EPI_PEXP, stat=stat, ld_stat=5, gate=gate)     # 3 n-tiles need 6 slots
    assert r and "ld_stat" in msg, msg
    r, msg = refused(520, svr2lib.EPI_PEXP, stat=stat, ld_stat=6, gate=gate)
    assert not r, msg
