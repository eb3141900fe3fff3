"""CPU: the native host runtime's geometry (csrc/engine.cu: window layouts and RoPE cos / sin tables, what
svr2_dit_forward builds per clip shape and svr2_dit_geometry returns) against the oracle's restatement of the reference
(oracle/dit_oracle.py: window boxes, window_token_index, rope_cos_sin_3b / _7b).  engine.cu is compiled with
SVR2_HOST_TEST (tables kept in host memory) by nvcc's host compiler; skipped where nvcc is missing."""
import math
import subprocess

import pytest
import torch

import native_trace
from oracle import dit_oracle

pytestmark = native_trace.needs_nvcc

# (regular, shifted) window counts of the SURVEY geometries (latent T, H/2, W/2)
SURVEY_WINDOWS = {(1, 32, 32): (4, 9), (5, 68, 120): (75, 90), (3, 135, 240): (243, 300), (17, 135, 240): (324, 400),
                  (2, 135, 240): (162, 200)}


@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    return native_trace.harness(tmp_path_factory, "geometry_dump", link_svr2=False)


def rope_freqs(variant, dtype):
    if variant == "3b":
        return (1.0 / (10000 ** (torch.arange(0, 42, 2)[:21].float() / 42))).to(dtype)
    return (torch.linspace(1.0, 128.0, 10) * math.pi).to(dtype)


def _assert_table(tab, rows, want, dtype, what):
    """tab [R, nf]: a table of the runtime; rows [N, k]: table rows; want [N, k, nf]: the oracle's values there."""
    nf = tab.shape[1]
    diff = (tab[rows] - want).abs()
    # cos / sin come from libm in engine.cu and from torch's vectorised kernels in the oracle: identical except where a
    # value sits within an fp32 ulp of a rounding tie of the table dtype (e.g. sin(300.0) in fp16) — at most a handful of
    # table entries (fp32 tables: the two libraries differ by an fp32 ulp in a few per cent of the entries)
    if dtype == torch.float32:
        assert diff.max().item() <= 2.4e-7, (what, diff.max().item())
    else:
        n, a, f = (diff > 0).nonzero().unbind(1)
        entries = (rows[n, a] * nf + f).unique()
        assert entries.numel() <= max(2, tab.numel() // 2000) and diff.max().item() <= 2 ** -9, (what, entries.numel())


def check_against_oracle(got, variant, T, Hp, Wp, l, shifted, freqs):
    """got: one layout and its cos / sin table as host tensors, named as in svr2_dit_geometry_desc.  Asserts that they
    are what the oracle derives from the reference's window boxes, every index exactly."""
    L = T * Hp * Wp
    boxes = dit_oracle.window_boxes(T, Hp, Wp, shifted)
    tgt, lens, loc = dit_oracle.window_token_index(T, Hp, Wp, boxes)
    n_win, tj = len(boxes), torch.arange(l)
    src, omap, o = [], [], 0
    for w, n in enumerate(lens.tolist()):           # each window's video tokens, then the l text tokens
        src += [tgt[o:o + n], -(tj + 1)]
        omap += [tgt[o:o + n], L + w * l + tj]
        o += n
    src, omap = torch.cat(src), torch.cat(omap)
    total = L + n_win * l
    assert [got["n_win"], got["total"], got["max_len"], got["n_txt_rows"]] == [n_win, total, int(lens.max()) + l, n_win * l]
    cu = got["cu_seqlens"].long()
    assert cu[0].item() == 0 and cu[-1].item() == total
    assert torch.equal(cu.diff(), lens + l)
    row_src = got["row_src"].long()
    vid = row_src >= 0
    # the window order and contents of the oracle's boxes, every token covered exactly once
    assert torch.equal(row_src, src)
    assert torch.equal(row_src[vid].sort().values, torch.arange(L))
    out_row_map = got["out_row_map"].long()
    assert torch.equal(out_row_map, omap) and torch.equal(out_row_map.sort().values, torch.arange(total))
    assert torch.equal(out_row_map[vid], row_src[vid])
    assert torch.equal(got["txt_rows"].long(), torch.nonzero(~vid).flatten())
    tok_dst = got["tok_dst"].long()
    assert torch.equal(row_src[tok_dst], torch.arange(L))
    rr = got["row_rope"].long().view(total, 3)
    assert torch.equal(got["tok_rope"].long().view(L, 3), rr[tok_dst])

    cos, sin = got["rope_cos"], got["rope_sin"]
    nf = freqs.numel()
    assert cos.shape == sin.shape == (got["rope_rows"], nf) and got["nfreq"] == nf
    assert torch.equal(rr[rr >= 0].unique(), torch.arange(cos.shape[0]))      # the table holds the rows used, no more
    if variant == "3b":
        assert torch.equal(rr[vid], loc[:, :3] + torch.tensor([l, 0, 0]))     # video (t + l, h, w), window-local
        assert torch.equal(rr[~vid], tj.repeat(n_win)[:, None].expand(-1, 3))  # text (j, j, j)
        (cv, sv), (ct, st) = dit_oracle.rope_cos_sin_3b(freqs, loc, l)
        for tab, want in ((cos, ct), (sin, st)):
            _assert_table(tab, rr[~vid][:l], want.view(l, 3, nf, 2)[..., 0], freqs.dtype, "text")
    else:
        assert (rr[~vid] == -1).all()
        for a in range(3):      # an axis of n tokens reads the n consecutive rows of the table kept for that size
            off, n = rr[vid, a] - loc[:, a], loc[:, 3 + a]
            for size in n.unique():
                assert (off[n == size] == off[n == size][0]).all()
        cv, sv = dit_oracle.rope_cos_sin_7b(freqs, loc)
    for tab, want in ((cos, cv), (sin, sv)):
        _assert_table(tab, rr[vid], want.view(L, 3, nf, 2)[..., 0], freqs.dtype, "video")


@pytest.mark.parametrize("variant,geom,dtype", [
    ("3b", (1, 32, 32), torch.float16), ("3b", (5, 68, 120), torch.float16), ("3b", (3, 135, 240), torch.float16),
    ("3b", (17, 135, 240), torch.float16), ("3b", (3, 20, 36), torch.bfloat16), ("3b", (2, 17, 23), torch.float32),
    ("7b", (2, 135, 240), torch.float16), ("7b", (3, 20, 36), torch.float16), ("7b", (5, 33, 47), torch.float16),
    # rounding the window size down instead of to nearest changes these windows; fp32 tables keep the linspace's last bit
    ("3b", (2, 8, 61), torch.float16), ("7b", (3, 20, 36), torch.float32),
])
def test_native_geometry_matches_oracle(dumper, variant, geom, dtype):
    T, Hp, Wp = geom
    l = 58
    fr = rope_freqs(variant, dtype)
    dt = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[dtype]
    out = subprocess.run([dumper, str(T), str(Hp), str(Wp), str(l), str(int(variant == "7b")), str(dt), str(fr.numel())]
                         + [repr(float(x)) for x in fr], capture_output=True, text=True, check=True).stdout.split("\n")
    it = iter(out)
    for s, shifted in ((0, False), (1, True)):
        hdr = next(it).split()
        assert hdr[:2] == ["layout", str(s)]
        got = dict(zip(("n_win", "total", "max_len", "n_txt_rows"), (int(x) for x in hdr[2:])))
        if geom in SURVEY_WINDOWS:
            assert got["n_win"] == SURVEY_WINDOWS[geom][s]
        for name in ("cu_seqlens", "row_src", "row_rope", "out_row_map", "tok_dst", "tok_rope", "txt_rows"):
            line = next(it).split()
            assert line[0] == name
            got[name] = torch.tensor([int(x) for x in line[1:]], dtype=torch.int32)
        got["rope_rows"], got["nfreq"] = int(next(it).split()[1]), fr.numel()
        tab = torch.tensor([[float(x) for x in next(it).split()] for _ in range(got["rope_rows"] * fr.numel())])
        got["rope_cos"], got["rope_sin"] = tab[:, 0].view(-1, fr.numel()), tab[:, 1].view(-1, fr.numel())
        check_against_oracle(got, variant, T, Hp, Wp, l, shifted, fr)
