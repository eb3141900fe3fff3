"""-m gpu: the bf16 GEMM / conv launches whose epilogue runs on the dedicated epilogue warps (the MMA warpgroups hand
over a bf16(acc + bias) tile and go on with the next tile) against a torch fp32 restatement: many tiles per CTA, fewer
tiles than SMs, ragged edges, residual + halo + GroupNorm statistics, the fused shortcut, the upsample with its dropped
head frame, and a replay inside a CUDA graph."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rnd(*shape, std=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * std).to(DEV)


def bf(x):
    return x.to(torch.bfloat16)


def assert_close(a, b, tol, what):
    a, b = a.float(), b.float()
    e = ((a - b).norm() / b.norm().clamp_min(1e-12)).item()
    assert math.isfinite(e) and e < tol, f"{what}: rel err {e:.3e} >= {tol}"


def _to_ndhwc(x_ncdhw, halo):
    x = x_ncdhw[0].permute(1, 2, 3, 0)
    if halo:
        x = torch.cat([x[:1]] * halo + [x], 0)
    return bf(x).contiguous()


def _conv_stats_call(lib, x_nd, T_in, H, W, Cin, w_k, Cout, T, bias, res, y, part, slots):
    args = (lib.ptr(x_nd), T_in, H, W, Cin, lib.ptr(w_k), Cout, 3, 3, 3, 1, 1, 1, T, lib.EPI_BIAS | lib.EPI_RESIDUAL,
            lib.ptr(bias), lib.ptr(res), lib.ptr(y), 2, 1, Cout)
    if part is None:
        assert lib.load().svr2_conv3d_stats_bf16(*args, None, 0, ctypes.byref(slots), lib.stream()) == 0
    else:
        lib.call("svr2_conv3d_stats_bf16", *args, lib.ptr(part), part.numel() * 4, ctypes.byref(slots), lib.stream())


# Cout 128: swap-AB tiles (128 channels x 256 pixels); Cout 256: 128 pixels x 256 channels.  The first shapes of each
# have more tiles than SMs (several tiles per CTA), the last ones fewer; H / W are not tile multiples.
@pytest.mark.parametrize("Cin,Cout,T,H,W", [(128, 128, 3, 70, 150), (64, 256, 2, 45, 139), (128, 128, 1, 9, 21),
                                            (128, 256, 1, 11, 13)])
def test_conv_residual_halo_stats(svr2lib, Cin, Cout, T, H, W):
    x = rnd(1, Cin, T, H, W, seed=1)
    w = rnd(Cout, Cin, 3, 3, 3, std=(27 * Cin) ** -0.5, seed=2)
    b, res = bf(rnd(Cout, seed=3)), bf(rnd(T, H, W, Cout, seed=4))
    xp = torch.cat([bf(x).float()[:, :, :1]] * 2 + [bf(x).float()], 2)
    ref = F.conv3d(xp, bf(w).float(), b.float(), padding=(0, 1, 1))[0].permute(1, 2, 3, 0)
    ref = bf(bf(ref).float() + res.float())
    x_nd = _to_ndhwc(x, 2)
    w_k = bf(w.permute(0, 2, 3, 4, 1).reshape(Cout, -1)).contiguous()
    res_h = torch.cat([res[:1], res[:1], res], 0).contiguous()
    y = torch.zeros(2 + T, H, W, Cout, device=DEV, dtype=torch.bfloat16)
    slots = ctypes.c_int(0)
    _conv_stats_call(svr2lib, x_nd, T + 2, H, W, Cin, w_k, Cout, T, b, res_h, y, None, slots)
    part = torch.full((T * slots.value * (Cout // 8) * 4,), float("nan"), device=DEV)
    _conv_stats_call(svr2lib, x_nd, T + 2, H, W, Cin, w_k, Cout, T, b, res_h, y, part, slots)
    torch.cuda.synchronize()
    assert_close(y[2:], ref, 4e-3, "conv + bias + residual")
    assert torch.equal(y[0], y[2]) and torch.equal(y[1], y[2]), "halo frames must replicate frame 0"
    assert torch.isfinite(part).all(), "every partial slot must be written"
    p4 = part.view(T, slots.value, Cout // 8, 4)
    yf = y[2:].float().view(T, -1, Cout // 8, 2, 4)          # channel octet halves: (x, y) and (z, w) partial sums
    assert_close(p4[..., [0, 2]].sum(1), yf.sum((1, 4)), 1e-4, "statistics (sum)")
    assert_close(p4[..., [1, 3]].sum(1), (yf * yf).sum((1, 4)), 1e-4, "statistics (sum of squares)")


@pytest.mark.parametrize("Cin,C2,Cout,T,H,W", [(128, 256, 128, 2, 66, 120), (256, 512, 256, 2, 37, 61)])
def test_conv_fused_shortcut_many_tiles(svr2lib, Cin, C2, Cout, T, H, W):
    h, x2 = rnd(1, Cin, T, H, W, seed=1), rnd(1, C2, T, H, W, seed=2)
    w = rnd(Cout, Cin, 3, 3, 3, std=(27 * Cin) ** -0.5, seed=3)
    wsc = rnd(Cout, C2, 1, 1, 1, std=C2 ** -0.5, seed=4)
    bsum = bf(rnd(Cout, seed=5))
    hp = torch.cat([bf(h).float()[:, :, :1]] * 2 + [bf(h).float()], 2)
    ref = F.conv3d(hp, bf(w).float(), bsum.float(), padding=(0, 1, 1)) + F.conv3d(bf(x2).float(), bf(wsc).float())
    h_nd, x_nd = _to_ndhwc(h, 2), _to_ndhwc(x2, 0)
    w_cat = torch.cat([bf(w.permute(0, 2, 3, 4, 1).reshape(Cout, -1)), bf(wsc.reshape(Cout, C2))], 1).contiguous()
    y = torch.zeros(2 + T, H, W, Cout, device=DEV, dtype=torch.bfloat16)
    args = (svr2lib.ptr(h_nd), T + 2, H, W, Cin, svr2lib.ptr(w_cat), Cout, 3, 3, 3, T, svr2lib.ptr(bsum),
            svr2lib.ptr(x_nd), C2, svr2lib.ptr(y), 2, 1)
    slots = ctypes.c_int(0)
    assert svr2lib.load().svr2_conv3d_shortcut_stats_bf16(*args, None, 0, ctypes.byref(slots), svr2lib.stream()) == 0
    part = torch.zeros(T * slots.value * (Cout // 8) * 4, device=DEV)
    svr2lib.call("svr2_conv3d_shortcut_stats_bf16", *args, svr2lib.ptr(part), part.numel() * 4, ctypes.byref(slots),
                 svr2lib.stream())
    torch.cuda.synchronize()
    assert_close(y[2:], ref[0].permute(1, 2, 3, 0), 4e-3, "conv + fused shortcut")
    assert torch.equal(y[0], y[2]) and torch.equal(y[1], y[2])
    sums = part.view(T, slots.value, Cout // 8, 4)[..., [0, 2]].sum((1, 2, 3))
    assert_close(sums, y[2:].float().sum((1, 2, 3)), 2e-3, "statistics (sum)")


@pytest.mark.parametrize("C,F_,H,W", [(256, 3, 40, 64), (512, 2, 9, 14)])
def test_upsample_drop_head(svr2lib, C, F_, H, W):
    r = 8
    x = rnd(1, C, F_, H, W, seed=1)
    w, b = rnd(r * C, C, std=C ** -0.5, seed=2), rnd(r * C, seed=3)
    y = F.conv3d(bf(x).float(), bf(w).float().view(r * C, C, 1, 1, 1), bf(b).float())
    y = y.view(1, 2, 2, 2, C, F_, H, W).permute(0, 4, 5, 3, 6, 1, 7, 2).reshape(1, C, F_ * 2, 2 * H, 2 * W)
    y = torch.cat([y[:, :, :1], y[:, :, 2:]], 2)
    out = torch.zeros(2 + y.shape[2], 2 * H, 2 * W, C, device=DEV, dtype=torch.bfloat16)
    x_nd, w16, b16 = _to_ndhwc(x, 0), bf(w).contiguous(), bf(b)
    svr2lib.call("svr2_upsample_shuffle_bf16", svr2lib.ptr(x_nd), F_, H, W, C, svr2lib.ptr(w16), svr2lib.ptr(b16), 1, 1,
                 svr2lib.ptr(out), 2, 1, svr2lib.stream())
    torch.cuda.synchronize()
    assert_close(out[2:], y[0].permute(1, 2, 3, 0), 4e-3, "upsample shuffle, dropped head frame")
    assert torch.equal(out[0], out[2]) and torch.equal(out[1], out[2])


# N = 2560: 256-column tiles, many per CTA; N = 200: 64 + ragged-column tiles; M = 40: narrow tiles, few CTAs
@pytest.mark.parametrize("M,N,K", [(3000, 2560, 320), (1500, 200, 256), (40, 72, 128)])
def test_linear_epilogues_many_tiles(svr2lib, M, N, K):
    a, w = bf(rnd(M, K, seed=1)), bf(rnd(N, K, std=K ** -0.5, seed=2))
    bias, gate, res = bf(rnd(N, seed=3)), rnd(N, seed=4), bf(rnd(M, N, seed=5))
    t0 = bf(a.float() @ w.float().T + bias.float()).float()
    out = svr2lib.linear(a, w, bias=bias, gate=gate, residual=res)
    assert_close(out, bf(bf(t0 * gate).float() + res.float()), 3e-3, "bias + gate + residual")
    out = svr2lib.linear(a, w, bias=bias, epi=svr2lib.EPI_GELU)
    assert_close(out, F.gelu(t0, approximate="tanh"), 4e-3, "gelu")
    out = svr2lib.linear(a, w, bias=bias, epi=svr2lib.EPI_SILU)
    assert_close(out, F.silu(t0), 4e-3, "silu")
    out = svr2lib.linear(a, w)
    assert_close(out, a.float() @ w.float().T, 4e-3, "plain")


def test_conv_graph_replay(svr2lib):
    """One conv launch captured in a CUDA graph and replayed gives the eager result bit for bit."""
    Cin, Cout, T, H, W = 128, 128, 2, 40, 72
    x_nd = _to_ndhwc(rnd(1, Cin, T, H, W, seed=1), 2)
    w_k = bf(rnd(Cout, 27 * Cin, std=(27 * Cin) ** -0.5, seed=2)).contiguous()
    b = bf(rnd(Cout, seed=3))
    eager = torch.zeros(T, H, W, Cout, device=DEV, dtype=torch.bfloat16)
    svr2lib.conv3d(x_nd, T + 2, H, W, Cin, w_k, Cout, (3, 3, 3), 1, 1, 1, T, eager, bias=b)
    torch.cuda.synchronize()
    y = torch.zeros_like(eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            svr2lib.conv3d(x_nd, T + 2, H, W, Cin, w_k, Cout, (3, 3, 3), 1, 1, 1, T, y, bias=b)
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, eager)
