"""-m gpu: every C-ABI op of libsvr2.so against a plain torch fp32 restatement of the same
reference op (floating point kernels; tolerances are stated per test)."""
import contextlib
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


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def assert_close(a, b, tol, what=""):
    e = rel_err(a, b)
    assert math.isfinite(e) and e < tol, f"{what}: rel err {e:.3e} >= {tol}"


# ------------------------------------------------------------------ linear
@pytest.mark.parametrize("M,N,K", [(300, 256, 192), (1000, 768, 256), (77, 64, 2560), (513, 384, 320),
                                   (2048, 7680, 2560), (129, 16, 128), (4, 2560, 256), (1, 1536, 256)])
def test_linear_plain(svr2lib, M, N, K):
    a, w = bf(rnd(M, K, seed=1)), bf(rnd(N, K, std=K ** -0.5, seed=2))
    out = svr2lib.linear(a, w)
    ref = a.float() @ w.float().T
    assert_close(out, ref, 4e-3, f"linear {M}x{N}x{K}")


def test_linear_epilogues(svr2lib):
    M, N, K = 777, 512, 448
    a, w = bf(rnd(M, K, seed=1)), bf(rnd(N, K, std=K ** -0.5, seed=2))
    bias, gate = bf(rnd(N, seed=3)), rnd(N, seed=4).float()
    res = bf(rnd(M, N, seed=5))
    acc = a.float() @ w.float().T
    # bias + gate + residual with the reference's rounding points
    out = svr2lib.linear(a, w, bias=bias, gate=gate, residual=res)
    t = bf(acc + bias.float()).float()
    t = bf(t * gate).float()
    ref = bf(t + res.float())
    assert_close(out, ref, 3e-3, "bias+gate+residual")
    out = svr2lib.linear(a, w, bias=bias, epi=svr2lib.EPI_GELU)
    assert_close(out, F.gelu(bf(acc + bias.float()).float(), approximate="tanh"), 4e-3, "gelu")
    out = svr2lib.linear(a, w, bias=bias, epi=svr2lib.EPI_SILU)
    assert_close(out, F.silu(bf(acc + bias.float()).float()), 4e-3, "silu")
    out = svr2lib.linear(a, w, epi=svr2lib.EPI_F32, out_scale=0.25)
    assert out.dtype == torch.float32
    assert_close(out, acc * 0.25, 1e-5, "f32")
    # SwiGLU: tile j of 256 weight rows = [128 gate rows ; 128 in rows]
    g, u = acc[:, :256], acc[:, 256:]
    wg, wu = w[:256], w[256:]
    w_il = torch.cat([wg[:128], wu[:128], wg[128:], wu[128:]], 0).contiguous()
    out = svr2lib.linear(a, w_il, epi=svr2lib.EPI_SWIGLU)
    ref = bf(F.silu(bf(g).float())).float() * bf(u).float()
    assert out.shape == (M, 256)
    assert_close(out, ref, 4e-3, "swiglu")


def test_linear_strided_and_big_k(svr2lib):
    M, N, K = 640, 256, 6912
    a_full = bf(rnd(M, K + 64, seed=7))
    a = a_full[:, :K]
    w = bf(rnd(N, K, std=K ** -0.5, seed=8))
    out = svr2lib.linear(a, w)
    assert_close(out, a.float() @ w.float().T, 4e-3, "strided A")


# ------------------------------------------------------------------ conv3d
def _to_ndhwc(x_ncdhw, halo):
    x = x_ncdhw[0].permute(1, 2, 3, 0)  # T,H,W,C
    if halo:
        x = torch.cat([x[:1]] * halo + [x], 0)
    return bf(x).contiguous()


@pytest.mark.parametrize("Cin,Cout,k,st,shw,T,H,W", [
    (64, 128, (3, 3, 3), 1, 1, 3, 20, 36),
    (128, 256, (1, 1, 1), 1, 1, 2, 10, 12),
    (128, 128, (1, 3, 3), 1, 2, 3, 16, 24),
    (128, 128, (3, 3, 3), 2, 2, 5, 16, 24),
    (512, 512, (3, 3, 3), 1, 1, 2, 6, 10),
    (128, 8, (3, 3, 3), 1, 1, 2, 12, 20),
    (256, 32, (3, 3, 3), 1, 1, 1, 4, 6),
    (128, 128, (3, 3, 3), 2, 2, 5, 48, 64),      # swap-AB + pair view
    (128, 128, (1, 3, 3), 1, 2, 2, 40, 72),      # swap-AB, spatial-only downsample
    (256, 128, (3, 3, 3), 1, 1, 2, 30, 44),      # swap-AB, ragged tile edges
    (128, 128, (1, 1, 1), 1, 1, 2, 24, 40),      # swap-AB 1x1x1
    (128, 128, (3, 3, 3), 1, 1, 3, 9, 256),      # swap-AB, wide rows
    (256, 128, (3, 3, 3), 1, 1, 2, 5, 520),      # swap-AB, wide rows, ragged last tile column
    (128, 96, (1, 3, 3), 1, 1, 2, 6, 512),       # swap-AB, kt = 1, Cout < 128
    (128, 128, (1, 3, 3), 1, 2, 2, 8, 1024),     # swap-AB, stride 2, wide rows
    (256, 256, (3, 3, 3), 1, 1, 2, 6, 256),      # 256-column tiles, wide rows
    (256, 512, (3, 3, 3), 1, 1, 1, 3, 128),      # two n-tiles, 128 x 1 pixel tiles (H_out < 8)
    (512, 256, (1, 3, 3), 1, 1, 2, 5, 200),      # kt = 1, 128 x 1 pixel tiles, ragged second tile
    (256, 256, (3, 3, 3), 2, 2, 3, 8, 512),      # 128 x 1 pixel tiles, stride 2
])
def test_conv3d(svr2lib, Cin, Cout, k, st, shw, T, H, W):
    x = rnd(1, Cin, T, H, W, seed=1)
    w = rnd(Cout, Cin, *k, std=(Cin * k[0] * k[1] * k[2]) ** -0.5, seed=2)
    b = rnd(Cout, seed=3)
    halo = k[0] - 1
    xb, wb, bb = bf(x).float(), bf(w).float(), bf(b).float()
    xp = torch.cat([xb[:, :, :1]] * halo + [xb], 2) if halo else xb
    if shw == 2:
        ref = F.conv3d(F.pad(xp, (0, 1, 0, 1)), wb, bb, stride=(st, 2, 2))
    else:
        ref = F.conv3d(xp, wb, bb, stride=(st, 1, 1), padding=(0, k[1] // 2, k[2] // 2))
    T_out, Ho, Wo = ref.shape[2:]
    x_nd = _to_ndhwc(x, halo)
    w_k = bf(w.permute(0, 2, 3, 4, 1).reshape(Cout, -1)).contiguous()
    res = bf(rnd(T_out, Ho, Wo, Cout, seed=4))
    y = torch.zeros(2 + T_out, Ho, Wo, Cout, device=DEV, dtype=torch.bfloat16)
    svr2lib.conv3d(x_nd, T + halo, H, W, Cin, w_k, Cout, k, st, shw, 1 if (shw == 1 and k[1] == 3) else 0, T_out, y,
                   bias=bf(b), residual=torch.cat([res[:1], res[:1], res], 0).contiguous(), out_t_pad=2,
                   out_dup_head=1)
    ref_nd = bf(bf(ref[0].permute(1, 2, 3, 0)).float() + res.float())
    assert_close(y[2:], ref_nd, 4e-3, "conv3d body")
    assert torch.equal(y[0], y[2]) and torch.equal(y[1], y[2]), "halo frames must replicate frame 0"


@pytest.mark.parametrize("Cin,C2,Cout,T,H,W", [
    (128, 256, 128, 2, 30, 44),     # decoder up3.res0: swap-AB, ragged tile edges
    (256, 512, 256, 3, 24, 40),     # decoder up2.res0: 256-column tiles
    (256, 128, 256, 2, 17, 33),     # encoder down1.res0 (odd sizes)
    (512, 256, 512, 1, 9, 16),      # encoder down2.res0, single frame
    (128, 256, 128, 2, 7, 512),     # swap-AB, wide rows, with the shortcut's extra k-blocks
    (256, 512, 256, 2, 5, 256),     # 256-column tiles, wide rows, with the shortcut's extra k-blocks
])
def test_conv3d_fused_shortcut(svr2lib, Cin, C2, Cout, T, H, W):
    """conv2(h) + conv_shortcut(x) as one contraction over [h ; x] (ResnetBlock3D, attn_video_vae.py:311-362) vs torch:
    fp32 reference of the two convolutions on bf16-rounded operands; statistics slots returned."""
    import ctypes
    h = rnd(1, Cin, T, H, W, seed=1)
    x2 = rnd(1, C2, T, H, W, seed=2)
    w = rnd(Cout, Cin, 3, 3, 3, std=(27 * Cin) ** -0.5, seed=3)
    wsc = rnd(Cout, C2, 1, 1, 1, std=C2 ** -0.5, seed=4)
    b, bsc = rnd(Cout, seed=5), rnd(Cout, seed=6)
    hb, xb = bf(h).float(), bf(x2).float()
    hp = torch.cat([hb[:, :, :1]] * 2 + [hb], 2)
    ref = F.conv3d(hp, bf(w).float(), None, padding=(0, 1, 1)) + F.conv3d(xb, bf(wsc).float(), None)
    bsum = bf(bf(b).float() + bf(bsc).float())
    ref = ref + bsum.float().view(1, -1, 1, 1, 1)
    h_nd, x_nd = _to_ndhwc(h, 2), _to_ndhwc(x2, 0)
    w_cat = torch.cat([bf(w.permute(0, 2, 3, 4, 1).reshape(Cout, -1)), bf(wsc.reshape(Cout, C2))], 1).contiguous()
    y = torch.zeros(2 + T, H, W, Cout, device=DEV, dtype=torch.bfloat16)
    args = (svr2lib.ptr(h_nd), T + 2, H, W, Cin, svr2lib.ptr(w_cat), Cout, 3, 3, 3, T, svr2lib.ptr(bsum),
            svr2lib.ptr(x_nd), C2, svr2lib.ptr(y), 2, 1)
    slots = ctypes.c_int(0)
    assert svr2lib.load().svr2_conv3d_shortcut_stats_bf16(*args, None, 0, ctypes.byref(slots), svr2lib.stream()) == 0
    part = torch.zeros(T * slots.value * (Cout // 8) * 4, device=DEV, dtype=torch.float32)
    svr2lib.call("svr2_conv3d_shortcut_stats_bf16", *args, svr2lib.ptr(part), part.numel() * 4, ctypes.byref(slots),
                 svr2lib.stream())
    assert_close(y[2:], ref[0].permute(1, 2, 3, 0), 4e-3, "conv + fused shortcut")
    assert torch.equal(y[0], y[2]) and torch.equal(y[1], y[2])
    # the statistics the epilogue emitted: per-frame sums of the stored values
    sums = part.view(T, slots.value, Cout // 8, 4)[..., [0, 2]].sum((1, 2, 3))
    assert_close(sums, y[2:].float().sum((1, 2, 3)), 2e-3, "epilogue statistics (sum)")


@pytest.mark.parametrize("C,temporal,F_,H,W", [(256, 0, 3, 6, 10), (512, 1, 3, 4, 6), (512, 1, 1, 4, 6),
                                                # W % 32 == 0: the TMA shuffle-store path (incl. a ragged last m-tile)
                                                (256, 0, 2, 5, 32), (512, 1, 3, 3, 64), (256, 1, 2, 7, 96)])
def test_upsample_shuffle(svr2lib, C, temporal, F_, H, W):
    z = 2 if temporal else 1
    r = 4 * z
    x = rnd(1, C, F_, H, W, seed=1)
    w = rnd(r * C, C, std=C ** -0.5, seed=2)
    b = rnd(r * C, seed=3)
    xb, wb, bb = bf(x).float(), bf(w).float(), bf(b).float()
    y = F.conv3d(xb, wb.view(r * C, C, 1, 1, 1), bb)
    y = y.view(1, 2, 2, z, C, F_, H, W).permute(0, 4, 5, 3, 6, 1, 7, 2).reshape(1, C, F_ * z, 2 * H, 2 * W)
    if temporal:
        y = torch.cat([y[:, :, :1], y[:, :, 2:]], 2)
    T_out = y.shape[2]
    out = torch.zeros(2 + T_out, 2 * H, 2 * W, C, device=DEV, dtype=torch.bfloat16)
    x_nd = _to_ndhwc(x, 0)
    w16, b16 = bf(w).contiguous(), bf(b)          # keep the operands alive across the launch
    svr2lib.call("svr2_upsample_shuffle_bf16", svr2lib.ptr(x_nd), F_, H, W, C, svr2lib.ptr(w16),
                 svr2lib.ptr(b16), temporal, 1, svr2lib.ptr(out), 2, 1, svr2lib.stream())
    assert_close(out[2:], y[0].permute(1, 2, 3, 0), 4e-3, "upsample shuffle")
    assert torch.equal(out[0], out[2]) and torch.equal(out[1], out[2])


# ------------------------------------------------------------------ elementwise
@pytest.mark.parametrize("dim", [256, 2560, 3072])
def test_rmsnorm_ada(svr2lib, dim):
    x = bf(rnd(333, dim, seed=1))
    scale, shift, wt = rnd(dim, seed=2) * 0.1 + 1, rnd(dim, seed=3) * 0.1, rnd(dim, seed=4) * 0.1 + 1
    r = x.float() / torch.sqrt(x.float().pow(2).mean(-1, keepdim=True) + 1e-5)
    out = svr2lib.rmsnorm_ada(x, scale, shift, mode=0)
    assert_close(out, r * scale + shift, 3e-3, "mode0")
    out = svr2lib.rmsnorm_ada(x, scale, shift, weight=wt, mode=0)
    assert_close(out, r * wt * scale + shift, 3e-3, "mode0+weight")
    out = svr2lib.rmsnorm_ada(x, scale, shift, mode=1)
    ref = bf(bf(bf(r).float() * scale).float() + shift)
    assert_close(out, ref, 3e-3, "mode1")


@contextlib.contextmanager
def geometry_handle(svr2lib, variant, heads, freqs, layers=4):
    """A DiT handle that holds nothing but every layer's RoPE frequencies: enough for svr2_dit_geometry."""
    desc = svr2lib.ModelDesc(variant=0 if variant == "3b" else 1, dim=heads * 128, heads=heads, layers=layers,
                             mm_layers=layers, txt_in_dim=64, in_ch=33, out_ch=16, mlp_kind=0, mlp_hidden=256, out_norm=1,
                             last_vid_only=0, eps=1e-5, timestep=1000.0)
    h = svr2lib.engine_create(desc, torch.cuda.current_device())
    try:
        svr2lib.engine_load(h, {f"{i}.rope_freqs": freqs for i in range(layers)}, copy=True)
        yield h
    finally:
        svr2lib.engine_destroy(h)


@pytest.mark.parametrize("variant", ["3b", "7b"])
def test_dit_geometry_entry_point(svr2lib, variant):
    """svr2_dit_geometry: the handle's device tables equal the oracle (as in tests/test_native_geometry_cpu.py); even
    layers use the regular windows, odd layers the shifted ones; fuse_qkv follows the heads and the RoPE width; and it
    refuses what svr2_dit_forward refuses, a VAE handle and a layer outside [0, layers)."""
    from test_native_geometry_cpu import check_against_oracle, rope_freqs
    freqs = rope_freqs(variant, torch.float16)
    l = 58
    ints = ("cu_seqlens", "row_src", "row_rope", "out_row_map", "tok_dst", "tok_rope", "txt_rows")
    with geometry_handle(svr2lib, variant, 2, freqs) as h:
        for T, Hp, Wp in ((3, 20, 36), (3, 135, 240)):
            for layer in (0, 1, 2, 3):
                g = svr2lib.dit_geometry(h, T, 2 * Hp, 2 * Wp, l, layer)
                L = T * Hp * Wp
                sizes = dict(cu_seqlens=g.n_win + 1, row_src=g.total, row_rope=3 * g.total, out_row_map=g.total,
                             tok_dst=L, tok_rope=3 * L, txt_rows=g.n_txt_rows)
                got = {n: getattr(g, n) for n in ("n_win", "total", "max_len", "n_txt_rows", "nfreq", "rope_rows")}
                got.update({n: svr2lib.host_copy(getattr(g, n), (sizes[n],), torch.int32) for n in ints})
                got.update({n: svr2lib.host_copy(getattr(g, n), (g.rope_rows, g.nfreq), torch.float32)
                            for n in ("rope_cos", "rope_sin")})
                check_against_oracle(got, variant, T, Hp, Wp, l, bool(layer & 1), freqs)
                assert g.fuse_qkv == 1
        for bad in ((3, 41, 72, l, 0), (3, 40, 72, l, 4), (3, 40, 72, l, -1), (3, 40, 72, 0, 0), (0, 40, 72, l, 0)):
            with pytest.raises(svr2lib.Svr2Error):
                svr2lib.dit_geometry(h, *bad)
    for heads, nfreq, fused in ((2, 21, 1), (2, 10, 1), (4, 21, 1), (3, 21, 0), (3, 10, 0), (2, 16, 0)):
        with geometry_handle(svr2lib, variant, heads, torch.linspace(0.5, 2.0, nfreq).half()) as h:
            assert svr2lib.dit_geometry(h, 1, 16, 24, l, 0).fuse_qkv == fused, (heads, nfreq)
    vae = svr2lib.engine_create(svr2lib.ModelDesc(variant=2), torch.cuda.current_device())
    try:
        with pytest.raises(svr2lib.Svr2Error, match="VAE"):
            svr2lib.dit_geometry(vae, 1, 16, 24, l, 0)
    finally:
        svr2lib.engine_destroy(vae)


@pytest.mark.parametrize("C,hw,frames,silu", [(128, 24 * 36, 3, 1), (256, 1000, 2, 1), (512, 77, 2, 0),
                                              (128, 300 * 200, 2, 1), (512, 20000, 1, 1)])
def test_groupnorm(svr2lib, C, hw, frames, silu):
    x = bf(rnd(frames, hw, C, seed=1) * 2 + 0.5)
    gamma, beta = bf(rnd(C, seed=2) * 0.1 + 1), bf(rnd(C, seed=3) * 0.1)
    y = torch.zeros(2 + frames, hw, C, device=DEV, dtype=torch.bfloat16)
    need = svr2lib.load().svr2_groupnorm_scratch_bytes(frames, hw, C)
    stats = torch.zeros(need // 8 + 1, device=DEV, dtype=torch.float64)
    args = (svr2lib.ptr(x), svr2lib.ptr(y), frames, hw, C, svr2lib.ptr(gamma), svr2lib.ptr(beta), 1e-6, silu, 2, 1,
            svr2lib.ptr(stats), stats.numel() * 8, svr2lib.stream())
    svr2lib.call("svr2_groupnorm_bf16", *args)
    y_first = y.clone()
    svr2lib.call("svr2_groupnorm_bf16", *args)
    assert torch.equal(y, y_first), "groupnorm must be bit-reproducible"
    ref = F.group_norm(x.float().permute(0, 2, 1), 32, gamma.float(), beta.float(), 1e-6)
    ref = bf(ref).float()
    if silu:
        ref = F.silu(ref)
    assert_close(y[2:], ref.permute(0, 2, 1), 3e-3, "groupnorm")
    assert torch.equal(y[0], y[2]) and torch.equal(y[1], y[2])


def test_transpose_misc(svr2lib):
    a = bf(rnd(70, 130, seed=2))
    t = torch.empty(130, 72, device=DEV, dtype=torch.bfloat16)
    svr2lib.call("svr2_transpose_bf16", svr2lib.ptr(a), 130, svr2lib.ptr(t), 72, 70, 130, svr2lib.stream())
    assert torch.equal(t[:, :70], a.T)
    # txt mean
    x = bf(rnd(9, 58, 256, seed=3))
    o = torch.empty(58, 256, device=DEV, dtype=torch.bfloat16)
    svr2lib.call("svr2_txt_window_mean_bf16", svr2lib.ptr(x), svr2lib.ptr(o), 9, 58, 256, svr2lib.stream())
    assert_close(o, x.float().mean(0), 3e-3, "txt mean")
    # patchify / unpatchify
    T, H, W, C = 2, 6, 8, 33
    vid = bf(rnd(T * H * W, C, seed=4))
    pt = torch.empty(T * 3 * 4, 192, device=DEV, dtype=torch.bfloat16)
    svr2lib.call("svr2_patchify_bf16", svr2lib.ptr(vid), svr2lib.ptr(pt), T, H, W, C, 192, svr2lib.stream())
    ref = vid.view(T, 3, 2, 4, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(T * 12, 4 * C)
    assert torch.equal(pt[:, :132], ref) and pt[:, 132:].abs().max() == 0
    back = torch.empty(T * H * W, 16, device=DEV, dtype=torch.bfloat16)
    v64 = bf(rnd(T * 12, 64, seed=5))
    svr2lib.call("svr2_unpatchify_bf16", svr2lib.ptr(v64), 64, svr2lib.ptr(back), T, H, W, 16, svr2lib.stream())
    ref = v64.view(T, 3, 4, 2, 2, 16).permute(0, 1, 3, 2, 4, 5).reshape(T * H * W, 16)
    assert torch.equal(back, ref)


def test_layout_and_im2col(svr2lib):
    C, T, H, W = 3, 2, 6, 8
    x = rnd(C, T, H, W, seed=1)
    out = torch.full((2 + T, H, W, 8), 7.0, device=DEV, dtype=torch.bfloat16)
    svr2lib.call("svr2_ncdhw_to_ndhwc_bf16", svr2lib.ptr(x), 0, C, T, H, W, svr2lib.ptr(out), 8, 2, 1.0,
                 svr2lib.stream())
    assert torch.equal(out[2:, ..., :3], bf(x).permute(1, 2, 3, 0)) and out[..., 3:].abs().max() == 0
    assert torch.equal(out[0], out[2]) and torch.equal(out[1], out[2])
    back = torch.empty(C, T, H, W, device=DEV, dtype=torch.float32)
    svr2lib.call("svr2_ndhwc_to_ncdhw", svr2lib.ptr(out[2:]), 8, C, T, H, W, svr2lib.ptr(back), 0, svr2lib.stream())
    assert torch.equal(back, bf(x).float())
    col = torch.empty(T * H * W, 128, device=DEV, dtype=torch.bfloat16)
    svr2lib.call("svr2_im2col3_bf16", svr2lib.ptr(out), T, H, W, C, 8, svr2lib.ptr(col), 128, svr2lib.stream())
    xp = F.pad(out[..., :3].float().permute(3, 0, 1, 2)[None], (1, 1, 1, 1))  # halo already in T
    ref = xp.unfold(2, 3, 1).unfold(3, 3, 1).unfold(4, 3, 1)  # 1,C,T,H,W,kt,kh,kw
    ref = ref[0].permute(1, 2, 3, 4, 5, 6, 0).reshape(T * H * W, 81)
    assert torch.equal(col[:, :81].float(), ref) and col[:, 81:].abs().max() == 0


@pytest.mark.parametrize("M,n", [(300, 160), (1000, 2052), (129, 36)])
def test_two_pass_attention_probabilities(svr2lib, M, n):
    """EPI_ROWSTAT + rowstat_combine + EPI_PEXP == softmax(q k^T * scale) (VAE mid-block attention)."""
    d = 512
    q, k = bf(rnd(M, d, seed=1)), bf(rnd(n, d, seed=2))
    scale = d ** -0.5
    s2 = scale * 1.4426950408889634
    slots = svr2lib.load().svr2_rowstat_slots(n)
    part = torch.empty(M, 2 * slots, device=DEV, dtype=torch.float32)
    svr2lib.linear(q, k, epi=svr2lib.EPI_ROWSTAT, out=part, out_scale=s2)
    lse = torch.empty(M, device=DEV, dtype=torch.float32)
    svr2lib.call("svr2_rowstat_combine", svr2lib.ptr(part), slots, slots, svr2lib.ptr(lse), M, svr2lib.stream())
    ldn = (n + 7) // 8 * 8
    P = torch.zeros(M, ldn, device=DEV, dtype=torch.bfloat16)
    k_pad = torch.zeros(ldn, d, device=DEV, dtype=torch.bfloat16)   # bf16 output needs N % 8 == 0
    k_pad[:n] = k
    svr2lib.linear(q, k_pad, epi=svr2lib.EPI_PEXP, gate=lse, out=P, out_scale=s2)
    S = (q.float() @ k.float().T) * scale
    assert_close(lse, torch.logsumexp(S, -1) * 1.4426950408889634, 1e-4, "lse2")
    assert_close(P[:, :n], torch.softmax(S, -1), 6e-3, "probabilities")
    assert (P[:, :n].float().sum(-1) - 1).abs().max() < 2e-2


@pytest.mark.parametrize("Cin,Cout,T,H,W", [(64, 128, 2, 20, 36), (128, 256, 2, 19, 30), (256, 512, 1, 12, 20)])
def test_conv_epilogue_groupnorm_stats(svr2lib, Cin, Cout, T, H, W):
    """svr2_conv3d_stats_bf16 + svr2_groupnorm_from_stats_bf16 == conv followed by per-frame GroupNorm + SiLU."""
    import ctypes
    x = rnd(1, Cin, T, H, W, seed=1)
    w = rnd(Cout, Cin, 3, 3, 3, std=(Cin * 27) ** -0.5, seed=2)
    b = rnd(Cout, seed=3)
    x_nd = _to_ndhwc(x, 2)
    w_k = bf(w.permute(0, 2, 3, 4, 1).reshape(Cout, -1)).contiguous()
    y = torch.zeros(T, H, W, Cout, device=DEV, dtype=torch.bfloat16)
    b16 = bf(b)                                   # must outlive the launch (a temporary's block gets reused by `part`)
    args = (svr2lib.ptr(x_nd), T + 2, H, W, Cin, svr2lib.ptr(w_k), Cout, 3, 3, 3, 1, 1, 1, T, svr2lib.EPI_BIAS,
            svr2lib.ptr(b16), None, svr2lib.ptr(y), 0, 0, Cout)
    slots = ctypes.c_int(0)
    assert svr2lib.load().svr2_conv3d_stats_bf16(*args, None, 0, ctypes.byref(slots), svr2lib.stream()) == 0
    part = torch.full((T * slots.value * (Cout // 8) * 4,), float("nan"), device=DEV)
    svr2lib.call("svr2_conv3d_stats_bf16", *args, svr2lib.ptr(part), part.numel() * 4, ctypes.byref(slots),
                 svr2lib.stream())
    assert torch.isfinite(part).all(), "every partial slot must be written"
    gamma, beta = bf(rnd(Cout, seed=4) * 0.1 + 1), bf(rnd(Cout, seed=5) * 0.1)
    z = torch.zeros(2 + T, H * W, Cout, device=DEV, dtype=torch.bfloat16)
    coef = torch.empty(T * Cout * 2, device=DEV)
    svr2lib.call("svr2_groupnorm_from_stats_bf16", svr2lib.ptr(y), svr2lib.ptr(z), T, H * W, Cout, svr2lib.ptr(gamma),
                 svr2lib.ptr(beta), 1e-6, 1, 2, 1, svr2lib.ptr(part), slots.value, svr2lib.ptr(coef), svr2lib.stream())
    ref = F.group_norm(y.float().view(T, H * W, Cout).permute(0, 2, 1), 32, gamma.float(), beta.float(), 1e-6)
    ref = F.silu(bf(ref).float()).permute(0, 2, 1)
    assert_close(z[2:], ref, 3e-3, "fused-stats groupnorm")
    assert torch.equal(z[0], z[2]) and torch.equal(z[1], z[2])
