"""-m gpu: the spatially tiled VAE passes on the native runtime.  The ramp tables equal the torch bf16 op chain of vae.py
_tiled for n = 1 .. 256; the seam variants of the final kernels equal "store the tile, then svr2_tile_accumulate_bf16"
element by element at edge and interior tiles; svr2_vae_encode_tiled / svr2_vae_decode_tiled equal the Python
tile-by-tile sequence (`.native = False`) bit for bit on the golden geometries, at a ragged 1080p geometry with forced
temporal slicing and for a decode of fewer frames; a 9-frame 4K batch from a 720p source upscales with both tilings on
one 80 GB GPU; graph replay and stream_video with tiling equal eager upscale_clip / upscale_video."""
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mods(pkg):
    name = "comfyui_seedvr2_videoupscaler_b200."
    return {m: importlib.import_module(name + m) for m in ("lib", "vae", "pipeline", "dit")}


def bits(t):
    return t.contiguous().view(torch.int16)


def torch_ramp(n):
    t = torch.linspace(0, 1, steps=n, device="cuda", dtype=torch.bfloat16)
    return 0.5 - 0.5 * torch.cos(t * torch.pi)


def test_ramp_tables_equal_torch(mods):
    lib = mods["lib"]
    for n in range(1, 257):
        m = 257 - n
        rh = torch.full((2 * n,), float("nan"), device="cuda", dtype=torch.bfloat16)
        rw = torch.full((2 * m,), float("nan"), device="cuda", dtype=torch.bfloat16)
        lib.call("svr2_tile_ramp_bf16", lib.ptr(rh), n, lib.ptr(rw), m, lib.stream())
        for tab, k in ((rh, n), (rw, m)):
            r = torch_ramp(k)
            assert torch.equal(bits(tab[:k]), bits(r)), (k, tab[:k], r)
            assert torch.equal(bits(tab[k:]), bits(1 - r)), k


def _weights(n, ov_len, lo, hi):
    """vae.py _tiled's edge weights of one axis."""
    w = torch.ones(n, device="cuda", dtype=torch.bfloat16)
    ov = max(0, min(ov_len, n - 1))
    if ov > 0:
        r = torch_ramp(ov_len)
        if lo:
            w[:ov] = r[:ov]
        if hi:
            w[-ov:] = 1 - r[:ov]
    return w


# (T, tile H, tile W, ramp lengths, edges, count updated): interior, corner and edge tiles, ramps longer than the tile
SEAM_CASES = [(2, 24, 40, (8, 16), 15, True), (3, 17, 9, (6, 6), 2 | 8, True), (1, 12, 30, (20, 4), 1 | 4 | 8, True),
              (2, 9, 13, (0, 5), 4, False), (1, 16, 16, (16, 16), 1 | 2, True)]


@pytest.mark.parametrize("T,h,w,lens,edges,with_count", SEAM_CASES)
def test_seam_variants_equal_store_then_accumulate(mods, T, h, w, lens, edges, with_count):
    lib = mods["lib"]
    g = torch.Generator(device="cuda").manual_seed(T * 1000 + h * 10 + w)
    Hr, Wr, y0, x0, F, t0 = h + 11, w + 7, 5, 3, T + 2, 1       # the tile at (y0, x0) of frames t0 .. t0 + T of F
    lh, lw = lens
    ramp_h = torch.zeros(max(1, 2 * lh), device="cuda", dtype=torch.bfloat16)
    ramp_w = torch.zeros(max(1, 2 * lw), device="cuda", dtype=torch.bfloat16)
    lib.call("svr2_tile_ramp_bf16", lib.ptr(ramp_h), lh, lib.ptr(ramp_w), lw, lib.stream())
    wh = _weights(h, lh, edges & 1, edges & 2)
    ww = _weights(w, lw, edges & 4, edges & 8)

    def run(kind, C):
        if kind == "gather":
            npix = (T + 2) * h * w
            ldz = (npix + 3) // 4 * 4
            src = torch.randn(81, ldz, generator=g, device="cuda") * 0.1
            bias = (torch.randn(C, generator=g, device="cuda") * 0.1).to(torch.bfloat16)
        else:
            src = (torch.randn(T, h, w, 32, generator=g, device="cuda")).to(torch.bfloat16)
        result = (torch.randn(C, F, Hr, Wr, generator=g, device="cuda")).to(torch.bfloat16)
        count = (torch.rand(Hr, Wr, generator=g, device="cuda") * 2).to(torch.bfloat16)
        # reference: the plain kernel stores the tile, svr2_tile_accumulate_bf16 adds it
        tile = torch.empty(C, T, h, w, device="cuda", dtype=torch.bfloat16)
        if kind == "gather":
            lib.call("svr2_conv_tap_gather", lib.ptr(src), ldz, C, lib.ptr(bias), T, h, w, lib.ptr(tile), 1, lib.stream())
        else:
            lib.call("svr2_ndhwc_to_ncdhw", lib.ptr(src), 32, C, T, h, w, lib.ptr(tile), 1, lib.stream())
        want_r, want_c = result.clone(), count.clone()
        scratch_c = count.clone()
        for c in range(C):        # the result's frames t0.. of channel c, as planes of an [F, Hr, Wr] block
            lib.call("svr2_tile_accumulate_bf16", lib.ptr(tile[c]), h * w, w, T, h, w, lib.ptr(wh), lib.ptr(ww),
                     lib.ptr(want_r[c, t0:]), lib.ptr(want_c if c == 0 else scratch_c), Hr, Wr, y0, x0, lib.stream())
        if not with_count:
            want_c = count.clone()
        got_r, got_c = result.clone(), count.clone()
        corner = (t0 * Hr * Wr + y0 * Wr + x0) * 2
        rp = got_r.data_ptr() + corner
        cp = got_c.data_ptr() + (y0 * Wr + x0) * 2 if with_count else None
        from ctypes import c_void_p
        args = (c_void_p(rp), F * Hr * Wr, Hr * Wr, Wr, None if cp is None else c_void_p(cp), lib.ptr(ramp_h), lh,
                lib.ptr(ramp_w), lw, edges, lib.stream())
        if kind == "gather":
            lib.call("svr2_conv_tap_gather_seam_bf16", lib.ptr(src), ldz, C, lib.ptr(bias), T, h, w, *args)
        else:
            lib.call("svr2_ndhwc_to_ncdhw_seam_bf16", lib.ptr(src), 32, C, T, h, w, *args)
        assert torch.equal(bits(got_r), bits(want_r)), (kind, (got_r.float() - want_r.float()).abs().max())
        assert torch.equal(bits(got_c), bits(want_c)), kind

    run("gather", 3)
    run("ndhwc", 16)


@pytest.fixture(scope="module")
def vae(pkg, mods):
    return mods["vae"].B200VideoVAE(pkg.weights.synth_vae_state_dict(seed=4321, dtype=torch.float16))


def _both(vae, fn):
    """fn() on the native tiled runtime and on the Python tile-by-tile sequence."""
    native = fn()
    vae.native = False
    try:
        python = fn()
    finally:
        vae.native = True
    return native, python


def test_native_tiled_equals_python_on_golden_geometries(vae):
    from oracle.make_golden import TILED_CASES
    for name, (kind, shp, tile, ov) in TILED_CASES.items():
        g = torch.Generator().manual_seed(7)
        if kind == "decode":
            src = torch.randn(1, 16, *shp, generator=g).cuda()
            a, b = _both(vae, lambda: vae.decode(src, tiled=True, tile_size=tile, tile_overlap=ov).sample)
        else:
            src = (torch.rand(1, 3, *shp, generator=g) * 2 - 1).cuda()
            a, b = _both(vae, lambda: vae.encode(src, tiled=True, tile_size=tile, tile_overlap=ov).latent)
        assert a.shape == b.shape and torch.equal(bits(a), bits(b)), name


def test_native_tiled_equals_python_1080p_sliced_and_frames(vae):
    """Ragged tiles at 1080p (1080 x 1920: 512-pixel tiles overlapping by 64 leave a short last row and column), every
    tile temporally sliced, and a decode of only the first frames."""
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(1, 3, 9, 1080, 1920, generator=g) * 2 - 1).cuda().to(torch.bfloat16)
    z = torch.randn(1, 16, 3, 135, 240, generator=g).cuda()
    vae.set_causal_slicing(split_size=4)
    try:
        a, b = _both(vae, lambda: vae.encode(x, tiled=True, tile_size=512, tile_overlap=64).latent)
        assert a.shape == (1, 16, 3, 135, 240) and torch.equal(bits(a), bits(b))
        a, b = _both(vae, lambda: vae.decode(z, tiled=True, tile_size=(512, 640), tile_overlap=(64, 96)).sample)
        assert a.shape == (1, 3, 9, 1080, 1920) and torch.equal(bits(a), bits(b))
        a, b = _both(vae, lambda: vae.decode(z, tiled=True, tile_size=(512, 640), tile_overlap=(64, 96), frames=6).sample)
        assert a.shape == (1, 3, 6, 1080, 1920) and torch.equal(bits(a), bits(b))
    finally:
        vae.set_causal_slicing(split_size=None)


def test_upscale_clip_4k_9_frames_tiled_fits(pkg, mods):
    """A 9-frame batch from a 720p source to 2160 x 3840 (3B, synthetic weights) with both VAE passes tiled at the
    loader's default 1024 / 128: 9 frames back, peak device memory under 80 GB."""
    eng = mods["pipeline"].build_synthetic_engine("3b")
    try:
        frames = torch.rand(9, 720, 1280, 3, generator=torch.Generator().manual_seed(1)).cuda()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        out = eng.upscale_clip(frames, resolution=2160, encode_tiled=True, decode_tiled=True)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_reserved()
        print(f"4K 9-frame tiled clip: peak reserved {peak / 1e9:.1f} GB, DiT workspace "
              f"{eng.dit.workspace_bytes(3, 270, 480, eng.txt.shape[0]) / 1e9:.1f} GB")
        assert out.shape == (9, 2160, 3840, 3) and torch.isfinite(out.float()).all()
        assert peak < 80e9
    finally:
        del eng
        mods["lib"].release_workspace()
        torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def engine(pkg, mods):
    cfg = mods["dit"].dit_config("3b", dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64)
    return mods["pipeline"].SeedVR2Engine(cfg, pkg.weights.synth_dit_state_dict(cfg, seed=1),
                                          pkg.weights.synth_vae_state_dict(seed=2), torch.randn(58, 64))


TILING = dict(encode_tiled=True, encode_tile_size=64, encode_tile_overlap=16, decode_tiled=True, decode_tile_size=(48, 64),
              decode_tile_overlap=(16, 24))


def test_graphed_tiled_clip_equals_eager(engine):
    frames = torch.rand(6, 48, 64, 3, generator=torch.Generator().manual_seed(5)).cuda()
    want = engine.upscale_clip(frames, seed=3, resolution=96, **TILING).clone()
    plain = engine.upscale_clip(frames, seed=3, resolution=96)
    assert want.shape == plain.shape == (6, 96, 128, 3) and not torch.equal(want, plain)     # tiling changes results
    graphed = engine.graphed(frames, seed=3, resolution=96, **TILING)
    assert torch.equal(graphed(frames, clone=True), want)
    assert torch.equal(graphed(frames, clone=True), want)
    del graphed


def test_stream_video_tiled_equals_upscale_video(engine):
    video = torch.rand(13, 48, 64, 3, generator=torch.Generator().manual_seed(6))
    kw = dict(batch_size=5, temporal_overlap=2, resolution=96, **TILING)
    want = engine.upscale_video(video.cuda(), **kw)
    got = torch.cat([t for _, t in engine.stream_video(video, out_dtype=torch.bfloat16, **kw)], 0)
    assert torch.equal(got.cuda(), want)
