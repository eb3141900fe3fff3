"""-m gpu: the VAE decode that returns only the first F output frames.  svr2_vae_decode_frames(F) must be bit-identical to
svr2_vae_decode followed by [:, :F] (un-sliced and temporally sliced, fp32 / bf16 / fp16 latents, engine-owned and caller
workspace, at a small size and at the 4K shard's 2 x 270 x 480 latent), and SeedVR2Engine.upscale_clip and its CUDA-graph
replay, which decode only the clip's real frames, bit-identical to the same clip decoded whole and cropped."""
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu

DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


@pytest.fixture(scope="module")
def mods(pkg):
    name = "comfyui_seedvr2_videoupscaler_b200."
    return {m: importlib.import_module(name + m) for m in ("lib", "vae", "pipeline", "dit")}


def _decode(lib, vae, z, T, h, w, sl, F, ws):
    """svr2_vae_decode (F None) or svr2_vae_decode_frames into a fresh (3, F, 8h, 8w) bf16 tensor."""
    L, hd = lib.load(), vae.native_handle()
    out = torch.full((3, 4 * T - 3 if F is None else F, 8 * h, 8 * w), float("nan"), device="cuda", dtype=torch.bfloat16)
    wp, wn = (None, 0) if ws is None else (lib.ptr(ws), ws.numel())
    if F is None:
        rc = L.svr2_vae_decode(hd, lib.ptr(z), DT[z.dtype], T, h, w, sl, lib.ptr(out), wp, wn, lib.stream())
    else:
        rc = L.svr2_vae_decode_frames(hd, lib.ptr(z), DT[z.dtype], T, h, w, sl, F, lib.ptr(out), wp, wn, lib.stream())
    assert rc == 0, L.svr2_engine_last_error(hd).decode()
    return out


def _check(lib, vae, T, h, w, sl, frames, dtypes, owners, seed=0):
    L, hd = lib.load(), vae.native_handle()
    g = torch.Generator().manual_seed(seed)
    z32 = torch.randn(16, T, h, w, generator=g)
    for dt in dtypes:
        z = z32.to(dt).cuda().contiguous()
        for owner in owners:
            ws = None
            if owner == "caller":
                full_need = L.svr2_vae_workspace_bytes(hd, 1, T, h, w, sl)
                assert L.svr2_vae_decode_frames_workspace_bytes(hd, T, h, w, sl, 4 * T - 3) == full_need
                need = {F: L.svr2_vae_decode_frames_workspace_bytes(hd, T, h, w, sl, F) for F in frames}
                assert min(need.values()) > 0
                ws = torch.empty(max(full_need, *need.values()), device="cuda", dtype=torch.uint8)
            full = _decode(lib, vae, z, T, h, w, sl, None, ws)
            for F in frames:
                if owner == "caller":
                    part = _decode(lib, vae, z, T, h, w, sl, F, ws[:need[F]])     # exactly the planned bytes
                else:
                    part = _decode(lib, vae, z, T, h, w, sl, F, None)
                torch.cuda.synchronize()
                assert torch.equal(part, full[:, :F]), (T, h, w, sl, F, dt, owner)
            del full, ws


@pytest.fixture(scope="module")
def vae_small(pkg, mods):
    return mods["vae"].B200VideoVAE(pkg.weights.synth_vae_state_dict(seed=3))


@pytest.mark.parametrize("T,h,w,sl,frames", [
    (3, 6, 10, 0, (9, 8, 7, 6, 1)),               # un-sliced
    (5, 6, 10, 2, (17, 16, 15, 14, 9, 8)),        # slices of 3 + 2 latent frames: the last trimmed, or not run at all
    (6, 5, 7, 1, (21, 20, 18, 13, 6)),            # five slices
])
def test_decode_frames_equals_cropped_decode_small(mods, vae_small, T, h, w, sl, frames):
    _check(mods["lib"], vae_small, T, h, w, sl, frames, (torch.float32, torch.bfloat16, torch.float16), ("engine", "caller"))


def test_decode_frames_equals_cropped_decode_4k_shard(pkg, mods):
    """The 4K shard's decode: latent 2 x 270 x 480, 5 frames of 2160 x 3840 decoded whole vs the first 4."""
    lib = mods["lib"]
    vae = mods["vae"].B200VideoVAE(pkg.weights.synth_vae_state_dict(seed=5))
    try:
        _check(lib, vae, 2, 270, 480, 0, (4,), (torch.bfloat16, torch.float32), ("caller",), seed=1)
        torch.cuda.empty_cache()
        _check(lib, vae, 2, 270, 480, 0, (4,), (torch.float16,), ("engine",), seed=2)
    finally:
        vae._drop_handle()                       # the engine-owned workspace goes back with the handle
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def test_vae_module_decode_frames(mods, vae_small):
    """B200VideoVAE.decode(frames=F) on the native runtime and on the Python sequencing: the first F frames of decode()."""
    z = torch.randn(1, 16, 5, 6, 10, generator=torch.Generator().manual_seed(4)).cuda()
    full = vae_small.decode(z).sample
    vae_small.set_causal_slicing(split_size=8)
    try:
        for F in (17, 15, 9, 3):
            assert torch.equal(vae_small.decode(z, frames=F).sample, full[:, :, :F])
            vae_small.native = False
            try:
                assert torch.equal(vae_small.decode(z, frames=F).sample, full[:, :, :F])
            finally:
                vae_small.native = True
    finally:
        vae_small.set_causal_slicing(split_size=None)
    with pytest.raises(ValueError):
        vae_small.decode(z, frames=18)


@pytest.fixture(scope="module")
def engine(pkg, mods):
    cfg = mods["dit"].dit_config("3b", dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64)
    return mods["pipeline"].SeedVR2Engine(cfg, pkg.weights.synth_dit_state_dict(cfg, seed=1),
                                          pkg.weights.synth_vae_state_dict(seed=2), torch.randn(58, 64))


@pytest.mark.parametrize("T", [4, 6, 8])                # padded to 5, 9, 9 frames
def test_upscale_clip_decodes_only_the_real_frames(mods, engine, T):
    SeedVR2Engine = mods["pipeline"].SeedVR2Engine
    frames = torch.rand(T, 36, 48, 3, generator=torch.Generator().manual_seed(T)).cuda()
    # the untrimmed path: the same engine with phase methods that decode (and plan) every frame, cropped afterwards
    engine.vae_decode = lambda latent, workspace=None: SeedVR2Engine.vae_decode(engine, latent, workspace=workspace)
    engine.clip_workspace = lambda T_, Hp, Wp: SeedVR2Engine.clip_workspace(engine, T_, Hp, Wp)
    try:
        want = engine.upscale_clip(frames, seed=11, resolution=72).clone()
    finally:
        del engine.vae_decode, engine.clip_workspace
    assert want.shape == (T, 72, 96, 3)
    got = engine.upscale_clip(frames, seed=11, resolution=72)
    assert torch.equal(got, want)
    graphed = engine.graphed(frames, seed=11, resolution=72)
    assert torch.equal(graphed(frames, clone=True), want)
    assert torch.equal(graphed(frames, clone=True), want)
    del graphed
