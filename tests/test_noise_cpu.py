"""CPU: the generation-noise restatement (oracle/noise_oracle.py) against the goldens made from the reference's code,
the C-ABI entry points of csrc/noise.cu and their argument refusal, and the engine's noise and batch options with the
GPU stages stubbed: frames reaching the encoder, output lengths, prepended-frame removal and the RNG draw order."""
import ctypes
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import noise_oracle as no
from oracle.make_noise_golden import INPUT_CASES, LATENT_CASES

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def bf(a):
    return torch.from_numpy(np.asarray(a)).to(torch.bfloat16)


@pytest.mark.parametrize("name", list(INPUT_CASES))
def test_input_noise_oracle_matches_golden(name):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    batches = len(g["encode_frames"])
    for bi in range(batches):
        tv, draw = bf(g[f"tv{bi}"]), bf(g[f"draw{bi}"])
        for s in g["scales"]:
            assert torch.equal(no.input_noise(tv, draw, float(s)), bf(g[f"out{bi}_{float(s)}"])), (bi, s)


def test_input_noise_golden_batches():
    """The node's batch_size 5: a full batch and a tail uniform-padded from 2 to 5 frames, both encoded as 5."""
    g = np.load(os.path.join(GOLD, "noise_input_video.npz"))
    assert list(g["batch_frames"]) == [5, 5] and list(g["encode_frames"]) == [5, 5]
    assert list(np.load(os.path.join(GOLD, "noise_input_tail.npz"))["batch_frames"]) == [5, 2]


@pytest.mark.parametrize("name", list(INPUT_CASES))
def test_engine_draws_in_the_reference_memory_order(pkg, name):
    """The engine's choice of layout per batch gives the strides of the reference's transformed clip and draw, in all
    three orders: (t h w c) for a batch of 4n+1 frames, (t c h w) for a padded batch that is resized or padded to 16,
    (c t h w) for a padded batch that is neither."""
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    gen_noise = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.noise")
    g = np.load(os.path.join(GOLD, name + ".npz"))
    _, h, w, _ = g["images"].shape
    for bi, T in enumerate(g["batch_frames"]):
        layout = pipeline.SeedVR2Engine.input_noise_layout(torch.zeros(int(T), h, w, 3), int(g["resolution"]))
        buf = gen_noise.input_noise_buffer(g[f"tv{bi}"].shape, "cpu", layout)
        assert buf.stride() == tuple(g[f"draw{bi}_strides"]), (name, bi, layout)


@pytest.mark.parametrize("name", list(LATENT_CASES))
def test_condition_oracle_matches_golden(name):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    latent, noise, r = bf(g["latent"]), bf(g["noise"]), bf(g["r"])
    Tl, h, w, c = latent.shape
    # the reference's latent and both draws are channels-last views of channel-major memory
    for k in ("latent_strides", "noise_strides", "r_strides"):
        assert tuple(g[k]) == (h * w, w, 1, Tl * h * w), k
    assert torch.equal(no.sr_condition(noise, latent), bf(g["vid_0.0"]))
    for s in g["scales"]:
        s = float(s)
        a, b = no.coefficients(s, latent.shape, "cpu")
        assert torch.equal(a, torch.from_numpy(g[f"A_{s}"])) and torch.equal(b, torch.from_numpy(g[f"B_{s}"]))
        assert torch.equal(no.sr_condition(noise, latent, r, s), bf(g[f"vid_{s}"])), s


def test_coefficients_follow_the_latent_shape_quirk():
    """_add_noise hands timestep_transform x.shape[1:] = (h, w, c): h = 1 is an 'image' whatever T' is."""
    a1, b1 = no.coefficients(0.5, (7, 1, 9, 16), "cpu")
    a2, b2 = no.coefficients(0.5, (1, 1, 9, 16), "cpu")
    assert torch.equal(a1, a2) and torch.equal(b1, b2)
    _, bv = no.coefficients(0.5, (1, 2, 9, 16), "cpu")
    assert not torch.equal(bv, b2)


def test_noise_entry_points_and_refusal(svr2lib):
    import __graft_entry__
    __graft_entry__.build()
    lib = svr2lib.load()
    assert len(svr2lib.SIGNATURES["svr2_input_noise_bf16"]) == 9
    assert len(svr2lib.SIGNATURES["svr2_sr_condition_bf16"]) == 9
    p = ctypes.c_void_p(16)
    bad_input = [
        ((p, p, 0, p, 0, 64, 1.0, 0.0, None), b"empty"),
        ((p, p, 0, p, 2, 0, 1.0, 0.0, None), b"empty"),
        ((p, p, 0, p, 1, 1 << 31, 1.0, 0.0, None), b"2^31"),
        ((None, p, 0, p, 1, 64, 1.0, 0.0, None), b"null"),
        ((p, None, 0, p, 1, 64, 1.0, 0.0, None), b"null"),
        ((p, p, 0, None, 1, 64, 1.0, 0.0, None), b"null"),
        ((p, p, 3, p, 1, 64, 1.0, 0.0, None), b"noise_layout"),
        ((p, p, -1, p, 1, 64, 1.0, 0.0, None), b"noise_layout"),
    ]
    for args, msg in bad_input:
        assert lib.svr2_input_noise_bf16(*args) == -1 and msg in lib.svr2_last_error(), args
    bad_cond = [
        ((p, p, None, None, None, p, 0, 16, None), b"empty"),
        ((p, p, None, None, None, p, 10, 0, None), b"empty"),
        ((p, p, None, None, None, p, 10, 65, None), b"64"),
        ((p, p, None, None, None, p, (1 << 31) // 33 + 1, 16, None), b"2^31"),
        ((None, p, None, None, None, p, 10, 16, None), b"null"),
        ((p, None, None, None, None, p, 10, 16, None), b"null"),
        ((p, p, None, None, None, None, 10, 16, None), b"null"),
        ((p, p, p, None, p, p, 10, 16, None), b"coefficients"),
        ((p, p, p, p, None, p, 10, 16, None), b"coefficients"),
    ]
    for args, msg in bad_cond:
        assert lib.svr2_sr_condition_bf16(*args) == -1 and msg in lib.svr2_last_error(), args


# ---------------------------------------------------------------------------------------------------------------
# engine host logic with the GPU stages stubbed
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture
def stub_engine(pkg, monkeypatch):
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    preprocess = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.preprocess")
    color_fix = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.color_fix")
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    gen_noise = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.noise")
    eng = object.__new__(pipeline.SeedVR2Engine)
    eng.device = torch.device("cpu")
    log = {"encode": [], "input_draws": [], "inference": []}

    def fake_run(self, x, channels_last):            # (T,h,w,3) -> (3,T,Hp,Wp): nearest resize, pad, [-1,1]
        (H, W), _ = preprocess.resized_size(x.shape[1], x.shape[2], self.resolution, self.max_resolution)
        y = torch.nn.functional.interpolate(x[..., :3].permute(0, 3, 1, 2).float(), size=(H, W)).permute(1, 0, 2, 3)
        y = torch.nn.functional.pad(y, (0, (16 - W % 16) % 16, 0, (16 - H % 16) % 16))
        return (y * 2 - 1).to(torch.bfloat16).contiguous()

    def fake_add(x, n, scale):
        if tuple(n.shape) != tuple(x.shape):
            raise ValueError("input_noise must have the clip's shape")
        log["input_draws"].append(n.clone())
        return no.input_noise(x, n, scale).contiguous()

    def fake_encode(x):
        log["encode"].append(x.clone())
        return x[0, ::4, ::8, ::8, None].expand(-1, -1, -1, 16).contiguous()          # (T', h, w, 16)

    def fake_inference(noise, latent, latent_noise=None, latent_noise_scale=0.0):
        log["inference"].append((noise.clone(), None if latent_noise is None else latent_noise.clone(), latent_noise_scale))
        return latent

    monkeypatch.setattr(preprocess.VideoTransform, "run", fake_run)
    monkeypatch.setattr(gen_noise, "add_input_noise", fake_add)
    eng.vae_encode = fake_encode
    eng.inference = fake_inference
    eng.clip_workspace = lambda T, Hp, Wp: None
    # decode: frame i of the output carries the encoder's input frame 4 * (i // 4) (enough to tell frames apart)
    eng.vae_decode = lambda z: z[..., 0].repeat_interleave(4, 0)[: 4 * z.shape[0] - 3, None].expand(-1, 3, -1, -1) \
        .repeat_interleave(8, -2).repeat_interleave(8, -1).permute(1, 0, 2, 3).contiguous()
    monkeypatch.setattr(color_fix, "sample_to_image", lambda s_: s_.permute(0, 2, 3, 1).contiguous())
    monkeypatch.setattr(shard, "blend_overlap", lambda p, c: ((p.float() + c.float()) / 2).to(p.dtype))
    return eng, pipeline, log


def test_uniform_batches_and_prepend_reach_the_encoder_as_the_reference_loop(stub_engine):
    """Frame counts reaching vae_encode and output lengths vs a literal restatement of generation_phases.py:344-402
    (batching, uniform padding, 4n+1 padding) and :1388-1397 (prepended frames removed unless p >= the output)."""
    eng, pipeline, log = stub_engine
    for total, bs, ov, uniform, p in ((13, 5, 0, True, 0), (13, 5, 0, False, 0), (11, 4, 1, True, 2),
                                      (7, 5, 2, True, 3), (3, 5, 0, True, 4), (2, 5, 0, False, 9), (9, 4, 0, True, 1)):
        frames = torch.rand(total, 16, 24, 3, generator=torch.Generator().manual_seed(total))
        log["encode"].clear()
        out = eng.upscale_video(frames, batch_size=bs, temporal_overlap=ov, resolution=16, uniform_batch_size=uniform,
                                prepend_frames=p)
        # ---- reference restatement
        n = total + p
        step = bs - ov if ov > 0 else bs
        eff = ov
        if step <= 0:
            step, eff = bs, 0
        counts, written = [], 0
        for idx in range(0, n, step):
            end = min(idx + bs, n)
            if idx > 0 and end - idx <= eff:
                break
            cur = end - idx
            t = bs if (uniform and cur < bs) else cur
            counts.append(t if t % 4 == 1 else ((t - 1) // 4 + 1) * 4 + 1)
            if idx > 0 and 0 < eff < cur and written >= eff:                 # overlap frames blended away
                cur -= eff
            written += cur
        expect_len = written - p if p < written else written
        assert [x.shape[1] for x in log["encode"]] == counts, (total, bs, ov, uniform, p)
        assert out.shape[0] == expect_len, (total, bs, ov, uniform, p)


def test_prepended_and_padded_frames_are_mirrors(stub_engine):
    eng, pipeline, log = stub_engine
    frames = torch.rand(9, 16, 24, 3, generator=torch.Generator().manual_seed(1))
    log["encode"].clear()
    eng.upscale_video(frames, batch_size=4, resolution=16, uniform_batch_size=True, prepend_frames=2)
    # video = [f2, f1, f0 .. f8] (generation_utils.py:196-198): batches [f2 f1 f0 f1], [f2 .. f5], and the tail
    # [f6 f7 f8] uniform-padded with its mirrored frame f7 to 4 frames, then 4n+1-padded with the next mirror, f8
    pre = pipeline.pad_video_temporal(frames, count=2, prepend=True)
    assert torch.equal(pre[:3], frames[[2, 1, 0]])
    enc = log["encode"]
    assert len(enc) == 3 and [x.shape[1] for x in enc] == [5, 5, 5]
    as_clip = lambda idx: (frames[idx].permute(3, 0, 1, 2) * 2 - 1).to(torch.bfloat16)
    assert torch.equal(enc[0][:, :4, :, :24], as_clip([2, 1, 0, 1]))          # 24 columns padded to 32
    assert torch.equal(enc[1][:, :4, :, :24], as_clip([2, 3, 4, 5]))
    assert torch.equal(enc[2][..., :24], as_clip([6, 7, 8, 7, 8]))


def test_draw_order_across_batches(stub_engine):
    """One seed + 1_000_000 generator feeds the input-noise draws of the batches in turn (generation_phases.py:329-330,
    419); every batch draws the DiT noise and then r from a generator seeded `seed` (:663, 680-683)."""
    eng, pipeline, log = stub_engine
    frames = torch.rand(12, 16, 24, 3, generator=torch.Generator().manual_seed(2))
    eng.upscale_video(frames, batch_size=5, resolution=16, seed=7, input_noise_scale=0.4, latent_noise_scale=0.3,
                      uniform_batch_size=True)
    shapes = [tuple(x.shape) for x in log["encode"]]
    assert len(shapes) == 3 and len(log["input_draws"]) == 3
    # every batch holds 5 frames (the tail is uniform-padded), so the reference's clip and draw are (t h w c) memory.
    # torch's CPU normal_ takes another algorithm for non-contiguous memory, so on the CPU the draws are restated
    # in memory order (the GPU tests compare the engine's draws with randn_like on the reference's strides)
    g = torch.Generator().manual_seed(7 + 1_000_000)
    for got, (c, T, Hp, Wp) in zip(log["input_draws"], shapes):
        ref = torch.randn((T, Hp, Wp, c), generator=g, dtype=torch.bfloat16)
        assert torch.equal(got.permute(1, 2, 3, 0), ref) and got.permute(1, 2, 3, 0).is_contiguous()
    g = torch.Generator().manual_seed(7)
    Tl, h, w, c = log["inference"][0][0].shape
    base = torch.randn((Tl, h, w, c), generator=g, dtype=torch.bfloat16)     # the engine's DiT noise
    r = torch.randn((c, Tl, h, w), generator=g, dtype=torch.bfloat16)        # then r, channel-major
    for noise, lat_noise, scale in log["inference"]:
        assert torch.equal(noise, base) and torch.equal(lat_noise.permute(3, 0, 1, 2), r) and scale == 0.3
    # the noisy copy goes to the encoder, the clean clip stays the style
    smp, sty = eng.clip_to_sample(frames[:5], resolution=16, input_noise_scale=0.4)
    clean = (frames[:5].permute(3, 0, 1, 2) * 2 - 1).to(torch.bfloat16)
    assert torch.equal(sty.permute(1, 0, 2, 3), clean)
    assert torch.equal(log["encode"][-1][:, :, :, :24], no.input_noise(
        torch.nn.functional.pad(clean, (0, 8)), log["input_draws"][-1], 0.4)[:, :, :, :24])


def test_scale_zero_draws_nothing_and_bad_scales_raise(stub_engine):
    eng, pipeline, log = stub_engine
    frames = torch.rand(5, 16, 24, 3, generator=torch.Generator().manual_seed(3))
    eng.clip_to_sample(frames, resolution=16)
    assert log["input_draws"] == [] and log["inference"][-1][1] is None
    for bad in (-0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            eng.clip_to_sample(frames, resolution=16, input_noise_scale=bad)
        with pytest.raises(ValueError):
            eng.upscale_video(frames, resolution=16, latent_noise_scale=bad)
    noise = torch.zeros(2, 2, 3, 16, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="latent_noise"):
        eng.clip_to_sample(frames, noise=noise, resolution=16, latent_noise_scale=0.5)
    eng.clip_to_sample(frames, noise=noise, latent_noise=noise, resolution=16, latent_noise_scale=1.5)   # > 1 is allowed
    assert log["inference"][-1][2] == 1.5
    x = torch.zeros(3, 5, 16, 32)
    with pytest.raises(ValueError, match="input_noise"):
        eng.clip_to_sample(frames, resolution=16, input_noise_scale=0.5, input_noise=x[:, :4])
