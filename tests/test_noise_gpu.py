"""-m gpu: the generation-noise kernels (csrc/noise.cu) bit for bit against the torch restatement run on the same GPU
(oracle/noise_oracle.py), the device coefficients, the draws against randn_like on the reference's strides, and the
noise and batch options inside the engine's clip runner."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import noise_oracle as no
from oracle.make_noise_golden import INPUT_CASES, LATENT_CASES

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
SCALES = (0.05, 0.3, 0.5, 1.0)


@pytest.fixture(scope="module")
def nz(pkg):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.noise")


def bf(a):
    return torch.from_numpy(np.asarray(a)).to(torch.bfloat16).cuda()


def relaid(nz, n, layout):
    buf = nz.input_noise_buffer(n.shape, "cuda", layout)
    buf.copy_(n)
    return buf


def test_input_noise_bit_exact(nz):
    """Every noise memory order the reference's clip can have, at the golden sizes and at 3x5x2160x3840."""
    clips = []
    for name in INPUT_CASES:
        g = np.load(os.path.join(GOLD, name + ".npz"))
        clips += [(bf(g[f"tv{i}"]), bf(g[f"draw{i}"])) for i in range(len(g["encode_frames"]))]
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.rand(3, 5, 2160, 3840, device="cuda", generator=gen) * 2 - 1).to(torch.bfloat16)
    clips.append((x, nz.draw_input_noise(x.shape, gen, "cuda")))
    clips.append((x[:, :, :36, :50].contiguous(), torch.randn(3, 5, 36, 50, device="cuda", generator=gen)))  # scalar path
    for tv, n in clips:
        tv = tv.contiguous()
        for layout in (nz.TCHW, nz.CTHW, nz.THWC):
            nl = relaid(nz, n.to(torch.bfloat16), layout)
            for s in SCALES:
                out = nz.add_input_noise(tv, nl, s)
                assert torch.equal(out, no.input_noise(tv, nl, s)), (tuple(tv.shape), layout, s)
    assert torch.equal(nz.add_input_noise(x, torch.zeros_like(x), 0.0), x)


def test_condition_bit_exact(nz):
    shapes = [(2, 270, 480, 16), (1, 135, 240, 16)] + [tuple(np.load(os.path.join(GOLD, n + ".npz"))["latent"].shape)
                                                        for n in LATENT_CASES]
    gen = torch.Generator(device="cuda").manual_seed(9)
    for shape in shapes:
        latent = torch.randn(shape, device="cuda", generator=gen).to(torch.bfloat16)
        noise = torch.randn(shape, device="cuda", generator=gen, dtype=torch.bfloat16)
        r = nz.draw_latent_noise(shape, gen, "cuda")
        T, h, w, c = shape
        old = torch.cat([noise, latent, torch.ones(T, h, w, 1, device="cuda", dtype=torch.bfloat16)], -1)
        plain = nz.sr_condition(noise, latent)
        assert torch.equal(plain, old.view(T * h * w, 2 * c + 1)) and torch.equal(plain, no.sr_condition(noise, latent))
        for s in SCALES:
            coef = nz.latent_noise_coefficients(s, shape, "cuda")
            got = nz.sr_condition(noise, latent, r, coef)
            assert torch.equal(got, no.sr_condition(noise, latent, r, s)), (shape, s)


def test_device_coefficients_equal_the_oracle(nz):
    for s in (0.01, 0.05, 0.3, 0.5, 0.77, 1.0, 1.5):
        for (h, w) in ((1, 1), (1, 9), (5, 7), (90, 160), (270, 480), (135, 240), (256, 256)):
            a, b = nz.latent_noise_coefficients(s, (3, h, w, 16), "cuda")
            ao, bo = no.coefficients(s, (3, h, w, 16), "cuda")
            assert torch.equal(a, ao) and torch.equal(b, bo), (s, h, w)


def test_draws_equal_randn_like_on_the_reference_strides(nz):
    """What set_seed + randn_like give on the reference's tensors: the transformed clips of four batches from one
    generator, in each memory order the reference's transform leaves ((t h w c), (t c h w), (c t h w)), then the DiT
    noise and r (channels-last views of c t h w memory)."""
    shape = (3, 5, 64, 96)
    layouts = [nz.THWC, nz.TCHW, nz.CTHW, nz.THWC]
    perms = {nz.TCHW: no.TCHW, nz.CTHW: no.CTHW, nz.THWC: no.THWC}
    latent = (2, 8, 12, 16)
    with torch.random.fork_rng(devices=[0]):
        torch.cuda.manual_seed(42 + 1_000_000)
        ref_in = [torch.randn_like(no.laid_out(shape, perms[lay], "cuda")) for lay in layouts]
        torch.cuda.manual_seed(42)
        lat = torch.empty((16, 2, 8, 12), device="cuda", dtype=torch.bfloat16).permute(1, 2, 3, 0)
        base = torch.randn_like(lat)
        ref_r = torch.randn_like(base)
    assert ref_in[0].stride() == (1, 64 * 96 * 3, 96 * 3, 3)
    g = nz.input_generator(42, "cuda")
    for ref, lay in zip(ref_in, layouts):
        got = nz.draw_input_noise(shape, g, "cuda", lay)
        assert torch.equal(got, ref) and got.stride() == ref.stride(), lay
    ins, base_o, r_o = no.draws(42, [(shape, perms[lay]) for lay in layouts], latent, "cuda")
    assert all(torch.equal(a, b) for a, b in zip(ins, ref_in)) and torch.equal(r_o, ref_r)
    g = torch.Generator(device="cuda").manual_seed(42)
    noise = torch.randn(latent, generator=g, device="cuda", dtype=torch.bfloat16)      # the engine's DiT noise
    assert torch.equal(noise.flatten(), base.permute(3, 0, 1, 2).flatten())           # same memory, other layout
    assert torch.equal(nz.draw_latent_noise(latent, g, "cuda"), ref_r)


def test_reference_transform_layouts_hold_on_the_gpu():
    """The memory orders the goldens record on the CPU are those of the reference's transform on the GPU as well: its
    steps (generation_utils.py:72-84: torchvision bicubic antialiased resize, clamp, zero pad to 16, normalise) and the
    4n+1 concatenation (generation_phases.py:109-124), run here on CUDA tensors."""
    import torchvision.transforms.functional as TVF

    def transform(v, size):
        v = TVF.resize(v, size, TVF.InterpolationMode.BICUBIC, antialias=True)
        v = torch.clamp(v, 0.0, 1.0)
        H, W = v.shape[-2:]
        if H % 16 or W % 16:
            v = torch.nn.functional.pad(v, (0, (16 - W % 16) % 16, 0, (16 - H % 16) % 16), mode="constant", value=0.0)
        v = TVF.normalize(v, [0.5], [0.5])
        return v.permute(1, 0, 2, 3)

    def padded_4n1(frames):                                                   # 4 frames -> [f0 .. f3, f2] as c t h w
        c = frames.permute(0, 3, 1, 2).permute(1, 0, 2, 3)
        return torch.cat([c, c[:, 2:3]], 1).permute(1, 0, 2, 3)

    frames = torch.rand(5, 20, 28, 3, device="cuda").to(torch.bfloat16)
    tv = transform(frames.permute(0, 3, 1, 2), 26)                            # 4n+1 frames: (t h w c)
    assert tv.stride() == no.laid_out(tv.shape, no.THWC, "cuda").stride()
    tv = transform(padded_4n1(frames[:4]), 26)                                # padded, resized: (t c h w)
    assert tv.stride() == no.laid_out(tv.shape, no.TCHW, "cuda").stride()
    same = torch.rand(4, 16, 32, 3, device="cuda").to(torch.bfloat16)
    tv = transform(padded_4n1(same), 16)                                      # padded, not resized or padded: (c t h w)
    assert tv.stride() == no.laid_out(tv.shape, no.CTHW, "cuda").stride()


@pytest.fixture(scope="module")
def engine(pkg):
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    cfg = dit.dit_config("3b", dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64)
    return pipeline.SeedVR2Engine(cfg, pkg.weights.synth_dit_state_dict(cfg, seed=1),
                                  pkg.weights.synth_vae_state_dict(seed=2), torch.randn(58, 64))


def test_engine_clip_with_both_noises(nz, engine):
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    preprocess = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.preprocess")
    frames4 = torch.rand(5, 36, 52, 4, generator=torch.Generator().manual_seed(3)).cuda()
    frames = frames4[..., :3].contiguous()
    kw = dict(resolution=72, input_noise_scale=0.6, latent_noise_scale=0.25)
    sample, style = engine.clip_to_sample(frames, seed=11, **kw)
    # composition of the public pieces with the oracle's blends and the same draws
    x = preprocess.VideoTransform(72, 0).run(frames, channels_last=True)
    layout = engine.input_noise_layout(frames, 72)
    assert layout == nz.THWC                                                    # 5 frames: no temporal padding
    n_in = nz.draw_input_noise(x.shape, nz.input_generator(11, "cuda"), "cuda", layout)
    latent = engine.vae_encode(no.input_noise(x, n_in, 0.6).contiguous())
    g = torch.Generator(device="cuda").manual_seed(11)
    noise = torch.randn(latent.shape, generator=g, device="cuda", dtype=torch.bfloat16)
    r = nz.draw_latent_noise(latent.shape, g, "cuda")
    T, h, w, c = latent.shape
    vid = no.sr_condition(noise, latent, r, 0.25)
    v = engine.dit(vid, engine.txt, [[T, h, w]], [[engine.txt.shape[0]]]).vid_sample
    y = engine.vae_decode(noise - v.view(T, h, w, c))
    H, W = preprocess.VideoTransform(72, 0).true_size(36, 52)
    assert torch.equal(sample, y[:, :5, :H, :W].permute(1, 0, 2, 3))
    assert torch.equal(style, x[:, :5, :H, :W].permute(1, 0, 2, 3))           # the style stays clean
    # explicit draws give the same result; no host synchronisation
    out = engine.upscale_clip(frames, seed=11, **kw)
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = engine.upscale_clip(frames, noise=noise, latent_noise=r, input_noise=n_in, **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(again, out)
    # RGBA: the noise touches the RGB only
    rgba = engine.upscale_clip(frames4, seed=11, keep_alpha=True, **kw)
    assert torch.equal(rgba[..., :3], out)
    # graph replay: the first replay sees the first input draw, the second the next one
    gc = engine.graphed(frames, seed=11, **kw)
    assert torch.equal(gc(frames, clone=True), out)
    g_in = nz.input_generator(11, "cuda")
    nz.draw_input_noise(x.shape, g_in, "cuda", layout)
    second = nz.draw_input_noise(x.shape, g_in, "cuda", layout)
    assert torch.equal(gc(frames, clone=True), engine.upscale_clip(frames, seed=11, input_noise=second, **kw))
    assert torch.equal(gc(frames, input_noise=n_in), out)
    # a 4-frame clip is 4n+1-padded and resized: its draw is (t c h w) memory
    assert engine.input_noise_layout(frames[:4], 72) == nz.TCHW
    n4 = nz.draw_input_noise(x.shape, nz.input_generator(11, "cuda"), "cuda", nz.TCHW)
    assert torch.equal(engine.upscale_clip(frames[:4], seed=11, **kw),
                       engine.upscale_clip(frames[:4], seed=11, input_noise=n4, **kw))


def test_engine_video_overlap_uniform_prepend_noise(engine):
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    nz = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.noise")
    frames = torch.rand(10, 36, 52, 3, generator=torch.Generator().manual_seed(7)).cuda()
    kw = dict(resolution=72, color_correction="wavelet", seed=5)
    vid = engine.upscale_video(frames, batch_size=5, temporal_overlap=2, uniform_batch_size=True, prepend_frames=2,
                               input_noise_scale=0.5, latent_noise_scale=0.2, **kw)
    pre = pipeline.pad_video_temporal(frames, count=2, prepend=True)
    gen = nz.input_generator(5, "cuda")

    def clip(a, b):
        batch = pre[a:b]
        if b - a < 5:
            batch = pipeline.pad_video_temporal(batch, count=5 - (b - a))
        s, st = engine.clip_to_sample(batch, seed=5, resolution=72, input_noise_scale=0.5, latent_noise_scale=0.2,
                                      input_generator=gen)
        return s[:b - a].contiguous(), st[:b - a].contiguous()

    post = lambda s, st: engine.finish_clip(s, st, color_correction="wavelet")
    ref = pipeline.run_batched(12, 5, 2, clip, shard.blend_overlap, post)[2:]
    assert vid.shape == (10, 72, 104, 3) and torch.equal(vid, ref)
