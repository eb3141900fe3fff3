"""-m gpu: the 8-bit output kernel (svr2_sample_to_image_u8) and the 8-bit input loads bit for bit against numpy
restatements of the reference CLI, SeedVR2Engine.stream_video against upscale_video on a small synthetic engine, and
its device memory against the video's length."""
import importlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mods(pkg):
    name = "comfyui_seedvr2_videoupscaler_b200."
    return {m: importlib.import_module(name + m) for m in ("color_fix", "preprocess", "alpha", "pipeline", "dit")}


def all_bf16():
    return torch.from_numpy(np.arange(65536, dtype=np.uint16).view(np.int16)).view(torch.bfloat16)


def cli_bytes(x: torch.Tensor) -> np.ndarray:
    """(frames.cpu().numpy() * 255.0).astype(np.uint8) of inference_cli.py:763 on a [0, 1] bf16 image."""
    return (x.float().cpu().numpy() * 255.0).astype(np.uint8)


def cli_frames(u8: np.ndarray) -> torch.Tensor:
    """The CLI's frames read from 8-bit RGB(A): fp32 / 255, then fp16 (inference_cli.py:613, 697)."""
    return torch.from_numpy(u8.astype(np.float32) / 255.0).to(torch.float16)


def test_u8_formatting_every_bf16_value(mods):
    cf = mods["color_fix"]
    v = all_bf16()
    for shape in ((1, 256, 256), (1, 1, 65537)):                 # the 4-pixel path and the one-pixel path
        n = shape[1] * shape[2]
        idx = torch.arange(n) % 65536
        # every pattern in every channel, at different pixels
        sample = torch.stack([v[(idx + k * 21845) % 65536] for k in range(3)]).view(1, 3, shape[1], shape[2])
        got = cf.sample_to_image_u8(sample.cuda()).cpu().numpy()
        assert got.shape == (1, shape[1], shape[2], 3)
        ref_t = sample.clamp(-1, 1).mul(0.5).add(0.5).permute(0, 2, 3, 1)       # the reference's bf16 ops, on the CPU
        finite = ~torch.isnan(ref_t)
        with np.errstate(invalid="ignore"):
            ref = cli_bytes(ref_t)
        assert np.array_equal(got[finite.numpy()], ref[finite.numpy()])
        # NaN samples clamp to -1 as in the bf16 formatting kernel: byte 0, the CLI's bytes of that kernel's image
        assert np.array_equal(got, cli_bytes(cf.sample_to_image(sample.cuda())))
        assert (got[~finite.numpy()] == 0).all()
        # alpha: channel 3 of the bf16 RGBA image, * 255 and truncated, no normalisation
        image = torch.zeros(1, shape[1], shape[2], 4, dtype=torch.bfloat16)
        image[..., 3] = v[idx].view(1, shape[1], shape[2])
        got4 = cf.sample_to_image_u8(sample.cuda(), image.cuda()).cpu().numpy()
        assert np.array_equal(got4[..., :3], got)
        with np.errstate(over="ignore", invalid="ignore"):
            a = image[..., 3].float().numpy() * np.float32(255.0)
            ref_a = a.astype(np.uint8)
        defined = np.isfinite(a) & (a > -1) & (a < 256)           # where numpy's float -> uint8 cast is defined
        assert np.array_equal(got4[..., 3][defined], ref_a[defined])
        assert (got4[..., 3][~defined] == np.where(a[~defined] >= 256, 255, 0)).all()   # saturated, NaN -> 0
    with pytest.raises(Exception):
        cf.sample_to_image_u8(torch.zeros(1, 3, 2, 2, dtype=torch.bfloat16))      # no CPU fallback


def byte_frames(T=2, h=16, w=16, binary=False):
    """Every byte value in every channel (RGB rotated against each other), alpha graded or a 0/255 mask."""
    v = np.arange(h * w * T) % 256
    rgba = np.stack([v, (v + 85) % 256, (v * 7 + 3) % 256, (v * 13) % 256], -1).reshape(T, h, w, 4).astype(np.uint8)
    if binary:
        rgba[..., 3] = np.where(np.arange(h * w * T).reshape(T, h, w) % 5 == 0, 0, 255)
    return rgba


def test_u8_input_loads_as_the_cli_reads_it(mods):
    pre, al = mods["preprocess"], mods["alpha"]
    u8 = byte_frames()
    f16 = cli_frames(u8)
    for res in (16, 40, 12):                                     # identity size, up- and down-scale
        for x8, x16 in ((u8, f16), (u8[..., :3], f16[..., :3])):
            a = pre.preprocess_frames(torch.from_numpy(np.ascontiguousarray(x8)).cuda(), res)
            b = pre.preprocess_frames(x16.contiguous().cuda(), res)
            assert torch.equal(a, b), res
        # the channels-first layout after the reference's cap (two resizes) too
        a = pre.VideoTransform(res, 20).run(torch.from_numpy(u8).cuda(), channels_last=True)
        assert torch.equal(a, pre.VideoTransform(res, 20).run(f16.cuda(), channels_last=True)), res
    g = torch.Generator().manual_seed(4)
    for binary in (False, True):
        u8 = byte_frames(binary=binary)
        f16 = cli_frames(u8)
        for H, W in ((16, 16), (40, 40)):
            sample = (torch.rand(2, 3, H, W, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
            img8 = torch.zeros(2, H, W, 4, dtype=torch.bfloat16, device="cuda")
            img16 = torch.zeros_like(img8)
            al.upscale_into_image(torch.from_numpy(u8).cuda(), sample, img8)
            al.upscale_into_image(f16.cuda(), sample, img16)
            assert torch.equal(img8, img16), (binary, H)


@pytest.fixture(scope="module")
def engine(pkg, mods):
    cfg = mods["dit"].dit_config("3b", dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64)
    return mods["pipeline"].SeedVR2Engine(cfg, pkg.weights.synth_dit_state_dict(cfg, seed=1),
                                          pkg.weights.synth_vae_state_dict(seed=2), torch.randn(58, 64))


def collect(pieces):
    nxt, out = 0, []
    for first, t in pieces:
        assert first == nxt and t.device.type == "cpu" and t.is_pinned()
        nxt += t.shape[0]
        out.append(t)
    return torch.cat(out, 0)


def test_stream_video_equals_upscale_video(engine):
    g = torch.Generator().manual_seed(7)
    frames = torch.rand(11, 36, 52, 4, generator=g)
    cases = [dict(temporal_overlap=0),
             dict(temporal_overlap=2, color_correction="lab", input_noise_scale=0.5, latent_noise_scale=0.2),
             dict(temporal_overlap=2, uniform_batch_size=True, prepend_frames=2, color_correction="wavelet_adaptive"),
             dict(temporal_overlap=2, keep_alpha=True, color_correction="lab", prepend_frames=1),
             dict(temporal_overlap=0, keep_alpha=True, uniform_batch_size=True, input_noise_scale=0.3)]
    sizes = [3, 1, 4, 2, 1]                                          # chunks of 3, 1, 4, 2 and 1 frames
    for case in cases:
        kw = dict(batch_size=5, resolution=72, seed=3, **case)
        video = frames if case.get("keep_alpha") else frames[..., :3].contiguous()
        ref = engine.upscale_video(video.cuda(), **kw)
        assert ref.shape == (11, 72, 104, video.shape[-1])
        chunks = lambda: iter(video.split(sizes))
        got = collect(engine.stream_video(video, out_dtype=torch.bfloat16, **kw))
        assert got.dtype == torch.bfloat16 and torch.equal(got, ref.cpu()), case
        got8 = collect(engine.stream_video(chunks(), **kw))
        assert got8.dtype == torch.uint8 and np.array_equal(got8.numpy(), cli_bytes(ref)), case
        assert torch.equal(collect(engine.stream_video(chunks(), out_dtype=torch.bfloat16, **kw)), ref.cpu()), case
        assert torch.equal(collect(engine.stream_video(video.cuda(), **kw)), got8), case


def test_u8_frames_equal_the_cli_float_frames(engine):
    u8 = np.random.default_rng(5).integers(0, 256, (7, 36, 52, 4), dtype=np.uint8)
    kw = dict(batch_size=5, temporal_overlap=2, resolution=72, seed=9, color_correction="lab", keep_alpha=True)
    ref = collect(engine.stream_video(cli_frames(u8), **kw))
    got = collect(engine.stream_video(iter(torch.from_numpy(u8).split(3)), **kw))
    assert got.shape == (7, 72, 104, 4) and torch.equal(got, ref)
    assert torch.equal(engine.upscale_video(torch.from_numpy(u8).cuda(), **kw), engine.upscale_video(cli_frames(u8).cuda(), **kw))


def test_device_memory_does_not_grow_with_the_video(engine):
    """1080p output, batches of 5 with overlap 2: 45 frames peak less than 32 MiB above 15 frames (one more held batch
    of output would be ~62 MiB of bf16 samples alone)."""
    src = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (45, 270, 480, 3), dtype=np.uint8))
    kw = dict(batch_size=5, temporal_overlap=2, resolution=1080, seed=1)

    def peak(n):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        frames = 0
        for _, t in engine.stream_video(iter(src[:n].split(4)), **kw):
            assert t.shape[1:] == (1080, 1920, 3)
            frames += t.shape[0]
        torch.cuda.synchronize()
        assert frames == n
        return torch.cuda.max_memory_allocated() - base

    peak(15)                                                    # shapes, tables and the resident workspace
    p15, p45 = peak(15), peak(45)
    print(f"peak above the resident state: 15 frames {p15 / 2**20:.1f} MiB, 45 frames {p45 / 2**20:.1f} MiB")
    assert p45 - p15 < 32 * 2 ** 20, (p15, p45)
