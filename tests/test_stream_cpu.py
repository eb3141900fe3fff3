"""CPU: the streaming batch loop (pipeline.final_slices / iter_batched / FrameSource) against run_batched, and
SeedVR2Engine.stream_video's host logic with the GPU stages stubbed (the kernels are covered by test_stream_gpu.py)."""
import importlib
import weakref

import pytest
import torch


@pytest.fixture(scope="module")
def pipeline(pkg):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")


def chunkings(frames, seed):
    """The same video as one tensor, as chunks of one frame and as chunks of random sizes (empty ones included)."""
    g = torch.Generator().manual_seed(seed)
    sizes, n = [], frames.shape[0]
    while n > 0:
        k = min(n, int(torch.randint(0, 7, (1,), generator=g)))
        sizes.append(k)
        n -= k
    pieces, pos = [], 0
    for k in sizes:
        pieces.append(frames[pos:pos + k])
        pos += k
    return {"tensor": frames, "ones": list(frames.split(1)), "random": iter(pieces)}


def decoded_for(a, b):
    g = torch.Generator().manual_seed(a * 1000 + b)
    return torch.rand(b - a, 3, 1, 2, generator=g).to(torch.bfloat16)


def test_generator_matches_run_batched_and_holds_a_bounded_number_of_frames(pipeline):
    blend = lambda p, c: (p.float() * 0.25 + c.float() * 0.75).to(torch.bfloat16)
    post = lambda smp, sty: (smp.float() * 0.5 + sty.float() * 0.25).permute(0, 2, 3, 1)
    for total in range(1, 41):
        frames = torch.rand(total, 3, 1, 2, generator=torch.Generator().manual_seed(total)).to(torch.bfloat16)
        for bs in range(1, 10):
            for ov in range(0, 11):
                ref = pipeline.run_batched(total, bs, ov, lambda a, b: (decoded_for(a, b), frames[a:b].clone()),
                                           blend, post)
                eff = pipeline.batch_ranges(total, bs, ov)[1]
                for name, video in chunkings(frames, total * 100 + bs * 11 + ov).items():
                    source = pipeline.FrameSource(video)
                    count = dict(returned=0, trimmed=0, posted=0)
                    alive = []

                    def clip(a, b):
                        held = count["returned"] - count["trimmed"] - count["posted"]
                        live = sum(t().shape[0] for t in alive if t() is not None)
                        assert held < bs + eff and live <= bs + eff, (total, bs, ov, name, a, held, live)
                        x = source.take(a, b)
                        assert torch.equal(x, frames[a:b]), (total, bs, ov, name, a, b)
                        s = decoded_for(a, b)
                        alive.append(weakref.ref(s))
                        count["returned"] += b - a
                        return s, x

                    def counted_blend(p, c):
                        count["trimmed"] += c.shape[0]
                        return blend(p, c)

                    def counted_post(smp, sty):
                        count["posted"] += smp.shape[0]
                        return post(smp, sty)

                    got = torch.cat(list(pipeline.iter_batched(source, bs, ov, clip, counted_blend, counted_post)), 0)
                    assert got.shape == ref.shape and torch.equal(got, ref), (total, bs, ov, name)


def test_frame_source_prepends_mirrored_frames_like_pad_video_temporal(pipeline):
    for total in range(1, 12):
        frames = torch.arange(total, dtype=torch.float32).view(total, 1, 1, 1)
        for p in range(0, 14):
            ref = pipeline.pad_video_temporal(frames, count=p, prepend=True) if p else frames
            for name, video in chunkings(frames, total * 31 + p).items():
                source = pipeline.FrameSource(video, prepend=p)
                assert source.fill(10 ** 6) == ref.shape[0] and source.channels == 1
                assert torch.equal(source.take(0, ref.shape[0]), ref), (total, p, name)
    source = pipeline.FrameSource(iter([torch.zeros(3, 1, 1, 1), torch.ones(4, 1, 1, 1)]))
    source.take(3, 5)
    with pytest.raises(IndexError):
        source.take(2, 4)                          # the first chunk has been let go


@pytest.fixture
def stub_engine(pkg, monkeypatch, pipeline):
    """Stages as in test_alpha_cpu.py's stand-ins, plus the 8-bit formatting as its torch restatement."""
    preprocess = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.preprocess")
    color_fix = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.color_fix")
    alpha = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.alpha")
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    gen_noise = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.noise")
    from oracle import noise_oracle as no
    eng = object.__new__(pipeline.SeedVR2Engine)
    eng.device = torch.device("cpu")

    def fake_run(self, x, channels_last):
        (H, W), _ = preprocess.resized_size(x.shape[1], x.shape[2], self.resolution, self.max_resolution)
        y = torch.nn.functional.interpolate(x[..., :3].permute(0, 3, 1, 2).float(), size=(H, W)).permute(1, 0, 2, 3)
        y = torch.nn.functional.pad(y, (0, (16 - W % 16) % 16, 0, (16 - H % 16) % 16))
        return (y * 2 - 1).to(torch.bfloat16).contiguous()

    def fake_alpha(src, sample, image):
        image[..., 3] = src[..., 3].float().mean(dim=(1, 2)).view(-1, 1, 1).to(image.dtype)
        return image

    to_image = lambda s_: (s_.float().permute(0, 2, 3, 1).clamp(-1, 1) * 0.5 + 0.5).to(torch.bfloat16)

    def fake_rgba(sample, image):
        image[..., :3] = to_image(sample)
        return image

    def fake_u8(sample, image_rgba=None):
        img = to_image(sample) if image_rgba is None else fake_rgba(sample, image_rgba.clone())
        return (img.float() * 255.0).to(torch.uint8)

    monkeypatch.setattr(preprocess.VideoTransform, "run", fake_run)
    monkeypatch.setattr(gen_noise, "add_input_noise", lambda x, n, scale: no.input_noise(x, n, scale).contiguous())
    # the decoded frame carries its encoder input (so that frames, batches and noise draws are told apart)
    eng.vae_encode = lambda x: x[0, ::4, ::8, ::8, None].expand(-1, -1, -1, 16).contiguous()
    eng.inference = lambda noise, latent, **kw: latent + noise * 0.01
    eng.clip_workspace = lambda T, Hp, Wp: None
    eng.vae_decode = lambda z: z[..., 0].repeat_interleave(4, 0)[: 4 * z.shape[0] - 3, None].expand(-1, 3, -1, -1) \
        .repeat_interleave(8, -2).repeat_interleave(8, -1).permute(1, 0, 2, 3).contiguous()
    monkeypatch.setattr(color_fix, "apply_color_correction",
                        lambda s_, st, mode, debug=None: ((s_.float() + st.float()) / 2).to(torch.bfloat16))
    monkeypatch.setattr(color_fix, "sample_to_image", to_image)
    monkeypatch.setattr(color_fix, "sample_to_image_rgba", fake_rgba)
    monkeypatch.setattr(color_fix, "sample_to_image_u8", fake_u8)
    monkeypatch.setattr(alpha, "upscale_into_image", fake_alpha)
    monkeypatch.setattr(shard, "blend_overlap", lambda p, c: ((p.float() + c.float()) / 2).to(p.dtype))
    return eng


def collect(pieces):
    """Concatenated frames of stream_video's output; the indices must follow each other from 0."""
    nxt, out = 0, []
    for first, t in pieces:
        assert first == nxt and t.shape[0] > 0 and t.device.type == "cpu"
        nxt += t.shape[0]
        out.append(t)
    return torch.cat(out, 0)


def test_stream_video_equals_upscale_video(stub_engine):
    eng = stub_engine
    g = torch.Generator().manual_seed(3)
    cases = [dict(total=13, batch_size=5, temporal_overlap=2), dict(total=13, batch_size=5, temporal_overlap=0),
             dict(total=11, batch_size=4, temporal_overlap=1, uniform_batch_size=True, prepend_frames=2),
             dict(total=7, batch_size=5, temporal_overlap=3, prepend_frames=3, keep_alpha=True),
             dict(total=3, batch_size=5, prepend_frames=4, uniform_batch_size=True),
             dict(total=2, batch_size=5, prepend_frames=9), dict(total=9, batch_size=4, prepend_frames=1, keep_alpha=True,
                                                               color_correction="lab"),
             dict(total=17, batch_size=5, temporal_overlap=4, input_noise_scale=0.3, latent_noise_scale=0.2)]
    for case in cases:
        total = case.pop("total")
        frames = torch.rand(total, 16, 24, 4, generator=g)
        frames[..., 3] = (torch.arange(total).float() / 16).view(total, 1, 1)
        kw = dict(resolution=16, seed=7, **case)
        ref = eng.upscale_video(frames, **kw)
        assert ref.shape[-1] == (4 if case.get("keep_alpha") else 3)
        for name, video in chunkings(frames, total).items():
            got = collect(eng.stream_video(video, out_dtype=torch.bfloat16, **kw))
            assert got.dtype == torch.bfloat16 and torch.equal(got, ref), (case, name)
        for name, video in chunkings(frames, total + 1).items():
            got = collect(eng.stream_video(video, **kw))
            assert got.dtype == torch.uint8 and torch.equal(got, (ref.float() * 255.0).to(torch.uint8)), (case, name)
    with pytest.raises(ValueError):
        next(eng.stream_video(frames, resolution=16, out_dtype=torch.float32))


def test_stream_video_yields_each_batch_before_reading_far_ahead(stub_engine, monkeypatch):
    """Slices come out while the input is still being read: with overlap 2 and batches of 5, the frames of the first
    batch are out before the input has gone past the third batch."""
    eng = stub_engine
    read = []

    def chunks():
        for i in range(30):
            read.append(i)
            yield torch.rand(1, 16, 24, 3)

    out = eng.stream_video(chunks(), batch_size=5, temporal_overlap=2, resolution=16)
    first, t = next(out)
    assert first == 0 and t.shape[0] == 5 and len(read) <= 11
    rest = collect(((f - 5, x) for f, x in out))
    assert rest.shape[0] == 25
