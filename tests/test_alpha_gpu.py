"""-m gpu: the alpha path of RGBA clips (csrc/alpha.cu through the C ABI and the ``alpha`` host mirror) against the
goldens made by the reference's alpha_upscaling.py and against the fp32 torch oracle on the GPU, and the engine's
RGBA clips (keep_alpha) with synthetic weights."""
import importlib
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import alpha_oracle as ao

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def am(pkg):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.alpha")


def run_kind(am, src, channels, rgb, kind):
    """svr2_alpha_upscale with an explicit out_kind; returns (out, scratch)."""
    T, h, w = src.shape[:3]
    H, W = rgb.shape[2:]
    out = torch.empty(T, H, W, device="cuda", dtype=torch.float32)
    scratch = am._scratch(T, h, w, H, W, "cuda")
    am._run(src, channels, rgb, out, kind, scratch)
    return out, scratch


def check_against(out, ref, taps, binary, tag):
    """Against the goldens, which the reference made on the CPU.  The kernel follows torch's CUDA rounding, as the
    reference does on its GPU tensors: the guide's mean is the channel sum times an fp32 factor there and a true
    division by 3 on the CPU, and the CPU's box sums need not add in the same order.  Those roundings move fp32 alphas
    by a few 1e-6 and flip a binary-mask threshold where q sits that close to it, hence bounds this loose; the exact
    checks are tests/test_alpha_elementwise_gpu.py and test_full_path_at_4k_vs_gpu_oracle.  Gradient alphas: max |d| <= 1e-4, bf16 casts >= 99.5 % equal and otherwise one bf16 ulp apart (the ulp taken at
    no less than 2^-8: below that, fp32 noise of 1e-9 is already several bf16 ulps of an invisible alpha).  Binary masks:
    <= 0.1 % of the pixels differ by more than 1e-4, each one where the oracle sat within 1e-4 of a threshold."""
    out, ref = out.float().cpu().reshape(ref.shape), ref.float().cpu()
    d = (out - ref).abs()
    if not binary:
        assert d.max().item() <= 1e-4, (tag, d.max().item())
        ob, rb = out.to(torch.bfloat16), ref.to(torch.bfloat16)
        same = (ob == rb).float().mean().item()
        ulp = rb.float().abs().clamp(min=2 ** -8) * 2 ** -7
        assert same >= 0.995 and ((ob.float() - rb.float()).abs() <= ulp).all(), (tag, same)
    else:
        bad = d > 1e-4
        assert bad.float().mean().item() <= 1e-3, (tag, bad.float().mean().item())
        near = ao.threshold_distance({k: v.float().cpu() for k, v in taps.items() if torch.is_tensor(v)}) <= 1e-4
        assert not (bad & ~near.reshape(bad.shape)).any(), (tag, int((bad & ~near.reshape(bad.shape)).sum()))


@pytest.mark.parametrize("name", list(ao.CASES))
def test_sobel_edges_bit_exact_on_golden_inputs(am, name):
    _, rgb = ao.make_inputs(**ao.CASES[name])
    got = am.detect_edges_batch(rgb.cuda())
    assert torch.equal(got.cpu(), ao.detect_edges_batch(rgb))


def test_sobel_edges_bit_exact_at_4k(am):
    g = torch.Generator(device="cuda").manual_seed(5)
    base = F.interpolate(torch.rand(2, 3, 68, 120, generator=g, device="cuda"), size=(2160, 3840), mode="bicubic")
    rgb = (base * 2.2 - 1.1 + 0.05 * torch.randn(2, 3, 2160, 3840, generator=g, device="cuda")).to(torch.bfloat16)
    assert torch.equal(am.detect_edges_batch(rgb), ao.detect_edges_batch(rgb))


@pytest.mark.parametrize("shape", [(2, 37, 53, 90, 128), (1, 90, 128, 37, 53), (3, 72, 128, 216, 384),
                                   (2, 100, 160, 40, 64), (1, 150, 75, 20, 10), (1, 1, 64, 9, 200)])
def test_alpha_resize_equals_torch_cuda(am, shape):
    """The base resize is torch's CUDA kernel (what the reference runs on its GPU alpha) bit for bit: the tap tables
    and accumulation of pre.cu's resize (tests/test_resize_elementwise_gpu.py), here on mask-like alphas, up, down
    (2.5x and the 7.5x limit) and from a one-pixel-high input.  torch's CPU kernel rounds its taps differently and lies
    up to ~6e-6 from the CUDA result; the bound against it is 1e-5."""
    T, h, w, H, W = shape
    g = torch.Generator().manual_seed(h * w)
    frames = torch.rand(T, h, w, 4, generator=g)
    frames[..., 3] = (torch.rand(T, h, w, generator=g) > 0.5).float() * 0.9 + 0.05 * torch.rand(T, h, w, generator=g)
    rgb = torch.zeros(T, 3, H, W, device="cuda", dtype=torch.bfloat16)
    for src in (frames.cuda(), frames.cuda().to(torch.bfloat16), frames.cuda().half()):
        got, _ = run_kind(am, src, 4, rgb, am.OUT_RESIZE)
        a = src[..., 3].to(torch.bfloat16).float()[:, None]
        ref_cuda = F.interpolate(a, size=(H, W), mode="bicubic", align_corners=False, antialias=True).clamp(0, 1)[:, 0]
        assert torch.equal(got, ref_cuda), (src.dtype, int((got != ref_cuda).sum()))
        ref = F.interpolate(a.cpu(), size=(H, W), mode="bicubic", align_corners=False, antialias=True).clamp(0, 1)[:, 0]
        assert (got.cpu() - ref).abs().max().item() <= 1e-5, src.dtype


@pytest.mark.parametrize("name", list(ao.CASES))
def test_full_path_vs_reference_goldens(am, name):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    alpha, rgb = ao.make_inputs(**ao.CASES[name])
    out = am.edge_guided_alpha_upscale(alpha.cuda(), None, rgb.cuda())
    assert out.shape == alpha.shape[:2] + rgb.shape[2:] and out.dtype == torch.float32
    taps = {}
    ao.edge_guided_alpha_upscale(alpha, rgb, taps)
    check_against(out, torch.from_numpy(g["out"]), taps, bool(g["meta"][-1]), name)


@pytest.mark.parametrize("kind", ["binary", "gradient"])
def test_full_path_at_4k_vs_gpu_oracle(am, kind):
    """The 4K shard shape: 5 frames, 720p alpha -> 2160 x 3840, bit for bit against the reference's op chain run by
    torch on the GPU, as the reference runs it."""
    alpha, rgb = ao.make_inputs(5, 720, 1280, 2160, 3840, kind, seed=11)
    alpha, rgb = alpha.cuda(), rgb.cuda()
    out = am.edge_guided_alpha_upscale(alpha, None, rgb)
    taps = {}
    ref = ao.edge_guided_alpha_upscale(alpha, rgb, taps)
    assert taps["binary"] == (kind == "binary")
    assert torch.equal(out, ref), (kind, int((out != ref).sum()))


# ---- the engine with synthetic weights
@pytest.fixture(scope="module")
def engine(pkg):
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    cfg = dit.dit_config("3b", dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64)
    return pipeline.SeedVR2Engine(cfg, pkg.weights.synth_dit_state_dict(cfg, seed=1),
                                  pkg.weights.synth_vae_state_dict(seed=2), torch.randn(58, 64))


def rgba_frames(T, seed):
    a, _ = ao.make_inputs(T, 36, 52, 36, 52, "binary", seed=seed)
    frames = torch.rand(T, 36, 52, 4, generator=torch.Generator().manual_seed(seed))
    frames[..., 3] = a[:, 0].float()
    return frames.cuda()


@pytest.mark.parametrize("cc", ["none", "wavelet", "lab"])
def test_engine_rgba_clip(am, engine, cc):
    frames4 = rgba_frames(5, 3)
    kw = dict(resolution=72, color_correction=cc)
    noise = torch.randn(engine.latent_shape(frames4, 72), generator=torch.Generator().manual_seed(1)).cuda()
    out = engine.upscale_clip(frames4, noise=noise, keep_alpha=True, **kw)
    plain = engine.upscale_clip(frames4, noise=noise, **kw)
    assert out.shape == (5, 72, 104, 4) and plain.shape == (5, 72, 104, 3)
    assert torch.equal(out[..., :3], plain)
    assert torch.equal(plain, engine.upscale_clip(frames4[..., :3].contiguous(), noise=noise, **kw))
    sample = engine.clip_to_sample(frames4, noise=noise, resolution=72)[0].contiguous()
    ref = am.edge_guided_alpha_upscale(frames4[..., 3][:, None], None, sample)[:, 0].to(torch.bfloat16)
    assert torch.equal(out[..., 3], ref)
    if cc == "lab":
        torch.cuda.set_sync_debug_mode("error")         # the RGBA clip makes no host synchronisation
        try:
            again = engine.upscale_clip(frames4, noise=noise, keep_alpha=True, **kw)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert torch.equal(again, out)
        gc = engine.graphed(frames4, noise=noise, keep_alpha=True, **kw)
        assert torch.equal(gc(frames4), out)
        frames_b = rgba_frames(5, 4)
        assert torch.equal(gc(frames_b), engine.upscale_clip(frames_b, noise=noise, keep_alpha=True, **kw))


def test_engine_rgba_video_per_slice_alpha(am, engine):
    """upscale_video with temporal_overlap = 2: the RGB is that of the RGB path, and every post-processed slice's alpha
    is the alpha of exactly that slice's input frames, refined against the slice's decoded RGB after the cross-fade."""
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    frames4 = rgba_frames(13, 7)
    kw = dict(resolution=72, color_correction="wavelet")
    vid = engine.upscale_video(frames4, batch_size=5, temporal_overlap=2, keep_alpha=True, **kw)
    assert vid.shape == (13, 72, 104, 4)
    assert torch.equal(vid[..., :3], engine.upscale_video(frames4, batch_size=5, temporal_overlap=2, **kw))
    slices = []

    def clip(a, b):
        s, st, src = engine.clip_to_sample(frames4[a:b], seed=42, resolution=72, keep_alpha=True)
        return s.contiguous(), (st.contiguous(), src)

    def post(sample, style):
        slices.append((sample.clone(), style[1]))
        return torch.empty(sample.shape[0], 1, device="cuda")

    pipeline.run_batched(13, 5, 2, clip, shard.blend_overlap, post)
    start = 0
    for sample, src in slices:
        n = sample.shape[0]
        assert torch.equal(src, frames4[start:start + n])
        ref = am.edge_guided_alpha_upscale(src[..., 3][:, None], None, sample)[:, 0].to(torch.bfloat16)
        assert torch.equal(vid[start:start + n, ..., 3], ref), start
        start += n
    assert start == 13
