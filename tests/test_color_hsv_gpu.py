"""-m gpu: the hsv and wavelet_adaptive colour corrections (csrc/hsv.cu, the fp32 wavelet level of csrc/post.cu, the
``color_fix`` host mirror) bit for bit against the fp32 torch restatement run on the same GPU (oracle/hsv_oracle.py),
against the goldens made by the reference's color_fix.py, and inside the engine's clip runner."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import color_oracle as co
from oracle import hsv_oracle as ho
from oracle.make_golden import color_inputs
from oracle.make_hsv_golden import HSV_CASES, edge_pixels

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def cf(pkg):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.color_fix")


def golden(name):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    return g, torch.from_numpy(g["content"]).to(torch.bfloat16), torch.from_numpy(g["style"]).to(torch.bfloat16)


def meets_golden(out, ref):
    """The reference's criterion for its own unstable sort: same saturation distribution, >= 35 dB."""
    sat = lambda x: co.saturation_map(x.float().cpu()).flatten().sort().values
    dsat = (sat(out) - sat(ref)).abs().mean().item()
    mse = ((out.float().cpu() - ref.float()) ** 2).mean().item()
    db = 99.0 if mse == 0 else 10 * np.log10(4.0 / mse)
    return dsat < 2e-3 and db > 35.0, (dsat, db)


def edge_clip(T, H, W, seed):
    """Random values plus the crafted corners of RGB -> HSV: gray, r=g / g=b ties, hues on both sides of every bin
    edge, h == 1 and maxc == 0."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(T, 3, H, W, generator=g) * 2 - 1
    px = [edge_pixels()]
    for b in range(12):            # hue b/12 +- a little: sector k = b // 2, fractional part (b % 2) / 2
        for d in (-1e-3, 0.0, 1e-3):
            h6 = (b / 2.0 + d * 6) % 6
            k, f = int(h6), h6 - int(h6)
            v, p, q, t = 1.0, 0.2, 1.0 - 0.8 * f, 0.2 + 0.8 * f
            rgb = [(v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q)][k]
            px.append(torch.tensor(rgb).view(3, 1) * 2 - 1)
    e = torch.cat(px, 1)
    flat = x.permute(1, 0, 2, 3).reshape(3, -1)
    flat[:, :e.shape[1]] = e
    return flat.reshape(3, T, H, W).permute(1, 0, 2, 3).contiguous().to(torch.bfloat16)


def test_rgb_hsv_round_trip_is_bit_exact(cf):
    """At most 100 pixels leave every bin unmatched: the output is the pure RGB -> HSV -> RGB round trip."""
    c = edge_clip(2, 7, 7, seed=1).cuda()
    s = edge_clip(2, 7, 7, seed=2).cuda()
    out = cf.hsv_saturation_histogram_match(c, s)
    h = ho._hsv(c)[:, 0]
    assert (h == 1.0).any() and ((h >= 11 / 12) & (h < 1)).any() and (h == 0).any()
    assert out.dtype == torch.bfloat16 and torch.equal(out.float(), ho.hsv_saturation_histogram_match(c, s))


def run_raw(svr2lib, c, s, wav=None):
    T, _, H, W = c.shape
    n = T * H * W
    need = svr2lib.load().svr2_hsv_scratch_bytes(n)
    scratch = torch.full((need,), 0xAB, device="cuda", dtype=torch.uint8)
    out = torch.empty_like(c)
    svr2lib.call("svr2_hsv_saturation_match_bf16", svr2lib.ptr(c), svr2lib.ptr(s), svr2lib.ptr(wav), svr2lib.ptr(out),
                 T, H * W, svr2lib.ptr(scratch), need, svr2lib.stream())
    hdr = scratch[:144].view(torch.int32).view(3, 12).cpu()
    return out, hdr


def test_bin_counts_and_qualify_flags(svr2lib):
    """The scratch header holds the reference's mask sizes (wrap pixels in bins 0 and 11) and the qualify flags;
    bins with exactly 100 and 101 pixels fall on both sides of the threshold."""
    def hue_pixels(b, k):        # k pixels of hue (b + 0.5) / 12 with varied saturation
        h6 = (b + 0.5) / 2.0
        i, f = int(h6), h6 - int(h6)
        sat = torch.linspace(0.2, 0.9, k)
        v, p, q, t = torch.ones(k), 1 - sat, 1 - sat * f, 1 - sat * (1 - f)
        rgb = [(v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q)][i]
        return torch.stack(rgb) * 2 - 1

    sizes_c = [150, 100, 101, 0, 120, 99, 101, 130, 101, 100, 200, 160]
    sizes_s = [140, 101, 101, 50, 101, 300, 100, 101, 111, 101, 0, 170]

    def clip(sizes):
        x = torch.cat([hue_pixels(b, k) for b, k in enumerate(sizes) if k], 1)
        n = x.shape[1]
        T, H = 2, 8
        W = -(-n // (T * H))
        pad = torch.full((3, T * H * W - n), -1.0)              # black: h = 0, bin 0
        x = torch.cat([x, pad], 1)[:, torch.randperm(T * H * W, generator=torch.Generator().manual_seed(n))]
        return x.reshape(3, T, H, W).permute(1, 0, 2, 3).contiguous().to(torch.bfloat16).cuda()

    c, s = clip(sizes_c), clip(sizes_s)
    out, hdr = run_raw(svr2lib, c, s)
    cc, sc = ho.bin_counts(c, s)
    assert hdr[0].tolist() == cc and hdr[1].tolist() == sc
    assert 100 in cc[1:] and 101 in cc and 100 in sc and 101 in sc
    assert hdr[2].tolist() == [int(a > 100 and b > 100) for a, b in zip(cc, sc)]
    assert torch.equal(out.float(), ho.hsv_saturation_histogram_match(c, s))


@pytest.mark.parametrize("name", list(HSV_CASES))
def test_hsv_goldens(cf, name):
    g, content, style = golden(name)
    c, s = content.cuda(), style.cuda()
    out = cf.hsv_saturation_histogram_match(c, s)
    diff = int((out.float() != ho.hsv_saturation_histogram_match(c, s)).sum())
    assert diff == 0, f"{diff} values differ from the GPU oracle"
    ok, why = meets_golden(out, torch.from_numpy(g["hsv"]))
    assert ok, why
    assert [ho.bin_counts(content, style)[0], ho.bin_counts(content, style)[1]] == g["counts"].tolist()


def single_hue_clip(T, H, W, seed):
    """A near-single-hue (warm red, h ~ 0.06-0.08) clip: bin 0 holds nearly every pixel."""
    g = torch.Generator().manual_seed(seed)
    r = 0.8 + 0.15 * torch.rand(T, 1, H, W, generator=g)
    gg = 0.1 + 0.02 * torch.rand(T, 1, H, W, generator=g)
    b = -0.5 + 0.05 * torch.rand(T, 1, H, W, generator=g)
    return torch.cat([r, gg, b], 1).to(torch.bfloat16)


@pytest.mark.parametrize("shape", [(2, 270, 480), (5, 2160, 3840), (5, 2160, 3840, "single_hue")])
def test_hsv_large_vs_gpu_oracle(cf, shape):
    T, H, W = shape[:3]
    if len(shape) == 4:
        content = single_hue_clip(T, H, W, 5)
        content[:, 0, :100], content[:, 2, :100] = -0.8, -0.9          # a green band: the two counts differ
        content = content.cuda()
        style = (single_hue_clip(T, H, W, 6).float() * 0.9).to(torch.bfloat16).cuda()
        cc, sc = ho.bin_counts(content, style)
        big = [b for b in range(12) if cc[b] > 2 ** 24]
        assert big and cc[big[0]] != sc[big[0]] and sc[big[0]] > 2 ** 24, (cc, sc)
    else:
        content, style = color_inputs(T, H, W, seed=11)
        content, style = content.cuda(), style.cuda()
    out = cf.hsv_saturation_histogram_match(content, style)
    ref = ho.hsv_saturation_histogram_match(content, style)
    diff = int((out.float() != ref).sum())
    assert diff == 0, f"{diff} of {out.numel()} values differ from the GPU oracle"


def test_wavelet_fp32_is_bit_exact(cf):
    for T, H, W in ((2, 40, 56), (1, 37, 53), (2, 270, 480)):
        content, style = color_inputs(T, H, W, seed=3)
        c, s = content.cuda(), style.cuda()
        assert torch.equal(cf._wavelet(c, s, fp32=True), ho.wavelet_reconstruction_fp32(c, s)), (T, H, W)


@pytest.mark.parametrize("case", list(HSV_CASES) + ["medium", "4k"])
def test_wavelet_adaptive_vs_gpu_oracle(cf, case):
    """Equal to the GPU oracle except where the mask (w_sat - s_sat) > 0.075 sits within 1e-6 of its threshold."""
    if case in HSV_CASES:
        g, content, style = golden(case)
    else:
        T, H, W = (2, 270, 480) if case == "medium" else (5, 2160, 3840)
        content, style = color_inputs(T, H, W, seed=12)
    c, s = content.cuda(), style.cuda()
    out = cf.wavelet_adaptive_color_correction(c, s)
    wav = ho.wavelet_reconstruction_fp32(c, s)
    res, margin = ho.adaptive_blend(c, s, wav, ho.hsv_saturation_histogram_match(c, s, out_bf16=False))
    ref = res.to(torch.bfloat16).float()
    differ = (out.float() != ref).any(1, keepdim=True)
    flips = (margin - 0.075).abs() <= 1e-6
    print(f"[{case}] wavelet_adaptive: {int(differ.sum())} pixels differ, {int(flips.sum())} near the mask threshold")
    assert not (differ & ~flips).any(), int((differ & ~flips).sum())
    if case in HSV_CASES:
        ok, why = meets_golden(out, torch.from_numpy(g["wavelet_adaptive"]))
        assert ok, why


def test_shape_mismatch_and_switch(cf):
    content, style = color_inputs(1, 40, 56)
    c, s = content.cuda(), style.cuda()
    for fn in (cf.hsv_saturation_histogram_match, cf.wavelet_adaptive_color_correction):
        with pytest.raises(NotImplementedError):
            fn(c, s[:, :, :20])
    with pytest.raises(NotImplementedError):
        cf.apply_color_correction(c, s, "hsv")
    assert torch.equal(cf.apply_color_correction(c, s, "wavelet_adaptive"), cf.wavelet_adaptive_color_correction(c, s))


# ---- the engine with synthetic weights
@pytest.fixture(scope="module")
def engine(pkg):
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    cfg = dit.dit_config("3b", dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64)
    return pipeline.SeedVR2Engine(cfg, pkg.weights.synth_dit_state_dict(cfg, seed=1),
                                  pkg.weights.synth_vae_state_dict(seed=2), torch.randn(58, 64))


def test_engine_wavelet_adaptive_clip(cf, engine):
    g = torch.Generator().manual_seed(3)
    frames4 = torch.rand(5, 36, 52, 4, generator=g).cuda()
    kw = dict(resolution=72, color_correction="wavelet_adaptive")
    noise = torch.randn(engine.latent_shape(frames4, 72), generator=torch.Generator().manual_seed(1)).cuda()
    out = engine.upscale_clip(frames4[..., :3].contiguous(), noise=noise, **kw)
    sample, style = engine.clip_to_sample(frames4[..., :3].contiguous(), noise=noise, resolution=72)
    assert torch.equal(out, cf.sample_to_image(cf.wavelet_adaptive_color_correction(sample, style)))
    torch.cuda.set_sync_debug_mode("error")             # the clip makes no host synchronisation
    try:
        again = engine.upscale_clip(frames4[..., :3].contiguous(), noise=noise, **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(again, out)
    gc = engine.graphed(frames4[..., :3].contiguous(), noise=noise, **kw)
    assert torch.equal(gc(frames4[..., :3].contiguous()), out)
    # RGBA: the correction stays RGB-only, the alpha is that of the uncorrected path
    rgba = engine.upscale_clip(frames4, noise=noise, keep_alpha=True, **kw)
    assert torch.equal(rgba[..., :3], out)
    assert torch.equal(rgba[..., 3], engine.upscale_clip(frames4, noise=noise, keep_alpha=True, resolution=72)[..., 3])
    gc4 = engine.graphed(frames4, noise=noise, keep_alpha=True, **kw)
    assert torch.equal(gc4(frames4), rgba)


def test_engine_wavelet_adaptive_video_with_overlap(engine):
    frames = torch.rand(13, 36, 52, 3, generator=torch.Generator().manual_seed(7)).cuda()
    vid = engine.upscale_video(frames, batch_size=5, temporal_overlap=2, resolution=72, color_correction="wavelet_adaptive")
    assert vid.shape == (13, 72, 104, 3) and vid.dtype == torch.bfloat16 and torch.isfinite(vid.float()).all()
