"""-m gpu: post-decode colour correction + image formatting (csrc/post.cu through the C ABI and the
``color_fix`` host mirror) against the goldens produced by the reference's src/utils/color_fix.py and
against the oracle at larger sizes.  Tolerances are stated per test."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import color_oracle
from oracle.make_golden import COLOR_CASES, color_inputs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def cf(pkg):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.color_fix")


def psnr(a, b, peak=2.0):
    mse = ((a.float().cpu() - b.float().cpu()) ** 2).mean().item()
    return 99.0 if mse == 0 else 10 * np.log10(peak * peak / mse)


def frac_equal(a, b):
    return (a.float().cpu() == b.float().cpu()).float().mean().item()


@pytest.mark.parametrize("name", list(COLOR_CASES))
def test_color_fix_vs_reference_golden(cf, name):
    T, H, W = COLOR_CASES[name]
    content, style = color_inputs(T, H, W)
    g = np.load(os.path.join(GOLD, name + ".npz"))
    c, s = content.cuda(), style.cuda()
    # wavelet: the 9-tap sum is order-independent up to the last fp32 bit -> bit-exact except (rarely) a 1-ulp bf16 tie
    w = cf.wavelet_reconstruction(c, s)
    ref = torch.from_numpy(g["wavelet"])
    assert w.dtype == torch.bfloat16 and frac_equal(w, ref) > 0.999 and psnr(w, ref) > 80.0
    # AdaIN: statistics in fp64 instead of torch's fp32 reduction; the bf16-rounded mean/std agree
    a = cf.adaptive_instance_normalization(c, s)
    ref = torch.from_numpy(g["adain"])
    assert frac_equal(a, ref) > 0.99 and psnr(a, ref) > 60.0
    # LAB: rank mapping; ties and 1e-7-level LAB differences move single elements to a neighbouring rank
    l = cf.lab_color_transfer(c, s, None, luminance_weight=0.8)
    ref = torch.from_numpy(g["lab"])
    assert frac_equal(l, ref) > 0.98 and psnr(l, ref) > 55.0, (frac_equal(l, ref), psnr(l, ref))


def test_histogram_match_is_exact_rank_mapping(svr2lib):
    """Size-independent properties at 4M elements: the output is a permutation of the reference values and
    preserves the order of the source."""
    n = 1 << 22
    g = torch.Generator().manual_seed(3)
    src = torch.randn(n, generator=g).cuda()
    ref = (torch.randn(n, generator=g) * 3 + 1).cuda()
    out = torch.empty_like(src)
    need = svr2lib.load().svr2_histogram_match_scratch_bytes(n)
    scratch = torch.empty(need, device="cuda", dtype=torch.uint8)
    svr2lib.call("svr2_histogram_match_f32", svr2lib.ptr(src), svr2lib.ptr(ref), svr2lib.ptr(out), n,
                 svr2lib.ptr(scratch), need, svr2lib.stream())
    assert torch.equal(out.sort().values, ref.sort().values)
    order = src.argsort()
    assert (out[order][1:] >= out[order][:-1]).all()
    # too-small scratch is an error, not a crash
    rc = svr2lib.load().svr2_histogram_match_f32(svr2lib.ptr(src), svr2lib.ptr(ref), svr2lib.ptr(out), n,
                                                  svr2lib.ptr(scratch), 16, svr2lib.stream())
    assert rc != 0 and b"scratch" in svr2lib.load().svr2_last_error()


def test_lab_round_trip_and_image_format(cf, svr2lib):
    """rgb -> LAB -> rgb is the identity up to bf16 rounding; sample_to_image equals the oracle bit for bit."""
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(2, 3, 33, 47, generator=g) * 2 - 1).to(torch.bfloat16)
    xc = x.cuda()
    n, hw = 2 * 33 * 47, 33 * 47
    lab = torch.empty(3, n, device="cuda", dtype=torch.float32)
    svr2lib.call("svr2_rgb_to_lab_f32", svr2lib.ptr(xc), svr2lib.ptr(lab), 2, hw, svr2lib.stream())
    ref_lab = color_oracle.rgb_to_lab(((x.float() + 1) * 0.5).clamp(0, 1)).permute(1, 0, 2, 3).reshape(3, n)
    assert (lab.cpu() - ref_lab).abs().max() < 2e-3          # L in [0,100], a/b in [-128,127]; fp32 pow differences
    back = torch.empty_like(xc)
    svr2lib.call("svr2_lab_to_rgb_bf16", svr2lib.ptr(lab[0]), None, svr2lib.ptr(lab[1]), svr2lib.ptr(lab[2]), 1.0,
                 svr2lib.ptr(back), 2, hw, svr2lib.stream())
    assert (back.float().cpu() - x.float()).abs().max() <= 2 ** -7      # one bf16 ulp near 1
    y = torch.cat([x, torch.tensor([-3.0, 2.0, 0.3]).view(1, 3, 1, 1).expand(1, 3, 33, 47).to(torch.bfloat16)])
    img = cf.sample_to_image(y.cuda())
    assert img.shape == (3, 33, 47, 3) and torch.equal(img.float().cpu(), color_oracle.sample_to_image(y))


def test_color_correction_switch(cf):
    content, style = color_inputs(1, 40, 56)
    c, s = content.cuda(), style.cuda()
    assert torch.equal(cf.apply_color_correction(c, s, "none"), c)
    assert torch.equal(cf.apply_color_correction(c, s, "wavelet"), cf.wavelet_reconstruction(c, s))
    with pytest.raises(NotImplementedError):
        cf.apply_color_correction(c, s, "hsv")
    with pytest.raises(NotImplementedError):
        cf.wavelet_reconstruction(c, s[:, :, :20])
    with pytest.raises(Exception):
        cf.wavelet_reconstruction(content, style)      # CPU tensors: no fallback


# ------------------------------------------------------------------ clip pre-processing (csrc/pre.cu)
@pytest.fixture(scope="module")
def pre(pkg):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.preprocess")


def _pre_cases():
    from oracle.make_golden import PRE_CASES
    return PRE_CASES


@pytest.mark.parametrize("name", list(_pre_cases()))
def test_preprocess_vs_reference_golden(pre, name):
    """prepare_video_transforms goldens: resize + clamp + pad-16 + normalise + c t h w in one kernel.  The goldens were
    made on the CPU, whose tap arithmetic differs from that of torch's CUDA kernel (which the kernel follows, see
    tests/test_resize_elementwise_gpu.py) in the last fp32 bits: equal up to one bf16 ulp where that flips a rounding."""
    from oracle.make_golden import pre_inputs
    T, h, w, res, mx = _pre_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    frames = pre_inputs(T, h, w)
    out = pre.preprocess_frames(frames.cuda(), res, mx)
    assert out.dtype == torch.bfloat16 and tuple(out.shape) == tuple(ref.shape)
    d = (out.float().cpu() - ref).abs()
    assert (d == 0).float().mean() > 0.999 and d.max() <= 2 ** -7, ((d == 0).float().mean().item(), d.max().item())
    # the t c h w entry point (the reference's Compose is called on t c h w) gives the same result
    out2 = pre.prepare_video_transforms(res, mx)(frames.cuda().to(torch.bfloat16).permute(0, 3, 1, 2))
    assert torch.equal(out, out2)


def test_preprocess_identity_size_and_padding(pre):
    """Frames already at the target size (the bench workload): exact clamp/normalise, padding holds -1."""
    g = torch.Generator().manual_seed(4)
    frames = (torch.rand(3, 72, 100, 3, generator=g) * 1.2 - 0.1).cuda()
    out = pre.preprocess_frames(frames, 72)
    assert tuple(out.shape) == (3, 3, 80, 112)
    ref = (frames.to(torch.bfloat16).float().clamp(0, 1) - 0.5).to(torch.bfloat16).float() / 0.5
    assert torch.equal(out[:, :, :72, :100].float(), ref.permute(3, 0, 1, 2))
    assert (out[:, :, 72:, :] == -1).all() and (out[:, :, :, 100:] == -1).all()


def test_blend_overlap_vs_reference_golden(pkg):
    """Temporal-overlap cross-fade kernel against the reference's blend_overlapping_frames goldens, bit for bit."""
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    gold = np.load(os.path.join(GOLD, "blend_overlap.npz"))
    g = torch.Generator().manual_seed(21)
    for ov in (1, 2, 3, 4, 7, 8):
        a = torch.rand(ov, 6, 8, 3, generator=g).to(torch.bfloat16)
        b = torch.rand(ov, 6, 8, 3, generator=g).to(torch.bfloat16)
        out = shard.blend_overlap(a.cuda(), b.cuda())
        assert torch.equal(out.float().cpu(), torch.from_numpy(gold[f"ov{ov}"])), ov
    # a 4K-sized pair of frames: same result as the oracle
    a = torch.rand(3, 270, 480, 3, generator=g).to(torch.bfloat16)
    b = torch.rand(3, 270, 480, 3, generator=g).to(torch.bfloat16)
    assert torch.equal(shard.blend_overlap(a.cuda(), b.cuda()).float().cpu(), color_oracle.blend_overlapping_frames(a, b, 3))
    # odd frame sizes (3 * 7 * 9 = 189 values per frame: neither % 8 nor % 4), both dtypes — the reference blends any size
    for dt in (torch.bfloat16, torch.float32):
        a = torch.rand(2, 7, 9, 3, generator=g).to(dt)
        b = torch.rand(2, 7, 9, 3, generator=g).to(dt)
        out = shard.blend_overlap(a.cuda(), b.cuda())
        assert out.shape == a.shape and torch.equal(out.cpu(), color_oracle.blend_overlapping_frames(a, b, 2).to(dt)), dt


def test_merge_shards_fp32_kernel(pkg):
    """Per-rank results merged with the fp32 cross-fade kernel == the oracle's merge (== inference_cli.py:1241-1274),
    bit for bit; the fp32 blend also matches the reference goldens."""
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    gold = np.load(os.path.join(GOLD, "blend_overlap.npz"))
    g = torch.Generator().manual_seed(21)
    for ov in (1, 2, 3, 4, 7, 8):                      # replay the generator of oracle/make_golden.py
        torch.rand(ov, 6, 8, 3, generator=g); torch.rand(ov, 6, 8, 3, generator=g)
    for ov in (2, 5):
        a, b = torch.rand(ov, 6, 8, 3, generator=g), torch.rand(ov, 6, 8, 3, generator=g)
        assert torch.equal(shard.blend_overlap(a.cuda(), b.cuda()).cpu(), torch.from_numpy(gold[f"f32_ov{ov}"]))
    g = torch.Generator().manual_seed(6)
    for total, world, ov in ((23, 3, 2), (16, 2, 4), (9, 4, 3)):
        parts = shard.partition_frames(total, world, ov)
        chunks = [torch.rand(b - a, 16, 24, 3, generator=g).to(torch.bfloat16) for a, b in parts]
        out = shard.merge_shards([c.cuda() for c in chunks], ov)
        assert out.dtype == torch.float32 and torch.equal(out.cpu(), color_oracle.merge_shards(chunks, ov))
