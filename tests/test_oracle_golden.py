"""CPU: the oracle restatements reproduce the committed golden vectors, which were produced
by the REFERENCE's own modules (oracle/make_golden.py).  Float tolerance 2e-4 of peak."""
import os

import numpy as np
import pytest
import torch

from oracle import color_oracle, dit_oracle, pre_oracle, vae_oracle
from oracle.make_golden import (COLOR_CASES, DIT_CASES, PRE_CASES, VAE_CASES, color_inputs, dit_inputs,
                                pre_inputs)

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("name", list(DIT_CASES))
def test_dit_oracle_matches_reference_golden(pkg, name):
    variant, over, (T, H, W), l = DIT_CASES[name]
    cfg = dit_oracle.dit_config(variant, **over)
    sd = {k: v.float() for k, v in pkg.weights.synth_dit_state_dict(cfg, seed=1234, dtype=torch.float16).items()}
    vid, txt = dit_inputs(cfg, T, H, W, l)
    g = np.load(os.path.join(GOLD, name + ".npz"))
    assert list(g["meta"]) == [T, H, W, l]
    taps = {}
    out = dit_oracle.dit_forward(sd, cfg, vid, txt, T, H, W, mode="fp32", taps=taps)
    ref = torch.from_numpy(g["out"])
    assert (out - ref).abs().max() < 2e-4 * ref.abs().max()
    assert (taps["emb"] - torch.from_numpy(g["emb"])).abs().max() < 1e-4
    assert (taps["block0"][::37] - torch.from_numpy(g["block0"])).abs().max() < 2e-4 * ref.abs().max()


@pytest.fixture(scope="module")
def vae_sd(pkg):
    return {k: v.float() for k, v in pkg.weights.synth_vae_state_dict(seed=4321, dtype=torch.float16).items()}


@pytest.mark.parametrize("name", list(VAE_CASES))
def test_vae_oracle_matches_reference_golden(vae_sd, name):
    kind, shp = VAE_CASES[name]
    g = torch.Generator().manual_seed(7)
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    if kind == "decode":
        z = torch.randn(1, 16, *shp, generator=g)
        out = vae_oracle.vae_decode(vae_sd, z)
    else:
        x = torch.rand(1, 3, *shp, generator=g) * 2 - 1
        out = vae_oracle.vae_encode(vae_sd, x)
    assert out.shape == ref.shape
    assert (out - ref).abs().max() < 2e-4 * max(ref.abs().max().item(), 1.0)


def test_bf16_mode_is_close_to_fp32(pkg):
    """ref_bf16 restates the reference's autocast flow; it must stay within bf16 noise of fp32."""
    variant, over, (T, H, W), l = DIT_CASES["dit3b_tiny_t5"]
    cfg = dit_oracle.dit_config(variant, **over)
    sd = {k: v.float() for k, v in pkg.weights.synth_dit_state_dict(cfg, seed=1234, dtype=torch.float16).items()}
    vid, txt = dit_inputs(cfg, T, H, W, l)
    a = dit_oracle.dit_forward(sd, cfg, vid, txt, T, H, W, mode="fp32")
    b = dit_oracle.dit_forward(sd, cfg, vid, txt, T, H, W, mode="ref_bf16").float()
    psnr = 10 * torch.log10(a.abs().max() ** 2 / (a - b).pow(2).mean())
    assert psnr > 45


@pytest.mark.parametrize("name", list(COLOR_CASES))
def test_color_oracle_matches_reference_golden(name):
    """src/utils/color_fix.py goldens: wavelet and AdaIN bit for bit; LAB up to the tie order of the reference's
    unstable torch.sort (a tied element may receive the adjacent reference value)."""
    T, H, W = COLOR_CASES[name]
    content, style = color_inputs(T, H, W)
    g = np.load(os.path.join(GOLD, name + ".npz"))
    assert torch.equal(color_oracle.wavelet_reconstruction(content, style), torch.from_numpy(g["wavelet"]))
    assert torch.equal(color_oracle.adaptive_instance_normalization(content, style), torch.from_numpy(g["adain"]))
    lab, ref = color_oracle.lab_color_transfer(content, style), torch.from_numpy(g["lab"])
    assert (lab == ref).float().mean() > 0.99
    assert 10 * torch.log10(4.0 / ((lab - ref) ** 2).mean()) > 60.0


def test_color_oracle_properties():
    """Histogram matching is an exact rank mapping; the wavelet split is a partition of the image."""
    g = torch.Generator().manual_seed(1)
    src, ref = torch.randn(5000, generator=g), torch.randn(5000, generator=g) * 3 + 1
    out = color_oracle.histogram_match(src, ref)
    assert torch.equal(out.sort().values, ref.sort().values)
    assert torch.equal(out.argsort(stable=True), src.argsort(stable=True))
    x = torch.rand(1, 3, 64, 80, generator=g) * 2 - 1
    high, low = color_oracle.wavelet_decomposition(x, mode="fp32")
    assert (high + low - x).abs().max() < 1e-5
    img = color_oracle.sample_to_image(torch.tensor([-2.0, -1.0, 0.0, 0.5, 3.0]).view(1, 1, 1, 5).expand(1, 3, 1, 5))
    assert img.shape == (1, 1, 5, 3) and torch.equal(img[0, 0, :, 0], torch.tensor([0.0, 0.0, 0.5, 0.75, 1.0]))


@pytest.mark.parametrize("name", list(PRE_CASES))
def test_pre_oracle_matches_reference_golden(name):
    """prepare_video_transforms goldens (reference transform classes on CPU): bit-equal except where the fp32
    accumulation order flips a bf16 rounding (at most one ulp)."""
    T, h, w, res, mx = PRE_CASES[name]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    out = pre_oracle.preprocess(pre_inputs(T, h, w), res, mx)
    assert out.shape == ref.shape
    d = (out - ref).abs()
    assert (d == 0).float().mean() > 0.999 and d.max() <= 2 ** -7


def test_pre_oracle_sizes_and_weights():
    assert pre_oracle.resized_size(720, 1280, 2160) == ((2160, 3840), False)
    assert pre_oracle.resized_size(1280, 720, 1080) == ((1920, 1080), False)
    assert pre_oracle.resized_size(540, 960, 1080, 1600) == ((900, 1600), True)
    first, count, w = pre_oracle.aa_weights(96, 40)          # 2.4x down-scale: the support widens to 4.8 taps
    assert count.max() >= 9 and np.allclose(w.sum(1), 1.0, atol=1e-6)
    assert pre_oracle.aa_weights(30, 90)[1].max() <= 5       # up-scale: plain 4-tap cubic (+1 zero-weight tap)
    first, count, w = pre_oracle.aa_weights(33, 33)          # identity: a single unit tap
    assert np.allclose(np.sort(w, 1)[:, -1], 1.0) and np.allclose(np.abs(w).sum(1), 1.0)


@pytest.mark.parametrize("T,h,w,res,mx", [(2, 30, 41, 90, 0), (2, 64, 48, 40, 0), (1, 36, 64, 108, 160),
                                          (2, 33, 57, 33, 0), (1, 61, 23, 47, 0), (1, 45, 80, 72, 100)])
def test_torch_op_chain_is_the_reference_compose(T, h, w, res, mx):
    """pre_oracle.preprocess_torch, the yardstick the GPU resize is held to bit for bit on the device, is the
    reference's own Compose (NaResize, clamp, DivisiblePad, Normalize, permute): bit-equal on the CPU, where both run
    the same torch kernels, so that every cast, the second resize of the cap and the padding are the reference's."""
    from oracle import make_golden, ref_import
    if not os.path.isdir(os.path.join(ref_import.REFERENCE_ROOT, "src")):
        pytest.skip("the reference sources are not installed")
    g = torch.Generator().manual_seed(h * w + res)
    clip = (torch.rand(T, 3, h, w, generator=g) * 1.2 - 0.1).to(torch.bfloat16)
    ref = make_golden.reference_compose(res, mx)(clip.clone())
    out = pre_oracle.preprocess_torch(clip.clone(), res, mx)
    assert out.dtype == ref.dtype == torch.bfloat16 and out.shape == ref.shape
    assert torch.equal(out, ref)


def test_blend_overlap_oracle_matches_reference_golden(pkg):
    """blend_overlapping_frames (generation_utils.py:284-312): same inputs as oracle/make_golden.py, bit for bit;
    the host-side weight table of shard.py is the same computation."""
    import importlib
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    gold = np.load(os.path.join(GOLD, "blend_overlap.npz"))
    g = torch.Generator().manual_seed(21)
    for ov in (1, 2, 3, 4, 7, 8):
        a = torch.rand(ov, 6, 8, 3, generator=g).to(torch.bfloat16)
        b = torch.rand(ov, 6, 8, 3, generator=g).to(torch.bfloat16)
        out = color_oracle.blend_overlapping_frames(a, b, ov)
        assert torch.equal(out, torch.from_numpy(gold[f"ov{ov}"]))
        w_prev, w_cur = shard.blend_weights(ov)
        ref = (a * w_prev.view(ov, 1, 1, 1) + b * w_cur.view(ov, 1, 1, 1)).float()
        assert torch.equal(ref, out)
    for ov in (2, 5):       # fp32 frames (multi-GPU merge)
        a, b = torch.rand(ov, 6, 8, 3, generator=g), torch.rand(ov, 6, 8, 3, generator=g)
        assert torch.equal(color_oracle.blend_overlapping_frames(a, b, ov), torch.from_numpy(gold[f"f32_ov{ov}"]))


def test_merge_shards_host_logic(pkg):
    """shard.merge_shards (inference_cli.py:1241-1274) with the oracle blend plugged in == the oracle's merge, incl. the
    'chunk not longer than the overlap' edge cases; partition + merge restores the frame count."""
    import importlib
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    g = torch.Generator().manual_seed(5)
    blend = lambda p, c: color_oracle.blend_overlapping_frames(p, c, p.shape[0])
    for total, world, ov in ((23, 3, 2), (16, 2, 4), (9, 4, 3), (5, 4, 2), (12, 2, 0)):
        parts = shard.partition_frames(total, world, ov)
        chunks = [torch.rand(b - a, 4, 6, 3, generator=g) for a, b in parts]
        out = shard.merge_shards(chunks, ov, blend=blend)
        assert torch.equal(out, color_oracle.merge_shards(chunks, ov))
        if all(c.shape[0] > ov for c in chunks):
            assert out.shape[0] == total


def test_hsv_and_adaptive_oracle_match_reference_as_distributions():
    """hsv / wavelet_adaptive (round-2 groundwork, not shipped by the engine): a third of the saturation values are
    tied, so the reference's unstable sort defines the result only up to the tie order — the oracle must agree with
    the reference golden as a distribution (sorted saturations) and to >= 35 dB, and its colour-space conversions
    must round-trip."""
    T, H, W = COLOR_CASES["color_t2_40x56"]
    content, style = color_inputs(T, H, W)
    tint = torch.tensor([1.0, 0.6, 0.3]).view(1, 3, 1, 1)
    c2, s2 = (content.float() * tint).to(torch.bfloat16), (style.float() * tint * 0.9).to(torch.bfloat16)
    g = np.load(os.path.join(GOLD, "color_t2_40x56.npz"))
    sat = lambda x: color_oracle.saturation_map(x.float()).flatten().sort().values
    for key, fn in (("hsv", color_oracle.hsv_saturation_histogram_match),
                    ("wavelet_adaptive", color_oracle.wavelet_adaptive_color_correction)):
        out, ref = fn(c2, s2), torch.from_numpy(g[key])
        assert (sat(out) - sat(ref)).abs().mean() < 2e-3
        assert 10 * torch.log10(4.0 / ((out - ref) ** 2).mean()) > 35.0
    c01 = ((c2.float() + 1.0) * 0.5).clamp(0.0, 1.0)
    assert (color_oracle.hsv_to_rgb(color_oracle.rgb_to_hsv(c01)) - c01).abs().max() < 1e-5


def test_tiled_vae_oracle_matches_reference_golden(pkg):
    """tiled_encode / tiled_decode restatement (attn_video_vae.py:1302-1630) vs goldens the reference's own tiled paths
    produced (oracle/make_golden.py --tiled-only): fp32, same inputs."""
    from oracle.make_golden import TILED_CASES
    sd32 = {k: v.float() for k, v in pkg.weights.synth_vae_state_dict(seed=4321, dtype=torch.float16).items()}
    for name, (kind, shp, tile, ov) in TILED_CASES.items():
        g = torch.Generator().manual_seed(7)
        gold = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
        if kind == "decode":
            out = vae_oracle.tiled_decode(sd32, torch.randn(1, 16, *shp, generator=g), tile, ov)
        else:
            out = vae_oracle.tiled_encode(sd32, torch.rand(1, 3, *shp, generator=g) * 2 - 1, tile, ov)
        assert out.shape == gold.shape and (out - gold).abs().max() < 2e-4 * max(gold.abs().max().item(), 1.0), name
