"""-m gpu: the CUDA path (through the C ABI) against the reference-pinned oracle and the
golden vectors.  Stated tolerances (bf16 compute): DiT output PSNR >= 50 dB vs the fp32
reference golden and >= 52 dB vs the oracle's ref_bf16 mode (north_star: latent PSNR >= 50 dB);
VAE (random weights amplify bf16 noise) >= 42 dB and never worse than 3 dB below what the
reference's own bf16 flow (oracle ref_bf16 on the same GPU) achieves."""
import importlib
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dit_oracle, vae_oracle
from oracle.make_golden import DIT_CASES, VAE_CASES, dit_inputs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def psnr(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return (10 * torch.log10(b.abs().max() ** 2 / (a - b).pow(2).mean())).item()


@pytest.mark.parametrize("name", list(DIT_CASES))
def test_dit_vs_golden(pkg, name):
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    variant, over, (T, H, W), l = DIT_CASES[name]
    cfg = dit.dit_config(variant, **over)
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=1234, dtype=torch.float16)
    vid, txt = dit_inputs(cfg, T, H, W, l)
    gold = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    eng = dit.B200NaDiT(cfg, sd)
    out = eng(vid.cuda(), txt.cuda(), torch.tensor([[T, H, W]]), torch.tensor([[l]])).vid_sample
    assert out.shape == gold.shape and torch.isfinite(out).all()
    obf = dit_oracle.dit_forward({k: v.float() for k, v in sd.items()}, cfg, vid, txt, T, H, W, mode="ref_bf16")
    p_gold, p_bf = psnr(out, gold), psnr(out, obf)
    assert p_gold >= 50.0, f"{name}: {p_gold:.1f} dB vs reference golden"
    assert p_bf >= 52.0, f"{name}: {p_bf:.1f} dB vs oracle ref_bf16"
    # determinism (README.md:144 "identical images with the same seed")
    out2 = eng(vid.cuda(), txt.cuda(), [[T, H, W]], [[l]]).vid_sample
    assert torch.equal(out, out2)


def test_dit_from_fp8_safetensors_file(pkg, tmp_path):
    """A *_fp8_e4m3fn.safetensors checkpoint (the reference CLI's default model file) loads straight into the engine:
    same output as the engine built from the de-quantised tensors, finite, close to the fp16 checkpoint's output."""
    from safetensors.torch import save_file
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    variant, over, (T, H, W), l = DIT_CASES["dit3b_tiny_t3"]
    cfg = dit.dit_config(variant, **over)
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=1234, dtype=torch.float16)
    path = str(tmp_path / "seedvr2_tiny_fp8_e4m3fn.safetensors")
    save_file({k: (v.to(torch.float8_e4m3fn) if (v.ndim == 2 and "freqs" not in k) else v).contiguous()
               for k, v in sd.items()}, path)
    sd8 = pkg.weights.load_state_dict(path)
    assert any(v.dtype == torch.float8_e4m3fn for v in sd8.values())
    vid, txt = dit_inputs(cfg, T, H, W, l)
    run = lambda d: dit.B200NaDiT(cfg, d)(vid.cuda(), txt.cuda(), [[T, H, W]], [[l]]).vid_sample
    out8 = run(sd8)
    out8_deq = run({k: (v.to(torch.float16) if v.dtype == torch.float8_e4m3fn else v) for k, v in sd8.items()})
    assert torch.isfinite(out8).all() and torch.equal(out8, out8_deq)
    assert psnr(out8, run(sd)) > 20.0          # fp8 storage costs precision, not sanity


@pytest.fixture(scope="module")
def vae_pair(pkg):
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    sd = pkg.weights.synth_vae_state_dict(seed=4321, dtype=torch.float16)
    return vae.B200VideoVAE(sd), {k: v.float().cuda() for k, v in sd.items()}


@pytest.mark.parametrize("name", list(VAE_CASES))
def test_vae_vs_golden(vae_pair, name):
    eng, sd32 = vae_pair
    kind, shp = VAE_CASES[name]
    g = torch.Generator().manual_seed(7)
    gold = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    if kind == "decode":
        z = torch.randn(1, 16, *shp, generator=g).cuda()
        out = eng.decode(z).sample
        obf = vae_oracle.vae_decode(sd32, z, mode="ref_bf16")
    else:
        x = (torch.rand(1, 3, *shp, generator=g) * 2 - 1).cuda()
        out = eng.encode(x).latent
        obf = vae_oracle.vae_encode(sd32, x, mode="ref_bf16")
    if out.ndim == 4:
        out = out.unsqueeze(2)
    assert out.shape == gold.shape
    p_eng, p_ref = psnr(out, gold), psnr(obf, gold)
    assert p_eng >= 42.0 and p_eng >= p_ref - 3.0, f"{name}: engine {p_eng:.1f} dB, reference bf16 flow {p_ref:.1f} dB"


def test_vae_roundtrip_shapes_and_slicing_property(vae_pair):
    """Size-independent properties at a larger size: decode of a longer clip equals decode of its
    prefix on the shared frames (causality), and encode->decode preserves shape."""
    eng, _ = vae_pair
    g = torch.Generator().manual_seed(3)
    z = torch.randn(1, 16, 4, 10, 16, generator=g).cuda()
    full = eng.decode(z).sample              # 13 frames
    pre = eng.decode(z[:, :, :2]).sample     # 5 frames
    assert full.shape == (1, 3, 13, 80, 128) and pre.shape == (1, 3, 5, 80, 128)
    assert psnr(full[:, :, :5], pre) > 60.0, "decoder must be causal in time"
    lat = eng.encode(full[:, :, :9]).latent
    assert lat.shape == (1, 16, 3, 10, 16)


@pytest.mark.parametrize("split", [4, 8])
def test_vae_temporal_slicing_is_exact(vae_pair, split):
    """set_causal_slicing (attn_video_vae.py:1709-1723, slicing_encode/_decode :1254-1300): slices whose halo
    is the previous slice's tail reproduce the un-sliced result bit for bit, in both directions."""
    eng, _ = vae_pair
    g = torch.Generator().manual_seed(11)
    z = torch.randn(1, 16, 5, 6, 10, generator=g).cuda()
    x = (torch.rand(1, 3, 17, 48, 80, generator=g) * 2 - 1).cuda()
    eng.set_causal_slicing(split_size=None, memory_device=None)
    dec_full, enc_full = eng.decode(z).sample, eng.encode(x).latent
    try:
        eng.set_causal_slicing(split_size=split, memory_device="same")
        dec_sl, enc_sl = eng.decode(z).sample, eng.encode(x).latent
    finally:
        eng.set_causal_slicing(split_size=None, memory_device=None)
    assert dec_full.shape == dec_sl.shape == (1, 3, 17, 48, 80)
    assert enc_full.shape == enc_sl.shape == (1, 16, 5, 6, 10)
    assert torch.equal(dec_full, dec_sl), f"sliced decode differs: {psnr(dec_full, dec_sl):.1f} dB"
    assert torch.equal(enc_full, enc_sl), f"sliced encode differs: {psnr(enc_full, enc_sl):.1f} dB"


def test_vae_slices_when_clip_exceeds_memory_model(vae_pair, monkeypatch):
    """With a tiny memory budget the engine slices on its own and still matches the un-sliced clip."""
    eng, _ = vae_pair
    g = torch.Generator().manual_seed(12)
    z = torch.randn(1, 16, 4, 6, 10, generator=g).cuda()
    full = eng.decode(z).sample
    monkeypatch.setattr(type(eng), "_frames_that_fit", lambda self, H, W, state_bytes_per_pixel=0: 4)
    assert torch.equal(eng.decode(z).sample, full)


def test_attention_seam_module(pkg):
    att = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.attention")
    m = att.B200FlashAttentionVarlen()
    lens = [463, 463, 120]
    total = sum(lens)
    g = torch.Generator().manual_seed(0)
    q, k, v = (torch.randn(total, 4, 128, generator=g).cuda() for _ in range(3))
    cu = torch.tensor([0, 463, 926, 1046], dtype=torch.int32).cuda()
    out = m(q, k, v, cu, cu, torch.tensor(463), torch.tensor(463), deterministic=False)
    o = 0
    for n in lens:
        qi, ki, vi = (x[o:o + n].bfloat16().float().permute(1, 0, 2)[None] for x in (q, k, v))
        ref = F.scaled_dot_product_attention(qi, ki, vi)[0].permute(1, 0, 2)
        assert psnr(out[o:o + n], ref) > 45
        o += n


def test_pipeline_clip_smoke(pkg):
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    cfg = dit.dit_config("3b", dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64)
    eng = pipeline.SeedVR2Engine(cfg, pkg.weights.synth_dit_state_dict(cfg, seed=1),
                                 pkg.weights.synth_vae_state_dict(seed=2), torch.randn(58, 64))
    frames = torch.rand(6, 70, 100, 3)
    out = eng.upscale_clip(frames)
    assert out.shape == (6, 70, 100, 3) and torch.isfinite(out).all()
    assert 0 <= out.min() and out.max() <= 1


def test_pipeline_resize_color_and_cuda_graph(pkg):
    """upscale_clip from source-resolution frames with LAB colour correction, eager vs one captured CUDA graph:
    bit-identical, and the graph replays on new frames."""
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    cfg = dit.dit_config("3b", dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64)
    eng = pipeline.SeedVR2Engine(cfg, pkg.weights.synth_dit_state_dict(cfg, seed=1),
                                 pkg.weights.synth_vae_state_dict(seed=2), torch.randn(58, 64))
    g = torch.Generator().manual_seed(0)
    frames = torch.rand(5, 36, 52, 3, generator=g).cuda()
    frames2 = torch.rand(5, 36, 52, 3, generator=g).cuda()
    kw = dict(resolution=72, color_correction="lab")
    noise = torch.randn(eng.latent_shape(frames, 72), generator=torch.Generator().manual_seed(1)).cuda()
    assert tuple(noise.shape) == (2, 10, 14, 16)         # 72 x 104 -> padded 80 x 112 -> /8
    eager1 = eng.upscale_clip(frames, noise=noise, **kw).clone()
    eager2 = eng.upscale_clip(frames2, noise=noise, **kw).clone()
    assert eager1.shape == (5, 72, 104, 3) and torch.isfinite(eager1).all() and 0 <= eager1.min() and eager1.max() <= 1
    gc = eng.graphed(frames, noise=noise, **kw)
    assert torch.equal(gc(frames), eager1)
    assert torch.equal(gc(frames2), eager2)
    assert torch.equal(gc(frames), eager1)


def test_upscale_video_batches_and_overlap(pkg):
    """Whole-video loop (generation_phases.py batching): one batch == upscale_clip bit for bit; with overlap the frames
    before the first cross-fade are those of the first batch; the output covers every input frame."""
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    cfg = dit.dit_config("3b", dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64)
    eng = pipeline.SeedVR2Engine(cfg, pkg.weights.synth_dit_state_dict(cfg, seed=1),
                                 pkg.weights.synth_vae_state_dict(seed=2), torch.randn(58, 64))
    frames = torch.rand(13, 36, 52, 3, generator=torch.Generator().manual_seed(2)).cuda()
    kw = dict(resolution=72, color_correction="wavelet")
    one = eng.upscale_video(frames[:5], batch_size=5, **kw)
    assert torch.equal(one, eng.upscale_clip(frames[:5], **kw))
    vid = eng.upscale_video(frames, batch_size=5, temporal_overlap=2, **kw)
    assert vid.shape == (13, 72, 104, 3) and torch.isfinite(vid).all() and 0 <= vid.min() and vid.max() <= 1
    plain = eng.upscale_video(frames, batch_size=5, temporal_overlap=0, **kw)
    assert plain.shape == (13, 72, 104, 3)
    assert torch.equal(plain[:5], one)                        # without overlap the first batch is untouched


def test_vae_medium_size_vs_oracle(vae_pair):
    """Larger spatial size than the goldens (ragged tile edges, swap-AB / fused-statistics paths):
    engine vs the oracle run on the same GPU in fp32 and in the reference's bf16 flow."""
    eng, sd32 = vae_pair
    g = torch.Generator().manual_seed(11)
    z = torch.randn(1, 16, 3, 34, 60, generator=g).cuda()            # -> 9 frames of 272 x 480
    out = eng.decode(z).sample
    ref32 = vae_oracle.vae_decode(sd32, z, mode="fp32")
    refbf = vae_oracle.vae_decode(sd32, z, mode="ref_bf16")
    assert out.shape == ref32.shape == (1, 3, 9, 272, 480)
    p_eng, p_ref = psnr(out, ref32), psnr(refbf, ref32)
    assert p_eng >= 40.0 and p_eng >= p_ref - 3.0, f"decode: engine {p_eng:.1f} dB vs reference-bf16 flow {p_ref:.1f} dB"
    x = out[:, :, :5].clamp(-1, 1)
    lat = eng.encode(x).latent
    ref32 = vae_oracle.vae_encode(sd32, x.float(), mode="fp32")
    refbf = vae_oracle.vae_encode(sd32, x.float(), mode="ref_bf16")
    p_eng, p_ref = psnr(lat, ref32), psnr(refbf, ref32)
    assert lat.shape == (1, 16, 2, 34, 60)
    assert p_eng >= 40.0 and p_eng >= p_ref - 3.0, f"encode: engine {p_eng:.1f} dB vs reference-bf16 flow {p_ref:.1f} dB"


def test_dit_medium_size_vs_oracle(pkg):
    """3B structure at width 512 (4 heads), 6 layers, 5 x 68 x 120 latent (75 / 90 windows of up to 810+58 tokens)."""
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    cfg = dit.dit_config("3b", dim=512, heads=4, layers=6, mm_layers=3, txt_in_dim=256)
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=99, dtype=torch.float16, device="cuda")
    T, H, W, l = 5, 68, 120, 58
    g = torch.Generator().manual_seed(5)
    vid, txt = torch.randn(T * H * W, 33, generator=g).cuda(), torch.randn(l, 256, generator=g).cuda()
    out = dit.B200NaDiT(cfg, sd)(vid, txt, [[T, H, W]], [[l]]).vid_sample
    sd32 = {k: v.float().cpu() for k, v in sd.items()}      # the oracle builds its index tables on the host
    ref32 = dit_oracle.dit_forward(sd32, cfg, vid.cpu(), txt.cpu(), T, H, W, mode="fp32")
    refbf = dit_oracle.dit_forward(sd32, cfg, vid.cpu(), txt.cpu(), T, H, W, mode="ref_bf16")
    p_eng, p_ref = psnr(out, ref32), psnr(refbf, ref32)
    assert p_eng >= 50.0, f"DiT medium: {p_eng:.1f} dB vs fp32 oracle (reference-bf16 flow: {p_ref:.1f} dB)"


def test_vae_tiled_vs_reference_golden_and_oracle(vae_pair):
    """tiled=True (a25; attn_video_vae.py:1302-1630): the engine's tile loop + seam kernels vs the goldens the reference's
    own tiled paths produced, and its seam arithmetic vs the oracle's bf16 blend fed with the ENGINE's own tiles
    (isolates plan / weights / rounding order: must agree to a bf16 ulp)."""
    from oracle.make_golden import TILED_CASES
    eng, sd32 = vae_pair
    for name, (kind, shp, tile, ov) in TILED_CASES.items():
        g = torch.Generator().manual_seed(7)
        gold = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
        if kind == "decode":
            src = torch.randn(1, 16, *shp, generator=g).cuda()
            out = eng.decode(src, tiled=True, tile_size=tile, tile_overlap=ov).sample
            obf = vae_oracle.tiled_decode(sd32, src, tile, ov, mode="ref_bf16")
            seam = vae_oracle.tiled_decode(None, src.bfloat16(), tile, ov, decode_fn=lambda t: eng.decode(t).sample)
        else:
            src = (torch.rand(1, 3, *shp, generator=g) * 2 - 1).cuda()
            out = eng.encode(src, tiled=True, tile_size=tile, tile_overlap=ov).latent
            obf = vae_oracle.tiled_encode(sd32, src, tile, ov, mode="ref_bf16")
            seam = vae_oracle.tiled_encode(None, src.bfloat16(), tile, ov, encode_fn=lambda t: eng.encode(t).latent)
        if out.ndim == 4:
            out, obf, seam = out.unsqueeze(2), obf.unsqueeze(2), (seam.unsqueeze(2) if seam.ndim == 4 else seam)
        assert out.shape == gold.shape, name
        p_eng, p_ref = psnr(out, gold), psnr(obf, gold)
        assert p_eng >= 42.0 and p_eng >= p_ref - 3.0, f"{name}: engine {p_eng:.1f} dB, reference bf16 flow {p_ref:.1f} dB"
        d = (out.float() - seam.float()).abs()
        assert (d == 0).float().mean() > 0.99 and d.max() <= 2 ** -6 * max(1.0, seam.abs().max().item()), \
            f"{name}: seam arithmetic differs from the reference's op order ({(d == 0).float().mean():.4f} equal, max {d.max():.4f})"


@pytest.mark.parametrize("name", ["dit3b_tiny_t3", "dit7b_tiny_t3"])
def test_dit_native_runtime_equals_python_sequencing(pkg, name):
    """svr2_dit_forward (C++ host runtime on a svr2_t handle: geometry, workspace plan, kernel sequence) against the
    same forward sequenced by the Python module: same kernels in the same order -> bit-identical output; the handle
    reports its workspace size and survives a second geometry."""
    dit = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.dit")
    variant, over, (T, H, W), l = DIT_CASES[name]
    cfg = dit.dit_config(variant, **over)
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=1234, dtype=torch.float16)
    vid, txt = dit_inputs(cfg, T, H, W, l)
    eng = dit.B200NaDiT(cfg, sd)
    eng.native = True
    out_n = eng(vid.cuda(), txt.cuda(), [[T, H, W]], [[l]]).vid_sample.clone()
    eng.native = False
    out_p = eng(vid.cuda(), txt.cuda(), [[T, H, W]], [[l]]).vid_sample
    # same kernels, same order, same tables (the Python sequencing reads the handle's, svr2_dit_geometry) -> bit-identical
    # output
    assert torch.equal(out_n, out_p), f"{name}: native vs python sequencing {psnr(out_n, out_p):.1f} dB"
    assert eng.workspace_bytes(T, H, W, l) > 0
    eng.native = True
    g = torch.Generator().manual_seed(9)
    vid2 = torch.randn(1 * 16 * 24, cfg["in_ch"], generator=g)
    o2 = eng(vid2.cuda(), txt.cuda(), [[1, 16, 24]], [[l]]).vid_sample
    eng.native = False
    assert torch.equal(o2, eng(vid2.cuda(), txt.cuda(), [[1, 16, 24]], [[l]]).vid_sample)
    assert torch.equal(out_n, dit.B200NaDiT(cfg, sd)(vid.cuda(), txt.cuda(), [[T, H, W]], [[l]]).vid_sample)


@pytest.mark.parametrize("split", [None, 4, 8])
def test_vae_native_runtime_equals_python_sequencing(vae_pair, split):
    """svr2_vae_encode / svr2_vae_decode (C++ host runtime on a svr2_t handle: kernel sequence, temporal slices with the
    conv memories, one first-fit activation arena) against the same clip sequenced by the Python module with torch
    allocations: same kernels, same order -> bit-identical results, un-sliced and sliced; the handle's workspace query is
    exact (one aligned block less is refused) and an engine-owned workspace gives the same result."""
    lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
    eng, _ = vae_pair
    g = torch.Generator().manual_seed(21)
    z = torch.randn(1, 16, 5, 18, 24, generator=g).cuda()                  # n = 432 keys: single-pass attention path
    x = (torch.rand(1, 3, 17, 144, 192, generator=g) * 2 - 1).cuda()
    eng.set_causal_slicing(split_size=split)
    try:
        eng.native = False
        dec_p, enc_p = eng.decode(z).sample.clone(), eng.encode(x).latent.clone()
        eng.native = True
        n0 = lib.LAUNCHES
        dec_n = eng.decode(z).sample.clone()
        launches = lib.LAUNCHES - n0
        enc_n = eng.encode(x).latent.clone()
    finally:
        eng.native = True
        eng.set_causal_slicing(split_size=None)
    assert launches >= 100          # kernels of one decode as counted by the native runtime (un-sliced: 153)
    assert dec_n.shape == dec_p.shape == (1, 3, 17, 144, 192) and enc_n.shape == enc_p.shape == (1, 16, 5, 18, 24)
    assert torch.equal(dec_n, dec_p), f"decode (split {split}): native vs python {psnr(dec_n, dec_p):.1f} dB"
    assert torch.equal(enc_n, enc_p), f"encode (split {split}): native vs python {psnr(enc_n, enc_p):.1f} dB"
    # fp16 input, engine-owned workspace, explicit too-small workspace
    h = eng.native_handle()
    sl = 0 if split is None else max(1, split // 4)
    need = eng.workspace_bytes(False, 5, 18, 24, sl)
    out = torch.empty_like(dec_n)
    zh = z[0].half().contiguous()
    ref = eng.decode(zh[None]).sample
    L = lib.load()
    assert L.svr2_vae_decode(h, lib.ptr(zh), 2, 5, 18, 24, sl, lib.ptr(out), None, 0, lib.stream()) == 0
    assert torch.equal(out, ref)
    ws = torch.empty(need, device="cuda", dtype=torch.uint8)
    assert L.svr2_vae_decode(h, lib.ptr(zh), 2, 5, 18, 24, sl, lib.ptr(out), lib.ptr(ws), need - 256, lib.stream()) != 0
    assert b"workspace" in L.svr2_engine_last_error(h)
    out.zero_()
    assert L.svr2_vae_decode(h, lib.ptr(zh), 2, 5, 18, 24, sl, lib.ptr(out), lib.ptr(ws), need, lib.stream()) == 0
    assert torch.equal(out, ref)


def test_engine_workspace_is_resident_and_goes_back_to_the_driver(pkg):
    """lib.workspace: one resident block per device (reused for smaller requests, regrown for larger ones), released to
    the driver — not to the caching allocator — by release_workspace()."""
    lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
    lib.release_workspace()
    a = lib.workspace(1 << 20, "cuda")
    assert a.is_cuda and a.dtype == torch.uint8 and a.numel() >= 1 << 20 and lib.workspace_held("cuda") == a.numel()
    ptr = a.data_ptr()
    b = lib.workspace(1 << 19, "cuda")
    assert b.data_ptr() == ptr
    del a, b
    c = lib.workspace(1 << 22, "cuda")
    assert c.numel() >= 1 << 22 and lib.workspace_held("cuda") == c.numel()
    del c
    reserved = torch.cuda.memory_reserved()
    lib.release_workspace("cuda")
    assert lib.workspace_held("cuda") == 0 and torch.cuda.memory_reserved() <= reserved


def test_vae_attention_single_pass_equals_two_pass_and_falls_back(vae_pair):
    """Mid-block attention (attn_video_vae.py:656-668): the single-pass path (sampled reference exponent, un-normalised
    probabilities, row-sum division in the P V epilogue) against the exact two-pass path on the same input, and the
    device-side fallback: keys crafted so that the true row maximum sits > 2^96 above every sampled key's score must
    still give the exact result (the conditional two-pass launches run)."""
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    eng, sd32 = vae_pair
    p = "decoder.mid_block.attentions.0."
    C, Hh, Ww = 512, 34, 60
    n = Hh * Ww
    g = torch.Generator(device="cuda").manual_seed(13)
    x = vae.Act(2, Hh, Ww, C, 0, "cuda")
    x.buf.copy_(torch.randn(x.buf.shape, generator=g, device="cuda", dtype=torch.bfloat16))

    def run(single):
        return eng._attention(x, p, single_pass=single).buf.clone()
    a, b = run(True), run(False)
    d = (a.float() - b.float()).abs()
    assert psnr(a, b) > 60.0 and d.max() <= 2 ** -5 * b.abs().max().item(), f"single vs two-pass: {psnr(a, b):.1f} dB, max {d.max():.4f}"
    # fallback: scale the K projection so that scores are huge and dominated by individual (mostly un-sampled) keys
    wk, bk = eng.W[p + "to_k.weight"], eng.W[p + "to_k.bias"]
    wk_saved, bk_saved = wk.clone(), bk.clone()
    try:
        wk.mul_(400.0)
        bk.mul_(400.0)
        a, b = run(True), run(False)
        assert torch.isfinite(a).all() and torch.isfinite(b).all()
        # chunks whose rows left the safe range are recomputed by the exact launches (bit-equal); the others stay single-pass
        assert psnr(a, b) > 60.0, f"extreme scores: single-pass + fallback vs exact path {psnr(a, b):.1f} dB"
        assert (a == b).float().mean() > 0.5, "the fallback launches did not run"
    finally:
        wk.copy_(wk_saved)
        bk.copy_(bk_saved)
