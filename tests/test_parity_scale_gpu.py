"""-m gpu: parity at the sizes that are benchmarked (VERDICT r1 item 1).

The oracle (oracle/dit_oracle.py, oracle/vae_oracle.py — pinned to the reference's own modules by
tests/test_oracle_golden.py) runs on the same GPU in true fp32 (TF32 off, tests/conftest.py) and in the reference's
bf16 rounding flow ("ref_bf16"); the engine goes through the C ABI.  Stated tolerances:

* full-width / full-depth DiT (3B: 2560 x 20 heads x 32 layers, 7B: 3072 x 24 x 36): output PSNR vs the fp32 oracle
  >= 50 dB (north_star "latent PSNR >= 50 dB") and never more than 1 dB below what the reference's own bf16 flow reaches
  on the same inputs (the reference-vs-reference floor is recorded beside it);
* VAE at 1088 x 1920: >= 40 dB vs fp32 and never more than 3 dB below the reference's bf16 flow (random weights
  amplify bf16 noise; the reference's bf16 flow is the bar);
* single ops at 4K shapes (band raster, swap-AB, fused GroupNorm statistics, pixel-shuffle store): every element within
  its rounding bound of the fp64 reference on the same bf16 operands; the conv also at relative L2 error <= 4e-3 (the
  mid-block attention at n = 129 600: tests/test_vae_attention_elementwise_gpu.py);
* whole clip (pre-process -> encode -> x0.9152 -> DiT -> noise - v -> /0.9152 -> decode -> crop) vs the oracle chain
  ``runner_encode -> dit_forward -> one_step_latent -> runner_decode`` (infer.py:54-78,117-199,315-395): not more than
  3 dB below the reference's bf16 flow.

Measured values are appended to the JSON file named by SVR2_PARITY_RECORD when it is set."""
import gc
import importlib
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import parity_record
from oracle import dit_oracle, vae_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda"


def psnr(a, b):
    a, b = a.float(), b.float()
    return (10 * torch.log10(b.abs().max() ** 2 / (a - b).pow(2).mean())).item()


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _mod(name):
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200." + name)


# ----------------------------------------------------------------------------------------------------------------
# (a) full-width, full-depth DiT
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant,geom", [("3b", (5, 136, 240)),      # BASELINE config 2: 40 800 tokens, 75 / 90 windows
                                          ("7b", (2, 136, 240))])     # 7B at a config-4-like 2-frame latent: 16 320 tokens
def test_dit_full_model_vs_oracle(pkg, variant, geom):
    dit = _mod("dit")
    cfg = dit.dit_config(variant)
    T, H, W = geom
    l = 58
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=77, dtype=torch.float16, device=DEV)
    g = torch.Generator().manual_seed(5)
    vid = torch.randn(T * H * W, 33, generator=g).to(DEV)
    txt = torch.randn(l, cfg["txt_in_dim"], generator=g).to(DEV)
    eng = dit.B200NaDiT(cfg, sd)
    out = eng(vid, txt, [[T, H, W]], [[l]]).vid_sample.float()
    out2 = eng(vid, txt, [[T, H, W]], [[l]]).vid_sample.float()
    assert torch.equal(out, out2), "engine must be deterministic"
    del eng, out2
    _free()
    sd32 = {k: v.float() for k, v in sd.items()}
    del sd
    _free()
    ocfg = dit_oracle.dit_config(variant)
    ref32 = dit_oracle.dit_forward(sd32, ocfg, vid, txt, T, H, W, mode="fp32")
    refbf = dit_oracle.dit_forward(sd32, ocfg, vid, txt, T, H, W, mode="ref_bf16").float()
    res = dict(tokens=T * (H // 2) * (W // 2), layers=cfg["layers"], dim=cfg["dim"],
               engine_vs_fp32=psnr(out, ref32), refbf16_vs_fp32=psnr(refbf, ref32), engine_vs_refbf16=psnr(out, refbf))
    # reference-vs-reference floor: the same bf16 flow with the reference's other attention backends
    for impl in ("sdpa", "flash_attn"):
        try:
            alt = dit_oracle.dit_forward(sd32, ocfg, vid, txt, T, H, W, mode="ref_bf16", attn_impl=impl).float()
            res[f"refbf16_{impl}_vs_fp32"] = psnr(alt, ref32)
            res[f"refbf16_{impl}_vs_refbf16_math"] = psnr(alt, refbf)
            res[f"engine_vs_refbf16_{impl}"] = psnr(out, alt)
            del alt
        except Exception as ex:   # noqa: BLE001 - a backend may be unavailable on the box; the floor is a report
            res[f"refbf16_{impl}"] = f"unavailable: {type(ex).__name__}"
    parity_record(f"dit_{variant}_full_{T}x{H}x{W}", **res)
    print(res)
    assert torch.isfinite(out).all()
    floor = min(50.0, res["refbf16_vs_fp32"] - 1.0)
    assert res["engine_vs_fp32"] >= floor, res


# ----------------------------------------------------------------------------------------------------------------
# (b) VAE at 1088 x 1920
# ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def vae_pair(pkg):
    vae = _mod("vae")
    sd = pkg.weights.synth_vae_state_dict(seed=4321, dtype=torch.float16)
    return vae.B200VideoVAE(sd), {k: v.float().to(DEV) for k, v in sd.items()}


def test_vae_1080p_vs_oracle(vae_pair):
    eng, sd32 = vae_pair
    g = torch.Generator().manual_seed(21)
    z = torch.randn(1, 16, 2, 136, 240, generator=g).to(DEV)             # -> 5 frames of 1088 x 1920
    out = eng.decode(z).sample
    assert out.shape == (1, 3, 5, 1088, 1920)
    ref32 = vae_oracle.vae_decode(sd32, z, mode="fp32")
    _free()
    refbf = vae_oracle.vae_decode(sd32, z, mode="ref_bf16")
    _free()
    d_eng, d_ref = psnr(out, ref32), psnr(refbf, ref32)
    x = out.clamp(-1, 1)
    del ref32, refbf
    _free()
    lat = eng.encode(x).latent
    assert lat.shape == (1, 16, 2, 136, 240)
    ref32 = vae_oracle.vae_encode(sd32, x.float(), mode="fp32")
    _free()
    refbf = vae_oracle.vae_encode(sd32, x.float(), mode="ref_bf16")
    e_eng, e_ref = psnr(lat, ref32), psnr(refbf, ref32)
    parity_record("vae_1080p_5f", decode_engine_vs_fp32=d_eng, decode_refbf16_vs_fp32=d_ref,
                  encode_engine_vs_fp32=e_eng, encode_refbf16_vs_fp32=e_ref)
    print(dict(d_eng=d_eng, d_ref=d_ref, e_eng=e_eng, e_ref=e_ref))
    assert d_eng >= 40.0 and d_eng >= d_ref - 3.0, f"decode: engine {d_eng:.1f} dB vs reference-bf16 flow {d_ref:.1f} dB"
    assert e_eng >= 40.0 and e_eng >= e_ref - 3.0, f"encode: engine {e_eng:.1f} dB vs reference-bf16 flow {e_ref:.1f} dB"


# ----------------------------------------------------------------------------------------------------------------
# (c) single ops at 4K shapes, through the engine's own layer wrappers (production dispatch: statistics-emitting conv,
#     band raster, swap-AB / CTA pairs, chunked attention)
# ----------------------------------------------------------------------------------------------------------------
def _conv_check_strips(x_buf, w, b, y, what):
    """Causal 3x3x3 conv (stride 1, padding 1) against the fp64 reference on the same bf16 operands, strip by strip
    (bounded memory): every element within the per-element bound of tests/test_conv_elementwise_gpu.py (one k-loop of
    K = 27 Cin, the bias add, one bf16 rounding); returns the relative L2 error against the bf16-rounded reference.
    x_buf (T+2,H,W,Cin) bf16 incl. the 2 halo frames; y (T,H,W,Cout) engine output."""
    from test_conv_elementwise_gpu import MAX_STRIP, U, check_elements, conv_ref_rows, raster, ulp_bf16, where
    Tt, H, W, Cin = x_buf.shape
    T, Cout = Tt - 2, w.shape[0]
    wb = w.to(torch.bfloat16).permute(0, 2, 3, 4, 1)                       # (Cout, kt, kh, kw, Cin)
    bd = b.to(torch.bfloat16).double()
    rs = raster(Cin, Cout, (3, 3, 3), 1, H, W)
    strip = max(1, MAX_STRIP // (T * W * Cout))
    num = den = 0.0
    for h0 in range(0, H, strip):
        h1 = min(H, h0 + strip)
        r, S = conv_ref_rows(x_buf, wb, 3, 3, 3, 1, 1, 1, T, W, h0, h1)
        r += bd
        S += bd.abs()
        check_elements(y[:, h0:h1], r, ulp_bf16(r) + (27 * Cin / 4 + 1) * U * S, what,
                       lambda t, h, w_: where(rs, t, h + h0, w_))
        rb = r.to(torch.bfloat16).double()
        num += (y[:, h0:h1].double() - rb).pow(2).sum().item()
        den += rb.pow(2).sum().item()
        del r, S, rb
    return math.sqrt(num / max(den, 1e-30))


@pytest.mark.parametrize("prefix,Cin,Cout", [("decoder.up_blocks.3.resnets.1.conv1", 128, 128),     # swap-AB, 4K
                                             ("decoder.up_blocks.3.resnets.0.conv1", 256, 128),     # swap-AB, K = 6912
                                             ("decoder.up_blocks.2.upsamplers.0.conv", 256, 256)])  # CTA pair, 4K
def test_conv3d_4k_band_raster_and_stats(vae_pair, prefix, Cin, Cout):
    vae = _mod("vae")
    eng, sd32 = vae_pair
    T, H, W = 2, 2160, 3840
    x = vae.Act(T, H, W, Cin, 2, DEV)
    g = torch.Generator(device=DEV).manual_seed(3)
    x.buf.copy_(torch.randn(x.buf.shape, generator=g, device=DEV, dtype=torch.bfloat16))
    y = eng._conv(x, prefix, stats=True)
    assert y.stats is not None and (y.T, y.H, y.W, y.C) == (T, H, W, Cout)
    e = _conv_check_strips(x.buf, sd32[prefix + ".weight"], sd32[prefix + ".bias"], y.body, f"conv {Cin}->{Cout} at 4K")
    # GroupNorm + SiLU from the statistics the conv epilogue produced, against torch on the engine's own conv output
    gn_prefix = {128: "decoder.up_blocks.3.resnets.1.norm2", 256: "decoder.up_blocks.2.resnets.2.norm2"}[Cout]
    gout = eng._gn(y, gn_prefix, True, 2)
    e_gn = 0.0
    for f in range(T):
        yf = y.body[f].permute(2, 0, 1)[None].float()
        r = F.group_norm(yf, 32, sd32[gn_prefix + ".weight"].bfloat16().float(), sd32[gn_prefix + ".bias"].bfloat16().float(), 1e-6)
        r = F.silu(r.bfloat16().float())[0].permute(1, 2, 0)
        e_gn = max(e_gn, rel_err(gout.body[f], r))
        del yf, r
    assert torch.equal(gout.buf[0], gout.buf[2]) and torch.equal(gout.buf[1], gout.buf[2])
    parity_record(f"conv3d_4k_{Cin}to{Cout}", rel_err=e, gn_from_stats_rel_err=e_gn)
    assert e < 4e-3, f"conv {Cin}->{Cout} at 4K: rel err {e:.3e}"
    assert e_gn < 6e-3, f"GroupNorm from epilogue statistics at 4K: rel err {e_gn:.3e}"


def test_upsample_shuffle_1080p_to_4k(vae_pair, svr2lib):
    """The 256-channel pixel-shuffle GEMM 1080p -> 4K, every element within the bound of
    tests/test_conv_elementwise_gpu.py::test_upsample_shuffle_elementwise (one k-loop of K = C, the bias add, one bf16
    rounding) against fp64, strip by strip; a guard frame before the halo and one after the body keep their sentinel."""
    from test_conv_elementwise_gpu import MAX_STRIP, U, check_elements, check_untouched, sentinel_fill, ulp_bf16
    eng, sd32 = vae_pair
    p = "decoder.up_blocks.2.upsamplers.0."
    C, Fr, H, W = 256, 2, 1080, 1920
    g = torch.Generator(device=DEV).manual_seed(4)
    x = torch.randn(Fr, H, W, C, generator=g, device=DEV, dtype=torch.bfloat16)
    obuf = sentinel_fill(torch.empty(1 + 2 + Fr + 1, 2 * H, 2 * W, C, device=DEV, dtype=torch.bfloat16))
    out = obuf[1:-1]
    w, b = eng.W[p + "upscale_conv.weight"], eng.W[p + "upscale_conv.bias"]
    svr2lib.call("svr2_upsample_shuffle_bf16", svr2lib.ptr(x), Fr, H, W, C, svr2lib.ptr(w), svr2lib.ptr(b), 0, 1,
                 svr2lib.ptr(out), 2, 1, svr2lib.stream())
    torch.cuda.synchronize()
    check_untouched(obuf[0], "shuffle 1080p->4K: guard frame")
    check_untouched(obuf[-1], "shuffle 1080p->4K: slack frame")
    assert torch.equal(out[0], out[2]) and torch.equal(out[1], out[2])
    wd, bd = w.reshape(4 * C, C).double(), b.double()
    strip = max(1, MAX_STRIP // (4 * W * C))
    for f in range(Fr):
        for h0 in range(0, H, strip):
            h1 = min(H, h0 + strip)
            xs = x[f, h0:h1].double().reshape(-1, C)
            r = (xs @ wd.T + bd).view(h1 - h0, W, 2, 2, C)                             # channel = ((x*2 + y)*1 + z)*C + c
            S = (xs.abs() @ wd.abs().T + bd.abs()).view(h1 - h0, W, 2, 2, C)
            r, S = (t.permute(0, 2, 1, 3, 4).reshape(1, 2 * (h1 - h0), 2 * W, C) for t in (r, S))   # (h x) (w y) c
            check_elements(out[2 + f:3 + f, 2 * h0:2 * h1], r, ulp_bf16(r) + (C / 4 + 1) * U * S,
                           "upsample shuffle 1080p->4K",
                           lambda t, h, w_: f"frame {f}, GEMM row {(h0 + h // 2) * W + w_ // 2} "
                                            f"(m-tile {((f * H + h0 + h // 2) * W + w_ // 2) // 128}), "
                                            f"column group (x {h % 2}, y {w_ % 2})")
            del xs, r, S


# ----------------------------------------------------------------------------------------------------------------
# (d) whole clip vs the oracle chain (a1 / a2 / a16)
# ----------------------------------------------------------------------------------------------------------------
def test_clip_chain_vs_oracle(pkg):
    pipeline, dit, preprocess = _mod("pipeline"), _mod("dit"), _mod("preprocess")
    over = dict(dim=512, heads=4, layers=6, mm_layers=3, txt_in_dim=256)
    cfg = dit.dit_config("3b", **over)
    dit_sd = pkg.weights.synth_dit_state_dict(cfg, seed=31, dtype=torch.float16)
    vae_sd = pkg.weights.synth_vae_state_dict(seed=4321, dtype=torch.float16)
    g = torch.Generator().manual_seed(8)
    txt = torch.randn(58, 256, generator=g)
    eng = pipeline.SeedVR2Engine(cfg, dit_sd, vae_sd, txt)
    T0, H, W = 8, 272, 480
    lo = torch.rand(T0, 3, H // 8, W // 8, generator=g)
    frames = F.interpolate(lo, size=(H, W), mode="bicubic", align_corners=False).clamp(0, 1).permute(0, 2, 3, 1).contiguous()
    frames = frames.to(DEV)
    noise = torch.randn(eng.latent_shape(frames), generator=g).to(DEV, torch.bfloat16)
    sample, _ = eng.clip_to_sample(frames, noise=noise)                       # (T0,3,H,W) bf16 in ~[-1,1]
    assert sample.shape == (T0, 3, H, W)
    # the oracle chain on the pre-processed clip (the transform itself is pinned bit-wise by tests/test_post_gpu.py)
    x = preprocess.VideoTransform(min(H, W)).run(pipeline.pad_video_temporal(frames), channels_last=True)   # (3,9,H,W)
    sdv32 = {k: v.float().to(DEV) for k, v in vae_sd.items()}
    sdd32 = {k: v.float().to(DEV) for k, v in dit_sd.items()}
    ocfg = dit_oracle.dit_config("3b", **over)
    res = {}
    outs = {}
    for mode in ("fp32", "ref_bf16"):
        lat = vae_oracle.runner_encode(sdv32, x[None].float(), mode)                          # (T',h,w,16) scaled
        Tl, h, w_, c = lat.shape
        nz = noise.float() if mode == "fp32" else noise
        vid = torch.cat([nz, lat.to(nz.dtype), torch.ones(Tl, h, w_, 1, device=DEV, dtype=nz.dtype)], -1)    # infer.py:54-78
        v = dit_oracle.dit_forward(sdd32, ocfg, vid.view(Tl * h * w_, 2 * c + 1), txt.to(DEV), Tl, h, w_, mode=mode)
        x0 = dit_oracle.one_step_latent(nz, v.view(Tl, h, w_, c).to(nz.dtype))                # euler.py:59-63
        y = vae_oracle.runner_decode(sdv32, x0, mode)[0, :, :T0].permute(1, 0, 2, 3)          # (T0,3,H,W)
        outs[mode] = y.float()
        if mode == "fp32":
            lat32 = lat
        else:
            res["latent_refbf16_vs_fp32"] = psnr(lat, lat32)
    lat_eng = eng.vae_encode(x)
    res["latent_engine_vs_fp32"] = psnr(lat_eng, lat32)
    res["clip_engine_vs_fp32"] = psnr(sample, outs["fp32"])
    res["clip_refbf16_vs_fp32"] = psnr(outs["ref_bf16"], outs["fp32"])
    res["clip_engine_vs_refbf16"] = psnr(sample, outs["ref_bf16"])
    parity_record("clip_chain_8f_272x480", **res)
    print(res)
    assert torch.isfinite(sample).all()
    assert res["latent_engine_vs_fp32"] >= res["latent_refbf16_vs_fp32"] - 3.0, res
    assert res["clip_engine_vs_fp32"] >= res["clip_refbf16_vs_fp32"] - 3.0, res
