"""CPU: the alpha path's oracle against the goldens made by the reference's own alpha_upscaling.py, its C-ABI entry
points, and the clip runner's RGBA sequencing with the GPU stages stubbed."""
import ctypes
import importlib
import os
import re

import numpy as np
import pytest
import torch

from oracle import alpha_oracle as ao

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
ALPHA_ENTRY_POINTS = {"svr2_alpha_upscale_scratch_bytes": 5, "svr2_alpha_upscale": 14, "svr2_sobel_edges_f32": 8,
                      "svr2_sample_to_image_rgba_bf16": 5}


@pytest.mark.parametrize("name", list(ao.CASES))
def test_alpha_oracle_matches_reference_goldens(name):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    alpha, rgb = ao.make_inputs(**ao.CASES[name])
    taps = {}
    out = ao.edge_guided_alpha_upscale(alpha, rgb, taps)
    assert torch.equal(taps["edges"], torch.from_numpy(g["edges"]))          # Sobel edges: bit for bit
    assert (out - torch.from_numpy(g["out"])).abs().max().item() <= 1e-6
    assert int(taps["binary"]) == int(g["meta"][-1])


def test_alpha_golden_cases_cover_every_branch():
    flags = {}
    for name in ao.CASES:
        taps = {}
        ao.edge_guided_alpha_upscale(*ao.make_inputs(**ao.CASES[name]), taps)
        flags[name] = (taps["binary"], taps["normalise"], taps["normalise_twice"], taps["edges"].amax().item())
    assert flags["alpha_grad_img"][0] is False and flags["alpha_bin_img"][0] is True
    assert flags["alpha_ratio95"][0] is False and abs(ao.binary_ratio(ao.make_inputs(**ao.CASES["alpha_ratio95"])[0])[0].item() - 0.95) < 1e-7
    assert flags["alpha_nonneg"][1] is False and flags["alpha_bin_t5"][2] is True
    assert flags["alpha_flat"][0] is True and flags["alpha_flat"][3] == 0.0


def test_alpha_entry_points_declared_and_bound(svr2lib):
    import __graft_entry__
    __graft_entry__.build()
    hdr = open(os.path.join(ROOT, "include", "svr2.h")).read()
    lib = svr2lib.load()
    for name, nargs in ALPHA_ENTRY_POINTS.items():
        assert re.search(rf"\b{name}\s*\(", hdr), name
        assert len(svr2lib.SIGNATURES[name]) == nargs and hasattr(lib, name)


def test_alpha_upscale_refuses_bad_arguments_without_touching_memory(svr2lib):
    """Argument checks run before any launch: a too-small scratch is an error status, not a fault."""
    lib = svr2lib.load()
    need = lib.svr2_alpha_upscale_scratch_bytes(5, 720, 1280, 2160, 3840)
    n = 5 * 2160 * 3840
    assert need >= 16 * n and need < 16 * n + (1 << 20)                    # 4 fp32 / u32 planes + tables
    assert lib.svr2_alpha_upscale_scratch_bytes(0, 1, 1, 1, 1) == 0
    fake = ctypes.c_void_p(1 << 20)
    rc = lib.svr2_alpha_upscale(fake, 1, 4, 5, 720, 1280, fake, 2160, 3840, fake, 1, fake, need - 1, None)
    assert rc == -1 and b"scratch too small" in lib.svr2_last_error()
    assert lib.svr2_alpha_upscale(fake, 1, 3, 5, 720, 1280, fake, 2160, 3840, fake, 1, fake, need, None) == -1
    assert lib.svr2_alpha_upscale(fake, 1, 4, 5, 720, 1280, fake, 2160, 3840, fake, 3, fake, need, None) == -1
    assert lib.svr2_sobel_edges_f32(fake, 5, 2160, 3840, fake, fake, 1024, None) == -1


def _stub_engine(pkg, monkeypatch, calls):
    """upscale_clip's GPU stages replaced by CPU stand-ins that log their names (as the host-logic test of
    test_abi_and_host.py does); the alpha stand-in writes each frame's mean input alpha into channel 3."""
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    preprocess = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.preprocess")
    color_fix = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.color_fix")
    alpha = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.alpha")
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    eng = object.__new__(pipeline.SeedVR2Engine)
    eng.device = torch.device("cpu")

    def log(name, fn):
        def wrapped(*a, **k):
            calls.append(name)
            return fn(*a, **k)
        return wrapped

    def fake_run(self, x, channels_last):
        assert x.shape[-1] in (3, 4)
        (H, W), _ = preprocess.resized_size(x.shape[1], x.shape[2], self.resolution, self.max_resolution)
        y = torch.nn.functional.interpolate(x[..., :3].permute(0, 3, 1, 2).float(), size=(H, W)).permute(1, 0, 2, 3)
        y = torch.nn.functional.pad(y, (0, (16 - W % 16) % 16, 0, (16 - H % 16) % 16))
        return (y * 2 - 1).to(torch.bfloat16)

    def fake_alpha(src, sample, image):
        assert src.shape[-1] == 4 and src.shape[0] == sample.shape[0] == image.shape[0]
        image[..., 3] = src[..., 3].float().mean(dim=(1, 2)).view(-1, 1, 1).to(image.dtype)
        return image

    def fake_rgba(sample, image):
        image[..., :3] = (sample.float().permute(0, 2, 3, 1).clamp(-1, 1) * 0.5 + 0.5).to(torch.bfloat16)
        return image

    monkeypatch.setattr(preprocess.VideoTransform, "run", log("preprocess", fake_run))
    eng.vae_encode = log("vae_encode", lambda x: torch.zeros((x.shape[1] - 1) // 4 + 1, x.shape[2] // 8, x.shape[3] // 8, 16,
                                                             dtype=torch.bfloat16))
    eng.inference = log("inference", lambda noise, latent: noise)
    eng.clip_workspace = lambda T, Hp, Wp: None
    eng.vae_decode = log("vae_decode", lambda z: torch.ones(3, 4 * z.shape[0] - 3, 8 * z.shape[1], 8 * z.shape[2],
                                                            dtype=torch.bfloat16) * 0.5)
    monkeypatch.setattr(color_fix, "apply_color_correction",
                        log("color", lambda s_, st, mode, debug=None: (s_.float() * 0 + st.float()).to(torch.bfloat16)))
    monkeypatch.setattr(color_fix, "sample_to_image",
                        log("to_image", lambda s_: (s_.float().permute(0, 2, 3, 1).clamp(-1, 1) * 0.5 + 0.5).to(torch.bfloat16)))
    monkeypatch.setattr(color_fix, "sample_to_image_rgba", log("to_image_rgba", fake_rgba))
    monkeypatch.setattr(alpha, "upscale_into_image", log("alpha", fake_alpha))
    monkeypatch.setattr(shard, "blend_overlap", lambda p, c: ((p.float() + c.float()) / 2).to(p.dtype))
    return eng


def test_rgba_frames_without_keep_alpha_run_the_rgb_sequence(pkg, monkeypatch):
    calls = []
    eng = _stub_engine(pkg, monkeypatch, calls)
    frames4 = torch.rand(6, 20, 30, 4)
    rgb_sequence = ["preprocess", "vae_encode", "inference", "vae_decode", "to_image"]
    for cc, seq in (("none", rgb_sequence), ("lab", rgb_sequence[:-1] + ["color", "to_image"])):
        del calls[:]
        out3 = eng.upscale_clip(frames4[..., :3].contiguous(), resolution=40, color_correction=cc)
        assert calls == seq
        del calls[:]
        out4 = eng.upscale_clip(frames4, resolution=40, color_correction=cc)
        assert calls == seq and torch.equal(out3, out4) and out4.shape == (6, 40, 60, 3)
    del calls[:]
    assert torch.equal(eng.upscale_video(frames4, batch_size=5, temporal_overlap=2, resolution=40),
                       eng.upscale_video(frames4[..., :3].contiguous(), batch_size=5, temporal_overlap=2, resolution=40))
    assert "alpha" not in calls and "to_image_rgba" not in calls


def test_keep_alpha_sequencing_and_per_slice_alpha(pkg, monkeypatch):
    calls = []
    eng = _stub_engine(pkg, monkeypatch, calls)
    frames4 = torch.rand(13, 20, 30, 4)
    frames4[..., 3] = (torch.arange(13).float() / 16).view(13, 1, 1)       # the alpha of frame t is t / 16
    out = eng.upscale_clip(frames4[:6], resolution=40, color_correction="lab", keep_alpha=True)
    # alpha before the colour correction, which stays RGB-only; the RGB channels are those of the RGB path
    assert calls == ["preprocess", "vae_encode", "inference", "vae_decode", "alpha", "color", "to_image_rgba"]
    assert out.shape == (6, 40, 60, 4)
    assert torch.equal(out[..., :3], eng.upscale_clip(frames4[:6], resolution=40, color_correction="lab"))
    assert torch.equal(out[..., 3], (torch.arange(6).float() / 16).view(6, 1, 1).expand(6, 40, 60).to(torch.bfloat16))
    assert eng.upscale_clip(frames4[:6, ..., :3], resolution=40, keep_alpha=True).shape == (6, 40, 60, 3)
    # whole video with overlap: every output frame's alpha comes from its own input frame
    vid = eng.upscale_video(frames4, batch_size=5, temporal_overlap=2, resolution=40, keep_alpha=True)
    assert vid.shape == (13, 40, 60, 4)
    assert torch.equal(vid[..., 3], (torch.arange(13).float() / 16).view(13, 1, 1).expand(13, 40, 60).to(torch.bfloat16))
    assert torch.equal(vid[..., :3], eng.upscale_video(frames4, batch_size=5, temporal_overlap=2, resolution=40))
