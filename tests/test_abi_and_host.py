"""CPU: the C-ABI library loads and exports every symbol include/svr2.h declares (no compute
calls without a GPU); host-side integer logic (padding, sharding, batching)."""
import importlib
import os
import re

import pytest
import torch

from oracle import dit_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(svr2lib):
    import __graft_entry__
    __graft_entry__.build()
    hdr = open(os.path.join(ROOT, "include", "svr2.h")).read()
    declared = set(re.findall(r"\b(svr2_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 19
    lib = svr2lib.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/svr2.h but not exported"
    assert set(svr2lib.SIGNATURES) | {"svr2_last_error", "svr2_engine_last_error"} == declared
    assert lib.svr2_version() >= 100
    assert isinstance(lib.svr2_last_error(), bytes)


def test_handle_api_fails_loudly_without_a_gpu(svr2lib):
    """svr2_create on a box without a B200 returns a status (never a usable handle, never a fallback); argument checks
    of the handle API work without a device."""
    import ctypes
    if torch.cuda.is_available():
        pytest.skip("needs a box without a GPU")
    lib = svr2lib.load()
    desc = svr2lib.ModelDesc(variant=0, dim=256, heads=2, layers=2, mm_layers=1, txt_in_dim=64, in_ch=33, out_ch=16,
                             mlp_kind=0, mlp_hidden=768, out_norm=1, last_vid_only=1, eps=1e-5, timestep=1000.0)
    h = ctypes.c_void_p()
    assert lib.svr2_create(ctypes.byref(h), 0, ctypes.byref(desc)) < 0 and not h.value
    assert lib.svr2_last_error()
    bad = svr2lib.ModelDesc(variant=0, dim=300, heads=2)
    assert lib.svr2_create(ctypes.byref(h), 0, ctypes.byref(bad)) == -1          # SVR2_ERR_ARG: dim != heads * 128
    assert lib.svr2_workspace_bytes(None, 3, 20, 36, 58) == 0
    with pytest.raises(svr2lib.Svr2Error):
        svr2lib.engine_create(desc, 0)


def test_product_path_has_no_oracle_or_fallback():
    pk = os.path.join(ROOT, "comfyui-seedvr2_videoupscaler_b200")
    for fn in os.listdir(pk):
        if fn.endswith(".py"):
            src = open(os.path.join(pk, fn)).read()
            assert "oracle" not in src.replace("oracle/", ""), f"{fn} must not import the oracle"
            assert "scaled_dot_product_attention" not in src and "F.conv3d" not in src


def test_padding_and_partition(pkg):
    import importlib
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    assert [pipeline.pad_4n1(n) for n in (1, 2, 4, 5, 8, 9, 16, 17, 64)] == [1, 5, 5, 5, 9, 9, 17, 17, 65]
    assert shard.partition_frames(64, 8) == [(8 * i, 8 * i + 8) for i in range(8)]
    assert shard.partition_frames(10, 4) == [(0, 3), (3, 6), (6, 8), (8, 10)]
    assert shard.partition_frames(10, 3, overlap=2) == [(0, 6), (4, 9), (7, 10)]
    assert shard.partition_frames(0, 2) == [(0, 0), (0, 0)]


def test_vae_slice_plan_matches_reference_split(pkg):
    """slicing_encode/_decode (attn_video_vae.py:1254-1300): frame 0 rides with the first slice."""
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    plan = vae.B200VideoVAE._plan
    assert plan(17, 4) == [(0, 5), (5, 9), (9, 13), (13, 17)]
    assert plan(5, 4) == [(0, 5)] and plan(1, 4) == [(0, 1)]
    assert plan(10, 3) == [(0, 4), (4, 7), (7, 10)]
    for T, size in ((33, 8), (21, 4), (6, 1)):
        cuts = plan(T, size)
        assert cuts[0][0] == 0 and cuts[-1][1] == T and all(a[1] == b[0] for a, b in zip(cuts, cuts[1:]))


def test_checkpoint_loader_formats(pkg, tmp_path):
    """weights.load_state_dict: safetensors in fp16 and fp8_e4m3fn storage, ComfyUI prefix stripping, .pth, GGUF refusal."""
    from safetensors.torch import save_file
    cfg = dit_oracle.dit_config("3b", layers=2, mm_layers=1, dim=256, heads=2)
    sd = pkg.weights.synth_dit_state_dict(cfg, seed=3, dtype=torch.float16)
    f16 = tmp_path / "dit_fp16.safetensors"
    save_file({k: v.contiguous() for k, v in sd.items()}, str(f16))
    got = pkg.weights.load_state_dict(str(f16))
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    f8 = tmp_path / "dit_fp8_e4m3fn.safetensors"
    save_file({"model.diffusion_model." + k: (v.to(torch.float8_e4m3fn) if v.ndim == 2 else v).contiguous()
               for k, v in sd.items()}, str(f8))
    got8 = pkg.weights.load_state_dict(str(f8))
    assert set(got8) == set(sd)
    k2 = next(k for k, v in sd.items() if v.ndim == 2)
    assert got8[k2].dtype == torch.float8_e4m3fn
    assert torch.equal(got8[k2].to(torch.bfloat16), sd[k2].to(torch.float8_e4m3fn).to(torch.bfloat16))
    pth = tmp_path / "vae.pth"
    torch.save({"a.weight": torch.ones(2, 2)}, str(pth))
    assert torch.equal(pkg.weights.load_state_dict(str(pth))["a.weight"], torch.ones(2, 2))
    with pytest.raises(NotImplementedError):
        pkg.weights.load_state_dict(str(tmp_path / "model.gguf"))
    full = {"vid_in.proj.weight": torch.empty(2560, 132)}
    assert pkg.weights.detect_dit_variant(full) == "3b"
    assert pkg.weights.detect_dit_variant({"vid_in.proj.weight": torch.empty(3072, 132)}) == "7b"


def test_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (the driver's reference arm) runs without a GPU and prints ONE JSON line with the
    keys of the bench contract, the same metric / unit / direction as the B200 arm and `impl: reference`."""
    import json
    import subprocess
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-800:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e", "impl"):
        assert k in d, k
    assert d["impl"] == "reference" and d["metric"] == "upscaled frames/sec SeedVR2-3B 720p->4K" and d["unit"] == "frames/s"
    assert d["higher_is_better"] is True and d["value"] > 0 and d["cpu_baseline"]["kind"] == "port"
    assert d["cpu_baseline"]["cores"] >= 1 and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]


def test_temporal_padding_mirrors_frames_like_the_reference(pkg):
    """pad_video_temporal (generation_utils.py:598-657): the 4n+1 padding appends REVERSED frames (excluding the edge
    frame), not copies of the last frame; goldens are frame-index sequences produced by the reference function."""
    import numpy as np
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    gold = np.load(os.path.join(ROOT, "tests", "golden", "pad_temporal.npz"))
    for t in range(1, 14):
        frames = torch.arange(t, dtype=torch.float32).view(t, 1, 1, 1)          # t h w c, value = frame index
        out = pipeline.pad_video_temporal(frames)
        assert out.shape[0] == pipeline.pad_4n1(t)
        assert out.flatten().tolist() == gold[f"auto_t{t}"].tolist()
        for count in (1, 3, t, t + 2):
            for prepend in (False, True):
                r = pipeline.pad_video_temporal(frames, count=count, prepend=prepend)
                assert r.flatten().tolist() == gold[f"t{t}_c{count}_{'pre' if prepend else 'app'}"].tolist()
    assert pipeline.pad_video_temporal(torch.arange(8.).view(8, 1, 1, 1)).flatten().tolist() == [0, 1, 2, 3, 4, 5, 6, 7, 6]


def test_partition_preloaded_matches_reference_chunking(pkg):
    """inference_cli.py:1196-1213 restated literally (torch.chunk / chunk-with-overlap) vs shard.partition_preloaded."""
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    for total in (1, 5, 16, 23, 64, 97):
        frames = torch.arange(total)
        for n in (1, 2, 3, 4, 8):
            for overlap in (0, 2, 4):
                for bs in (1, 5):
                    if overlap > 0 and n > 1:
                        cwo = total // n + overlap
                        if bs > 1:
                            cwo = ((cwo + bs - 1) // bs) * bs
                        base = cwo - overlap
                        ref = [frames[i * base: (total if i == n - 1 else min(i * base + cwo, total))] for i in range(n)]
                    else:
                        ref = list(torch.chunk(frames, n, dim=0))
                    got = shard.partition_preloaded(total, n, overlap, bs)
                    assert [frames[a:b].tolist() for a, b in got] == [r.tolist() for r in ref], (total, n, overlap, bs)


def test_batched_video_loop_matches_reference_phases(pkg):
    """pipeline.batch_ranges / run_batched vs a literal restatement of the reference's loops: batch indices
    (generation_phases.py:271-289, 344-358), overlap cross-fade into the already written tail and trimming (:969-1000),
    per-batch post-processing against the input frames minus the overlap (:1249-1263)."""
    from oracle import color_oracle
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    blend = lambda p, c: color_oracle.blend_overlapping_frames(p, c, p.shape[0]).to(torch.bfloat16)
    for total, bs, ov in ((23, 5, 0), (23, 5, 2), (17, 9, 4), (12, 5, 3), (9, 5, 4), (6, 5, 7), (5, 5, 2), (30, 13, 1)):
        g = torch.Generator().manual_seed(total * 100 + bs * 10 + ov)
        frames = torch.rand(total, 3, 4, 8, generator=g).to(torch.bfloat16)               # stands for the input clip
        decoded = {}

        def clip(a, b):
            if (a, b) not in decoded:
                decoded[(a, b)] = torch.rand(b - a, 3, 4, 8, generator=g).to(torch.bfloat16)
            return decoded[(a, b)].clone(), frames[a:b].clone()

        post = lambda smp, sty: (smp.float() * 0.5 + sty.float() * 0.25).permute(0, 2, 3, 1)
        got = pipeline.run_batched(total, bs, ov, clip, blend, post)
        # ---- reference restatement
        step = bs - ov if ov > 0 else bs
        eff = ov
        if step <= 0:
            step, eff = bs, 0
        ranges = []
        for idx in range(0, total, step):
            end = min(idx + bs, total)
            if idx > 0 and end - idx <= eff:
                break
            ranges.append((idx, end))
        assert pipeline.batch_ranges(total, bs, ov) == (ranges, eff)
        final = torch.zeros(0, 3, 4, 8, dtype=torch.bfloat16)
        slices = []
        for i, (a, b) in enumerate(ranges):
            smp = decoded[(a, b)].clone()
            start = final.shape[0]
            if i > 0 and eff > 0 and eff < smp.shape[0] and start >= eff:
                final[start - eff:start] = blend(final[start - eff:start], smp[:eff])
                smp = smp[eff:]
            final = torch.cat([final, smp], 0)
            slices.append((start, final.shape[0], a, i))
        outs = []
        for start, stop, a, i in slices:
            sty = frames[a:a + bs][(eff if i > 0 else 0):][: stop - start]
            outs.append(post(final[start:stop], sty))
        ref = torch.cat(outs, 0)
        assert got.shape == ref.shape and torch.equal(got, ref), (total, bs, ov)
        if eff < bs:
            assert got.shape[0] == total or ranges[-1][1] < total


def test_clip_runner_control_flow_with_stubbed_kernels(pkg, monkeypatch):
    """upscale_clip / clip_to_sample / upscale_video sequencing on CPU with the GPU stages stubbed (the kernels are
    covered by the -m gpu tests): shapes, cropping, padding, batching and the colour-correction hook."""
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    preprocess = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.preprocess")
    color_fix = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.color_fix")
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    eng = object.__new__(pipeline.SeedVR2Engine)
    eng.device = torch.device("cpu")
    seen = {}

    def fake_run(self, x, channels_last):                                  # (T,h,w,3) -> (3,T,Hp,Wp), 2x nearest up-scale
        (H, W), _ = preprocess.resized_size(x.shape[1], x.shape[2], self.resolution, self.max_resolution)
        y = torch.nn.functional.interpolate(x.permute(0, 3, 1, 2).float(), size=(H, W)).permute(1, 0, 2, 3)
        y = torch.nn.functional.pad(y, (0, (16 - W % 16) % 16, 0, (16 - H % 16) % 16))
        seen["frames_in"] = x.shape[0]
        return (y * 2 - 1).to(torch.bfloat16)

    monkeypatch.setattr(preprocess.VideoTransform, "run", fake_run)
    eng.vae_encode = lambda x: torch.zeros((x.shape[1] - 1) // 4 + 1, x.shape[2] // 8, x.shape[3] // 8, 16, dtype=torch.bfloat16)
    eng.inference = lambda noise, latent: noise
    eng.clip_workspace = lambda T, Hp, Wp: None                             # no native runtime on the CPU
    eng.vae_decode = lambda z: torch.ones(3, 4 * z.shape[0] - 3, 8 * z.shape[1], 8 * z.shape[2], dtype=torch.bfloat16) * 0.5
    monkeypatch.setattr(color_fix, "apply_color_correction", lambda s_, st, mode, debug=None: (s_.float() * 0 + st.float()).to(torch.bfloat16))
    monkeypatch.setattr(color_fix, "sample_to_image", lambda s_: (s_.float().permute(0, 2, 3, 1).clamp(-1, 1) * 0.5 + 0.5).to(torch.bfloat16))
    monkeypatch.setattr(shard, "blend_overlap", lambda p, c: ((p.float() + c.float()) / 2).to(p.dtype))
    frames = torch.rand(6, 20, 30, 3)
    out = eng.upscale_clip(frames, resolution=40)
    assert out.shape == (6, 40, 60, 3) and seen["frames_in"] == 9           # 6 -> 9 frames (4n+1), cropped back to 6
    assert torch.allclose(out.float(), torch.full_like(out.float(), 0.75))
    out = eng.upscale_clip(frames, resolution=40, color_correction="lab")    # colour hook receives the transformed input
    ref = torch.nn.functional.interpolate(frames.permute(0, 3, 1, 2), size=(40, 60)).permute(0, 2, 3, 1)
    assert out.shape == (6, 40, 60, 3) and (out.float() - ref).abs().max() < 0.02
    smp, sty = eng.clip_to_sample(frames[:5], resolution=40)
    assert smp.shape == sty.shape == (5, 3, 40, 60) and seen["frames_in"] == 5
    vid = eng.upscale_video(torch.rand(13, 20, 30, 3), batch_size=5, temporal_overlap=2, resolution=40)
    assert vid.shape == (13, 40, 60, 3)
    assert tuple(eng.latent_shape(frames, 40)) == (3, 6, 8, 16)


def test_vae_slice_search_picks_the_longest_slice_that_fits(pkg, monkeypatch):
    """B200VideoVAE.plan_slices: un-sliced first, then set_causal_slicing's split, then shorter slices — the first whose
    exact workspace (stubbed here: the native dry run needs no GPU but the module's constructor does) fits the budget."""
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    eng = object.__new__(vae.B200VideoVAE)
    eng.split_size = None
    asked = []

    def fake_ws(encode, T, H, W, sl=0):
        asked.append(sl)
        frames = (T if sl == 0 else min(T, sl + 1))
        return 100 * frames + (50 if sl else 0)            # bytes grow with the slice length; slicing state costs 50

    monkeypatch.setattr(eng, "workspace_bytes", fake_ws, raising=False)
    assert eng.plan_slices(False, 17, 8, 8, budget=10 ** 6) == (0, 1700) and asked == [0]
    del asked[:]
    sz, need = eng.plan_slices(False, 17, 8, 8, budget=1000)            # 100 * (sz + 1) + 50 <= 1000 -> sz = 8
    assert (sz, need) == (8, 950) and asked[0] == 0 and asked[1:] == list(range(15, 7, -1))      # shrinks one frame at a time
    sz, need = eng.plan_slices(True, 33, 64, 64, budget=1400)           # encode: multiples of 4: 100 * 13 + 50 = 1350
    assert (sz, need) == (12, 1350)
    assert eng.plan_slices(True, 10, 64, 64, budget=10)[0] == 0         # not 4n+1 frames: never sliced
    eng.split_size = 16                                                 # set_causal_slicing(split_size=16 sample frames)
    assert eng.plan_slices(False, 17, 8, 8, budget=10 ** 6) == (4, 550)
    assert eng.plan_slices(True, 33, 64, 64, budget=10 ** 6) == (16, 1750)
    assert eng.plan_slices(False, 4, 8, 8, budget=10 ** 6) == (0, 400)  # the clip is shorter than the split
