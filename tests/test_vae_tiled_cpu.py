"""CPU: the spatially tiled VAE passes of the native runtime (svr2_vae_encode_tiled / svr2_vae_decode_tiled, csrc/vae_engine.cu
compiled with SVR2_HOST_TEST through tests/native/vae_trace.cu) against the Python module's tile-by-tile sequence
(vae.py B200VideoVAE._tiled, `.native = False`): the same tiles in the same order and every kernel with the same scalars,
except two substitutions made exactly where expected — a tile's crop copy + input conversion is the windowed conversion
(svr2_ncdhw_to_ndhwc_window reading the tile's rectangle of the clip), and a tile's final kernel +
svr2_tile_accumulate_bf16 is the final kernel's seam variant (per temporal slice, at the tile's corner of the result).
The exact workspace covers the run and a 256-byte smaller one is refused.  Also: the clip runner's tiling settings."""
import importlib

import pytest
import torch

import native_trace
from native_trace import assert_same_ops, launches, needs_nvcc, run, summary


@pytest.fixture(scope="module")
def tracer(tmp_path_factory):
    return native_trace.harness(tmp_path_factory, "vae_trace")


@pytest.fixture(scope="module")
def cpu_vae(tmp_path_factory):
    """The recording Python VAE module and its weights manifest."""
    with native_trace.recording_vae() as (eng, log):
        yield eng, log, native_trace.write_manifest(eng, str(tmp_path_factory.mktemp("vae_manifest") / "weights.txt"))


def _plan(encode, H, W, tile, ov):
    """vae.py _tiled's plan, written out independently: (whole, Hl, Wl, s, ramp lengths, [(y0, y1, x0, x1)])."""
    f = 8
    th, tw = max(1, tile[0] // f), max(1, tile[1] // f)
    whole = (H <= tile[0] and W <= tile[1]) if encode else (H <= th and W <= tw)
    loh, low = max(0, min(ov[0] // f, th - 1)), max(0, min(ov[1] // f, tw - 1))
    Hl, Wl = ((H + 7) // 8, (W + 7) // 8) if encode else (H, W)
    tiles = []
    for y0 in range(0, Hl, max(1, th - loh)):
        for x0 in range(0, Wl, max(1, tw - low)):
            y1, x1 = min(y0 + th, Hl), min(x0 + tw, Wl)
            if not ((y0 > 0 and y1 - y0 <= loh) or (x0 > 0 and x1 - x0 <= low)):
                tiles.append((y0, y1, x0, x1))
    return whole, Hl, Wl, (1 if encode else 8), ((loh, low) if encode else tuple(ov)), tiles


# (direction, T, H, W, tile, overlap, split_size, frames): H x W sample pixels for encode, latent pixels for decode
CASES = {
    "dec_ragged_skip": ("dec", 2, 10, 14, (32, 48), (8, 16), None, None),     # last row and column inside the overlap
    "dec_one_row": ("dec", 2, 3, 20, (64, 64), (16, 16), None, None),         # the frame is one tile high
    "dec_overlap_clamped": ("dec", 2, 5, 6, (16, 24), (40, 40), None, None),  # overlap >= tile: clamped, ramps truncated
    "dec_sliced": ("dec", 5, 6, 9, (32, 40), (8, 8), 8, None),                # 2 latent frames per temporal slice
    "dec_frames": ("dec", 3, 7, 9, (32, 32), (8, 8), None, 6),                # 6 of 9 output frames
    "dec_sliced_frames": ("dec", 5, 6, 9, (32, 40), (8, 8), 4, 10),           # slices past the wanted frames do not run
    "dec_whole": ("dec", 2, 4, 6, (32, 48), (8, 8), None, None),              # a tile as large as the frame: un-tiled
    "enc_ragged_skip": ("enc", 5, 56, 72, (24, 32), (8, 8), None, None),
    "enc_sliced": ("enc", 9, 40, 48, (24, 24), (8, 16), 4, None),
    "enc_overlap_clamped": ("enc", 1, 32, 40, (16, 16), (64, 64), None, None),
    "enc_whole": ("enc", 5, 32, 40, (32, 48), (8, 8), None, None),
}


@needs_nvcc
@pytest.mark.parametrize("name", list(CASES))
def test_tiled_sequence_matches_python(cpu_vae, tracer, name):
    kind, T, H, W, tile, ov, split, frames = CASES[name]
    enc = kind == "enc"
    eng, log, manifest = cpu_vae
    del log[:]
    eng.set_causal_slicing(split_size=split)
    try:
        if enc:
            out = eng.encode(torch.zeros(1, 3, T, H, W, dtype=torch.bfloat16), tiled=True, tile_size=tile, tile_overlap=ov).latent
        else:
            out = eng.decode(torch.zeros(1, 16, T, H, W, dtype=torch.bfloat16), tiled=True, tile_size=tile, tile_overlap=ov,
                             frames=frames).sample
    finally:
        eng.set_causal_slicing(split_size=None)
    F = (T - 1) // 4 + 1 if enc else (4 * T - 3 if frames is None else frames)
    assert tuple(out.shape) == ((1, 16, F, H // 8, W // 8) if enc else (1, 3, F, 8 * H, 8 * W))
    want = list(log)
    slice_frames = 0 if split is None else (max(4, split // 4 * 4) if enc else max(1, split // 4))
    rc, got, err = run(tracer, manifest, "tiled", kind, T, H, W, *tile, *ov, slice_frames, F)
    assert rc == 0, (rc, err[-2000:])
    need, touched, n_launches = summary(got.pop())
    assert 0 < touched < need and need % 256 == 0                  # the dry run covers the run (a 256 B smaller one is refused)

    whole, Hl, Wl, s, (lh, lw), tiles = _plan(enc, H, W, tile, ov)
    if whole:                                                       # the un-tiled pass, exactly
        assert_same_ops(got, want)
        assert not any("accumulate" in ln for ln in want)
        assert n_launches == launches(want)
        return
    assert got[0] == f"svr2_tile_ramp_bf16 {'p1' if lh else 'p0'} {lh} {'p1' if lw else 'p0'} {lw} p0", got[0]
    Hr, Wr, C = Hl * s, Wl * s, (16 if enc else 3)
    Hin, Win = (H, W)
    f = 8 if enc else 1
    final_name = "svr2_ndhwc_to_ncdhw" if enc else "svr2_conv_tap_gather"
    gi, tile_i, inputs, finals = 1, 0, [], []
    n_window = n_seam = 0
    for w_ in want:
        name_ = w_.split()[0]
        if name_ == "svr2_tile_accumulate_bf16":                   # closes the tile: check its substitutions
            tok = w_.split()
            planes, eh, ew, rH, rW, y0s, x0s = (int(t) for t in (tok[4], tok[5], tok[6], tok[11], tok[12], tok[13], tok[14]))
            y0, y1, x0, x1 = tiles[tile_i]
            assert (rH, rW, y0s, x0s, eh, ew, planes) == (Hr, Wr, y0 * s, x0 * s, (y1 - y0) * s, (x1 - x0) * s, C * F), w_
            edges = (1 if y0 > 0 else 0) | (2 if y1 < Hl else 0) | (4 if x0 > 0 else 0) | (8 if x1 < Wl else 0)
            a = 0
            for py, nat in inputs:                                  # the tile's window of the clip, slice by slice
                cs, fs, rs, off = (int(t) for t in nat.split(" | ")[1].split())
                assert (cs, fs, rs) == (T * Hin * Win, Hin * Win, Win), nat
                assert off == a * Hin * Win + y0 * f * Win + x0 * f, (nat, a, y0, x0)
                a += int(py.split()[4])
            o = 0
            for k, (py, nat) in enumerate(finals):                  # the seam per temporal slice, count plane in the first
                off, cs, fs, rs = (int(t) for t in nat.split(" | ")[1].split()[:4])
                cnt, l_h, l_w, e = nat.split(" | ")[1].split()[4:]
                assert (off, cs, fs, rs) == (o * Hr * Wr + y0 * s * Wr + x0 * s, F * Hr * Wr, Hr * Wr, Wr), nat
                assert (cnt, int(l_h), int(l_w), int(e)) == ("p1" if k == 0 else "p0", lh, lw, edges), nat
                o += int(py.split()[4 if enc else 5])
            assert o == F, (o, F)
            tile_i += 1
            inputs, finals = [], []
            continue
        g = got[gi]
        gi += 1
        if name_ == "svr2_ncdhw_to_ndhwc_bf16":
            assert g.split(" | ")[0] == w_.replace("svr2_ncdhw_to_ndhwc_bf16", "svr2_ncdhw_to_ndhwc_window"), (g, w_)
            inputs.append((w_, g))
            n_window += 1
        elif name_ == final_name:
            head = g.split(" | ")[0].split()
            py = w_.split()
            assert head[0] == final_name + "_seam", (g, w_)
            n = 7 if enc else 8                                     # in/z .. W (the plain call's output pointer dropped)
            assert head[1:n] == py[1:n] and head[-1] == py[-1], (g, w_)
            finals.append((w_, g))
            n_seam += 1
        else:
            assert g == w_, f"op {gi - 1}: native `{g}` vs python `{w_}`"
    assert gi == len(got) and tile_i == len(tiles)
    assert n_window == n_seam                                       # one of each per temporal slice
    n_acc = sum(w_.startswith("svr2_tile_accumulate_bf16") for w_ in want)
    assert n_launches == launches(want) - n_acc + 1


@needs_nvcc
def test_tiled_arguments_refused(cpu_vae, tracer):
    _, _, manifest = cpu_vae
    for args in (("dec", 2, 8, 8, 0, 64, 8, 8, 0, 5), ("dec", 2, 8, 8, 64, 64, -8, 8, 0, 5), ("dec", 2, 8, 8, 32, 32, 8, 8, 0, 6),
                 ("enc", 5, 36, 40, 32, 32, 8, 8, 0, 0)):
        rc, _, err = run(tracer, manifest, "tiled", *args)
        assert rc == 3 and "refused" in err, (args, rc, err)


@needs_nvcc
def test_tiled_4k_needs_fit_one_gpu(cpu_vae, tracer):
    """Exact needs of the 4K batch passes (2160 x 3840 from a 720p source: latent 270 x 480) at the loader's default tile
    1024 / overlap 128: a 9-frame encode and a 3-latent-frame decode, tiled, against the same passes un-tiled."""
    _, _, manifest = cpu_vae

    def need(*args):
        rc, lines, err = run(tracer, manifest, "tiled", *args, "plan")
        assert rc == 0, err[-2000:]
        return int(lines[-1].split()[2])

    enc_tiled, enc_whole = need("enc", 9, 2160, 3840, 1024, 1024, 128, 128, 0, 0), need("enc", 9, 2160, 3840, 8192, 8192, 0, 0, 0, 0)
    dec_tiled, dec_whole = need("dec", 3, 270, 480, 1024, 1024, 128, 128, 0, 9), need("dec", 3, 270, 480, 8192, 8192, 0, 0, 0, 9)
    print(f"4K 9 frames: encode {enc_tiled / 1e9:.1f} GB tiled vs {enc_whole / 1e9:.1f} GB; "
          f"decode {dec_tiled / 1e9:.1f} GB tiled vs {dec_whole / 1e9:.1f} GB")
    assert enc_tiled < 20e9 and dec_tiled < 20e9 and enc_whole > 60e9 and dec_whole > 100e9


def test_clip_runner_tiling_settings_with_stubbed_kernels(pkg, monkeypatch):
    """The clip runner's tiling settings on the CPU with the GPU stages stubbed: which phases tile with which
    (tile_h, tile_w, overlap_h, overlap_w), one workspace per clip sized for the tiled passes, and the untouched calls
    when tiling is off."""
    pipeline = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.pipeline")
    preprocess = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.preprocess")
    color_fix = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.color_fix")
    shard = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.shard")
    eng = object.__new__(pipeline.SeedVR2Engine)
    eng.device = torch.device("cpu")
    calls = []

    def fake_run(self, x, channels_last):
        (H, W), _ = preprocess.resized_size(x.shape[1], x.shape[2], self.resolution, self.max_resolution)
        y = torch.nn.functional.interpolate(x.permute(0, 3, 1, 2).float(), size=(H, W)).permute(1, 0, 2, 3)
        y = torch.nn.functional.pad(y, (0, (16 - W % 16) % 16, 0, (16 - H % 16) % 16))
        return (y * 2 - 1).to(torch.bfloat16)

    monkeypatch.setattr(preprocess.VideoTransform, "run", fake_run)

    def vae_encode(x, workspace=None, tiles=None):
        calls.append(("encode", workspace, tiles))
        return torch.zeros((x.shape[1] - 1) // 4 + 1, x.shape[2] // 8, x.shape[3] // 8, 16, dtype=torch.bfloat16)

    def vae_decode(z, workspace=None, frames=None, tiles=None):
        calls.append(("decode", workspace, tiles))
        return torch.zeros(3, frames, 8 * z.shape[1], 8 * z.shape[2], dtype=torch.bfloat16)

    def clip_workspace(T, Hp, Wp, frames=None, **tiling):
        calls.append(("workspace", pipeline.tiling_settings(tiling)))
        return "WS"

    eng.vae_encode, eng.vae_decode, eng.clip_workspace = vae_encode, vae_decode, clip_workspace
    eng.inference = lambda noise, latent, workspace=None: noise
    monkeypatch.setattr(color_fix, "sample_to_image", lambda s_: (s_.float().permute(0, 2, 3, 1) * 0.5 + 0.5).to(torch.bfloat16))
    monkeypatch.setattr(shard, "blend_overlap", lambda p, c: p)
    frames = torch.rand(5, 20, 30, 3)

    eng.upscale_clip(frames, resolution=40)
    assert calls == [("workspace", {}), ("encode", "WS", None), ("decode", "WS", None)]
    del calls[:]
    eng.upscale_clip(frames, resolution=40, decode_tiled=True)
    assert [c[0] for c in calls] == ["workspace", "encode", "decode"]
    assert calls[0][1]["decode_tiled"] and not calls[0][1]["encode_tiled"]
    assert calls[1][2] is None and calls[2][2] == (1024, 1024, 128, 128)
    del calls[:]
    eng.upscale_clip(frames, resolution=40, encode_tiled=True, encode_tile_size=(512, 768), encode_tile_overlap=64,
                     decode_tiled=True, decode_tile_size=256, decode_tile_overlap=(32, 16))
    assert calls[1][2] == (512, 768, 64, 64) and calls[2][2] == (256, 256, 32, 16)
    assert sum(c[0] == "workspace" for c in calls) == 1                 # one workspace per clip
    del calls[:]
    vid = eng.upscale_video(torch.rand(13, 20, 30, 3), batch_size=5, temporal_overlap=2, resolution=40, encode_tiled=True)
    assert vid.shape == (13, 40, 60, 3)
    n_ws = sum(c[0] == "workspace" for c in calls)
    assert n_ws == sum(c[0] == "encode" for c in calls) == 4            # one workspace per batch
    assert all(c[2] == (1024, 1024, 128, 128) for c in calls if c[0] == "encode")
    assert all(c[2] is None for c in calls if c[0] == "decode")
    del calls[:]
    got = list(eng.stream_video(torch.rand(13, 20, 30, 3), batch_size=5, temporal_overlap=2, resolution=40, decode_tiled=True,
                                out_dtype=torch.bfloat16))
    assert sum(t.shape[0] for _, t in got) == 13
    assert all(c[2] == (1024, 1024, 128, 128) for c in calls if c[0] == "decode")
    with pytest.raises(TypeError, match="tiling"):
        eng.upscale_clip(frames, resolution=40, decode_tile=512)
    with pytest.raises(ValueError, match="tile_overlap"):
        eng.upscale_clip(frames, resolution=40, decode_tiled=True, decode_tile_overlap=-8)
