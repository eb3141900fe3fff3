"""CPU: the VAE decode that returns only the first F output frames (svr2_vae_decode_frames / B200VideoVAE.decode(frames=F)).
The native runtime (csrc/vae_engine.cu, compiled with SVR2_HOST_TEST through tests/native/vae_trace.cu) must
enqueue the same kernels with the same scalar arguments as the Python module's sequencing (vae.py); F = 4T-3 must be
exactly svr2_vae_decode; every layer after the last temporal upsampler must run on the slice's wanted frames only; the
workspace plan must cover the run and be exact; F outside 1 .. 4T-3 must be refused."""
import pytest
import torch

import native_trace
from native_trace import assert_same_ops, launches, run, summary

pytestmark = native_trace.needs_nvcc


@pytest.fixture(scope="module")
def tracer(tmp_path_factory):
    return native_trace.harness(tmp_path_factory, "vae_trace")


@pytest.fixture(scope="module")
def cpu_vae(tmp_path_factory):
    """The recording Python VAE module and its weights manifest."""
    with native_trace.recording_vae() as (eng, log):
        yield eng, log, native_trace.write_manifest(eng, str(tmp_path_factory.mktemp("vae_manifest") / "weights.txt"))


def _slices(T, slice_frames):
    """[(first latent frame, latent frames, output frames)] of the native decode (vae_engine.cu Run::decode)."""
    if slice_frames <= 0 or T - 1 <= slice_frames:
        return [(0, T, 4 * T - 3)]
    out, a, b = [], 0, 1 + slice_frames
    while a < T:
        out.append((a, b - a, 4 * (b - a) - (3 if a == 0 else 0)))
        a, b = b, min(b + slice_frames, T)
    return out


def _keeps(T, slice_frames, F):
    """Output frames each slice computes when only the first F are wanted: later slices do not run, the last is trimmed."""
    keeps, o0 = [], 0
    for _, _, n_out in _slices(T, slice_frames):
        if F <= o0:
            break
        keeps.append(min(F - o0, n_out))
        o0 += n_out
    return keeps


# (T, h, w, slice_frames, F): un-sliced T = 2, 3, 5 with F = 4T-3 - {0, 1, 2, 3}; sliced decodes whose last slice is trimmed
# by 1 - 3 frames, and ones where later slices do not run at all
CASES = ([(T, 4, 6, 0, 4 * T - 3 - d) for T in (2, 3, 5) for d in range(4)]
         + [(5, 6, 10, 2, 17 - d) for d in (1, 2, 3)]             # slices of 3 + 2 latent frames: 9 + 8 output frames
         + [(6, 5, 7, 1, 21 - d) for d in (1, 2, 3)]              # 2 + 1 + 1 + 1 + 1 latent frames: 5 + 4 x 4 output frames
         + [(6, 5, 7, 1, 9), (6, 5, 7, 1, 7), (6, 5, 7, 1, 3), (5, 6, 10, 2, 9)])


@pytest.mark.parametrize("T,h,w,slice_frames,F", CASES)
def test_trimmed_decode_sequence_matches_python(cpu_vae, tracer, T, h, w, slice_frames, F):
    eng, log, manifest = cpu_vae
    del log[:]
    eng.set_causal_slicing(split_size=None if slice_frames == 0 else 4 * slice_frames)
    try:
        out = eng.decode(torch.zeros(1, 16, T, h, w, dtype=torch.bfloat16), frames=F).sample
    finally:
        eng.set_causal_slicing(split_size=None)
    assert out.shape == (1, 3, F, 8 * h, 8 * w)
    want = list(log)
    rc, lines, err = run(tracer, manifest, "frames", T, h, w, slice_frames, F)
    assert rc == 0, (rc, err[-2000:])
    need, touched, n_launches = summary(lines.pop())
    assert_same_ops(lines, want)                                   # without the channel-stride suffix of the strided converters
    assert 0 < touched < need and need % 256 == 0                  # the dry run covers the run (a 256 B smaller one is refused)
    assert n_launches == launches(want)

    # per slice: identical to the untrimmed decode up to the last temporal upsampler's shuffle, then every layer on `keep`
    keeps = _keeps(T, slice_frames, F)
    rc, full, err = run(tracer, manifest, "dec", T, h, w, slice_frames)
    assert rc == 0, err[-2000:]
    full.pop()
    split = lambda ls: [[ln for ln in s.split("\n") if ln] for s in "\n".join(ls).split("svr2_ncdhw_to_ndhwc_bf16")[1:]]
    trimmed, untrimmed = split(lines), split(full)
    assert len(trimmed) == len(keeps) and len(untrimmed) == len(_slices(T, slice_frames))
    for s, (keep, ops, ref) in enumerate(zip(keeps, trimmed, untrimmed)):
        shuffles = [i for i, ln in enumerate(ops) if ln.startswith("svr2_upsample_shuffle_bf16")]
        assert len(shuffles) == 3
        cut = shuffles[1] + 1                                       # up_blocks.1 (the last temporal upsampler) and before
        assert ops[:cut] == ref[:cut], f"slice {s}: the work before the trim point changed"
        n_conv = 0
        for ln in ops[cut:]:
            tok = ln.split(" | ")[0].split()
            if tok[0] in ("svr2_conv3d_bf16", "svr2_conv3d_stats_bf16"):
                assert int(tok[14]) == keep, (s, ln)
                n_conv += 1
            elif tok[0] == "svr2_conv3d_shortcut_stats_bf16":
                assert int(tok[11]) == keep, (s, ln)
                n_conv += 1
            elif tok[0] in ("svr2_groupnorm_from_stats_bf16", "svr2_groupnorm_bf16", "svr2_upsample_shuffle_bf16"):
                assert int(tok[3 if "groupnorm" in tok[0] else 2]) == keep, (s, ln)
            elif tok[0] == "svr2_conv_tap_gather":
                assert int(tok[5]) == keep and int(ln.split(" | ")[1]) == F * 64 * h * w, (s, ln)   # (3, F, 8h, 8w) output
        assert n_conv == 1 + 3 * 2 + 1 + 3 * 2                      # up_blocks.1 conv, up_blocks.2, its upsampler, up_blocks.3


@pytest.mark.parametrize("T,h,w,slice_frames", [(2, 4, 6, 0), (3, 6, 10, 0), (5, 6, 10, 2), (6, 5, 7, 1), (1, 40, 24, 0)])
def test_all_frames_is_the_untrimmed_decode(cpu_vae, tracer, T, h, w, slice_frames):
    """svr2_vae_decode_frames(F = 4T-3) enqueues exactly what svr2_vae_decode does, channel strides included, in a workspace
    of the same exact size."""
    _, _, manifest = cpu_vae
    rc, got, err = run(tracer, manifest, "frames", T, h, w, slice_frames, 4 * T - 3)
    assert rc == 0, err[-2000:]
    rc, want, err = run(tracer, manifest, "dec", T, h, w, slice_frames)
    assert rc == 0, err[-2000:]
    assert got == want


@pytest.mark.parametrize("T,F", [(2, 0), (2, 6), (2, -1), (1, 2), (5, 18)])
def test_frames_out_of_range_are_refused(cpu_vae, tracer, T, F):
    eng, _, manifest = cpu_vae
    rc, _, err = run(tracer, manifest, "frames", T, 4, 6, 0, F)
    assert rc == 3 and err.count(f"frames = {F}") == 2, (rc, err)   # the workspace query and the decode both refuse
    with pytest.raises(ValueError, match="frames"):
        eng.decode(torch.zeros(1, 16, T, 4, 6, dtype=torch.bfloat16), frames=F)


def test_trimmed_workspace_of_the_flagship_shapes(cpu_vae, tracer):
    """Exact decode workspaces of the 4K shard (latent 2 x 270 x 480: 5 frames decoded, 4 wanted) and of the 1080p clip
    (latent 5 x 135 x 240: 17 decoded, 16 wanted), untrimmed and trimmed."""
    _, _, manifest = cpu_vae

    def need(T, h, w, F):
        rc, lines, err = run(tracer, manifest, "frames", T, h, w, 0, F, "plan")
        assert rc == 0, err[-2000:]
        return int(lines[-1].split()[2])

    for T, h, w, F in ((2, 270, 480, 4), (5, 135, 240, 16)):
        full, trimmed = need(T, h, w, 4 * T - 3), need(T, h, w, F)
        print(f"decode workspace latent {T}x{h}x{w}: {full} B for {4 * T - 3} frames, {trimmed} B for {F}")
        assert trimmed < full
