"""CPU: the native VAE runtime's kernel sequence (csrc/vae_engine.cu, what svr2_vae_encode / svr2_vae_decode enqueue) against
the Python module's (vae.py, the sequence the -m gpu tests pin to the oracle), op by op with every scalar argument, for
un-sliced and temporally sliced clips; and its workspace plan (the dry run must equal what the real run touches, and a
smaller workspace must be refused).  vae_engine.cu is compiled with SVR2_HOST_TEST by nvcc's host compiler
(tests/native/vae_trace.cu); the GPU test test_vae_native_runtime_equals_python_sequencing checks the results bit for bit."""
import pytest
import torch

import native_trace
from native_trace import assert_same_ops, launches, run, summary, write_manifest

pytestmark = native_trace.needs_nvcc


@pytest.fixture(scope="module")
def tracer(tmp_path_factory):
    return native_trace.harness(tmp_path_factory, "vae_trace")


@pytest.fixture(scope="module")
def cpu_vae():
    with native_trace.recording_vae() as vae_log:
        yield vae_log


@pytest.mark.parametrize("direction,T,H,W,split", [
    ("dec", 3, 6, 10, None), ("dec", 5, 6, 10, 8), ("dec", 6, 5, 7, 4), ("dec", 1, 40, 24, None),
    ("dec", 1, 270, 480, None),         # the 4K latent: mid-block attention at n = 129 600 in 16 query chunks
    ("enc", 9, 48, 80, None), ("enc", 17, 48, 80, 8), ("enc", 13, 32, 48, 4), ("enc", 6, 32, 48, 4), ("enc", 1, 128, 160, None),
])
def test_native_vae_sequence_matches_python(cpu_vae, tracer, tmp_path, direction, T, H, W, split):
    eng, log = cpu_vae
    manifest = write_manifest(eng, str(tmp_path / "weights.txt"))
    del log[:]
    eng.set_causal_slicing(split_size=split)
    try:
        if direction == "dec":
            out = eng.decode(torch.zeros(1, 16, T, H, W, dtype=torch.bfloat16)).sample
            assert out.shape == (1, 3, 4 * T - 3, 8 * H, 8 * W)
            slice_frames = 0 if split is None else max(1, split // 4)
        else:
            out = eng.encode(torch.zeros(1, 3, T, H, W, dtype=torch.bfloat16)).latent
            assert out.shape == (1, 16, (T - 1) // 4 + 1, H // 8, W // 8)
            slice_frames = 0 if split is None else max(4, split // 4 * 4)
    finally:
        eng.set_causal_slicing(split_size=None)
    want = list(log)
    rc, lines, err = run(tracer, manifest, direction, T, H, W, slice_frames)
    assert rc == 0, (rc, err[-2000:])
    need, touched, n_launches = summary(lines.pop())
    assert_same_ops(lines, want)                                   # without the channel-stride suffix of the strided converters
    assert 0 < touched < need and need % 256 == 0
    assert n_launches == launches(want)
    sliced = any(ln.split(" | ")[1] != str((T if direction == "dec" else T) * H * W) for ln in lines if ln.startswith("svr2_ncdhw"))
    assert not sliced                                              # the input channel stride is always the whole clip's
    n_in = sum(ln.startswith("svr2_ncdhw_to_ndhwc") for ln in lines)
    if slice_frames and T - 1 > slice_frames and (direction == "dec" or (T - 1) % 4 == 0):
        assert n_in == 1 + -(-(T - 1 - slice_frames) // slice_frames)
    else:
        assert n_in == 1


def test_native_vae_plan_shrinks_with_slices(cpu_vae, tracer, tmp_path):
    """The exact workspace of a sliced pass is smaller than the un-sliced one and grows with the slice length."""
    eng, _ = cpu_vae
    manifest = write_manifest(eng, str(tmp_path / "weights.txt"))

    def need(direction, T, H, W, s):
        rc, lines, err = run(tracer, manifest, direction, T, H, W, s)
        assert rc == 0, err[-2000:]
        return int(lines[-1].split()[2])

    full, s2, s1 = need("dec", 9, 34, 60, 0), need("dec", 9, 34, 60, 2), need("dec", 9, 34, 60, 1)
    assert s1 < s2 < full
    full, s8, s4 = need("enc", 33, 272, 480, 0), need("enc", 33, 272, 480, 8), need("enc", 33, 272, 480, 4)
    assert s4 < s8 < full


def test_native_vae_arena_fuzz(tracer):
    """The activation arena: 200 random alloc / release / top-allocation scripts replayed on the unbounded (dry-run) arena
    and on one capped at the dry run's size — identical placements, no overlap of live blocks, nothing beyond the cap."""
    rc, lines, err = run(tracer, "fuzz")
    assert rc == 0 and "arena fuzz ok" in lines, (rc, err[-500:])
