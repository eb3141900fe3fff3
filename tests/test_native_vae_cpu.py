"""CPU: the native VAE runtime's kernel sequence (csrc/vae_engine.cu, what svr2_vae_encode / svr2_vae_decode enqueue) against
the Python module's (vae.py, the sequence the -m gpu tests pin to the oracle), op by op with every scalar argument, for
un-sliced and temporally sliced clips; and its workspace plan (the dry run must equal what the real run touches, and a
smaller workspace must be refused).  vae_engine.cu is compiled with SVR2_HOST_TEST by nvcc's host compiler
(tests/native/vae_trace.cu); the GPU test test_vae_native_runtime_equals_python_sequencing checks the results bit for bit."""
import ctypes
import importlib
import os
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def tracer(tmp_path_factory, pkg):
    lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
    lib.load()                                                     # builds nothing; fails loudly if libsvr2.so is missing
    exe = str(tmp_path_factory.mktemp("vae") / "vae_trace")
    csrc = os.path.join(ROOT, "comfyui-seedvr2_videoupscaler_b200", "csrc")
    # kernel entry points are the harness's stubs; the pure helpers (svr2_conv_stat_slots, svr2_rowstat_slots,
    # svr2_groupnorm_scratch_bytes) come from the real library
    r = subprocess.run([NVCC, "-std=c++17", "-O1", "-I", csrc, "-o", exe, os.path.join(ROOT, "tests", "native", "vae_trace.cu"),
                        "-L", csrc, "-lsvr2", "-Xlinker", "-rpath", "-Xlinker", csrc], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


@pytest.fixture(scope="module")
def cpu_vae(pkg):
    """The Python VAE module on the CPU with the kernel layer replaced by a recorder."""
    lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    mp = pytest.MonkeyPatch()
    mp.setattr(lib, "device_check", lambda: (132, 9, 0))
    eng = vae.B200VideoVAE(pkg.weights.synth_vae_state_dict(seed=1, dtype=torch.float16), device="cpu")
    eng.native = False
    log = []

    def fmt(a):
        if a is None:
            return "p0"
        if isinstance(a, ctypes.c_void_p):
            return "p1" if a.value else "p0"
        if isinstance(a, bool):
            return str(int(a))
        if isinstance(a, int):
            return str(a)
        if isinstance(a, float):
            return "%.5g" % a
        return "p1"                                                # ctypes.byref(...)

    def record(name, *args, flops=0.0, nbytes=0.0, tag=""):
        log.append(" ".join([name] + [fmt(a) for a in args]))

    mp.setattr(lib, "call", record)
    mp.setattr(lib, "stream", lambda: None)
    mp.setattr(lib, "_bf16c", lambda t, name: t)
    mp.setattr(type(eng), "_require_cuda", lambda self, what: None)
    mp.setattr(type(eng), "_frames_that_fit", lambda self, H, W, state_bytes_per_pixel=0: 10 ** 6)
    mp.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    mp.setattr(torch.cuda, "memory_reserved", lambda d=None: 0)
    mp.setattr(torch.cuda, "memory_allocated", lambda d=None: 0)
    mp.setattr(torch.cuda, "empty_cache", lambda: None)
    mp.setattr(torch.cuda, "get_device_properties", lambda d=None: type("P", (), {"total_memory": 1 << 40})())
    yield eng, log
    mp.undo()


def _manifest(eng, path):
    with open(path, "w") as f:
        for k, t in eng._native_tensors().items():
            f.write(" ".join([k, str(max(t.ndim, 1))] + [str(n) for n in (t.shape if t.ndim else (1,))]) + "\n")


@pytest.mark.parametrize("direction,T,H,W,split", [
    ("dec", 3, 6, 10, None), ("dec", 5, 6, 10, 8), ("dec", 6, 5, 7, 4), ("dec", 1, 40, 24, None),
    ("enc", 9, 48, 80, None), ("enc", 17, 48, 80, 8), ("enc", 13, 32, 48, 4), ("enc", 6, 32, 48, 4), ("enc", 1, 128, 160, None),
])
def test_native_vae_sequence_matches_python(cpu_vae, tracer, tmp_path, direction, T, H, W, split):
    eng, log = cpu_vae
    manifest = str(tmp_path / "weights.txt")
    _manifest(eng, manifest)
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
    r = subprocess.run([tracer, manifest, direction, str(T), str(H), str(W), str(slice_frames)], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    lines = r.stdout.strip().split("\n")
    summary = lines.pop().split()
    got = [ln.split(" | ")[0] for ln in lines]                     # drop the channel-stride suffix of the strided converters
    assert len(got) == len(want), (len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"op {i}: native `{g}` vs python `{w}`"
    need, touched, launches = int(summary[2]), int(summary[4]), int(summary[6])
    assert 0 < touched < need and need % 256 == 0
    lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
    assert launches == sum(lib.KERNELS_PER_CALL.get(w.split()[0], 1) for w in want)
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
    manifest = str(tmp_path / "weights.txt")
    _manifest(eng, manifest)

    def need(direction, T, H, W, s):
        r = subprocess.run([tracer, manifest, direction, str(T), str(H), str(W), str(s)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        return int(r.stdout.strip().split("\n")[-1].split()[2])

    full, s2, s1 = need("dec", 9, 34, 60, 0), need("dec", 9, 34, 60, 2), need("dec", 9, 34, 60, 1)
    assert s1 < s2 < full
    full, s8, s4 = need("enc", 33, 272, 480, 0), need("enc", 33, 272, 480, 8), need("enc", 33, 272, 480, 4)
    assert s4 < s8 < full


def test_native_vae_arena_fuzz(tracer):
    """The activation arena: 200 random alloc / release / top-allocation scripts replayed on the unbounded (dry-run) arena
    and on one capped at the dry run's size — identical placements, no overlap of live blocks, nothing beyond the cap."""
    r = subprocess.run([tracer, "fuzz"], capture_output=True, text=True)
    assert r.returncode == 0 and "arena fuzz ok" in r.stdout, (r.returncode, r.stderr[-500:])
