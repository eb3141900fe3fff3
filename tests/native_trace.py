"""Shared by the CPU tests that trace the native runtimes: the host-compiled harnesses under tests/native, and the Python
VAE module (vae.py) on the CPU recording its kernel launches in the same text format as tests/native/vae_trace.cu's stubs."""
import contextlib
import ctypes
import importlib
import os
import shutil
import subprocess

import pytest
import torch

from svr2_import import load_package

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "comfyui-seedvr2_videoupscaler_b200", "csrc")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
needs_nvcc = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
_harnesses = {}


def _lib():
    load_package()
    return importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")


def harness(tmp_path_factory, name, link_svr2=True):
    """tests/native/<name>.cu compiled by nvcc's host compiler, once per pytest process.  Linked with libsvr2, the kernel
    entry points are the harness's stubs and the pure helpers (svr2_conv_stat_slots, svr2_rowstat_slots,
    svr2_groupnorm_scratch_bytes) come from the real library; otherwise nothing is linked."""
    if name not in _harnesses:
        exe = str(tmp_path_factory.mktemp(name) / name)
        cmd = [NVCC, "-std=c++17", "-O1", "-I", CSRC, "-o", exe, os.path.join(ROOT, "tests", "native", name + ".cu")]
        if link_svr2:
            _lib().load()                                          # builds nothing; fails loudly if libsvr2.so is missing
            cmd += ["-L", CSRC, "-lsvr2", "-Xlinker", "-rpath", "-Xlinker", CSRC]
        else:
            cmd += ["-Xlinker", "--unresolved-symbols=ignore-all"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        _harnesses[name] = exe
    return _harnesses[name]


def _fmt(a):
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
    return "p1"                                                    # ctypes.byref(...)


@contextlib.contextmanager
def recording_vae():
    """The Python VAE module on the CPU (`.native = False`) with the kernel layer replaced by a recorder: yields (eng, log),
    log getting one line per kernel call as the harness prints it.  Every patch is undone on exit."""
    lib = _lib()
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(lib, "device_check", lambda: (132, 9, 0))
        eng = vae.B200VideoVAE(load_package().weights.synth_vae_state_dict(seed=1, dtype=torch.float16), device="cpu")
        eng.native = False
        log = []
        mp.setattr(lib, "call", lambda name, *args, flops=0.0, nbytes=0.0, tag="": log.append(" ".join([name] + [_fmt(a) for a in args])))
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


def write_manifest(eng, path, heads=True):
    """The weights manifest the harness reads (name rank d0 d1 ... per line); heads=False leaves out the folded head
    weights (`:head`), as a module loaded without them."""
    with open(path, "w") as f:
        for k, t in eng._native_tensors().items():
            if heads or not k.endswith(":head"):
                f.write(" ".join([k, str(max(t.ndim, 1))] + [str(n) for n in (t.shape if t.ndim else (1,))]) + "\n")
    return path


def run(exe, *args):
    """(exit code, stdout lines, stderr) of one harness run."""
    r = subprocess.run([exe, *map(str, args)], capture_output=True, text=True)
    return r.returncode, r.stdout.strip().split("\n"), r.stderr


def summary(line):
    """(workspace bytes, touched max offset, launches) of a pass's last line."""
    tok = line.split()
    assert tok[:2] == ["#", "workspace"] and tok[3::2] == ["touched_max_offset", "launches"], line
    return int(tok[2]), int(tok[4]), int(tok[6])


def launches(want):
    """Kernels the Python module's recorded calls launch."""
    return sum(_lib().KERNELS_PER_CALL.get(w.split()[0], 1) for w in want)


def assert_same_ops(got, want):
    """The harness's trace lines, each without its ' | ' suffix, are the recorded calls op by op."""
    got = [ln.split(" | ")[0] for ln in got]
    assert len(got) == len(want), (len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"op {i}: native `{g}` vs python `{w}`"
