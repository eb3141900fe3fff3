"""CPU: the causal convs' folded head taps (include/svr2.h SVR2_EPI_FOLD_HEAD).

The weights folded at load (B200VideoVAE._fold_head) have the layout the kernel reads; exactly the kt = 3 convs the
sequence runs get them; the native runtime (csrc/vae_engine.cu, compiled with SVR2_HOST_TEST through
tests/native/vae_trace.cu) sets the fold on those convs in the first temporal slice of a clip and nowhere else, and its
workspace plan does not change.  test_native_vae_cpu.py compares its launch sequence with the Python module's op by op."""
import importlib

import pytest
import torch

import native_trace
from native_trace import run, write_manifest

pytestmark = native_trace.needs_nvcc
EPI_FOLD_HEAD = 2048


@pytest.fixture(scope="module")
def cpu_vae():
    with native_trace.recording_vae() as (eng, _):
        yield eng


@pytest.fixture(scope="module")
def tracer(tmp_path_factory):
    return native_trace.harness(tmp_path_factory, "vae_trace")


def test_folded_weights_layout(cpu_vae, pkg):
    """[2 Cout, K]: the regular rows (the conv's weight buffer itself), then [bf16(W0+W1) bf16(W2) | bf16(W0+W1+W2)] with
    the sums in fp32 over the checkpoint's (fp16) weights in that order; one per kt = 3 conv that runs through
    svr2_conv3d_bf16 / _stats (not encoder.conv_in, decoder.conv_out or the conv2 that runs fused with its block's
    shortcut)."""
    eng = cpu_vae
    sd = pkg.weights.synth_vae_state_dict(seed=1, dtype=torch.float16)
    want = {k for k in eng.W.keys() if k.endswith(".weight") and eng.meta.get(k + ".k", (0,))[0] == 3
            and k not in ("encoder.conv_in.weight", "decoder.conv_out.weight")
            and not (k.endswith("conv2.weight") and k.replace("conv2.weight", "conv_shortcut.weight") in eng.W)}
    heads = {k[: -len(":head")] for k in eng.W.keys() if k.endswith(":head")}
    assert heads == want and len(heads) > 40
    extra = 0
    for k in sorted(heads):
        w, wf = eng.W[k], eng.W[k + ":head"]
        Cout, K = w.shape
        n = K // 3
        assert wf.shape == (2 * Cout, K) and wf.is_contiguous()
        assert w.data_ptr() == wf.data_ptr() and torch.equal(wf[:Cout], w), k
        src = sd[k].float().permute(0, 2, 3, 4, 1)                           # [Cout, kt, kh, kw, Cin] fp16 -> fp32
        src = torch.nn.functional.pad(src, (0, w.shape[1] // 27 - src.shape[-1])).reshape(Cout, K)
        w0, w1, w2 = (src[:, i * n:(i + 1) * n] for i in range(3))
        f = wf[Cout:]
        assert torch.equal(f[:, :n], (w0 + w1).to(torch.bfloat16)), k
        assert torch.equal(f[:, n:2 * n], w[:, 2 * n:3 * n]), k
        assert torch.equal(f[:, 2 * n:], ((w0 + w1) + w2).to(torch.bfloat16)), k
        extra += f.numel() * 2
    print(f"folded head weights: {len(heads)} convs, {extra / 2 ** 20:.1f} MiB of bf16 beyond the regular weights")


def test_folded_weights_stay_views_after_a_device_move(pkg):
    """A device move copies every buffer on its own; afterwards each folded conv's weight is again the first Cout rows of
    its :head buffer (one copy of the weights resident, not two)."""
    lib = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.lib")
    vae = importlib.import_module("comfyui_seedvr2_videoupscaler_b200.vae")
    mp = pytest.MonkeyPatch()
    mp.setattr(lib, "device_check", lambda: (132, 9, 0))
    try:
        eng = vae.B200VideoVAE(pkg.weights.synth_vae_state_dict(seed=2, dtype=torch.float16), device="cpu")
    finally:
        mp.undo()
    before = {k: eng.W[k].clone() for k in eng.W.keys()}
    eng._apply(lambda t: t.clone())                                    # what .to(other device) does, buffer by buffer
    heads = [k for k in eng.W.keys() if k.endswith(":head")]
    assert heads
    for k in heads:
        w, head = eng.W[k[: -len(":head")]], eng.W[k]
        assert w.data_ptr() == head.data_ptr() and w.shape[0] * 2 == head.shape[0], k
    assert all(torch.equal(eng.W[k], t) for k, t in before.items())
    live = {b.untyped_storage().data_ptr() for b in eng.buffers()}
    assert len(live) == len(list(eng.buffers())) - len(heads)


def _trace(*args):
    rc, lines, err = run(*args)
    assert rc == 0, (rc, err[-2000:])
    return lines


def _convs_per_slice(lines):
    """[[(kt, epilogue flags)] per temporal slice] of the conv launches, from the trace's scalars."""
    slices = []
    for ln in lines:
        tok = ln.split(" | ")[0].split()
        if tok[0] == "svr2_ncdhw_to_ndhwc_bf16":
            slices.append([])
        elif tok[0] in ("svr2_conv3d_bf16", "svr2_conv3d_stats_bf16"):
            slices[-1].append((int(tok[8]), int(tok[15])))
    return slices


@pytest.mark.parametrize("direction,T,H,W,slice_frames", [
    ("dec", 3, 6, 10, 0), ("dec", 5, 6, 10, 2), ("dec", 6, 5, 7, 1), ("dec", 1, 40, 24, 0),
    ("enc", 9, 48, 80, 0), ("enc", 17, 48, 80, 8), ("enc", 13, 32, 48, 4), ("enc", 1, 128, 160, 0),
])
def test_fold_runs_in_the_first_slice_only(cpu_vae, tracer, tmp_path, direction, T, H, W, slice_frames):
    with_heads = _trace(tracer, write_manifest(cpu_vae, str(tmp_path / "w.txt")), direction, T, H, W, slice_frames)
    without = _trace(tracer, write_manifest(cpu_vae, str(tmp_path / "w0.txt"), heads=False), direction, T, H, W, slice_frames)
    slices = _convs_per_slice(with_heads[:-1])
    assert len(slices) == (1 if slice_frames == 0 else len(_convs_per_slice(without[:-1])))
    for s, convs in enumerate(slices):
        for i, (kt, flags) in enumerate(convs):
            assert bool(flags & EPI_FOLD_HEAD) == (s == 0 and kt == 3), (s, i, kt, flags)
    assert any(kt == 3 for kt, _ in slices[0])
    # loaded without the folded weights: the same launches, every conv with all its taps
    for s, convs in enumerate(_convs_per_slice(without[:-1])):
        assert all(not (flags & EPI_FOLD_HEAD) for _, flags in convs)
        assert [(kt, flags & ~EPI_FOLD_HEAD) for kt, flags in convs] == [(kt, flags & ~EPI_FOLD_HEAD) for kt, flags in slices[s]]
    assert len(with_heads) == len(without)
    # the workspace plan and the launch count do not change
    assert with_heads[-1].split()[2] == without[-1].split()[2] and with_heads[-1].split()[6] == without[-1].split()[6]


def test_workspace_of_the_flagship_shapes_unchanged(cpu_vae, tracer, tmp_path):
    """The exact decode workspace of the 4K shard (latent 2 x 270 x 480, 4 of 5 frames) and of the 1080p clip (latent
    5 x 135 x 240, 16 of 17 frames), and of two encodes, with and without the folded weights: the fold allocates nothing."""
    m1, m0 = write_manifest(cpu_vae, str(tmp_path / "w.txt")), write_manifest(cpu_vae, str(tmp_path / "w0.txt"), heads=False)
    for T, h, w, F in ((2, 270, 480, 4), (5, 135, 240, 16)):
        got = [_trace(tracer, m, "frames", T, h, w, 0, F, "plan")[-1] for m in (m1, m0)]
        assert got[0] == got[1], (T, h, w, got)
    for T, H, W in ((5, 96, 160), (17, 64, 96)):
        got = [_trace(tracer, m, "enc", T, H, W, 0)[-1].split()[2] for m in (m1, m0)]
        assert got[0] == got[1], (T, H, W, got)
