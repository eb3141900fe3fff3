"""TEST INFRASTRUCTURE ONLY — generates tests/golden/noise_*.npz from the REFERENCE.

Run where the reference checkout is available (``ref_import.REFERENCE_ROOT``):

    python -m oracle.make_noise_golden

The batch preparation (``_prepare_video_batch``, ``_apply_4n1_padding``, the video transform), ``set_seed``,
``timestep_transform``, ``LinearInterpolationSchedule`` and ``get_condition`` are the reference's own code, on the
CPU.  The inline noise lines of ``encode_all_batches`` (generation_phases.py:416-429) and ``upscale_all_batches``
(:663, 680-697) are restated here with their citations, so the draw order across batches is pinned by this
restatement, not by running the phase functions themselves.  Every file stores the inputs, the raw draws, the latent
strides the reference really sees and the outputs; the restatement in ``oracle/noise_oracle.py`` is checked against
them bit for bit before they are written.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import noise_oracle as no  # noqa: E402
from oracle import ref_import  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SEED = 42
INPUT_SCALES = (0.05, 0.3, 1.0)
LATENT_SCALES = (0.1, 0.5, 1.0)

# name: (frames, h, w, resolution, batch_size, uniform_batch_size)
INPUT_CASES = {
    "noise_input_video": (7, 20, 28, 26, 5, True),    # the node's batch_size 5: a full batch and a tail uniform-padded
                                                      # from 2 to 5 frames, both 4n+1 as they come: (t h w c) memory
    "noise_input_tail": (7, 20, 28, 26, 5, False),    # the 2-frame tail 4n+1-padded to 5, then resized: (t c h w)
    "noise_input_same_size": (6, 32, 48, 32, 4, False),  # 4n+1-padded, neither resized nor padded: (c t h w)
    "noise_input_img": (1, 18, 22, 24, 1, False),     # an image: (t h w c)
}
# name: latent (T', h, w, c)
LATENT_CASES = {
    "noise_latent_video": (2, 6, 8, 16),
    "noise_latent_img": (1, 5, 7, 16),            # T' = 1
    "noise_latent_h1": (2, 1, 9, 16),             # h = 1: timestep_transform sees one frame, so the image shift
}


def _import_reference():
    ref_import.install_stubs()
    if "omegaconf" not in sys.modules:                    # imported by the config modules only, never called here
        class _OmegaConf:
            @staticmethod
            def register_new_resolver(*_a, **_k):
                pass
        m = types.ModuleType("omegaconf")
        m.DictConfig, m.ListConfig, m.OmegaConf = dict, list, _OmegaConf
        sys.modules["omegaconf"] = m
    from src.common.diffusion.schedules.lerp import LinearInterpolationSchedule
    from src.common.seed import set_seed
    from src.core import generation_phases as gp
    from src.core.generation_utils import prepare_video_transforms
    from src.core.infer import VideoDiffusionInfer
    from src.optimization.performance import optimized_channels_to_last
    return types.SimpleNamespace(lerp=LinearInterpolationSchedule, set_seed=set_seed, gp=gp,
                                 transforms=prepare_video_transforms, infer=VideoDiffusionInfer,
                                 channels_to_last=optimized_channels_to_last)


def input_case(ref, name, T, h, w, res, batch_size, uniform):
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    images = torch.rand(T, h, w, 3, generator=g)
    transform = ref.transforms(resolution=res)
    out = {"images": images.numpy(), "resolution": np.array(res)}
    clips, draws, counts, frames = [], [], [], []
    ref.set_seed(SEED + 1000000)                                               # :329-330
    for bi, start in enumerate(range(0, T, batch_size)):                       # :345-356, no overlap
        end = min(start + batch_size, T)
        cur = end - start
        pad = batch_size - cur if uniform and cur < batch_size else 0         # :361
        video = ref.gp._prepare_video_batch(images=images, start_idx=start, end_idx=end, uniform_padding=pad)
        video = video.to(torch.bfloat16)                                       # manage_tensor, compute dtype
        frames.append(video.size(0))
        if video.size(0) % 4 != 1:
            video = ref.gp._apply_4n1_padding(video)                           # :395-402
        tv = transform(video)                                                  # :411
        noise = torch.randn_like(tv)                                           # :419
        (H, W), twice = _resized_size(h, w, res)
        layout = no.clip_layout(frames[-1], (h, w), (H, W), twice, tv.shape[2:])
        print(f"{name}: batch {bi} of {frames[-1]} frames: transformed_video {tuple(tv.shape)} strides {tv.stride()}, "
              f"memory order {layout}")
        assert noise.stride() == tv.stride() == no.laid_out(tv.shape, layout, "cpu").stride(), "clip_layout"
        clips.append((tuple(tv.shape), layout))
        draws.append(noise)
        counts.append(tv.shape[1])
        out[f"tv{bi}"] = tv.float().numpy()
        out[f"draw{bi}"] = noise.float().numpy()
        out[f"draw{bi}_strides"] = np.array(noise.stride())
        for s in INPUT_SCALES:
            n = noise * 0.05                                                   # :422
            blend_factor = s * 0.5                                             # :425
            res_ = tv * (1 - blend_factor) + (tv + n) * blend_factor           # :428
            assert torch.equal(res_, no.input_noise(tv, noise, s))
            out[f"out{bi}_{s}"] = res_.float().numpy()
    ins, _, _ = no.draws(SEED, clips, (1, 1, 1, 16), "cpu")
    for d, ref_d in zip(ins, draws):
        assert torch.equal(d, ref_d) and d.stride() == ref_d.stride(), "draw order / memory order of the restatement"
    out["batch_frames"] = np.array(frames)
    out["encode_frames"] = np.array(counts)
    out["scales"] = np.array(INPUT_SCALES)
    return out


def _resized_size(h, w, res):
    """SideResize's output size without a max_resolution (torchvision's _compute_resized_output_size)."""
    short, long = min(h, w), max(h, w)
    new_long = int(res * long / short)
    return ((new_long, res) if w <= h else (res, new_long)), False


class _Runner:
    """What ``timestep_transform`` reads of VideoDiffusionInfer: the transform flag and the VAE factors (the
    configs set transform: True and leave the factors at their defaults, configs_3b/main.yaml:66-80)."""

    def __init__(self, ref):
        self.config = types.SimpleNamespace(diffusion=types.SimpleNamespace(timesteps={"transform": True}),
                                            vae=types.SimpleNamespace(model={}))
        self.schedule = ref.lerp(T=1000.0)


def latent_case(ref, name, shape):
    Tl, h, w, c = shape
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    z = torch.randn(1, c, Tl, h, w, generator=g).to(torch.bfloat16)           # the encoder's (b c t h w) output
    latent = ref.channels_to_last(z)                                           # infer.py:187
    latent = ((latent - 0.0) * 0.9152).squeeze(0)                             # infer.py:188, 196
    latent = latent.to(torch.bfloat16)                                         # manage_tensor (keeps strides)
    print(f"{name}: latent {tuple(latent.shape)} strides {latent.stride()}")
    runner = _Runner(ref)
    out = {"latent": latent.float().numpy(), "latent_strides": np.array(latent.stride())}
    ref.set_seed(SEED)                                                         # :663
    base_noise = torch.randn_like(latent, dtype=torch.bfloat16)                # :680
    r = torch.randn_like(base_noise)                                           # :683
    aug = base_noise * 0.1 + r * 0.05
    out.update(noise=base_noise.float().numpy(), r=r.float().numpy(), noise_strides=np.array(base_noise.stride()),
               r_strides=np.array(r.stride()))
    _, base_o, r_o = no.draws(SEED, [], shape, "cpu")
    assert torch.equal(base_o, base_noise) and torch.equal(r_o, r) and r_o.stride() == r.stride()
    for s in (0.0,) + LATENT_SCALES:
        x = latent
        if s != 0.0:                                                           # _add_noise, :686-693
            t = torch.tensor([1000.0], dtype=torch.bfloat16) * s
            shp = torch.tensor(latent.shape[1:])[None]
            t = ref.infer.timestep_transform(runner, t, shp)
            x = runner.schedule.forward(latent, aug, t)
            a_o, b_o = no.coefficients(s, shape, "cpu")
            assert torch.equal(runner.schedule.A(t), a_o) and torch.equal(runner.schedule.B(t), b_o)
            out[f"A_{s}"], out[f"B_{s}"], out[f"t_{s}"] = a_o.numpy(), b_o.numpy(), t.numpy()
        cond = ref.infer.get_condition(None, base_noise, task="sr", latent_blur=x)     # :696-700
        vid = torch.cat([base_noise, cond], -1).reshape(Tl * h * w, 2 * c + 1)         # the DiT's input rows
        assert torch.equal(vid, no.sr_condition(base_noise, latent, r, s))
        out[f"vid_{s}"] = vid.float().numpy()
    out["scales"] = np.array(LATENT_SCALES)
    return out


def main():
    ref = _import_reference()
    os.makedirs(GOLD, exist_ok=True)
    for name, (T, h, w, res, bs, uni) in INPUT_CASES.items():
        np.savez_compressed(os.path.join(GOLD, name + ".npz"), **input_case(ref, name, T, h, w, res, bs, uni))
    for name, shape in LATENT_CASES.items():
        np.savez_compressed(os.path.join(GOLD, name + ".npz"), **latent_case(ref, name, shape))
    print("wrote", ", ".join(list(INPUT_CASES) + list(LATENT_CASES)))


if __name__ == "__main__":
    main()
