"""Clip-level runner over the H100 engines.

Mirrors ``VideoDiffusionInfer`` (reference ``src/core/infer.py``): ``vae_encode``
(:117-199), ``inference`` (:315-395, one Euler step, cfg = 1: x0 = x_t - v,
``samplers/euler.py:59-63``), ``vae_decode`` (:203-278), with the latents handed
between phases on the device (no host bounce).  ``upscale_clip`` strings them
together the way ``generation_phases.py`` does for one clip: 4n+1 temporal pad
(:109-124), clamp + pad-16 + normalise (``generation_utils.py:72-84``), encode,
condition = [latent | 1] (``infer.py:54-78``), DiT, decode, crop, optional colour
correction against the input clip (``generation_phases.py:1249-1319``), [0,1] image format.  With ``keep_alpha`` an
RGBA clip keeps its alpha: edge-guided upscaling against the decoded RGB before colour correction (:1142-1217,
``alpha.py``).  ``input_noise_scale`` / ``latent_noise_scale`` blend noise into the encoder's input and the DiT's
condition (:415-431, 679-704, ``noise.py``); ``upscale_video`` also takes the batch options ``uniform_batch_size`` and
``prepend_frames`` (:95-101, 360-378, 949-958, 1388-1397).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import alpha, color_fix, noise as gen_noise, preprocess
from .dit import B200NaDiT, dit_config
from .vae import B200VideoVAE

SCALING_FACTOR = 0.9152   # configs_3b/main.yaml:60
SHIFTING_FACTOR = 0.0


def pad_4n1(n: int) -> int:
    """frames -> next 4n+1 (generation_phases.py:109-124)."""
    return n if n % 4 == 1 else n + (4 - (n - 1) % 4)


def pad_video_temporal(frames: torch.Tensor, count: int = 0, prepend: bool = False) -> torch.Tensor:
    """Temporal padding along dim 0 with REVERSED frames, the reference's single source of truth for the 4n+1
    constraint and for prepended frames (``pad_video_temporal``, generation_utils.py:598-657): ``count == 0`` pads the
    end up to the next 4n+1; the mirror excludes the edge frame itself ([f0..f7] -> [f0..f7, f6]); when more frames
    are needed than the clip has, the far-edge frame is repeated."""
    t = frames.shape[0]
    if count == 0 and not prepend:
        if t % 4 == 1:
            return frames
        count = ((t - 1) // 4 + 1) * 4 + 1 - t
    if count <= 0:
        return frames
    if count >= t:
        last = frames[-1:]
        repeated = last.expand(count - t + 1, *frames.shape[1:])
        rev = frames[1:].flip(0) if t > 1 else last[:0]
        return torch.cat([repeated, rev, frames] if prepend else [frames, rev, repeated], 0)
    rev = frames[1:count + 1].flip(0) if prepend else frames[-count - 1:-1].flip(0)
    return torch.cat([rev, frames] if prepend else [frames, rev], 0)


class SeedVR2Engine:
    def __init__(self, dit_cfg: dict, dit_sd: Dict[str, torch.Tensor], vae_sd: Dict[str, torch.Tensor],
                 txt_embed: torch.Tensor, device="cuda"):
        self.device = torch.device(device)
        self.dit = B200NaDiT(dit_cfg, dit_sd, device=device)
        self.vae = B200VideoVAE(vae_sd, device=device)
        self.txt = txt_embed.to(self.device, torch.bfloat16).contiguous()

    # ---- VideoDiffusionInfer.vae_encode ---------------------------------
    @torch.no_grad()
    def vae_encode(self, clip: torch.Tensor, workspace=None) -> torch.Tensor:
        """clip (3,T,H,W) in [-1,1] -> latent (T',h,w,16) bf16, scaled."""
        z = self.vae.encode(clip[None].to(self.device, torch.bfloat16), workspace=workspace).latent   # (1,16,T',h,w)
        z = (z - SHIFTING_FACTOR) * SCALING_FACTOR
        return z[0].permute(1, 2, 3, 0).contiguous()

    # ---- VideoDiffusionInfer.inference ------------------------------------
    @torch.no_grad()
    def inference(self, noise: torch.Tensor, latent: torch.Tensor, workspace=None,
                  latent_noise: Optional[torch.Tensor] = None, latent_noise_scale: float = 0.0) -> torch.Tensor:
        """noise, latent (T',h,w,16) -> x0 (T',h,w,16).  DiT input = [noise | condition | 1] (task 'sr'); with
        ``latent_noise_scale`` > 0 the condition is moved toward noise * 0.1 + latent_noise * 0.05 along the lerp
        schedule at the shifted timestep scale * 1000 (generation_phases.py:680-697)."""
        T, h, w, c = latent.shape
        coef = None
        if gen_noise.check_scale("latent_noise_scale", latent_noise_scale) > 0:
            if latent_noise is None:
                raise ValueError("latent_noise_scale > 0 needs latent_noise (the second draw of the DiT noise generator)")
            coef = gen_noise.latent_noise_coefficients(latent_noise_scale, latent.shape, self.device)
        else:
            latent_noise = None
        vid = gen_noise.sr_condition(noise.to(self.device), latent.to(self.device), latent_noise, coef)
        v = self.dit(vid, self.txt, [[T, h, w]], [[self.txt.shape[0]]], workspace=workspace).vid_sample
        return noise.to(self.device, torch.bfloat16) - v.view(T, h, w, c)

    # ---- VideoDiffusionInfer.vae_decode -----------------------------------
    @torch.no_grad()
    def vae_decode(self, latent: torch.Tensor, workspace=None) -> torch.Tensor:
        """latent (T',h,w,16) -> sample (3,T,H,W) bf16 in ~[-1,1]."""
        z = latent.permute(3, 0, 1, 2)[None]
        z = z / SCALING_FACTOR + SHIFTING_FACTOR
        return self.vae.decode(z, workspace=workspace).sample[0]

    def clip_workspace(self, T: int, Hp: int, Wp: int) -> Optional[torch.Tensor]:
        """ONE workspace for the three phases of a clip of T (4n+1) frames at Hp x Wp (multiples of 16): the maximum of
        the exact needs of VAE encode, the DiT forward and VAE decode (svr2_vae_workspace_bytes / svr2_workspace_bytes),
        with the VAE passes temporally sliced until they fit the free HBM.  The phases run one after the other on one
        stream, so they can share the bytes; the block is the engine's resident workspace (lib.workspace: kept between clips,
        grown on demand; the capture pool inside a CUDA graph).  None when a phase runs on the Python sequencing (profiling)."""
        from . import lib
        if not (self.vae._use_native() and self.dit.native and lib.PROFILER is None):
            return None
        Tl, h, w = (T - 1) // 4 + 1, Hp // 8, Wp // 8
        budget = int(0.92 * self.vae._free_bytes()) - 2 * 3 * T * Hp * Wp * 2      # the decoded clip and its crop
        need = max(self.vae.plan_slices(True, T, Hp, Wp, budget)[1], self.vae.plan_slices(False, Tl, h, w, budget)[1],
                   self.dit.workspace_bytes(Tl, h, w, self.txt.shape[0]))
        return lib.workspace(need, self.device)

    def latent_shape(self, frames: torch.Tensor, resolution: Optional[int] = None, max_resolution: int = 0):
        """(T', h, w, 16) of the latent ``upscale_clip`` will produce for ``frames`` (T,h,w,3)."""
        res = resolution if resolution is not None else min(frames.shape[1], frames.shape[2])
        H, W = preprocess.resized_size(frames.shape[1], frames.shape[2], res, max_resolution)[0]
        Hp, Wp = (H + 15) // 16 * 16, (W + 15) // 16 * 16
        return ((pad_4n1(frames.shape[0]) - 1) // 4 + 1, Hp // 8, Wp // 8, 16)

    @staticmethod
    def input_noise_layout(frames: torch.Tensor, resolution: Optional[int] = None, max_resolution: int = 0) -> int:
        """Memory order (``noise.TCHW`` / ``CTHW`` / ``THWC``) of the reference's transformed clip for the clip
        ``frames`` (T,h,w,C), which its input-noise draw follows (``noise.input_noise_layout``)."""
        h, w = frames.shape[1], frames.shape[2]
        res = resolution if resolution is not None else min(h, w)
        (H, W), twice = preprocess.resized_size(h, w, res, max_resolution)
        return gen_noise.input_noise_layout(frames.shape[0], (h, w), (H, W), twice,
                                            ((H + 15) // 16 * 16, (W + 15) // 16 * 16))

    def graphed(self, frames: torch.Tensor, **kw) -> "GraphedClip":
        """Capture ``upscale_clip`` for this clip shape into a CUDA graph (see ``GraphedClip``)."""
        return GraphedClip(self, frames, **kw)

    # ---- one clip end to end ------------------------------------------------
    @torch.no_grad()
    def upscale_clip(self, frames: torch.Tensor, noise: Optional[torch.Tensor] = None, seed: int = 42,
                     color_correction: str = "none", resolution: Optional[int] = None,
                     max_resolution: int = 0, keep_alpha: bool = False, input_noise_scale: float = 0.0,
                     latent_noise_scale: float = 0.0, input_noise: Optional[torch.Tensor] = None,
                     latent_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """frames (T,h,w,3) in [0,1]; ``resolution`` = target shortest edge (None: keep the size, i.e. the frames
        are already at the target resolution).  Returns (T,H,W,3) bf16 in [0,1] on the device.
        ``color_correction``: "none", "lab" (the reference CLI default), "wavelet", "adain" or "wavelet_adaptive" —
        matched against the transformed input clip (generation_phases.py:1299-1317).
        ``keep_alpha``: frames (T,h,w,4) are RGBA; returns (T,H,W,4) with the alpha upscaled against the decoded RGB
        (generation_phases.py:1142-1217).  Without it a 4th channel is ignored.
        ``input_noise_scale``, ``latent_noise_scale``, ``input_noise``, ``latent_noise``: see ``clip_to_sample``."""
        rgba = keep_alpha and frames.shape[-1] == 4
        out = self.clip_to_sample(frames, noise=noise, seed=seed, resolution=resolution, max_resolution=max_resolution,
                                  keep_alpha=rgba, input_noise_scale=input_noise_scale,
                                  latent_noise_scale=latent_noise_scale, input_noise=input_noise,
                                  latent_noise=latent_noise)
        return self.finish_clip(*out, color_correction=color_correction)

    @staticmethod
    def finish_clip(sample: torch.Tensor, style: torch.Tensor, src: Optional[torch.Tensor] = None,
                    color_correction: str = "none") -> torch.Tensor:
        """Phase 4 for one clip (or slice): optional colour correction, [0,1] image format (T,H,W,3).  ``src``: the
        input RGBA frames (T,h,w,4) of these output frames; their alpha is upscaled against the decoded sample before
        the colour correction (which stays RGB-only) and becomes channel 3 of a (T,H,W,4) image."""
        if src is None:
            if color_correction != "none":
                sample = color_fix.apply_color_correction(sample, style, color_correction)
            return color_fix.sample_to_image(sample)                # t h w c in [0,1]
        sample = sample.to(torch.bfloat16).contiguous()
        T, _, H, W = sample.shape
        image = torch.empty(T, H, W, 4, device=sample.device, dtype=torch.bfloat16)
        alpha.upscale_into_image(src, sample, image)
        if color_correction != "none":
            sample = color_fix.apply_color_correction(sample, style, color_correction)
        return color_fix.sample_to_image_rgba(sample, image)

    @torch.no_grad()
    def clip_to_sample(self, frames: torch.Tensor, noise: Optional[torch.Tensor] = None, seed: int = 42,
                       resolution: Optional[int] = None, max_resolution: int = 0, keep_alpha: bool = False,
                       input_noise_scale: float = 0.0, latent_noise_scale: float = 0.0,
                       input_noise: Optional[torch.Tensor] = None, latent_noise: Optional[torch.Tensor] = None,
                       input_generator: Optional[torch.Generator] = None):
        """Phases 1-3 for one clip: frames (T,h,w,3) in [0,1] -> (sample, style), both (T,3,H,W) bf16 in [-1,1]:
        the decoded clip and the transformed input clip it is colour-matched against in phase 4.  ``keep_alpha``
        (frames (T,h,w,4)): (sample, style, src) with src the input frames on the device, unpadded, whose alpha
        phase 4 upscales.

        ``input_noise_scale`` > 0: the encoder reads the transformed clip blended with Gaussian noise (:415-431); the
        style stays the clean clip (:1249-1256).  The draw is ``input_noise`` (3, T4n+1, Hp, Wp) when given, else from
        ``input_generator``, else from a fresh generator seeded ``seed + 1_000_000`` (the reference's first batch).
        ``latent_noise_scale`` > 0: the DiT condition is augmented (:679-704) with ``latent_noise`` (T',h,w,16) when
        given, else with a second draw of the DiT noise generator right after ``noise``; an explicit ``noise`` needs
        an explicit ``latent_noise``.  Both scales must be finite and >= 0; at 0 nothing extra is drawn."""
        input_noise_scale = gen_noise.check_scale("input_noise_scale", input_noise_scale)
        latent_noise_scale = gen_noise.check_scale("latent_noise_scale", latent_noise_scale)
        if latent_noise_scale > 0 and noise is not None and latent_noise is None:
            raise ValueError("an explicit noise with latent_noise_scale > 0 needs an explicit latent_noise as well")
        T0 = frames.shape[0]
        x = src = frames.to(self.device)
        x = pad_video_temporal(x)                                   # mirrored tail frames, generation_phases.py:109-124
        # resize (identity when the frames already have the target size) + clamp + pad-16 + normalise + c t h w
        # in one kernel (prepare_video_transforms, generation_utils.py:72-84)
        res = resolution if resolution is not None else min(frames.shape[1], frames.shape[2])
        tf = preprocess.VideoTransform(res, max_resolution)
        H0, W0 = tf.true_size(frames.shape[1], frames.shape[2])
        x = tf.run(x, channels_last=True)                           # (3, T, Hp, Wp) bf16 in [-1,1]
        ws = self.clip_workspace(x.shape[1], x.shape[2], x.shape[3])
        kw = {} if ws is None else {"workspace": ws}
        x_enc = x
        if input_noise_scale > 0:
            if input_noise is None:
                g = input_generator if input_generator is not None else gen_noise.input_generator(seed, self.device)
                layout = self.input_noise_layout(frames, resolution, max_resolution)
                input_noise = gen_noise.draw_input_noise(x.shape, g, self.device, layout)
            x_enc = gen_noise.add_input_noise(x, input_noise, input_noise_scale)
        latent = self.vae_encode(x_enc, **kw)
        del x_enc
        if noise is None:
            g = torch.Generator(device=self.device).manual_seed(seed)
            noise = torch.randn(latent.shape, generator=g, device=self.device, dtype=torch.bfloat16)
            if latent_noise_scale > 0 and latent_noise is None:
                latent_noise = gen_noise.draw_latent_noise(latent.shape, g, self.device)
        aug = dict(latent_noise=latent_noise, latent_noise_scale=latent_noise_scale) if latent_noise_scale > 0 else {}
        x0 = self.inference(noise, latent, **kw, **aug)
        y = self.vae_decode(x0, **kw)                               # (3,T,H,W)
        del ws, kw
        sample = y[:, :T0, :H0, :W0].permute(1, 0, 2, 3)            # t c h w, the layout of phase 4
        style = x[:, :T0, :H0, :W0].permute(1, 0, 2, 3)            # the transformed input clip in [-1,1]
        return (sample, style, src) if keep_alpha else (sample, style)

    @torch.no_grad()
    def upscale_video(self, frames: torch.Tensor, batch_size: int = 5, temporal_overlap: int = 0, seed: int = 42,
                      color_correction: str = "none", resolution: Optional[int] = None,
                      max_resolution: int = 0, keep_alpha: bool = False, input_noise_scale: float = 0.0,
                      latent_noise_scale: float = 0.0, uniform_batch_size: bool = False,
                      prepend_frames: int = 0) -> torch.Tensor:
        """A whole video on one GPU the way the reference's four phases do it (generation_phases.py:271-289, 344-358,
        969-1000, 1236-1345): batches of ``batch_size`` frames stepping by ``batch_size - temporal_overlap``, every batch
        seeded identically, the overlap cross-faded into the previous batch's tail, colour correction per batch
        against its own input frames, [0,1] image format.  Returns (T,H,W,3) bf16.  ``keep_alpha`` with RGBA frames:
        (T,H,W,4); the alpha of every post-processed slice is upscaled from the input alpha of exactly that slice's
        frames against its decoded RGB after the cross-fade.

        ``input_noise_scale`` / ``latent_noise_scale``: as in ``clip_to_sample``; one input-noise generator seeded
        ``seed + 1_000_000`` feeds the batches in turn (:329-330), the DiT noise is reseeded per batch (:663).
        ``uniform_batch_size``: a batch shorter than ``batch_size`` is padded to it with mirrored frames before encoding
        and its output trimmed back to the real frames (:95-101, 360-378, 949-958).  ``prepend_frames`` = p: p mirrored
        frames are put in front of the video and the first p output frames dropped, unless p is not smaller than the
        output (generation_utils.py:196-198, generation_phases.py:1388-1397).  A multi-GPU caller prepends once,
        before sharding."""
        from . import shard
        rgba = keep_alpha and frames.shape[-1] == 4
        input_noise_scale = gen_noise.check_scale("input_noise_scale", input_noise_scale)
        latent_noise_scale = gen_noise.check_scale("latent_noise_scale", latent_noise_scale)
        if prepend_frames < 0:
            raise ValueError(f"prepend_frames must be >= 0, got {prepend_frames}")
        if prepend_frames > 0:
            frames = pad_video_temporal(frames, count=prepend_frames, prepend=True)
        gen = gen_noise.input_generator(seed, self.device) if input_noise_scale > 0 else None
        noise_kw = dict(input_noise_scale=input_noise_scale, latent_noise_scale=latent_noise_scale, input_generator=gen)

        def clip(a, b):
            batch = frames[a:b]
            if uniform_batch_size and b - a < batch_size:
                batch = pad_video_temporal(batch, count=batch_size - (b - a))
            out = self.clip_to_sample(batch, seed=seed, resolution=resolution, max_resolution=max_resolution,
                                      keep_alpha=rgba, **noise_kw)
            s, st = out[0][:b - a].contiguous(), out[1][:b - a].contiguous()
            return (s, (st, out[2][:b - a])) if rgba else (s, st)

        def post(sample, style):
            style, src = style if rgba else (style, None)
            return self.finish_clip(sample, style, src, color_correction=color_correction)

        out = run_batched(frames.shape[0], batch_size, temporal_overlap, clip, shard.blend_overlap, post)
        if 0 < prepend_frames < out.shape[0]:
            out = out[prepend_frames:]
        return out



def batch_ranges(total: int, batch_size: int, temporal_overlap: int = 0):
    """([start, end) per batch, effective overlap) of generation_phases.py:271-289, 344-358: step =
    batch_size - overlap (overlap reset to 0 when it is not smaller than the batch); a trailing batch that would hold
    nothing but overlap frames is dropped."""
    step = batch_size - temporal_overlap if temporal_overlap > 0 else batch_size
    if step <= 0:
        step, temporal_overlap = batch_size, 0
    out = []
    for idx in range(0, total, step):
        end = min(idx + batch_size, total)
        if idx > 0 and end - idx <= temporal_overlap:
            break
        out.append((idx, end))
    return out, temporal_overlap


def _frames(x, sl: slice):
    return tuple(t[sl] for t in x) if isinstance(x, tuple) else x[sl]


def run_batched(total: int, batch_size: int, temporal_overlap: int, clip_fn, blend_fn, post_fn) -> torch.Tensor:
    """The reference's batch loop with the engine plugged in as callables: ``clip_fn(start, end) -> (sample, style)``
    ((t,3,H,W) in [-1,1]; ``style`` may be a tuple of per-frame tensors, all sliced along frames alike),
    ``blend_fn(prev_tail, cur_head)``, ``post_fn(sample, style) -> (t,H,W,C)``.  Decoded batches are
    laid end to end; from the second batch on the first ``overlap`` frames are cross-faded into the tail already written
    and dropped (generation_phases.py:969-1000), and phase 4 then post-processes every batch's slice against its own
    input frames minus those overlap frames (:1249-1263)."""
    ranges, overlap = batch_ranges(total, batch_size, temporal_overlap)
    samples, styles = [], []
    written = 0
    for i, (a, b) in enumerate(ranges):
        sample, style = clip_fn(a, b)
        if i > 0 and overlap > 0 and overlap < sample.shape[0] and written >= overlap:
            # the tail lives in the previous batches' slices (it may span more than one when batches are short)
            tail = torch.cat(samples, 0)[-overlap:] if samples[-1].shape[0] < overlap else samples[-1][-overlap:]
            blended = blend_fn(tail.contiguous(), sample[:overlap].contiguous())
            k = overlap
            for j in range(len(samples) - 1, -1, -1):          # write the blended frames back, last slice first
                n = min(k, samples[j].shape[0])
                samples[j][samples[j].shape[0] - n:] = blended[k - n:k].to(samples[j].dtype)
                k -= n
                if k == 0:
                    break
            sample, style = sample[overlap:], _frames(style, slice(overlap, None))
        samples.append(sample)
        styles.append(_frames(style, slice(None, sample.shape[0])))
        written += sample.shape[0]
    return torch.cat([post_fn(s_, st_) for s_, st_ in zip(samples, styles)], 0)


class GraphedClip:
    """CUDA-graph replay of ``SeedVR2Engine.upscale_clip`` for one clip shape.

    The reference pays Python + launch overhead for every op of every clip (and so does the eager path here:
    ~3 000 kernel launches per 4K clip, ~1 700 for a single image, where the GPU work is shorter than the launch
    train).  All launches go through the C ABI on the current stream with pre-built tensor maps, nothing on the path
    synchronises with the host and the window / RoPE tables are cached per shape, so the whole clip — pre-processing,
    VAE encode, DiT, VAE decode, colour correction, formatting — captures into ONE graph whose intermediates live in
    the graph's private pool.  ``__call__`` copies the new frames into the static input and replays.  ``clip_kwargs``
    are those of ``upscale_clip``; ``keep_alpha=True`` captures the alpha path of RGBA frames as well."""

    def __init__(self, engine: "SeedVR2Engine", frames: torch.Tensor, noise: Optional[torch.Tensor] = None,
                 seed: int = 42, warmup: int = 2, latent_noise: Optional[torch.Tensor] = None, **clip_kwargs):
        from . import lib
        if lib.PROFILER is not None:
            raise lib.Svr2Error("per-call event profiling cannot run inside a graph capture")
        self.engine, self.kw = engine, clip_kwargs
        dev = engine.device
        self.static_in = frames.to(dev).clone()
        in_scale = gen_noise.check_scale("input_noise_scale", clip_kwargs.get("input_noise_scale", 0.0))
        lat_scale = gen_noise.check_scale("latent_noise_scale", clip_kwargs.get("latent_noise_scale", 0.0))
        if clip_kwargs.get("input_noise") is not None:
            raise ValueError("GraphedClip draws its input noise per replay; pass input_noise to __call__")
        if lat_scale > 0 and noise is not None and latent_noise is None:
            raise ValueError("an explicit noise with latent_noise_scale > 0 needs an explicit latent_noise as well")
        shape = engine.latent_shape(frames, clip_kwargs.get("resolution"), clip_kwargs.get("max_resolution", 0))
        if noise is None:
            g = torch.Generator(device=dev).manual_seed(seed)
            noise = torch.randn(shape, generator=g, device=dev, dtype=torch.bfloat16)
            if lat_scale > 0 and latent_noise is None:
                latent_noise = gen_noise.draw_latent_noise(shape, g, dev)
        self.noise = noise.to(dev, torch.bfloat16).clone()
        # static draws the graph reads: the DiT's augmentation noise (the same for every clip, as every batch of the
        # reference reseeds), and the input noise, refilled before each replay from one seed + 1_000_000 generator
        self.latent_noise = latent_noise.to(dev, torch.bfloat16).clone() if lat_scale > 0 else None
        self.input_noise, self._input_gen = None, None
        if in_scale > 0:
            self._input_gen = gen_noise.input_generator(seed, dev)
            self._input_layout = engine.input_noise_layout(frames, clip_kwargs.get("resolution"),
                                                           clip_kwargs.get("max_resolution", 0))
            clip_shape = (3, pad_4n1(frames.shape[0]), 8 * shape[1], 8 * shape[2])
            self.input_noise = gen_noise.input_noise_buffer(clip_shape, dev, self._input_layout)
        kw = dict(clip_kwargs, noise=self.noise, latent_noise=self.latent_noise, input_noise=self.input_noise)
        if warmup > 0:                          # shape-dependent tables and kernel attributes (skip with warmup=0
            side = torch.cuda.Stream(device=dev)    # when the engine has already run this clip shape eagerly)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                for _ in range(warmup):
                    engine.upscale_clip(self.static_in, **self._noise_kw(kw))
            torch.cuda.current_stream(dev).wait_stream(side)
        # the graph's private pool holds one whole clip of intermediates (~100 GB at 4K): hand the eager path's resident
        # workspace and cached blocks back first so both never have to coexist
        torch.cuda.synchronize(dev)
        lib.release_workspace(dev)
        torch.cuda.empty_cache()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.static_out = engine.upscale_clip(self.static_in, **self._noise_kw(kw))

    def _noise_kw(self, kw):
        """upscale_clip kwargs without the noise arguments a clip without those options never took."""
        return {k: v for k, v in kw.items() if v is not None or k not in ("latent_noise", "input_noise")}

    def refill_input_noise(self, input_noise: Optional[torch.Tensor] = None) -> None:
        """The static input-noise buffer for the next replay: ``input_noise`` (3, T, Hp, Wp) when given, else the next
        draw of the clip's ``seed + 1_000_000`` generator, in the memory order of ``noise.draw_input_noise``."""
        if input_noise is None:
            input_noise = gen_noise.draw_input_noise(self.input_noise.shape, self._input_gen, self.input_noise.device,
                                                     self._input_layout)
        elif tuple(input_noise.shape) != tuple(self.input_noise.shape):
            raise ValueError(f"input_noise must have shape {tuple(self.input_noise.shape)}, got {tuple(input_noise.shape)}")
        self.input_noise.copy_(input_noise, non_blocking=True)

    def __call__(self, frames: torch.Tensor, clone: bool = False, input_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Replay on new frames of the captured shape.  The returned tensor is the graph's STATIC output buffer: the
        next replay overwrites it — pass ``clone=True`` (or copy it out, as bench.py does into pinned host memory)
        when results of several clips are kept.  With ``input_noise_scale`` > 0 every replay first takes the next
        input-noise draw (successive replays see successive batches of the reference), or ``input_noise``."""
        if tuple(frames.shape) != tuple(self.static_in.shape):
            raise ValueError(f"GraphedClip captured frames of shape {tuple(self.static_in.shape)}, got {tuple(frames.shape)}")
        if self.input_noise is not None:
            self.refill_input_noise(input_noise)
        self.static_in.copy_(frames, non_blocking=True)
        self.graph.replay()
        return self.static_out.clone() if clone else self.static_out


def build_synthetic_engine(variant="3b", device="cuda", seed=1234, txt_len=58) -> SeedVR2Engine:
    """Random-init weights of the named architecture (no checkpoints exist offline)."""
    from . import weights
    cfg = dit_config(variant)
    dit_sd = weights.synth_dit_state_dict(cfg, seed=seed, dtype=torch.float16, device=device)
    vae_sd = weights.synth_vae_state_dict(seed=seed + 1, dtype=torch.float16, device=device)
    g = torch.Generator().manual_seed(seed + 2)
    txt = torch.randn(txt_len, cfg["txt_in_dim"], generator=g)
    eng = SeedVR2Engine(cfg, dit_sd, vae_sd, txt, device=device)
    del dit_sd, vae_sd
    return eng


def build_engine(dit_checkpoint: str, vae_checkpoint: str, txt_embed, device="cuda") -> SeedVR2Engine:
    """Engine from checkpoint files: DiT ``seedvr2_ema_{3b,7b}_{fp16,fp8_e4m3fn}.safetensors`` or a GGUF file
    (``seedvr2_ema_{3b,7b}-Q4_K_M.gguf`` …, dequantised on the device while the engine loads it), VAE
    ``ema_vae_fp16.safetensors`` (``model_registry.py:40-75``) and the positive text embedding (``pos_emb.pt``,
    ``generation_utils.py:load_text_embeddings``) given as a path or tensor."""
    from . import weights
    if dit_checkpoint.lower().endswith(".gguf"):
        dit_sd = weights.load_gguf(dit_checkpoint)
    else:
        dit_sd = weights.load_state_dict(dit_checkpoint)
    cfg = dit_config(weights.detect_dit_variant(dit_sd))
    vae_sd = weights.load_state_dict(vae_checkpoint)
    txt = torch.load(txt_embed, map_location="cpu", weights_only=True) if isinstance(txt_embed, str) else txt_embed
    if txt.ndim == 3:
        txt = txt[0]
    return SeedVR2Engine(cfg, dit_sd, vae_sd, txt, device=device)
