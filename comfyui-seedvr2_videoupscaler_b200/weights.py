"""Deterministic synthetic checkpoints with the key layout of the real files.

No network and no real weights exist in the build/bench environment
(BASELINE.json: "random-init weights of that architecture"), so tests, the
benchmark and the golden-vector generator all draw weights from here.  Key
names/shapes are those of ``seedvr2_ema_{3b,7b}_fp16.safetensors`` and
``ema_vae_fp16.safetensors`` as produced by the reference module constructors
(SURVEY.md §8(a) "Synthetic-checkpoint key layout"; reference
``src/models/dit_3b/nadit.py:49-186``, ``src/models/video_vae_v3/modules/attn_video_vae.py:671-1035``).

Initialisation is *not* the reference's default init: gates / projections are
scaled so every block contributes O(1) to the residual stream — otherwise a
parity test would only exercise the skip path.
"""
from __future__ import annotations

import math
from typing import Dict

import torch


def _gen(seed: int, device="cpu") -> torch.Generator:
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    return g


class _Maker:
    def __init__(self, seed: int, dtype: torch.dtype, device: str):
        self.g = _gen(seed, device)
        self.dtype = dtype
        self.device = device
        self.sd: Dict[str, torch.Tensor] = {}

    def randn(self, *shape, std=1.0, mean=0.0):
        x = torch.randn(*shape, generator=self.g, device=self.device, dtype=torch.float32)
        return (x * std + mean).to(self.dtype)

    def linear(self, name: str, out_f: int, in_f: int, bias: bool = True, gain: float = 1.0):
        self.sd[name + ".weight"] = self.randn(out_f, in_f, std=gain / math.sqrt(in_f))
        if bias:
            self.sd[name + ".bias"] = self.randn(out_f, std=0.1)

    def conv(self, name: str, out_c: int, in_c: int, k=(3, 3, 3), gain: float = 1.0):
        fan_in = in_c * k[0] * k[1] * k[2]
        self.sd[name + ".weight"] = self.randn(out_c, in_c, *k, std=gain / math.sqrt(fan_in))
        self.sd[name + ".bias"] = self.randn(out_c, std=0.05)

    def norm(self, name: str, c: int):
        self.sd[name + ".weight"] = self.randn(c, std=0.1, mean=1.0)
        self.sd[name + ".bias"] = self.randn(c, std=0.1)


def swiglu_hidden(dim: int, expand_ratio: int = 4, multiple_of: int = 256) -> int:
    h = int(2 * dim * expand_ratio / 3)
    return multiple_of * ((h + multiple_of - 1) // multiple_of)


def synth_dit_state_dict(cfg: dict, seed: int = 1234, dtype=torch.float16, device="cpu") -> Dict[str, torch.Tensor]:
    """cfg: see ``dit.dit_config``; keys as the reference NaDiT.state_dict()."""
    m = _Maker(seed, dtype, device)
    d, heads, hd = cfg["dim"], cfg["heads"], cfg["head_dim"]
    inner = heads * hd
    is7 = cfg["variant"] == "7b"
    m.linear("vid_in.proj", d, cfg["in_ch"] * 4)
    m.linear("txt_in", d, cfg["txt_in_dim"])
    m.linear("emb_in.proj_in", d, 256)
    m.linear("emb_in.proj_hid", d, d)
    m.linear("emb_in.proj_out", 6 * d, d, gain=0.5)
    nfreq = (hd // 2 // 3) // 2 if is7 else (hd // 3) // 2
    if is7:
        freqs = torch.linspace(1.0, 256 / 2, nfreq) * math.pi          # freqs_for="pixel", max_freq=256
    else:
        rd = hd // 3
        freqs = 1.0 / (10000 ** (torch.arange(0, rd, 2)[: rd // 2].float() / rd))  # freqs_for="lang"
    for i in range(cfg["layers"]):
        shared = i >= cfg["mm_layers"]
        last = cfg.get("last_vid_only", False) and i == cfg["layers"] - 1
        p = f"blocks.{i}."
        for s in (("all",) if shared else ("vid", "txt")):
            m.linear(p + f"attn.proj_qkv.{s}", 3 * inner, d, bias=False)
            m.linear(p + f"attn.proj_out.{s}", d, inner)
            m.sd[p + f"attn.norm_q.{s}.weight"] = m.randn(hd, std=0.1, mean=1.0)
            m.sd[p + f"attn.norm_k.{s}.weight"] = m.randn(hd, std=0.1, mean=1.0)
        m.sd[p + "attn.rope.rope.freqs"] = freqs.to(dtype).to(device)
        for s in (("all",) if shared else (("vid",) if last else ("vid", "txt"))):
            if cfg["mlp"] == "swiglu":
                hid = swiglu_hidden(d)
                m.linear(p + f"mlp.{s}.proj_in_gate", hid, d, bias=False, gain=1.5)
                m.linear(p + f"mlp.{s}.proj_out", d, hid, bias=False)
                m.linear(p + f"mlp.{s}.proj_in", hid, d, bias=False)
            else:
                m.linear(p + f"mlp.{s}.proj_in", 4 * d, d, gain=1.5)
                m.linear(p + f"mlp.{s}.proj_out", d, 4 * d)
            for layer in ("attn", "mlp"):
                m.sd[p + f"ada.{s}.{layer}_shift"] = m.randn(d, std=0.1)
                m.sd[p + f"ada.{s}.{layer}_scale"] = m.randn(d, std=0.1, mean=1.0)
                m.sd[p + f"ada.{s}.{layer}_gate"] = m.randn(d, std=0.3)
    if cfg["out_norm"]:
        m.sd["vid_out_norm.weight"] = m.randn(d, std=0.1, mean=1.0)
        m.sd["vid_out_ada.out_shift"] = m.randn(d, std=0.1)
        m.sd["vid_out_ada.out_scale"] = m.randn(d, std=0.1, mean=1.0)
    m.linear("vid_out.proj", cfg["out_ch"] * 4, d)
    return m.sd


VAE_CHANNELS = (128, 256, 512, 512)


def synth_vae_state_dict(seed: int = 4321, dtype=torch.float16, device="cpu",
                         channels=VAE_CHANNELS, latent: int = 16) -> Dict[str, torch.Tensor]:
    """Keys of VideoAutoencoderKLWrapper.state_dict() for
    s8_c16_t4_inflation_sd3.yaml (attn_video_vae.py:671-1035)."""
    m = _Maker(seed, dtype, device)
    c = list(channels)

    def resnet(p, ci, co):
        m.norm(p + "norm1", ci)
        m.conv(p + "conv1", co, ci, gain=1.4)
        m.norm(p + "norm2", co)
        m.conv(p + "conv2", co, co, gain=0.7)
        if ci != co:
            m.conv(p + "conv_shortcut", co, ci, k=(1, 1, 1))

    def mid(p, ch):
        resnet(p + "resnets.0.", ch, ch)
        a = p + "attentions.0."
        m.norm(a + "group_norm", ch)
        for n in ("to_q", "to_k", "to_v"):
            m.linear(a + n, ch, ch, gain=1.5 if n != "to_v" else 1.0)
        m.linear(a + "to_out.0", ch, ch, gain=0.7)
        resnet(p + "resnets.1.", ch, ch)

    # encoder
    m.conv("encoder.conv_in", c[0], 3)
    ci = c[0]
    for i, co in enumerate(c):
        for j in range(2):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}.", ci if j == 0 else co, co)
        ci = co
        if i < len(c) - 1:
            temporal = i >= len(c) - 2 - 1      # Encoder3D: is_temporal_down_block
            k = (3, 3, 3) if temporal else (1, 3, 3)
            m.conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", co, co, k=k)
    mid("encoder.mid_block.", c[-1])
    m.norm("encoder.conv_norm_out", c[-1])
    m.conv("encoder.conv_out", 2 * latent, c[-1])
    # decoder
    rc = list(reversed(c))
    m.conv("decoder.conv_in", rc[0], latent)
    mid("decoder.mid_block.", rc[0])
    ci = rc[0]
    for i, co in enumerate(rc):
        for j in range(3):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}.", ci if j == 0 else co, co)
        ci = co
        if i < len(rc) - 1:
            temporal = i < 2
            r = 8 if temporal else 4
            p = f"decoder.up_blocks.{i}.upsamplers.0."
            eye = torch.eye(co, device=device).repeat(r, 1).reshape(co * r, co, 1, 1, 1)
            w = eye + torch.randn(co * r, co, 1, 1, 1, generator=m.g, device=device) * (0.3 / math.sqrt(co))
            m.sd[p + "upscale_conv.weight"] = w.to(dtype)
            m.sd[p + "upscale_conv.bias"] = m.randn(co * r, std=0.05)
            m.conv(p + "conv", co, co)
    m.norm("decoder.conv_norm_out", rc[-1])
    m.conv("decoder.conv_out", 3, rc[-1], gain=0.5)
    return m.sd


# ----------------------------------------------------------------------------------------------------------
# checkpoint files (SURVEY.md §8(f) rank 4)
def load_state_dict(path: str, device="cpu") -> Dict[str, torch.Tensor]:
    """Checkpoint file -> state dict with the reference key layout (``load_quantized_state_dict``,
    ``src/core/model_loader.py:84-153``): ``.safetensors`` in fp16 / bf16 / fp32 or fp8_e4m3fn storage (the CLI default
    model is ``*_fp8_e4m3fn.safetensors``, ``model_registry.py:56``) and ``.pth`` / ``.pt``.  The engines cast every
    tensor to their bf16 / fp32 layouts on the GPU, so fp8 and fp16 storage need no separate path.  GGUF (block-quantised)
    checkpoints are not part of the engine's path."""
    low = path.lower()
    if low.endswith(".safetensors"):
        from safetensors.torch import load_file
        sd = load_file(path, device=str(device))
    elif low.endswith((".pth", ".pt")):
        sd = torch.load(path, map_location=device, weights_only=True)
        if isinstance(sd, dict) and "state_dict" in sd and all(not torch.is_tensor(v) for v in sd.values()):
            sd = sd["state_dict"]
    elif low.endswith(".gguf"):
        raise NotImplementedError("GGUF checkpoints are not supported by the engine (use the safetensors files)")
    else:
        raise ValueError(f"unknown checkpoint format: {path}")
    prefix = "model.diffusion_model."          # ComfyUI-style exports (model_loader.py:143-147)
    if any(k.startswith(prefix) for k in sd):
        sd = {(k[len(prefix):] if k.startswith(prefix) else k): v for k, v in sd.items()}
    return sd


def detect_dit_variant(sd: Dict[str, torch.Tensor]) -> str:
    """3B (dim 2560, 32 layers) or 7B (dim 3072, 36 layers) from the checkpoint itself."""
    dim = sd["vid_in.proj.weight"].shape[0]
    if dim == 2560:
        return "3b"
    if dim == 3072:
        return "7b"
    raise ValueError(f"unrecognised NaDiT width {dim}")
