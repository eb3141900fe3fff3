"""Host side of the H100 causal 3-D conv video VAE (encode + decode).

Mirrors the reference operator interface
``VideoAutoencoderKLWrapper.encode(x).latent`` / ``.decode(z).sample``
(reference ``src/models/video_vae_v3/modules/attn_video_vae.py:1680-1698``) and
replaces ``Encoder3D`` (``:808-856``), ``Decoder3D`` (``:983-1035``),
``ResnetBlock3D`` (``:311-362``), ``Upsample3D`` (``:110-174``), ``Downsample3D``
(``:226-250``), ``UNetMidBlock3D`` + diffusers ``Attention`` (``:656-668``),
``InflatedCausalConv3d`` and ``causal_norm_wrapper``
(``causal_inflation_lib.py:213-305, 354-409``) with calls into libsvr2.so.

Data layout: activations are NDHWC bf16.  A tensor that feeds a causal 3x3x3
conv carries its temporal halo as two real frames in front of frame 0
(``pad = 2``); the kernel that produces it writes frame 0 into the halo as well
(first-frame replication, ``extend_head``, ``causal_inflation_lib.py:423-438``).
The reference's temporal slicing (``slicing_encode/_decode``, ``:1254-1300``) is
numerically exact; clips that fit in HBM are processed un-sliced, longer ones
in temporal chunks whose halo frames are the previous chunk's last two frames
at the same layer (the reference's ``InflatedCausalConv3d.memory``,
``causal_inflation_lib.py:306-352``) -- bit-identical to the un-sliced result.
"""
from __future__ import annotations

import os
from ctypes import c_void_p
from typing import Dict, Optional

import torch

from . import lib
from .module import EngineModule


class Act:
    """[pad + T, H, W, C] bf16 activation; ``pad`` halo frames replicate frame 0 (``rep``: its producer wrote them so, in
    the clip's first temporal slice) or hold the previous slice's tail."""

    def __init__(self, T, H, W, C, pad, device, buf=None, rep=False):
        self.T, self.H, self.W, self.C, self.pad = T, H, W, C, pad
        self.buf = buf if buf is not None else torch.empty(pad + T, H, W, C, device=device, dtype=torch.bfloat16)
        self.stats = None     # (partial sums tensor, slots) written by the producing conv's epilogue
        self.rep = rep

    @property
    def frame_elems(self):
        return self.H * self.W * self.C

    def body_ptr(self):
        return self.buf.data_ptr() + self.pad * self.frame_elems * 2

    @property
    def body(self):
        return self.buf[self.pad:]


def tile_settings(tile_size, tile_overlap) -> tuple:
    """(tile_h, tile_w, overlap_h, overlap_w) in sample pixels from a spatial tile size and overlap, each an int or an
    (h, w) pair (the VAE loader's ``*_tile_size`` / ``*_tile_overlap``)."""
    def pair(v, name, lo):
        h, w = (v, v) if isinstance(v, int) else tuple(v)
        if int(h) != h or int(w) != w or h < lo or w < lo:
            raise ValueError(f"{name} must be an int >= {lo} or a pair of them, got {v!r}")
        return int(h), int(w)
    return pair(tile_size, "tile_size", 1) + pair(tile_overlap, "tile_overlap", 0)


class VAEOutput:
    def __init__(self, **kw):
        self.__dict__.update(kw)


class B200VideoVAE(EngineModule):
    """Drop-in for the reference ``runner.vae`` (model-slot seam, infer.py:125-266): an ``nn.Module`` with the weights
    as buffers in the kernels' layout (``module.EngineModule``)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda"):
        super().__init__(device)
        lib.device_check()
        self.meta: Dict[str, tuple] = {}     # per conv: kernel size, un-padded (Cout, Cin)
        self._load(state_dict)
        self._chunk = None          # {"first": bool, "state": {layer key: last two frames}} while slicing
        self._sliced_plans = set()  # (direction, clip shape, cuts) that already ran sliced once
        self.split_size = None      # explicit temporal slice length in sample frames (set_causal_slicing)
        self.debug = None           # set by apply_model_specific_config (model_configuration.py:1270-1272)
        self.tensor_offload_device = None
        # encode / decode sequenced by the native runtime (csrc/vae_engine.cu; default) or by this module's Python
        # methods (per-call profiling, tests against the native runtime)
        self.native = True
        self._ws_bytes: Dict[tuple, int] = {}

    # ---- native runtime (csrc/vae_engine.cu): the same sequences in C++ on a svr2_t handle -------------------
    def _device_state_moved(self):
        self._drop_handle()
        # a device move copies every buffer on its own: make each folded conv's weight a view of its :head rows again
        W = self.__dict__.get("W")
        for k in [k for k in W.keys() if k.endswith(":head")] if W is not None else ():
            head = W[k]
            self._buffers[W._names[k[: -len(":head")]]] = head[: head.shape[0] // 2]

    def _drop_handle(self):
        h = self.__dict__.get("_handle")
        if h:
            lib.engine_destroy(h)
        self.__dict__["_handle"] = None
        if "_ws_bytes" in self.__dict__:
            self._ws_bytes.clear()

    def __del__(self):
        try:
            self._drop_handle()
        except Exception:   # noqa: BLE001 - interpreter shutdown
            pass

    def native_handle(self):
        """svr2_t* (variant 2) that borrows this module's weight buffers; conv weights are described with their
        [Cout, kt, kh, kw, Cin] shape (the buffers are those K-major rows)."""
        if self.__dict__.get("_handle"):
            return self._handle
        h = lib.engine_create(lib.ModelDesc(variant=2), self.device.index if self.device.index is not None
                              else torch.cuda.current_device())
        try:
            lib.engine_load(h, self._native_tensors(), copy=False)
        except Exception:
            lib.engine_destroy(h)
            raise
        self.__dict__["_handle"] = h
        return h

    def _native_tensors(self) -> Dict[str, torch.Tensor]:
        """The weight buffers under their checkpoint names, conv weights viewed as [Cout, kt, kh, kw, Cin]."""
        tensors = {}
        for k in self.W.keys():
            t = self.W[k]
            if (k + ".k") in self.meta and t.ndim == 2 and k not in ("encoder.conv_in.weight", "decoder.conv_out.weight"):
                kt, kh, kw = self.meta[k + ".k"]
                t = t.view(t.shape[0], kt, kh, kw, t.shape[1] // (kt * kh * kw))
            tensors[k] = t
        return tensors

    def workspace_bytes(self, encode: bool, T: int, H: int, W: int, slice_frames: int = 0,
                        frames: Optional[int] = None, tiles: Optional[tuple] = None) -> int:
        """Exact workspace of one native encode (T sample frames of H x W) / decode (T latent frames of H x W latent
        pixels) with temporal slices of ``slice_frames`` (0 = un-sliced); ``frames``: the decoded frames wanted (None:
        all 4T-3); ``tiles``: (tile_h, tile_w, overlap_h, overlap_w) of a spatially tiled pass (None: un-tiled)."""
        frames = None if encode else (4 * T - 3 if frames is None else frames)
        key = (bool(encode), T, H, W, slice_frames, frames, tiles)
        if key not in self._ws_bytes:
            L, h = lib.load(), self.native_handle()
            if tiles is not None:
                n = int(L.svr2_vae_tiled_workspace_bytes(h, 0 if encode else 1, T, H, W, *tiles, slice_frames,
                                                         0 if encode else frames))
            else:
                n = int(L.svr2_vae_workspace_bytes(h, 0, T, H, W, slice_frames) if encode
                        else L.svr2_vae_decode_frames_workspace_bytes(h, T, H, W, slice_frames, frames))
            if n <= 0:
                raise lib.Svr2Error("svr2_vae workspace query failed: " + L.svr2_engine_last_error(h).decode())
            self._ws_bytes[key] = n
        return self._ws_bytes[key]

    def _use_native(self) -> bool:
        return self.native and lib.PROFILER is None

    def _free_bytes(self) -> int:
        """Free HBM incl. torch's cached blocks and the engine's resident workspace (it is regrown on demand)."""
        free, _ = torch.cuda.mem_get_info(self.device)
        held = 0 if torch.cuda.is_current_stream_capturing() else lib.workspace_held(self.device)
        return free + torch.cuda.memory_reserved(self.device) - torch.cuda.memory_allocated(self.device) + held

    def plan_slices(self, encode: bool, T: int, H: int, W: int, budget: Optional[int] = None,
                    frames: Optional[int] = None, tiles: Optional[tuple] = None):
        """(slice_frames, workspace bytes) of a native encode (T sample frames of H x W) / decode (T latent frames of
        H x W latent pixels; ``frames``: the decoded frames wanted, None: all): the longest temporal slice — un-sliced
        first, then set_causal_slicing's split, then shorter ones — whose EXACT workspace fits ``budget`` bytes (default:
        92 % of the free HBM incl. torch's cached blocks).  ``tiles``: (tile_h, tile_w, overlap_h, overlap_w) — the
        same search for a spatially tiled pass, whose every tile is sliced alike."""
        step = 4 if encode else 1
        cap = None if self.split_size is None else (max(4, self.split_size // 4 * 4) if encode else max(1, self.split_size // 4))
        can_slice = not (encode and (T - 1) % 4)       # only 4n+1-frame clips continue the temporal stride phase
        sz = 0 if (cap is None or T - 1 <= cap or not can_slice) else cap
        fr = {} if frames is None else {"frames": frames}
        if tiles is not None:
            fr["tiles"] = tiles
        need = self.workspace_bytes(encode, T, H, W, sz, **fr)
        if can_slice:
            if budget is None:
                budget = int(0.92 * self._free_bytes())
            while need > budget:                       # each candidate is one dry run of the C++ sequence (no launches)
                cur = sz if sz else (T - 1 + step - 1) // step * step
                if cur <= step:
                    break
                sz = cur - step
                need = self.workspace_bytes(encode, T, H, W, sz, **fr)
        return sz, need

    def _native_run(self, encode: bool, src: torch.Tensor, T: int, H: int, W: int, out: torch.Tensor, workspace=None,
                    frames: Optional[int] = None, tiles: Optional[tuple] = None):
        """``workspace``: a uint8 CUDA tensor shared by the phases of a clip (pipeline.SeedVR2Engine.clip_workspace) or None —
        then the engine's resident block (lib.workspace; the capture pool inside a CUDA graph).  ``frames``: decode only
        the first ``frames`` output frames (None: all).  ``tiles``: (tile_h, tile_w, overlap_h, overlap_w), a spatially
        tiled pass (svr2_vae_encode_tiled / svr2_vae_decode_tiled)."""
        if workspace is not None:
            sz, need = self.plan_slices(encode, T, H, W, budget=workspace.numel(), frames=frames, tiles=tiles)
            if need > workspace.numel():
                raise lib.Svr2Error(f"B200VideoVAE: workspace of {workspace.numel()} bytes given, {need} needed")
            ws = workspace
        else:
            sz, need = self.plan_slices(encode, T, H, W, frames=frames, tiles=tiles)
            ws = lib.workspace(need, self.device)
        dt = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[src.dtype]
        if tiles is not None:
            if encode:
                lib.call("svr2_vae_encode_tiled", self.native_handle(), lib.ptr(src), dt, T, H, W, *tiles, sz, lib.ptr(out),
                         lib.ptr(ws), ws.numel(), lib.stream())
            else:
                lib.call("svr2_vae_decode_tiled", self.native_handle(), lib.ptr(src), dt, T, H, W, *tiles, sz,
                         4 * T - 3 if frames is None else frames, lib.ptr(out), lib.ptr(ws), ws.numel(), lib.stream())
        elif encode:
            lib.call("svr2_vae_encode", self.native_handle(), lib.ptr(src), dt, T, H, W, sz, lib.ptr(out), lib.ptr(ws),
                     ws.numel(), lib.stream())
        else:
            lib.call("svr2_vae_decode_frames", self.native_handle(), lib.ptr(src), dt, T, H, W, sz,
                     4 * T - 3 if frames is None else frames, lib.ptr(out), lib.ptr(ws), ws.numel(), lib.stream())
        lib.LAUNCHES += int(lib.load().svr2_vae_last_launches(self.native_handle())) - 1
        return out

    # ---- weights ---------------------------------------------------------
    def _conv_w(self, w, cin_pad=None, cout_pad=None, dtype=torch.bfloat16):
        """[O,I,kt,kh,kw] -> [O, kt*kh*kw*I] bf16 (K-major, tap-major then channel)."""
        O, I = w.shape[:2]
        w = w.to(self.device, dtype).permute(0, 2, 3, 4, 1)  # O,kt,kh,kw,I
        if cin_pad and cin_pad > I:
            w = torch.nn.functional.pad(w, (0, cin_pad - I))
        w = w.reshape(O, -1)
        if cout_pad and cout_pad > O:
            w = torch.nn.functional.pad(w, (0, 0, 0, cout_pad - O))
        return w.contiguous()

    def _vec(self, v, pad_to=None):
        v = v.to(self.device, torch.bfloat16)
        if pad_to and pad_to > v.numel():
            v = torch.nn.functional.pad(v, (0, pad_to - v.numel()))
        return v.contiguous()

    def _load(self, sd):
        sd = dict(sd)
        # deprecated diffusers attention key names (attn_video_vae.py:1647-1657)
        for k in list(sd.keys()):
            for old, new in ((".query.", ".to_q."), (".key.", ".to_k."), (".value.", ".to_v."),
                             (".proj_attn.", ".to_out.0.")):
                if ".attentions." in k and old in k:
                    sd[k.replace(old, new)] = sd.pop(k)
                    break
        W: Dict[str, torch.Tensor] = {}
        for k, v in sd.items():
            if k.endswith("upscale_conv.weight"):
                W[k] = v.to(self.device, torch.bfloat16).reshape(v.shape[0], v.shape[1]).contiguous()
            elif k == "encoder.conv_in.weight":      # im2col GEMM: K = 81 padded to 128
                W[k] = torch.nn.functional.pad(self._conv_w(v), (0, 128 - 81)).contiguous()
            elif k == "decoder.conv_in.weight":
                W[k] = self._conv_w(v, cin_pad=64)
            elif k == "decoder.conv_out.weight":
                # tap-major GEMM operand: row = tap*3 + co, K = 128 input channels (see decode())
                O, I = v.shape[:2]
                W[k] = v.to(self.device, torch.bfloat16).permute(2, 3, 4, 0, 1).reshape(27 * O, I).contiguous()
            elif k.endswith(".weight") and v.ndim == 5:
                W[k] = self._conv_w(v)
            elif k.endswith(".weight") and v.ndim == 4:   # 2-D checkpoint: "tail" inflation (causal_inflation_lib.py:440-457)
                raise NotImplementedError("2-D VAE checkpoints are not supported by the engine")
            else:
                W[k] = self._vec(v) if v.ndim == 1 else v.to(self.device, torch.bfloat16).contiguous()
            if k.endswith(".weight") and v.ndim == 5:
                self.meta[k + ".k"] = tuple(v.shape[2:])
                self.meta[k + ".real"] = (v.shape[0], v.shape[1])   # un-padded (Cout, Cin) for the FLOP model

        # ResnetBlock3D with a channel change: conv2 and the 1x1x1 conv_shortcut become ONE contraction
        # [hidden ; x] . [W2 ; Wsc] (svr2_conv3d_shortcut_stats_bf16): concatenate the K-major weight rows, sum the biases
        for k in [k for k in W if k.endswith("conv_shortcut.weight")]:
            p = k[: -len("conv_shortcut.weight")]
            wsc = W[k].reshape(W[k].shape[0], -1)                                   # [Cout, Cin] (1x1x1)
            W[p + "conv2+shortcut.weight"] = torch.cat([W[p + "conv2.weight"], wsc], 1).contiguous()
            W[p + "conv2+shortcut.bias"] = (W[p + "conv2.bias"].float() + W[p + "conv_shortcut.bias"].float()
                                            ).to(torch.bfloat16).contiguous()
        # Every kt = 3 conv that runs through svr2_conv3d_bf16 / _stats gets its folded head taps (include/svr2.h
        # SVR2_EPI_FOLD_HEAD) for the first temporal slice, whose input halo replicates frame 0; the regular weight is the
        # first Cout rows of that buffer.  (conv2 of a block with a shortcut runs unfolded as conv2+shortcut.)  The sums are
        # taken over the checkpoint's own weights, so a folded weight is rounded to bf16 once, like each unfolded tap.
        for k in [k for k in W if k.endswith(".weight")]:
            if (self.meta.get(k + ".k", (0,))[0] != 3 or k in ("encoder.conv_in.weight", "decoder.conv_out.weight")
                    or (k.endswith("conv2.weight") and k.replace("conv2.weight", "conv_shortcut.weight") in W)):
                continue
            W[k + ":head"] = self._fold_head(self._conv_w(sd[k], cin_pad=64 if k == "decoder.conv_in.weight" else None,
                                                          dtype=torch.float32))
            W[k] = W[k + ":head"][: W[k].shape[0]]
        self.W = self._register("w", W)

    @staticmethod
    def _fold_head(w: torch.Tensor) -> torch.Tensor:
        """[Cout, 3n] K-major rows of a kt = 3 conv (n = kh*kw*Cin per temporal tap; any float dtype) -> [2 Cout, 3n] bf16:
        bf16(rows), then [bf16(W0+W1) bf16(W2) | bf16(W0+W1+W2)], the sums in fp32 in that order."""
        n = w.shape[1] // 3
        w01, w2 = w[:, :n].float() + w[:, n:2 * n].float(), w[:, 2 * n:].float()
        fold = torch.cat([w01, w2, w01 + w2], 1)
        return torch.cat([w, fold], 0).to(torch.bfloat16).contiguous()

    # ---- temporal slicing state -------------------------------------------
    @property
    def _first(self) -> bool:
        return self._chunk is None or self._chunk["first"]

    def _halo(self, y: Act, key: str) -> None:
        """Slice boundary: the halo of a tensor that feeds a causal conv is the previous slice's tail at the
        same layer (InflatedCausalConv3d.memory, causal_inflation_lib.py:306-352); remember this slice's tail."""
        c = self._chunk
        if c is None or y.pad == 0:
            return
        if not c["first"]:
            y.buf[: y.pad].copy_(c["state"][key])
        c["state"][key] = y.buf[-y.pad:].clone()

    # ---- primitive wrappers ----------------------------------------------
    def _gn(self, x: Act, prefix: str, silu: bool, pad: int) -> Act:
        y = Act(x.T, x.H, x.W, x.C, pad, self.device, rep=pad > 0 and self._first)
        if x.stats is not None:     # statistics came out of the producing conv's epilogue: finalize + apply only
            part, slots = x.stats
            coef = torch.empty(x.T * x.C * 2, device=self.device, dtype=torch.float32)
            lib.call("svr2_groupnorm_from_stats_bf16", c_void_p(x.body_ptr()), lib.ptr(y.buf), x.T, x.H * x.W, x.C,
                     lib.ptr(self.W[prefix + ".weight"]), lib.ptr(self.W[prefix + ".bias"]), 1e-6, int(silu), pad,
                     int(pad > 0 and self._first), lib.ptr(part), slots, lib.ptr(coef), lib.stream(),
                     nbytes=4.0 * x.T * x.H * x.W * x.C)
            self._halo(y, prefix)
            return y
        # per-call scratch (a few hundred KB): engine-level scratch would be baked into a captured CUDA graph by address
        # and could be rebound by a later, larger eager clip while the graph still writes to the old block
        need = lib.load().svr2_groupnorm_scratch_bytes(x.T, x.H * x.W, x.C)
        stats = torch.empty((need + 7) // 8, device=self.device, dtype=torch.float64)
        lib.call("svr2_groupnorm_bf16", c_void_p(x.body_ptr()), lib.ptr(y.buf), x.T, x.H * x.W, x.C,
                 lib.ptr(self.W[prefix + ".weight"]), lib.ptr(self.W[prefix + ".bias"]), 1e-6, int(silu), pad,
                 int(pad > 0 and self._first), lib.ptr(stats), stats.numel() * 8, lib.stream(),
                 nbytes=6.0 * x.T * x.H * x.W * x.C)
        self._halo(y, prefix)
        return y

    def _conv(self, x: Act, prefix: str, *, out_pad=0, residual: Optional[Act] = None, stride_t=1, stride_hw=1,
              stats=False) -> Act:
        w = self.W[prefix + ".weight"]
        kt, kh, kw = self.meta[prefix + ".weight.k"]
        assert x.pad == kt - 1, f"{prefix}: conv with kt={kt} needs a {kt - 1}-frame halo, got {x.pad}"
        x_ptr, T_in_total = lib.ptr(x.buf), x.pad + x.T
        if stride_t == 2 and not self._first:
            # a later slice of a temporally strided conv continues the global stride phase: one frame of
            # memory instead of two (kernel - stride, causal_inflation_lib.py:306-352), T_out = T / 2
            assert x.T % 2 == 0, "temporal slices after the first must hold a multiple of 4 frames"
            x_ptr, T_in_total = c_void_p(x.buf.data_ptr() + x.frame_elems * 2), x.pad - 1 + x.T
            T_out = x.T // 2
        else:
            T_out = (x.T - 1) // stride_t + 1
        Ho, Wo = (x.H, x.W) if stride_hw == 1 else (x.H // 2, x.W // 2)
        y = Act(T_out, Ho, Wo, w.shape[0], out_pad, self.device, rep=out_pad > 0 and self._first)
        res_ptr = None
        if residual is not None:
            assert (residual.T, residual.H, residual.W, residual.C) == (T_out, Ho, Wo, w.shape[0])
            # the kernel indexes the residual with the output's offsets (which include out_pad halo frames)
            res_ptr = c_void_p(residual.body_ptr() - out_pad * y.frame_elems * 2)
        # a halo that replicates frame 0: frames 0 and 1 run folded taps (vae_engine.cu Run::head_weight)
        wf = self.W.get(prefix + ".weight:head") if (x.rep and kt == 3) else None
        folded = 0 if wf is None else (3 if stride_t == 1 and T_out >= 2 else 2)      # temporal taps the fold skips
        epi = lib.EPI_BIAS | (lib.EPI_RESIDUAL if residual is not None else 0) | (lib.EPI_FOLD_HEAD if wf is not None else 0)
        pad_hw = 1 if (stride_hw == 1 and kh == 3) else 0
        args = (x_ptr, T_in_total, x.H, x.W, x.C, lib.ptr(w if wf is None else wf), w.shape[0], kt, kh, kw, stride_t, stride_hw,
                pad_hw, T_out, epi, lib.ptr(self.W[prefix + ".bias"]), res_ptr, lib.ptr(y.buf), out_pad,
                int(out_pad > 0 and self._first), w.shape[0])
        name, extra = "svr2_conv3d_bf16", ()
        if stats and w.shape[0] in (128, 256, 512):
            import ctypes
            slots = ctypes.c_int(lib.load().svr2_conv_stat_slots(w.shape[0], Ho, Wo))
            part = torch.empty(T_out * slots.value * (w.shape[0] // 8) * 4, device=self.device, dtype=torch.float32)
            y.stats = (part, slots.value)
            name, extra = "svr2_conv3d_stats_bf16", (lib.ptr(part), part.numel() * 4, ctypes.byref(slots))
        lib.call(name, *args, *extra, lib.stream(),
                 flops=2.0 * (kt * T_out - folded) * Ho * Wo * self.meta[prefix + ".weight.real"][0] * kh * kw
                 * self.meta[prefix + ".weight.real"][1],
                 tag=(f"|{x.C}>{w.shape[0]}|k{kt}{kh}{kw}|s{stride_t}{stride_hw}|{T_out}x{Ho}x{Wo}"
                      if (lib.PROFILER is not None and lib.PROFILER.detail) else ""))
        self._halo(y, prefix + ":out")
        return y

    def _resnet(self, x: Act, p: str, out_pad=0) -> Act:
        """ResnetBlock3D.forward (attn_video_vae.py:311-362)."""
        h = self._gn(x, p + "norm1", True, 2)
        h = self._conv(h, p + "conv1", stats=True)
        h = self._gn(h, p + "norm2", True, 2)
        if (p + "conv_shortcut.weight") in self.W:
            return self._conv_shortcut(h, x, p, out_pad)
        return self._conv(h, p + "conv2", out_pad=out_pad, residual=x, stats=True)

    def _conv_shortcut(self, h: Act, x: Act, p: str, out_pad: int) -> Act:
        """conv2(h) + conv_shortcut(x) as one implicit GEMM over [h ; x] (see _load); statistics for the next GroupNorm."""
        import ctypes
        w, b = self.W[p + "conv2+shortcut.weight"], self.W[p + "conv2+shortcut.bias"]
        kt, kh, kw = self.meta[p + "conv2.weight.k"]
        Cout, C2 = w.shape[0], x.C
        assert h.pad == kt - 1 and (h.T, h.H, h.W) == (x.T, x.H, x.W) and h.C == Cout
        y = Act(h.T, h.H, h.W, Cout, out_pad, self.device, rep=out_pad > 0 and self._first)
        args = (lib.ptr(h.buf), h.pad + h.T, h.H, h.W, h.C, lib.ptr(w), Cout, kt, kh, kw, h.T, lib.ptr(b),
                c_void_p(x.body_ptr()), C2, lib.ptr(y.buf), out_pad, int(out_pad > 0 and self._first))
        slots = ctypes.c_int(lib.load().svr2_conv_stat_slots(Cout, h.H, h.W))
        part = torch.empty(h.T * slots.value * (Cout // 8) * 4, device=self.device, dtype=torch.float32)
        y.stats = (part, slots.value)
        lib.call("svr2_conv3d_shortcut_stats_bf16", *args, lib.ptr(part), part.numel() * 4, ctypes.byref(slots), lib.stream(),
                 flops=2.0 * h.T * h.H * h.W * Cout * (kt * kh * kw * h.C + C2),
                 tag=(f"|{h.C}+{C2}>{Cout}|k{kt}{kh}{kw}|s11|{h.T}x{h.H}x{h.W}"
                      if (lib.PROFILER is not None and lib.PROFILER.detail) else ""))
        self._halo(y, p + "conv2:out")
        return y

    def _attention(self, x: Act, p: str, single_pass: bool = True) -> Act:
        """UNetMidBlock3D per-frame attention (attn_video_vae.py:656-668): GN -> q,k,v -> 1-head
        softmax(q k^T / sqrt(C)) v -> out proj -> + x.  ``single_pass=False`` runs only the exact two-pass launches."""
        C, n = x.C, x.H * x.W
        dev = self.device
        y = self._gn(x, p + "group_norm", False, 0)
        yf = y.buf.view(x.T * n, C)
        q = lib.linear(yf, self.W[p + "to_q.weight"], bias=self.W[p + "to_q.bias"])
        # K carries 8 spare rows: pass 2 runs with N rounded up to a multiple of 8 (16-byte stores);
        # the extra score columns are never read by the P @ V GEMM (its K extent is n)
        k_buf = torch.empty(x.T * n + 8, C, device=dev, dtype=torch.bfloat16)
        k_buf[x.T * n:].zero_()
        lib.linear(yf, self.W[p + "to_k.weight"], bias=self.W[p + "to_k.bias"], out=k_buf[: x.T * n])
        v = lib.linear(yf, self.W[p + "to_v.weight"], bias=self.W[p + "to_v.bias"])
        del y, yf
        o = self._softmax_v(q, k_buf, v, x.T, n, single_pass)
        out = Act(x.T, x.H, x.W, C, 0, dev)
        xb = x.body.reshape(x.T * n, C)
        lib.linear(o, self.W[p + "to_out.0.weight"], bias=self.W[p + "to_out.0.bias"], residual=xb,
                   out=out.buf.view(x.T * n, C))
        return out

    @staticmethod
    def _attention_chunk_rows(n: int) -> int:
        """Query rows per chunk of _softmax_v (vae_engine.cu attention computes the same): whole waves of m-tiles, as many
        as keep the chunk's bf16 P under 4 GiB, never more rows than the frame's m-tiles hold."""
        ldn = (n + 7) // 8 * 8
        wave_rows = 66 * 128                       # 66 m-tiles x 2 n-tiles (d = 512) = one full wave of 132 CTAs
        k = max(1, (1 << 32) // (wave_rows * ldn * 2))
        return min(wave_rows * k, (n + 127) // 128 * 128)

    def _softmax_v(self, q, k_buf, v, T: int, n: int, single_pass: bool = True, *, o=None, vt=None, P=None,
                   flag_log=None):
        """softmax(q k^T / sqrt(C)) v per frame for T frames of n tokens: q, v (T n, C); k_buf (T n + 8, C) whose last 8
        rows are zero.  Returns o (T n, C) bf16.  Tests may pass the output `o`, the scratch `vt` (C, >= ceil8(n)) and
        `P` (>= min(cq, n) rows, ldn columns) to guard them, and `flag_log` (int32, one entry per frame and query chunk) to
        receive the single-pass fallback flag as each chunk's svr2_pexp_stat_combine left it."""
        C, dev = q.shape[1], self.device
        # Two GEMM passes per query chunk, never materialising the fp32 score matrix:
        #   pass 1: per-row (max, sum exp2) partials of q k^T * scale  -> log2-sum-exp per row
        #   pass 2: P = bf16(exp2(q k^T * scale - lse))  (normalised probabilities)
        #   then   O = P @ V  (V consumed through its transpose, K-major)
        ldn = (n + 7) // 8 * 8
        cq = self._attention_chunk_rows(n)
        slots = lib.load().svr2_rowstat_slots(n)
        if vt is None:
            vt = torch.empty(C, ldn, device=dev, dtype=torch.bfloat16)
        part = torch.empty(min(cq, n), 2 * slots, device=dev, dtype=torch.float32)
        lse = torch.empty(min(cq, n), device=dev, dtype=torch.float32)
        if P is None:
            P = torch.empty(min(cq, n), ldn, device=dev, dtype=torch.bfloat16)
        if o is None:
            o = torch.empty(T * n, C, device=dev, dtype=torch.bfloat16)
        k_ = k_buf[:T * n]
        scale2 = (1.0 / (C ** 0.5)) * 1.4426950408889634
        # Default (n >= 256, n % 8 == 0): ONE Q K^T pass.  A 1/16-cost GEMM over every 16th key yields a reference
        # exponent per row; the full pass writes un-normalised bf16(exp2(s - ref)) and fp32 row sums; P~ @ V is divided
        # by the row sum in its epilogue.  Exact (softmax is shift-invariant; bf16 rounding is relative) as long as every
        # row sum lies in (1e-30, 1e30) — checked on the device; the exact two-pass launches below are conditional on
        # that flag.
        single = single_pass and n >= 256 and n % 8 == 0
        if single:
            k_sub_stride = 16
            n_sub = (n + k_sub_stride - 1) // k_sub_stride
            slots_s = lib.load().svr2_rowstat_slots(n_sub)
            slots_p = 2 * ((n + 255) // 256)
            rows_max = min(cq, n)
            part_s = torch.empty(rows_max, 2 * slots_s, device=dev, dtype=torch.float32)
            stat = torch.empty(rows_max, 2 * slots_p, device=dev, dtype=torch.float32)
            mhat = torch.empty(rows_max, device=dev, dtype=torch.float32)
            rscale = torch.empty(rows_max, device=dev, dtype=torch.float32)
            flag = torch.zeros(1, device=dev, dtype=torch.int32)
        for f in range(T):
            qf, kf, vf = q[f * n:(f + 1) * n], k_[f * n:(f + 1) * n], v[f * n:(f + 1) * n]
            lib.call("svr2_transpose_bf16", lib.ptr(vf), C, lib.ptr(vt), vt.stride(0), n, C, lib.stream())
            for r0 in range(0, n, cq):
                rows = min(cq, n - r0)
                qc, oc = qf[r0:r0 + rows], o[f * n + r0: f * n + r0 + rows]
                if single:
                    lib.linear(qc, kf[::k_sub_stride], epi=lib.EPI_ROWSTAT, out=part_s[:rows], out_scale=scale2, count_flops=False)
                    lib.call("svr2_rowstat_max", lib.ptr(part_s), slots_s, slots_s, lib.ptr(mhat), rows, lib.ptr(flag), lib.stream())
                    lib.linear(qc, kf, epi=lib.EPI_PEXP, gate=mhat, out=P[:rows], out_scale=scale2, stat_out=stat[:rows])
                    lib.call("svr2_pexp_stat_combine", lib.ptr(stat), slots_p, slots_p, lib.ptr(mhat), lib.ptr(rscale), rows,
                             lib.ptr(flag), lib.stream())
                    if flag_log is not None:
                        flag_log[f * -(-n // cq) + r0 // cq].copy_(flag[0])
                    lib.linear(P[:rows, :n], vt[:, :n], out=oc, rowscale=rscale)
                run_if = flag if single else None        # exact path: unconditional, or the device-side fallback
                lib.linear(qc, kf, epi=lib.EPI_ROWSTAT, out=part[:rows], out_scale=scale2, count_flops=False, run_if=run_if)
                lib.call("svr2_rowstat_combine", lib.ptr(part), slots, slots, lib.ptr(lse), rows, lib.stream())
                lib.linear(qc, k_buf[f * n: f * n + ldn], epi=lib.EPI_PEXP, gate=lse, out=P[:rows], out_scale=scale2,
                           run_if=run_if, count_flops=not single)
                lib.linear(P[:rows, :n], vt[:, :n], out=oc, run_if=run_if, count_flops=not single)
        return o

    def _mid(self, x: Act, p: str) -> Act:
        x = self._resnet(x, p + "resnets.0.")
        x = self._attention(x, p + "attentions.0.")
        return self._resnet(x, p + "resnets.1.")

    def _upsample(self, x: Act, p: str, temporal: bool, keep: Optional[int] = None) -> Act:
        """Upsample3D.forward (attn_video_vae.py:110-174).  ``keep``: only the first ``keep`` shuffled frames are wanted
        (the decoder's last temporal upsampler; every later layer is causal frame by frame): the conv and everything
        after it run on those frames alone."""
        z = 2 if temporal else 1
        first = self._first                       # remove_head only drops (f=0, z=1) of the clip's first slice
        T_out = x.T * z - (1 if temporal and first else 0)
        y = Act(T_out, 2 * x.H, 2 * x.W, x.C, 2, self.device, rep=first)
        lib.call("svr2_upsample_shuffle_bf16", c_void_p(x.body_ptr()), x.T, x.H, x.W, x.C,
                 lib.ptr(self.W[p + "upscale_conv.weight"]), lib.ptr(self.W[p + "upscale_conv.bias"]), int(temporal),
                 int(first), lib.ptr(y.buf), 2, int(first), lib.stream(),
                 flops=2.0 * x.T * x.H * x.W * x.C * 4 * z * x.C)
        if keep is not None and keep < y.T:
            y = Act(keep, y.H, y.W, y.C, y.pad, self.device, buf=y.buf[:y.pad + keep], rep=y.rep)
        self._halo(y, p + "shuffle")
        return self._conv(y, p + "conv", stats=True)

    # ---- temporal slice planning -------------------------------------------
    BYTES_PER_PIXEL_FRAME = 1500     # measured peak working set of one full-resolution frame (decode or encode)
    # Slicing keeps, for every tensor that feeds a causal conv, the last two frames of the previous slice (the
    # reference's per-conv `memory`).  Summed over the decoder that is 4.3 kB per full-resolution pixel and frame
    # (1280 channels at full resolution, 2304 at 1/2, 3584 at 1/4, ~5200 at 1/8), 2.0 kB for the encoder.
    DEC_STATE_BYTES_PER_PIXEL = 2 * 4400
    ENC_STATE_BYTES_PER_PIXEL = 2 * 2100

    def _frames_that_fit(self, H: int, W: int, state_bytes_per_pixel: int = 0) -> int:
        """Full-resolution frames one pass may hold, from the free HBM (minus the slicing state when slicing)."""
        free, _ = torch.cuda.mem_get_info(self.device)
        free += torch.cuda.memory_reserved(self.device) - torch.cuda.memory_allocated(self.device)
        budget = int(0.85 * free) - state_bytes_per_pixel * H * W
        return max(1, budget // (self.BYTES_PER_PIXEL_FRAME * H * W))

    @staticmethod
    def _plan(T: int, size: int):
        """[start, stop) slices like the reference (slicing_encode/_decode, attn_video_vae.py:1254-1300):
        the first slice is frame 0 plus ``size`` frames, every later one ``size`` frames."""
        if T - 1 <= size:
            return [(0, T)]
        cuts = [(0, 1 + size)]
        while cuts[-1][1] < T:
            cuts.append((cuts[-1][1], min(T, cuts[-1][1] + size)))
        return cuts

    @staticmethod
    def _decoded_per_slice(cuts, frames: int):
        """Output frames each decode slice of ``cuts`` computes when only the first ``frames`` are wanted (slice_decode
        of the native runtime): slices past them are dropped, the last one that runs is trimmed."""
        keep, o0 = [], 0
        for a, b in cuts:
            n_out = 4 * (b - a) - (3 if a == 0 else 0)
            if frames <= o0:
                break
            keep.append(min(frames - o0, n_out))
            o0 += n_out
        return keep

    def _run_sliced(self, fn, src: torch.Tensor, cuts, keep=None):
        """``keep`` (decode): per slice, the output frames ``fn(slice, keep[i])`` computes; slices without an entry do not
        run.  None: ``fn(slice)`` for every slice."""
        extra = [()] * len(cuts) if keep is None else [(k,) for k in keep]
        if len(cuts) == 1:
            return fn(src, *extra[0])
        cuts = cuts[:len(extra)]
        outs = []
        key = (fn.__name__, tuple(src.shape), tuple(cuts))
        if not torch.cuda.is_current_stream_capturing():
            # long clips run close to the HBM limit: the FIRST sliced pass of a shape starts from an unfragmented pool.
            # Repeats of the same shape find their blocks in the caching allocator; the cache is emptied again only when
            # it holds a large share of the device un-allocated (fragmentation risk) and the allocator is not the
            # non-fragmenting one (PYTORCH_CUDA_ALLOC_CONF=expandable_segments:True, which bench.py selects for these
            # workloads) — every empty_cache puts synchronous cudaFree / cudaMalloc calls in front of the layers.
            expandable = "expandable_segments:True" in os.environ.get("PYTORCH_CUDA_ALLOC_CONF", "")
            idle = torch.cuda.memory_reserved(self.device) - torch.cuda.memory_allocated(self.device)
            total = torch.cuda.get_device_properties(self.device).total_memory
            if key not in self._sliced_plans or (not expandable and idle > 0.25 * total):
                torch.cuda.empty_cache()
            self._sliced_plans.add(key)
        self._chunk = {"first": True, "state": {}}
        try:
            for (a, b), args in zip(cuts, extra):
                outs.append(fn(src[:, a:b].contiguous(), *args))
                self._chunk["first"] = False
        finally:
            self._chunk = None
        return torch.cat(outs, dim=2)

    # ---- public API --------------------------------------------------------
    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict=True, tiled=False, tile_size=None, tile_overlap=None, workspace=None,
               frames: Optional[int] = None):
        """z (1,16,T,h,w) or (1,16,h,w) -> .sample (1,3,4T-3,8h,8w) bf16 (Decoder3D.forward).  ``frames``: return only
        the first ``frames`` (1 .. 4T-3) output frames, the same values; the decoder is causal in time, so the layers
        after the last temporal upsampler run on those frames alone.  ``tiled``: spatial tiles of ``tile_size`` sample
        pixels overlapping by ``tile_overlap`` (each an int or an (h, w) pair; default 512 / 64), see ``_tiled``; on
        the native runtime by default (svr2_vae_decode_tiled)."""
        self._require_cuda("B200VideoVAE.decode")
        squeeze = z.ndim == 4
        if squeeze:
            z = z.unsqueeze(2)
        T = z.shape[2]
        if frames is not None and not 1 <= frames <= 4 * T - 3:
            raise ValueError(f"frames = {frames}: a decode of {T} latent frames returns 1 .. {4 * T - 3} frames")
        if tiled:
            tiles = tile_settings(tile_size or 512, 64 if tile_overlap is None else tile_overlap)
            if self._use_native():
                _, _, T, h, w = z.shape
                F = 4 * T - 3 if frames is None else frames
                out = torch.empty(1, 3, F, 8 * h, 8 * w, device=self.device, dtype=torch.bfloat16)
                self._native_run(False, z[0].to(self.device).contiguous(), T, h, w, out, workspace, frames=F, tiles=tiles)
            else:
                out = self._tiled(z, False, tiles[:2], tiles[2:], frames=frames)
            return VAEOutput(sample=out.squeeze(2) if squeeze else out)
        assert z.shape[0] == 1 and z.shape[1] == 16
        _, _, T, h, w = z.shape
        F = 4 * T - 3 if frames is None else frames
        zin = z[0].to(self.device)
        if self._use_native():
            out = torch.empty(1, 3, F, 8 * h, 8 * w, device=self.device, dtype=torch.bfloat16)
            self._native_run(False, zin.contiguous(), T, h, w, out, workspace, frames=F)
            return VAEOutput(sample=out.squeeze(2) if squeeze else out)
        if 4 * T - 3 <= self._frames_that_fit(8 * h, 8 * w):         # the whole clip fits: no slicing state needed
            size = T
        else:
            size = max(1, self._frames_that_fit(8 * h, 8 * w, self.DEC_STATE_BYTES_PER_PIXEL) // 4)   # latent frames
        if self.split_size is not None:
            size = min(size, max(1, self.split_size // 4))
        cuts = self._plan(T, size)
        out = self._run_sliced(self._decode_slice, zin, cuts, self._decoded_per_slice(cuts, F))
        if squeeze:
            out = out.squeeze(2)
        return VAEOutput(sample=out)

    def _decode_slice(self, zin: torch.Tensor, keep: int) -> torch.Tensor:
        """One temporal slice: zin (16,T,h,w) -> (1,3,keep,8h,8w), the first ``keep`` of its T' output frames (T' = 4T-3
        for the clip's first slice else 4T)."""
        dev = self.device
        zin = zin.contiguous()
        _, T, h, w = zin.shape
        dt = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[zin.dtype]
        x = Act(T, h, w, 64, 2, dev, rep=self._first)
        lib.call("svr2_ncdhw_to_ndhwc_bf16", lib.ptr(zin), dt, 16, T, h, w, lib.ptr(x.buf), 64, 2, 1.0, lib.stream())
        self._halo(x, "decoder.in")
        x = self._conv(x, "decoder.conv_in", stats=True)
        x = self._mid(x, "decoder.mid_block.")
        for i in range(4):
            for j in range(3):
                x = self._resnet(x, f"decoder.up_blocks.{i}.resnets.{j}.")
            if i < 3:
                x = self._upsample(x, f"decoder.up_blocks.{i}.upsamplers.0.", temporal=i < 2, keep=keep if i == 1 else None)
        assert x.T == keep
        x = self._gn(x, "decoder.conv_norm_out", True, 2)
        # conv_out (128 -> 3): per-tap channel contraction as ONE GEMM over all input pixels (x read once, not
        # 27 times), fp32 z[tap*3+co][pixel], then the 27-tap spatial/temporal gather writes NCDHW directly.
        wt = self.W["decoder.conv_out.weight"]                      # [81, 128]
        npix = (x.pad + x.T) * x.H * x.W
        ldz = (npix + 3) // 4 * 4
        z = torch.empty(wt.shape[0], ldz, device=dev, dtype=torch.float32)
        lib.linear(wt, x.buf.view(npix, x.C), epi=lib.EPI_F32, out=z[:, :npix] if ldz != npix else z)
        out = torch.empty(1, 3, x.T, x.H, x.W, device=dev, dtype=torch.bfloat16)
        lib.call("svr2_conv_tap_gather", lib.ptr(z), ldz, 3, lib.ptr(self.W["decoder.conv_out.bias"]), x.T, x.H, x.W,
                 lib.ptr(out), 1, lib.stream(), nbytes=4.0 * 81 * npix)
        return out

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict=True, tiled=False, tile_size=None, tile_overlap=None, workspace=None):
        """x (1,3,T,H,W) or (1,3,H,W) in [-1,1] -> .latent (1,16,(T-1)/4+1,H/8,W/8) bf16 = posterior mode
        (Encoder3D.forward + DiagonalGaussianDistribution.mode, attn_video_vae.py:1680-1689).  ``tiled``: as in
        ``decode`` (svr2_vae_encode_tiled; frames whose sides are not multiples of 8 run ``_tiled``)."""
        self._require_cuda("B200VideoVAE.encode")
        squeeze = x.ndim == 4
        if squeeze:
            x = x.unsqueeze(2)
        if tiled:
            tiles = tile_settings(tile_size or 512, 64 if tile_overlap is None else tile_overlap)
            _, _, T, H, Wd = x.shape
            if self._use_native() and H % 8 == 0 and Wd % 8 == 0:
                out = torch.empty(1, 16, (T - 1) // 4 + 1, H // 8, Wd // 8, device=self.device, dtype=torch.bfloat16)
                self._native_run(True, x[0].to(self.device).contiguous(), T, H, Wd, out, workspace, tiles=tiles)
            else:
                out = self._tiled(x, True, tiles[:2], tiles[2:])
            return VAEOutput(latent=out.squeeze(2) if squeeze else out, latent_dist=None)
        assert x.shape[0] == 1 and x.shape[1] == 3
        _, _, T, H, Wd = x.shape
        xin = x[0].to(self.device)
        if self._use_native() and H % 8 == 0 and Wd % 8 == 0:
            out = torch.empty(1, 16, (T - 1) // 4 + 1, H // 8, Wd // 8, device=self.device, dtype=torch.bfloat16)
            self._native_run(True, xin.contiguous(), T, H, Wd, out, workspace)
            return VAEOutput(latent=out.squeeze(2) if squeeze else out, latent_dist=None)
        if T <= self._frames_that_fit(H, Wd):
            size = max(4, (T + 3) // 4 * 4)
        else:                                                        # sample frames per slice, a multiple of 4
            size = max(4, self._frames_that_fit(H, Wd, self.ENC_STATE_BYTES_PER_PIXEL) // 4 * 4)
        if self.split_size is not None:
            size = min(size, max(4, self.split_size // 4 * 4))
        # slices continue the stride-2 phase of the temporal downsamplers only for clips of 4n+1 frames
        cuts = self._plan(T, size) if (T - 1) % 4 == 0 else [(0, T)]
        out = self._run_sliced(self._encode_slice, xin, cuts)
        if squeeze:
            out = out.squeeze(2)
        return VAEOutput(latent=out, latent_dist=None)

    def _encode_slice(self, xin: torch.Tensor) -> torch.Tensor:
        """One temporal slice: xin (3,T,H,W) -> (1,16,T',H/8,W/8); T = 1+4k for the first slice, 4k after."""
        dev = self.device
        xin = xin.contiguous()
        _, T, H, Wd = xin.shape
        dt = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[xin.dtype]
        x8 = torch.empty(2 + T, H, Wd, 8, device=dev, dtype=torch.bfloat16)
        lib.call("svr2_ncdhw_to_ndhwc_bf16", lib.ptr(xin), dt, 3, T, H, Wd, lib.ptr(x8), 8, 2, 1.0, lib.stream())
        self._halo(Act(T, H, Wd, 8, 2, dev, buf=x8), "encoder.in")
        col = torch.empty(T * H * Wd, 128, device=dev, dtype=torch.bfloat16)
        lib.call("svr2_im2col3_bf16", lib.ptr(x8), T, H, Wd, 3, 8, lib.ptr(col), 128, lib.stream())
        h = Act(T, H, Wd, 128, 0, dev)
        lib.linear(col, self.W["encoder.conv_in.weight"], bias=self.W["encoder.conv_in.bias"],
                   out=h.buf.view(T * H * Wd, 128))
        del col, x8
        for i in range(4):
            p = f"encoder.down_blocks.{i}."
            temporal = i in (1, 2)
            h = self._resnet(h, p + "resnets.0.")
            h = self._resnet(h, p + "resnets.1.", out_pad=2 if (i < 3 and temporal) else 0)
            if i < 3:
                h = self._conv(h, p + "downsamplers.0.conv", stride_t=2 if temporal else 1, stride_hw=2, stats=True)
        h = self._mid(h, "encoder.mid_block.")
        h = self._gn(h, "encoder.conv_norm_out", True, 2)
        h = self._conv(h, "encoder.conv_out")
        out = torch.empty(1, 16, h.T, h.H, h.W, device=dev, dtype=torch.bfloat16)
        lib.call("svr2_ndhwc_to_ncdhw", lib.ptr(h.buf), 32, 16, h.T, h.H, h.W, lib.ptr(out), 1, lib.stream())
        return out

    # ---- spatial tiling (a25) ------------------------------------------------
    def _tiled(self, src: torch.Tensor, encode: bool, tile_size, tile_overlap, frames: Optional[int] = None) -> torch.Tensor:
        """VideoAutoencoderKL.tiled_encode / tiled_decode (attn_video_vae.py:1302-1630): the frame is cut into latent
        tiles of ``tile_size // 8`` stepping by ``tile - overlap // 8``; every tile runs through the whole (temporally
        sliced) encoder / decoder on its own and the results are cross-faded with raised-cosine ramps on interior
        edges — in latent space for encode, in sample space for decode — then normalised by the accumulated weights.
        Tiling changes results by design (tiles do not see their neighbours); it exists to bound memory.  The seam
        arithmetic runs in bf16 with the reference's rounding points (``svr2_tile_accumulate_bf16``).  ``frames``
        (decode): each tile decodes only the first ``frames`` output frames.  The tile-by-tile sequencing in Python
        (``.native = False``, profiling) of what svr2_vae_encode_tiled / svr2_vae_decode_tiled run natively."""
        dev = self.device
        _, _, _, H, W = src.shape
        f = 8
        th, tw = max(1, tile_size[0] // f), max(1, tile_size[1] // f)
        run = (lambda t: self.encode(t).latent) if encode else (lambda t: self.decode(t, frames=frames).sample)
        if (encode and H <= tile_size[0] and W <= tile_size[1]) or (not encode and H <= th and W <= tw):
            return run(src)
        loh, low = max(0, min(tile_overlap[0] // f, th - 1)), max(0, min(tile_overlap[1] // f, tw - 1))
        sh, sw = max(1, th - loh), max(1, tw - low)
        Hl, Wl = ((H + f - 1) // f, (W + f - 1) // f) if encode else (H, W)
        s = 1 if encode else f                                     # result samples per latent sample
        ovh, ovw = (loh, low) if encode else tuple(tile_overlap)   # ramp lengths in result samples
        bf = torch.bfloat16

        def ramp(n):
            t = torch.linspace(0, 1, steps=n, device=dev, dtype=bf)
            return 0.5 - 0.5 * torch.cos(t * torch.pi)
        ramps = (ramp(ovh) if ovh > 0 else None, ramp(ovw) if ovw > 0 else None)

        def weights(n, ov, r, lo, hi):
            w = torch.ones(n, device=dev, dtype=bf)
            if ov > 0 and lo:
                w[:ov] = r[:ov]
            if ov > 0 and hi:
                w[-ov:] = 1 - r[:ov]
            return w
        result = count = None
        for y0 in range(0, Hl, sh):
            y1 = min(y0 + th, Hl)
            for x0 in range(0, Wl, sw):
                x1 = min(x0 + tw, Wl)
                if (y0 > 0 and y1 - y0 <= loh) or (x0 > 0 and x1 - x0 <= low):
                    continue                                        # wholly inside the previous tile's overlap
                if encode:
                    tile = run(src[:, :, :, y0 * f:min(y1 * f, H), x0 * f:min(x1 * f, W)])
                else:
                    tile = run(src[:, :, :, y0:y1, x0:x1])
                tile = tile.contiguous()
                if result is None:
                    C, T = tile.shape[1], tile.shape[2]
                    result = torch.zeros(1, C, T, Hl * s, Wl * s, device=dev, dtype=bf)
                    count = torch.zeros(Hl * s, Wl * s, device=dev, dtype=bf)
                eh = min((y1 - y0) * s, tile.shape[3], Hl * s - y0 * s)
                ew = min((x1 - x0) * s, tile.shape[4], Wl * s - x0 * s)
                wh = weights(eh, max(0, min(ovh, eh - 1)), ramps[0], y0 > 0, y1 < Hl)
                ww = weights(ew, max(0, min(ovw, ew - 1)), ramps[1], x0 > 0, x1 < Wl)
                lib.call("svr2_tile_accumulate_bf16", lib.ptr(tile), tile.shape[3] * tile.shape[4], tile.shape[4],
                         C * T, eh, ew, lib.ptr(wh), lib.ptr(ww), lib.ptr(result), lib.ptr(count), Hl * s, Wl * s,
                         y0 * s, x0 * s, lib.stream(), nbytes=6.0 * C * T * eh * ew)
        lib.call("svr2_tile_normalize_bf16", lib.ptr(result), lib.ptr(count), result.shape[1] * result.shape[2],
                 Hl * s * Wl * s, lib.stream(), nbytes=4.0 * result.numel())
        return result

    # reference wrapper surface used by the pipeline (model_configuration.py:1247-1276)
    def preprocess(self, x):
        return x

    def postprocess(self, x):
        return x

    def set_causal_slicing(self, *, split_size=None, memory_device=None):
        """attn_video_vae.py:1709-1723: ``split_size`` sample frames per temporal slice (latent slices hold
        split_size // 4).  Slicing is exact; None lets the engine slice only when the clip does not fit in HBM."""
        self.split_size = split_size

    def set_memory_limit(self, conv_max_mem=None, norm_max_mem=None):
        pass
