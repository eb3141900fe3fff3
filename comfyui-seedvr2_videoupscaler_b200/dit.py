"""Host side of the H100 NaDiT forward (3B and 7B).

Mirrors the reference operator interface ``NaDiT.forward(vid, txt, vid_shape,
txt_shape, timestep) -> NaDiTOutput.vid_sample`` (reference
``src/models/dit_3b/nadit.py:190-248``, ``src/models/dit_7b/nadit.py:152-190``)
for b = 1, and replaces everything below it — ``NaMMSRTransformerBlock``
(``nablocks/mmsr_block.py:84-128``), ``NaSwinAttention`` (``mmattn.py:161-271``),
``FlashAttentionVarlen`` (``attention.py:114-148``), ``AdaSingle``
(``modulation.py:65-118``), ``CustomRMSNorm`` (``normalization.py:88-109``),
``SwiGLUMLP`` (``mlp.py:46-62``), ``NaPatchIn/Out`` (``patch/patch_v1.py:76-127``),
``TimeEmbedding`` (``embedding.py:25-62``) — with calls into libsvr2.so.

Python here does only: weight re-layout at load, buffer allocation and kernel
sequencing.  The window / RoPE index tables (``window.py:28-83``, ``na.py:583-641``,
``rope.py:130-176``) are the native runtime's, read through ``svr2_dit_geometry``.
No torch op touches activations on the hot path.
"""
from __future__ import annotations

import math
from typing import Dict, List, NamedTuple, Optional, Tuple

import torch

from . import lib, weights
from .attention import FlashAttentionVarlen
from .lib import EPI_GELU, EPI_SILU, EPI_SWIGLU
from .module import EngineModule


def dit_config(variant: str = "3b", **over) -> dict:
    """configs_3b/main.yaml:6-37, configs_7b/main.yaml:6-33."""
    if variant == "3b":
        cfg = dict(variant="3b", dim=2560, heads=20, head_dim=128, layers=32, mm_layers=10,
                   mlp="swiglu", txt_in_dim=5120, in_ch=33, out_ch=16, eps=1e-5,
                   out_norm=True, last_vid_only=True)
    elif variant == "7b":
        cfg = dict(variant="7b", dim=3072, heads=24, head_dim=128, layers=36, mm_layers=36,
                   mlp="gelu", txt_in_dim=5120, in_ch=33, out_ch=16, eps=1e-5,
                   out_norm=False, last_vid_only=False)
    else:
        raise ValueError(variant)
    cfg.update(over)
    return cfg


# --------------------------------------------------------------------------
# weights that stay compressed in device memory (resident="compressed")
# --------------------------------------------------------------------------
RESIDENT_MODES = ("expanded", "compressed")


class MatrixPart(NamedTuple):
    """One state-dict entry of a compressed block matrix and where svr2_weight_expand_bf16 puts its rows."""
    key: str
    format: int        # svr2_tensor_desc dtype code: lib.FMT_F16, lib.FMT_F8_E4M3 or lib.FMT_GGML + GGML type
    rows: int
    cols: int
    row_group: int
    group_stride: int
    row_offset: int


def storage_format(v) -> Optional[int]:
    """Format code of a state-dict entry that can stay as stored: a GGUF-quantized entry (a ``load_gguf`` record or the
    reference's ``GGUFTensor``) of a type the kernel decodes, or an fp8_e4m3fn tensor.  None for a dense entry."""
    if weights._is_quantized(v):
        return lib.FMT_GGML + int(v.tensor_type) if weights._known_block(int(v.tensor_type)) else None
    if isinstance(v, torch.Tensor) and v.dtype == torch.float8_e4m3fn:
        return lib.FMT_F8_E4M3
    return None


def _matrix_parts(sd, keys, swiglu: bool) -> Optional[List[MatrixPart]]:
    entries = [sd[k] for k in keys]
    fmts = [storage_format(v) for v in entries]
    if all(f is None for f in fmts):
        return None
    parts = []
    for j, (k, v, f) in enumerate(zip(keys, entries, fmts)):
        if f is None:      # the dense half of a SwiGLU pair whose other half is compressed: fp16 expands to the same bf16
            if not (isinstance(v, torch.Tensor) and v.dtype == torch.float16):
                return None
            f = lib.FMT_F16
        shape = tuple(int(n) for n in (v.tensor_shape if weights._is_quantized(v) else v.shape))
        block = weights.gguf_type_size(f - lib.FMT_GGML)[0] if f >= lib.FMT_GGML else 1
        if len(shape) != 2 or shape[1] % max(block, 8):
            return None
        rows, cols = shape
        if swiglu and (rows % 128 or (j and (rows, cols) != (parts[0].rows, parts[0].cols))):
            return None
        parts.append(MatrixPart(k, f, rows, cols, *((128, 256, 128 * j) if swiglu else (rows, rows, 0))))
    return parts


def compressed_matrices(cfg: dict, sd) -> Dict[str, List[MatrixPart]]:
    """What ``resident="compressed"`` keeps in its storage format: engine-layout matrix name -> its state-dict
    entries.  Only the four matrices of a block's stream qualify (``attn.proj_qkv``, ``attn.proj_out``, the MLP input
    and output weights: over 99 % of the bytes), and only when their entries are quantized or fp8; a SwiGLU input matrix
    is its ``proj_in_gate`` and ``proj_in`` entries, interleaved per 128 rows by the expansion.  Layers whose video
    and text streams share weights (``all``) are listed once, under the video name."""
    out: Dict[str, List[MatrixPart]] = {}
    swiglu = cfg["mlp"] == "swiglu"
    for i in range(cfg["layers"]):
        shared = i >= cfg["mm_layers"]
        last = cfg["last_vid_only"] and i == cfg["layers"] - 1
        for s in (("vid",) if shared else ("vid", "txt")):
            key, p = ("all" if shared else s), f"blocks.{i}."
            mats = {"qkv.w": [p + f"attn.proj_qkv.{key}.weight"], "out.w": [p + f"attn.proj_out.{key}.weight"]}
            if not (last and s == "txt"):
                mats["mlp_in.w"] = [p + f"mlp.{key}.proj_in_gate.weight", p + f"mlp.{key}.proj_in.weight"] if swiglu \
                    else [p + f"mlp.{key}.proj_in.weight"]
                mats["mlp_out.w"] = [p + f"mlp.{key}.proj_out.weight"]
            for n, keys in mats.items():
                parts = _matrix_parts(sd, keys, swiglu and n == "mlp_in.w")
                if parts:
                    out[f"{i}.{s}.{n}"] = parts
    return out


def slot_layout(cfg: dict, plan: Dict[str, List[MatrixPart]]) -> Tuple[List[Dict[str, int]], int]:
    """(per layer: matrix name -> byte offset in the staging slot, slot bytes): a block's compressed matrices in bf16
    one after the other, each rounded up to 256 bytes; the slot is the largest block (csrc/engine.cu plans the same)."""
    offsets: List[Dict[str, int]] = [{} for _ in range(cfg["layers"])]
    ends = [0] * cfg["layers"]
    for name, parts in plan.items():
        i = int(name.split(".", 1)[0])
        offsets[i][name] = ends[i]
        ends[i] += (sum(p.rows for p in parts) * parts[0].cols * 2 + 255) // 256 * 256
    return offsets, max(ends, default=0)


# --------------------------------------------------------------------------
# the engine
# --------------------------------------------------------------------------
class NaDiTOutput:
    def __init__(self, vid_sample):
        self.vid_sample = vid_sample


class B200NaDiT(EngineModule):
    """Drop-in for the reference ``runner.dit`` (VideoDiffusionInfer model slot, infer.py:361-367): an ``nn.Module``
    whose weights are buffers in the kernels' layout (see ``module.EngineModule`` for the lifecycle it survives) and
    which holds one ``FlashAttentionVarlen`` submodule, the class ``apply_model_specific_config`` looks for.

    ``resident``: ``"expanded"`` (default) expands every weight to bf16 once, at load.  ``"compressed"`` keeps the
    block matrices of a GGUF-quantized or fp8_e4m3fn state dict in their storage format in device memory
    (``compressed_matrices``) and expands each block's matrices to bf16 into a staging slot of the workspace just before
    the block runs: the GEMMs read the same bf16 bytes, so the output is bit-identical, the resident weights shrink to
    about the checkpoint's size and every forward pays the expansion.  A dense checkpoint has nothing to keep
    compressed and loads the same in both modes."""

    K_IN_PAD = 192  # 4*33 = 132 patch channels padded to 3 k-blocks of 64

    def __init__(self, cfg: dict, state_dict: Dict[str, torch.Tensor], device="cuda", timestep: float = 1000.0,
                 resident: str = "expanded"):
        if resident not in RESIDENT_MODES:
            raise ValueError(f"resident must be one of {RESIDENT_MODES}, got {resident!r}")
        super().__init__(device)
        self.resident = resident
        lib.device_check()
        self.cfg = cfg
        self.timestep = timestep
        self._window_flops: Dict[tuple, List[float]] = {}
        self.attention = FlashAttentionVarlen()
        self._load(state_dict)
        # forward sequenced by the native runtime (default) or by this module's Python loop (per-call profiling, tests
        # against the native runtime)
        self.native = True

    def _device_state_moved(self):
        if hasattr(self, "_window_flops"):
            self._window_flops.clear()
        self.__dict__.pop("_stage", None)
        self._drop_handle()

    # ---- native runtime (csrc/engine.cu): the same forward sequenced in C++ on a svr2_t handle ---------------
    def _drop_handle(self):
        h = self.__dict__.get("_handle")
        if h:
            lib.engine_destroy(h)
        self.__dict__["_handle"] = None

    def __del__(self):
        try:
            self._drop_handle()
        except Exception:   # noqa: BLE001 - interpreter shutdown
            pass

    def native_handle(self):
        """svr2_t* that borrows this module's weight buffers (they stay under nn.Module lifecycle control) and owns
        its workspace and the window / RoPE tables both sequencings read; rebuilt after a device move."""
        if self.__dict__.get("_handle"):
            return self._handle
        cfg = self.cfg
        desc = lib.ModelDesc(variant=0 if cfg["variant"] == "3b" else 1, dim=cfg["dim"], heads=cfg["heads"],
                             layers=cfg["layers"], mm_layers=cfg["mm_layers"], txt_in_dim=cfg["txt_in_dim"],
                             in_ch=cfg["in_ch"], out_ch=cfg["out_ch"], mlp_kind=0 if cfg["mlp"] == "swiglu" else 1,
                             mlp_hidden=self.mlp_hidden, out_norm=int(cfg["out_norm"]), last_vid_only=int(cfg["last_vid_only"]),
                             eps=cfg["eps"], timestep=self.timestep)
        h = lib.engine_create(desc, self.device.index if self.device.index is not None else torch.cuda.current_device())
        try:
            lib.engine_load(h, {k: self.W[k] for k in self.W.keys()}, copy=False)
            if self._formats:
                lib.engine_load(h, {k: self.C[k] for k in self.C.keys()}, copy=False, formats=self._formats)
            lib.engine_load(h, {k: self.M[k] for k in self.M.keys()}, copy=False)
            lib.engine_load(h, {f"{i}.rope_freqs": f for i, f in enumerate(self.rope_freqs)}, copy=True)
        except Exception:
            lib.engine_destroy(h)
            raise
        self.__dict__["_handle"] = h
        return h

    def workspace_bytes(self, T: int, H: int, W: int, txt_len: int = 58) -> int:
        return int(lib.load().svr2_workspace_bytes(self.native_handle(), T, H, W, txt_len))

    # ---- weights ---------------------------------------------------------
    def _w(self, sd, key):
        return sd[key].to(self.device, torch.bfloat16).contiguous()

    def _f(self, sd, key):
        return sd[key].to(self.device, torch.float32).contiguous()

    def _stored_bytes(self, v) -> torch.Tensor:
        """The bytes of a quantized or fp8 entry as stored, 1-D uint8 on the device (4-byte aligned for the kernel)."""
        t = weights._raw_blocks(v) if weights._is_quantized(v) else v.contiguous().view(torch.uint8).reshape(-1)
        t = t.to(self.device)
        return t.clone() if t.data_ptr() % 4 else t

    def _load(self, sd):
        cfg, dev = self.cfg, self.device
        plan = compressed_matrices(cfg, sd) if self.resident == "compressed" else {}
        stored = sd
        sd = weights.dequantizing(sd, self.device)   # GGUF entries: dense fp16 on the device, one key at a time
        d = cfg["dim"]
        W: Dict[str, torch.Tensor] = {}
        C: Dict[str, torch.Tensor] = {}                      # compressed matrices: the bytes of their entries
        formats: Dict[str, Tuple[int, Tuple[int, int]]] = {}  # their format codes and logical shapes

        def keep_compressed(name):
            parts = plan.get(name)
            for part, suffix in zip(parts or (), ("",) if parts and len(parts) == 1 else (".gate", ".in")):
                C[name + suffix] = self._stored_bytes(stored[part.key])
                formats[name + suffix] = (part.format, (part.rows, part.cols))
            return parts is not None
        w_in = sd["vid_in.proj.weight"].to(dev, torch.bfloat16)
        w_pad = torch.zeros(d, self.K_IN_PAD, device=dev, dtype=torch.bfloat16)
        w_pad[:, : w_in.shape[1]] = w_in
        W["vid_in.w"], W["vid_in.b"] = w_pad, self._w(sd, "vid_in.proj.bias")
        W["txt_in.w"], W["txt_in.b"] = self._w(sd, "txt_in.weight"), self._w(sd, "txt_in.bias")
        W["vid_out.w"], W["vid_out.b"] = self._w(sd, "vid_out.proj.weight"), self._w(sd, "vid_out.proj.bias")
        self.rope_freqs = []
        for i in range(cfg["layers"]):
            shared = i >= cfg["mm_layers"]
            last = cfg["last_vid_only"] and i == cfg["layers"] - 1
            p = f"blocks.{i}."
            for s in ("vid", "txt"):
                key = "all" if shared else s
                if shared and s == "txt":   # alias
                    for n in ("qkv.w", "out.w", "out.b", "nq", "nk", "nqk", "mlp_in.w", "mlp_in.b", "mlp_out.w", "mlp_out.b"):
                        if f"{i}.vid.{n}" in W:
                            W[f"{i}.txt.{n}"] = W[f"{i}.vid.{n}"]
                    for n in [k[len(f"{i}.vid."):] for k in C if k.startswith(f"{i}.vid.")]:
                        C[f"{i}.txt.{n}"], formats[f"{i}.txt.{n}"] = C[f"{i}.vid.{n}"], formats[f"{i}.vid.{n}"]
                    continue
                if not keep_compressed(f"{i}.{s}.qkv.w"):
                    W[f"{i}.{s}.qkv.w"] = self._w(sd, p + f"attn.proj_qkv.{key}.weight")
                if not keep_compressed(f"{i}.{s}.out.w"):
                    W[f"{i}.{s}.out.w"] = self._w(sd, p + f"attn.proj_out.{key}.weight")
                W[f"{i}.{s}.out.b"] = self._w(sd, p + f"attn.proj_out.{key}.bias")
                W[f"{i}.{s}.nq"] = self._f(sd, p + f"attn.norm_q.{key}.weight")
                W[f"{i}.{s}.nk"] = self._f(sd, p + f"attn.norm_k.{key}.weight")
                W[f"{i}.{s}.nqk"] = torch.cat([W[f"{i}.{s}.nq"], W[f"{i}.{s}.nk"]]).contiguous()   # [2][128]
                if last and s == "txt":
                    continue
                if cfg["mlp"] == "swiglu":
                    if not keep_compressed(f"{i}.{s}.mlp_in.w"):
                        g = sd[p + f"mlp.{key}.proj_in_gate.weight"].to(dev, torch.bfloat16)
                        u = sd[p + f"mlp.{key}.proj_in.weight"].to(dev, torch.bfloat16)
                        hid = g.shape[0]
                        assert hid % 128 == 0
                        # interleave 128-row groups: tile j of 256 rows = [gate_j ; in_j]  (EPI_SWIGLU)
                        il = torch.stack([g.view(hid // 128, 128, d), u.view(hid // 128, 128, d)], 1)
                        W[f"{i}.{s}.mlp_in.w"] = il.reshape(2 * hid, d).contiguous()
                    if not keep_compressed(f"{i}.{s}.mlp_out.w"):
                        W[f"{i}.{s}.mlp_out.w"] = self._w(sd, p + f"mlp.{key}.proj_out.weight")
                else:
                    if not keep_compressed(f"{i}.{s}.mlp_in.w"):
                        W[f"{i}.{s}.mlp_in.w"] = self._w(sd, p + f"mlp.{key}.proj_in.weight")
                    W[f"{i}.{s}.mlp_in.b"] = self._w(sd, p + f"mlp.{key}.proj_in.bias")
                    if not keep_compressed(f"{i}.{s}.mlp_out.w"):
                        W[f"{i}.{s}.mlp_out.w"] = self._w(sd, p + f"mlp.{key}.proj_out.weight")
                    W[f"{i}.{s}.mlp_out.b"] = self._w(sd, p + f"mlp.{key}.proj_out.bias")
            fr = sd.get(p + "attn.rope.rope.freqs")
            if fr is None:
                # the reference zero-fills persistent buffers a checkpoint does not carry (initialize_meta_buffers_impl,
                # model_loader.py:777-815; SURVEY G4): zero frequencies = identity rotation — reproduce that
                import warnings
                warnings.warn(f"{p}attn.rope.rope.freqs missing from the checkpoint: zero-filled like the reference "
                              "(RoPE becomes the identity)")
                nfreq = (128 // 2 // 3) // 2 if cfg["variant"] == "7b" else (128 // 3) // 2
                fr = torch.zeros(nfreq, dtype=sd["vid_in.proj.weight"].dtype)
            self.rope_freqs.append(fr.detach().cpu())
        self.W = self._register("w", W)
        self.C, self._formats, self._plan = self._register("c", C), formats, plan
        self._slot_offsets, self.slot_bytes = slot_layout(cfg, plan)
        self.mlp_hidden = plan["0.vid.mlp_in.w"][0].rows if "0.vid.mlp_in.w" in plan else \
            W["0.vid.mlp_in.w"].shape[0] // (2 if cfg["mlp"] == "swiglu" else 1)
        # ---- time embedding (constant: t == 1000, SURVEY.md fact 2) and AdaSingle vectors
        half = 128
        f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
        a = torch.tensor([self.timestep], dtype=torch.float32)[:, None] * f[None]
        e = torch.cat([a.sin(), a.cos()], -1).to(dev, torch.bfloat16)
        e = lib.linear(e, self._w(sd, "emb_in.proj_in.weight"), bias=self._w(sd, "emb_in.proj_in.bias"), epi=EPI_SILU)
        e = lib.linear(e, self._w(sd, "emb_in.proj_hid.weight"), bias=self._w(sd, "emb_in.proj_hid.bias"), epi=EPI_SILU)
        e = lib.linear(e, self._w(sd, "emb_in.proj_out.weight"), bias=self._w(sd, "emb_in.proj_out.bias"))
        E = e.float().view(d, 2, 3)     # [channel, layer{attn,mlp}, {shift,scale,gate}]  modulation.py:76
        M: Dict[str, torch.Tensor] = {}
        ones, zeros = torch.ones(d, device=dev), torch.zeros(d, device=dev)
        for i in range(cfg["layers"]):
            shared = i >= cfg["mm_layers"]
            last = cfg["last_vid_only"] and i == cfg["layers"] - 1
            for s in ("vid", "txt"):
                if last and s == "txt":
                    M[f"{i}.txt.attn_scale"], M[f"{i}.txt.attn_shift"] = ones, zeros
                    continue
                key = "all" if shared else s
                for li, layer in enumerate(("attn", "mlp")):
                    for gi, g in enumerate(("shift", "scale", "gate")):
                        M[f"{i}.{s}.{layer}_{g}"] = (E[:, li, gi] + self._f(sd, f"blocks.{i}.ada.{key}.{layer}_{g}")).contiguous()
        if cfg["out_norm"]:
            # G1: vid_out_ada reuses the attention slice of emb
            M["out_shift"] = (E[:, 0, 0] + self._f(sd, "vid_out_ada.out_shift")).contiguous()
            M["out_scale"] = (E[:, 0, 1] + self._f(sd, "vid_out_ada.out_scale")).contiguous()
            M["out_weight"] = self._f(sd, "vid_out_norm.weight")
        self.M = self._register("m", M)
        self.emb = None          # the raw time embedding is folded into M

    def _attn_flops(self, key: tuple, geo) -> List[float]:
        """Per layout parity: Σ over the windows of 4·len²·128, the attention FLOPs of one head (profiler records)."""
        if key not in self._window_flops:
            cu = [lib.host_copy(g.cu_seqlens, (g.n_win + 1,), torch.int32) for g in geo[:2]]
            self._window_flops[key] = [float((c.diff().double() ** 2).sum()) * 4 * 128 for c in cu]
        return self._window_flops[key]

    # ---- forward -----------------------------------------------------------
    @torch.no_grad()
    def forward(self, vid, txt, vid_shape, txt_shape, timestep=None, disable_cache=False, workspace=None):
        """vid (T*H*W, 33), txt (l, 5120); vid_shape [[T,H,W]], txt_shape [[l]] (b = 1)."""
        self._require_cuda("B200NaDiT.forward")
        if timestep is not None:
            t_in = float(torch.as_tensor(timestep).reshape(-1)[0])
            if abs(t_in - self.timestep) > 1e-3:
                raise lib.Svr2Error(f"B200NaDiT folds the time embedding of t = {self.timestep} into its AdaSingle vectors "
                                    f"at load (one-step sampling, SURVEY.md fact 2); got t = {t_in}")
        cfg, W, M = self.cfg, self.W, self.M
        vs = vid_shape.tolist() if torch.is_tensor(vid_shape) else list(vid_shape)
        ts = txt_shape.tolist() if torch.is_tensor(txt_shape) else list(txt_shape)
        if len(vs) != 1:
            raise ValueError("B200NaDiT: batch size 1 only (the reference pipeline always passes b = 1)")
        T, H, Wd = (int(v) for v in vs[0])
        l = int(ts[0][0])
        dev, d, heads = self.device, cfg["dim"], cfg["heads"]
        inner = heads * 128
        Hp, Wp = H // 2, Wd // 2
        L = T * Hp * Wp
        vid = vid.to(dev, torch.bfloat16).contiguous()
        txt = txt.to(dev, torch.bfloat16).contiguous()
        if self.native and lib.PROFILER is None:
            out = torch.empty(T * H * Wd, cfg["out_ch"], device=dev, dtype=torch.bfloat16)
            # the workspace comes from torch's caching allocator (and from the capture pool inside a CUDA graph) and goes
            # back to it after the forward: the VAE phases need those bytes (35 GB at a 65-frame 4K clip)
            # (or is the clip's shared workspace, pipeline.SeedVR2Engine.clip_to_sample)
            need = self.workspace_bytes(T, H, Wd, l)
            ws = workspace if (workspace is not None and workspace.numel() >= need) else \
                torch.empty(need, device=dev, dtype=torch.uint8)
            lib.call("svr2_dit_forward_ws", self.native_handle(), lib.ptr(vid), lib.ptr(txt), T, H, Wd, l, lib.ptr(out),
                     lib.ptr(ws), ws.numel(), lib.stream())
            n_l = cfg["layers"]
            lib.LAUNCHES += 15 * n_l - (3 if cfg["last_vid_only"] else 0) + 5 + (1 if cfg["out_norm"] else 0) - 1
            lib.LAUNCHES += sum(len(parts) for parts in self._plan.values())     # one expansion per compressed entry
            return NaDiTOutput(out)
        # the tables svr2_dit_forward uses, layer by layer, from the handle
        geo = [lib.dit_geometry(self.native_handle(), T, H, Wd, l, i) for i in range(cfg["layers"])]
        attn_flops = self._attn_flops((T, H, Wd, l), geo)
        st = lib.stream()

        # stem
        xp = torch.empty(L, self.K_IN_PAD, device=dev, dtype=torch.bfloat16)
        lib.call("svr2_patchify_bf16", lib.ptr(vid), lib.ptr(xp), T, H, Wd, cfg["in_ch"], self.K_IN_PAD, st)
        x = lib.linear(xp, W["vid_in.w"], bias=W["vid_in.b"])
        t = lib.linear(txt, W["txt_in.w"], bias=W["txt_in.b"])
        del xp

        max_total = max(g.total for g in geo)
        qb = torch.empty(max_total, heads, 128, device=dev, dtype=torch.bfloat16)
        kb, vb = torch.empty_like(qb), torch.empty_like(qb)
        max_rows = L + max(g.n_win for g in geo) * l
        o_all = torch.empty(max_rows, inner, device=dev, dtype=torch.bfloat16)
        o_t = torch.empty(l, inner, device=dev, dtype=torch.bfloat16)

        for i in range(cfg["layers"]):
            last = cfg["last_vid_only"] and i == cfg["layers"] - 1
            g = geo[i]
            Wb = self._expand_block(i)     # this block's compressed matrices, as bf16 in the staging tensor
            k = lambda s, n: Wb[f"{i}.{s}.{n}"] if f"{i}.{s}.{n}" in Wb else W[f"{i}.{s}.{n}"]
            m = lambda n: M[f"{i}.{n}"]
            # ---- attention branch
            a_v = lib.rmsnorm_ada(x, m("vid.attn_scale"), m("vid.attn_shift"), mode=0, eps=cfg["eps"])
            a_t = lib.rmsnorm_ada(t, m("txt.attn_scale"), m("txt.attn_shift"), mode=0, eps=cfg["eps"])
            qkv_t = lib.linear(a_t, k("txt", "qkv.w"))
            q, kk, v = qb[: g.total], kb[: g.total], vb[: g.total]
            rope_args = (g.rope_cos, g.rope_sin, g.nfreq)
            if g.fuse_qkv:
                # video rows: q/k RMSNorm + RoPE + window scatter inside the QKV GEMM's epilogue; text rows (the same
                # 58 rows appended to every window) by the row-subset form of the stand-alone kernel
                lib.call("svr2_linear_qkv_rope_bf16", lib.ptr(a_v), a_v.stride(0), lib.ptr(k("vid", "qkv.w")), d, L, heads, d,
                         g.tok_dst, g.tok_rope, *rope_args, lib.ptr(k("vid", "nqk")), cfg["eps"],
                         lib.ptr(q), lib.ptr(kk), lib.ptr(v), st, flops=2.0 * L * 3 * inner * d)
                lib.call("svr2_qk_norm_rope_rows_bf16", None, lib.ptr(qkv_t), g.row_src, g.row_rope, *rope_args,
                         lib.ptr(k("vid", "nq")), lib.ptr(k("vid", "nk")), lib.ptr(k("txt", "nq")), lib.ptr(k("txt", "nk")),
                         cfg["eps"], g.txt_rows, g.n_txt_rows, heads, lib.ptr(q), lib.ptr(kk), lib.ptr(v), st,
                         nbytes=12.0 * g.n_txt_rows * inner)
            else:
                qkv_v = lib.linear(a_v, k("vid", "qkv.w"))
                lib.call("svr2_qk_norm_rope_window_bf16", lib.ptr(qkv_v), lib.ptr(qkv_t), g.row_src, g.row_rope,
                         *rope_args, lib.ptr(k("vid", "nq")), lib.ptr(k("vid", "nk")), lib.ptr(k("txt", "nq")),
                         lib.ptr(k("txt", "nk")), cfg["eps"], g.total, heads, lib.ptr(q), lib.ptr(kk), lib.ptr(v), st,
                         nbytes=12.0 * g.total * inner)
                del qkv_v
            del a_v
            lib.call("svr2_attn_varlen_bf16", lib.ptr(q), lib.ptr(kk), lib.ptr(v), lib.ptr(o_all), g.cu_seqlens, g.n_win,
                     g.total, heads, g.max_len, g.out_row_map, st, flops=attn_flops[i % 2] * heads)
            lib.call("svr2_txt_window_mean_bf16", lib.ptr(o_all[L:]), lib.ptr(o_t), g.n_win, l, inner, st)
            h_v = lib.linear(o_all[:L], k("vid", "out.w"), bias=k("vid", "out.b"), gate=m("vid.attn_gate"), residual=x)
            h_t = lib.linear(o_t, k("txt", "out.w"), bias=k("txt", "out.b"),
                             gate=None if last else m("txt.attn_gate"), residual=t)
            # ---- MLP branch
            x = self._mlp(i, "vid", h_v, k)
            t = h_t if last else self._mlp(i, "txt", h_t, k)   # last layer: text output is unused downstream
            del h_v

        if cfg["out_norm"]:
            xo = lib.rmsnorm_ada(x, M["out_scale"], M["out_shift"], weight=M["out_weight"], mode=0, eps=cfg["eps"])
        else:
            xo = x
        v64 = lib.linear(xo, W["vid_out.w"], bias=W["vid_out.b"])
        out = torch.empty(T * H * Wd, cfg["out_ch"], device=dev, dtype=torch.bfloat16)
        lib.call("svr2_unpatchify_bf16", lib.ptr(v64), v64.stride(0), lib.ptr(out), T, H, Wd, cfg["out_ch"], st)
        return NaDiTOutput(out)

    def _expand_block(self, i: int) -> Dict[str, torch.Tensor]:
        """Block i's compressed matrices expanded to bf16 (svr2_weight_expand_bf16) into the staging tensor the module
        keeps, by name; the stream orders this after the previous block's GEMMs, which read the same tensor."""
        offsets = self._slot_offsets[i]
        if not offsets:
            return {}
        stage = self.__dict__.get("_stage")
        if stage is None:
            stage = self.__dict__["_stage"] = torch.empty(self.slot_bytes // 2, device=self.device, dtype=torch.bfloat16)
        out = {}
        for name, off in offsets.items():
            parts = self._plan[name]
            cols = parts[0].cols
            dst = stage[off // 2: off // 2 + sum(p.rows for p in parts) * cols].view(-1, cols)
            for part, suffix in zip(parts, ("",) if len(parts) == 1 else (".gate", ".in")):
                src = self.C[name + suffix]
                lib.call("svr2_weight_expand_bf16", part.format, lib.ptr(src), part.rows, cols, lib.ptr(dst),
                         part.row_group, part.group_stride, part.row_offset, lib.stream(),
                         nbytes=float(src.numel() + 2 * part.rows * cols))
            out[name] = dst
            if i >= self.cfg["mm_layers"]:      # shared weights: the text stream reads the same bytes
                out[name.replace(".vid.", ".txt.", 1)] = dst
        return out

    def _mlp(self, i, s, h, k):
        cfg, W, M = self.cfg, self.W, self.M
        mm = lib.rmsnorm_ada(h, M[f"{i}.{s}.mlp_scale"], M[f"{i}.{s}.mlp_shift"], mode=1, eps=cfg["eps"])
        if cfg["mlp"] == "swiglu":
            z = lib.linear(mm, k(s, "mlp_in.w"), epi=EPI_SWIGLU)
            return lib.linear(z, k(s, "mlp_out.w"), gate=M[f"{i}.{s}.mlp_gate"], residual=h)
        z = lib.linear(mm, k(s, "mlp_in.w"), bias=W[f"{i}.{s}.mlp_in.b"], epi=EPI_GELU)
        return lib.linear(z, k(s, "mlp_out.w"), bias=W[f"{i}.{s}.mlp_out.b"], gate=M[f"{i}.{s}.mlp_gate"],
                          residual=h)

