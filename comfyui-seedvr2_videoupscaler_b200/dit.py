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

Python here does only: weight re-layout at load, integer window/RoPE index
bookkeeping (``window.py:28-83``, ``na.py:583-641``, ``rope.py:130-176``), buffer
allocation and kernel sequencing.  No torch op touches activations on the hot path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from math import ceil
from typing import Dict, List, Tuple

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
# window geometry (integer bookkeeping, host)
# --------------------------------------------------------------------------
def window_boxes(t: int, h: int, w: int, shifted: bool, num_windows=(4, 3, 3)) -> List[Tuple[int, ...]]:
    """Window boxes in the reference's enumeration order (w-major, then h, then t):
    make_720Pwindows_bysize / make_shifted_720Pwindows_bysize, dit_3b/window.py:28-83."""
    rnt, rnh, rnw = num_windows
    scale = math.sqrt((45 * 80) / (h * w))
    rh, rw = round(h * scale), round(w * scale)
    wh, ww = ceil(rh / rnh), ceil(rw / rnw)
    wt = ceil(min(t, 30) / rnt)
    if shifted:
        st, sh, sw = (0.5 if wt < t else 0, 0.5 if wh < h else 0, 0.5 if ww < w else 0)
        nt, nh, nw = ceil((t - st) / wt), ceil((h - sh) / wh), ceil((w - sw) / ww)
        nt, nh, nw = (nt + 1 if st > 0 else 1, nh + 1 if sh > 0 else 1, nw + 1 if sw > 0 else 1)

        def rng(i, s, win, ext):
            return max(int((i - s) * win), 0), min(int((i - s + 1) * win), ext)
    else:
        st = sh = sw = 0
        nt, nh, nw = ceil(t / wt), ceil(h / wh), ceil(w / ww)

        def rng(i, s, win, ext):
            return i * win, min((i + 1) * win, ext)
    out = []
    for iw in range(nw):
        w0, w1 = rng(iw, sw, ww, w)
        if w1 <= w0:
            continue
        for ih in range(nh):
            h0, h1 = rng(ih, sh, wh, h)
            if h1 <= h0:
                continue
            for it in range(nt):
                t0, t1 = rng(it, st, wt, t)
                if t1 <= t0:
                    continue
                out.append((t0, t1, h0, h1, w0, w1))
    return out


@dataclass
class WindowLayout:
    n_win: int
    total: int            # L + n_win * l rows in window order
    max_len: int
    cu_seqlens: torch.Tensor   # int32 [n_win+1]
    row_src: torch.Tensor      # int32 [total]   >=0 video token, <0 -(text idx + 1)
    row_rope: torch.Tensor     # int32 [total,3] rows of the cos/sin tables (or -1)
    out_row_map: torch.Tensor  # int32 [total]   video rows -> token idx, text rows -> L + w*l + j
    attn_flops: float = 0.0    # sum over windows of 4 * len^2 * 128 (per head)
    tok_dst: torch.Tensor = None    # int32 [L]    window-order row of every video token (inverse of row_src)
    tok_rope: torch.Tensor = None   # int32 [L,3]  row_rope in token order
    txt_rows: torch.Tensor = None   # int32 [n_win*l] window-order rows that hold text tokens


def build_layout(T: int, Hp: int, Wp: int, l: int, shifted: bool, variant: str, device) -> Tuple[WindowLayout, dict]:
    boxes = window_boxes(T, Hp, Wp, shifted)
    L = T * Hp * Wp
    grid = torch.arange(L, dtype=torch.int64).view(T, Hp, Wp)
    src, rope, omap, lens = [], [], [], []
    size_rows: Dict[int, int] = {}   # 7B: table offset for every distinct window-axis size
    if variant == "7b":
        off = 0
        for b in boxes:
            for n in (b[1] - b[0], b[3] - b[2], b[5] - b[4]):
                if n not in size_rows:
                    size_rows[n] = off
                    off += n
    tj = torch.arange(l, dtype=torch.int64)
    for wi, (t0, t1, h0, h1, w0, w1) in enumerate(boxes):
        sub = grid[t0:t1, h0:h1, w0:w1].reshape(-1)
        tt, hh, ww_ = torch.meshgrid(torch.arange(t1 - t0), torch.arange(h1 - h0), torch.arange(w1 - w0),
                                     indexing="ij")
        if variant == "3b":   # rope.py:172-173: video (t + l, h, w) window-local; text (j, j, j)
            r_v = torch.stack([tt.reshape(-1) + l, hh.reshape(-1), ww_.reshape(-1)], -1)
            r_t = torch.stack([tj, tj, tj], -1)
        else:                 # dit_7b/rope.py:73-111: video only
            r_v = torch.stack([tt.reshape(-1) + size_rows[t1 - t0], hh.reshape(-1) + size_rows[h1 - h0],
                               ww_.reshape(-1) + size_rows[w1 - w0]], -1)
            r_t = torch.full((l, 3), -1, dtype=torch.int64)
        src += [sub, -(tj + 1)]
        rope += [r_v, r_t]
        omap += [sub, L + wi * l + tj]
        lens.append(sub.numel() + l)
    lens_t = torch.tensor(lens, dtype=torch.int64)
    cu = torch.zeros(len(lens) + 1, dtype=torch.int32)
    cu[1:] = lens_t.cumsum(0).int()
    src_all, rope_all = torch.cat(src), torch.cat(rope)
    rows = torch.arange(src_all.numel())
    is_vid = src_all >= 0
    tok_dst = torch.empty(L, dtype=torch.int64)
    tok_dst[src_all[is_vid]] = rows[is_vid]                  # the windows partition the tokens: a bijection
    tok_rope = torch.empty(L, 3, dtype=torch.int64)
    tok_rope[src_all[is_vid]] = rope_all[is_vid]
    lay = WindowLayout(
        n_win=len(boxes), total=int(lens_t.sum()), max_len=int(lens_t.max()),
        cu_seqlens=cu.to(device), row_src=torch.cat(src).int().to(device),
        row_rope=torch.cat(rope).int().contiguous().to(device), out_row_map=torch.cat(omap).int().to(device),
        attn_flops=float((lens_t.double() ** 2).sum()) * 4 * 128,
        tok_dst=tok_dst.int().to(device), tok_rope=tok_rope.int().contiguous().to(device),
        txt_rows=rows[~is_vid].int().to(device))
    return lay, size_rows


def rope_tables(freqs: torch.Tensor, variant: str, npos: int, size_rows: Dict[int, int]):
    """cos/sin tables [R, nfreq] fp32, evaluated the way rotary_embedding_torch does:
    angle = pos.type(freqs.dtype) * freqs, cos/sin in that dtype (SURVEY.md §8 G4)."""
    f = freqs.detach().cpu()
    if variant == "3b":
        pos = torch.arange(npos).type(f.dtype)
    else:
        rows = max((o + n for n, o in size_rows.items()), default=0)
        pos = torch.zeros(rows, dtype=f.dtype)
        for n, o in size_rows.items():
            pos[o:o + n] = torch.linspace(-1, 1, steps=n).type(f.dtype)
    ang = torch.einsum("p,f->pf", pos, f)
    return ang.cos().float().contiguous(), ang.sin().float().contiguous()


# --------------------------------------------------------------------------
# the engine
# --------------------------------------------------------------------------
class NaDiTOutput:
    def __init__(self, vid_sample):
        self.vid_sample = vid_sample


class B200NaDiT(EngineModule):
    """Drop-in for the reference ``runner.dit`` (VideoDiffusionInfer model slot, infer.py:361-367): an ``nn.Module``
    whose weights are buffers in the kernels' layout (see ``module.EngineModule`` for the lifecycle it survives) and
    which holds one ``FlashAttentionVarlen`` submodule, the class ``apply_model_specific_config`` looks for."""

    K_IN_PAD = 192  # 4*33 = 132 patch channels padded to 3 k-blocks of 64

    def __init__(self, cfg: dict, state_dict: Dict[str, torch.Tensor], device="cuda", timestep: float = 1000.0):
        super().__init__(device)
        lib.device_check()
        self.cfg = cfg
        self.timestep = timestep
        self._layouts: Dict[tuple, tuple] = {}
        self.attention = FlashAttentionVarlen()
        self._load(state_dict)
        # the fused QKV epilogue needs 256-column tiles to be whole head pairs and one of the two shipped RoPE widths
        # (the same rule as fuse_qkv_ok in csrc/engine.cu)
        self.fuse_qkv = cfg["heads"] % 2 == 0 and self.rope_freqs[0].numel() in (21, 10)
        # forward sequenced by the native runtime (default) or by this module's Python loop (per-call profiling, tests
        # against the native runtime)
        self.native = True

    def _device_state_moved(self):
        if hasattr(self, "_layouts"):
            self._layouts.clear()      # window / RoPE tables live on the old device
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
        its workspace; rebuilt after a device move."""
        if self.__dict__.get("_handle"):
            return self._handle
        cfg = self.cfg
        mlp_hidden = (self.W["0.vid.mlp_in.w"].shape[0] // 2) if cfg["mlp"] == "swiglu" else self.W["0.vid.mlp_in.w"].shape[0]
        desc = lib.ModelDesc(variant=0 if cfg["variant"] == "3b" else 1, dim=cfg["dim"], heads=cfg["heads"],
                             layers=cfg["layers"], mm_layers=cfg["mm_layers"], txt_in_dim=cfg["txt_in_dim"],
                             in_ch=cfg["in_ch"], out_ch=cfg["out_ch"], mlp_kind=0 if cfg["mlp"] == "swiglu" else 1,
                             mlp_hidden=mlp_hidden, out_norm=int(cfg["out_norm"]), last_vid_only=int(cfg["last_vid_only"]),
                             eps=cfg["eps"], timestep=self.timestep)
        h = lib.engine_create(desc, self.device.index if self.device.index is not None else torch.cuda.current_device())
        try:
            lib.engine_load(h, {k: self.W[k] for k in self.W.keys()}, copy=False)
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

    def _load(self, sd):
        sd = weights.dequantizing(sd, self.device)   # GGUF entries: dense fp16 on the device, one key at a time
        cfg, dev = self.cfg, self.device
        d = cfg["dim"]
        W: Dict[str, torch.Tensor] = {}
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
                    continue
                W[f"{i}.{s}.qkv.w"] = self._w(sd, p + f"attn.proj_qkv.{key}.weight")
                W[f"{i}.{s}.out.w"] = self._w(sd, p + f"attn.proj_out.{key}.weight")
                W[f"{i}.{s}.out.b"] = self._w(sd, p + f"attn.proj_out.{key}.bias")
                W[f"{i}.{s}.nq"] = self._f(sd, p + f"attn.norm_q.{key}.weight")
                W[f"{i}.{s}.nk"] = self._f(sd, p + f"attn.norm_k.{key}.weight")
                W[f"{i}.{s}.nqk"] = torch.cat([W[f"{i}.{s}.nq"], W[f"{i}.{s}.nk"]]).contiguous()   # [2][128]
                if last and s == "txt":
                    continue
                if cfg["mlp"] == "swiglu":
                    g = sd[p + f"mlp.{key}.proj_in_gate.weight"].to(dev, torch.bfloat16)
                    u = sd[p + f"mlp.{key}.proj_in.weight"].to(dev, torch.bfloat16)
                    hid = g.shape[0]
                    assert hid % 128 == 0
                    # interleave 128-row groups: tile j of 256 rows = [gate_j ; in_j]  (EPI_SWIGLU)
                    il = torch.stack([g.view(hid // 128, 128, d), u.view(hid // 128, 128, d)], 1)
                    W[f"{i}.{s}.mlp_in.w"] = il.reshape(2 * hid, d).contiguous()
                    W[f"{i}.{s}.mlp_out.w"] = self._w(sd, p + f"mlp.{key}.proj_out.weight")
                else:
                    W[f"{i}.{s}.mlp_in.w"] = self._w(sd, p + f"mlp.{key}.proj_in.weight")
                    W[f"{i}.{s}.mlp_in.b"] = self._w(sd, p + f"mlp.{key}.proj_in.bias")
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

    # ---- geometry cache ----------------------------------------------------
    def _geometry(self, T, Hp, Wp, l):
        key = (T, Hp, Wp, l)
        if key not in self._layouts:
            variant = self.cfg["variant"]
            lays, tabs = [], {}
            for shifted in (False, True):
                lay, size_rows = build_layout(T, Hp, Wp, l, shifted, variant, self.device)
                lays.append((lay, size_rows))
            tables = []
            for i in range(self.cfg["layers"]):
                lay, size_rows = lays[i % 2]
                fr = self.rope_freqs[i]
                tk = (i % 2, fr.dtype, tuple(fr.tolist()))
                if tk not in tabs:
                    npos = int(lay.row_rope.max().item()) + 1
                    c, s = rope_tables(fr, variant, npos, size_rows)
                    tabs[tk] = (c.to(self.device), s.to(self.device))
                tables.append(tabs[tk])
            self._layouts[key] = ([x[0] for x in lays], tables)
        return self._layouts[key]

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
            return NaDiTOutput(out)
        layouts, tables = self._geometry(T, Hp, Wp, l)
        st = lib.stream()

        # stem
        xp = torch.empty(L, self.K_IN_PAD, device=dev, dtype=torch.bfloat16)
        lib.call("svr2_patchify_bf16", lib.ptr(vid), lib.ptr(xp), T, H, Wd, cfg["in_ch"], self.K_IN_PAD, st)
        x = lib.linear(xp, W["vid_in.w"], bias=W["vid_in.b"])
        t = lib.linear(txt, W["txt_in.w"], bias=W["txt_in.b"])
        del xp

        max_total = max(lay.total for lay in layouts)
        qb = torch.empty(max_total, heads, 128, device=dev, dtype=torch.bfloat16)
        kb, vb = torch.empty_like(qb), torch.empty_like(qb)
        max_rows = L + max(lay.n_win for lay in layouts) * l
        o_all = torch.empty(max_rows, inner, device=dev, dtype=torch.bfloat16)
        o_t = torch.empty(l, inner, device=dev, dtype=torch.bfloat16)
        nfreq = tables[0][0].shape[1]

        for i in range(cfg["layers"]):
            last = cfg["last_vid_only"] and i == cfg["layers"] - 1
            lay = layouts[i % 2]
            cos_t, sin_t = tables[i]
            k = lambda s, n: W[f"{i}.{s}.{n}"]
            m = lambda n: M[f"{i}.{n}"]
            # ---- attention branch
            a_v = lib.rmsnorm_ada(x, m("vid.attn_scale"), m("vid.attn_shift"), mode=0, eps=cfg["eps"])
            a_t = lib.rmsnorm_ada(t, m("txt.attn_scale"), m("txt.attn_shift"), mode=0, eps=cfg["eps"])
            qkv_t = lib.linear(a_t, k("txt", "qkv.w"))
            q, kk, v = qb[: lay.total], kb[: lay.total], vb[: lay.total]
            rope_args = (lib.ptr(cos_t), lib.ptr(sin_t), nfreq)
            if self.fuse_qkv:
                # video rows: q/k RMSNorm + RoPE + window scatter inside the QKV GEMM's epilogue; text rows (the same
                # 58 rows appended to every window) by the row-subset form of the stand-alone kernel
                lib.call("svr2_linear_qkv_rope_bf16", lib.ptr(a_v), a_v.stride(0), lib.ptr(k("vid", "qkv.w")), d, L, heads, d,
                         lib.ptr(lay.tok_dst), lib.ptr(lay.tok_rope), *rope_args, lib.ptr(k("vid", "nqk")), cfg["eps"],
                         lib.ptr(q), lib.ptr(kk), lib.ptr(v), st, flops=2.0 * L * 3 * inner * d)
                lib.call("svr2_qk_norm_rope_rows_bf16", None, lib.ptr(qkv_t), lib.ptr(lay.row_src), lib.ptr(lay.row_rope),
                         *rope_args, lib.ptr(k("vid", "nq")), lib.ptr(k("vid", "nk")), lib.ptr(k("txt", "nq")),
                         lib.ptr(k("txt", "nk")), cfg["eps"], lib.ptr(lay.txt_rows), lay.txt_rows.numel(), heads,
                         lib.ptr(q), lib.ptr(kk), lib.ptr(v), st, nbytes=12.0 * lay.txt_rows.numel() * inner)
            else:
                qkv_v = lib.linear(a_v, k("vid", "qkv.w"))
                lib.call("svr2_qk_norm_rope_window_bf16", lib.ptr(qkv_v), lib.ptr(qkv_t), lib.ptr(lay.row_src),
                         lib.ptr(lay.row_rope), *rope_args, lib.ptr(k("vid", "nq")),
                         lib.ptr(k("vid", "nk")), lib.ptr(k("txt", "nq")), lib.ptr(k("txt", "nk")), cfg["eps"],
                         lay.total, heads, lib.ptr(q), lib.ptr(kk), lib.ptr(v), st, nbytes=12.0 * lay.total * inner)
                del qkv_v
            del a_v
            o_view = o_all.view(-1, heads, 128)
            self.attention.run(q, kk, v, lay.cu_seqlens, lay.max_len, out=o_view, out_row_map=lay.out_row_map,
                               flops=lay.attn_flops * heads)
            lib.call("svr2_txt_window_mean_bf16", lib.ptr(o_all[L:]), lib.ptr(o_t), lay.n_win, l, inner, st)
            h_v = lib.linear(o_all[:L], k("vid", "out.w"), bias=k("vid", "out.b"), gate=m("vid.attn_gate"), residual=x)
            h_t = lib.linear(o_t, k("txt", "out.w"), bias=k("txt", "out.b"),
                             gate=None if last else m("txt.attn_gate"), residual=t)
            # ---- MLP branch
            x = self._mlp(i, "vid", h_v)
            t = h_t if last else self._mlp(i, "txt", h_t)   # last layer: text output is unused downstream
            del h_v

        if cfg["out_norm"]:
            xo = lib.rmsnorm_ada(x, M["out_scale"], M["out_shift"], weight=M["out_weight"], mode=0, eps=cfg["eps"])
        else:
            xo = x
        v64 = lib.linear(xo, W["vid_out.w"], bias=W["vid_out.b"])
        out = torch.empty(T * H * Wd, cfg["out_ch"], device=dev, dtype=torch.bfloat16)
        lib.call("svr2_unpatchify_bf16", lib.ptr(v64), v64.stride(0), lib.ptr(out), T, H, Wd, cfg["out_ch"], st)
        return NaDiTOutput(out)

    def _mlp(self, i, s, h):
        cfg, W, M = self.cfg, self.W, self.M
        mm = lib.rmsnorm_ada(h, M[f"{i}.{s}.mlp_scale"], M[f"{i}.{s}.mlp_shift"], mode=1, eps=cfg["eps"])
        if cfg["mlp"] == "swiglu":
            z = lib.linear(mm, W[f"{i}.{s}.mlp_in.w"], epi=EPI_SWIGLU)
            return lib.linear(z, W[f"{i}.{s}.mlp_out.w"], gate=M[f"{i}.{s}.mlp_gate"], residual=h)
        z = lib.linear(mm, W[f"{i}.{s}.mlp_in.w"], bias=W[f"{i}.{s}.mlp_in.b"], epi=EPI_GELU)
        return lib.linear(z, W[f"{i}.{s}.mlp_out.w"], bias=W[f"{i}.{s}.mlp_out.b"], gate=M[f"{i}.{s}.mlp_gate"],
                          residual=h)

