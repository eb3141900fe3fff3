"""The literal ``attention_mode`` seam: a drop-in for the reference's
``FlashAttentionVarlen`` (``src/models/dit_3b/attention.py:77-148``) backed by the
wgmma kernel ``svr2_attn_varlen_bf16`` — same call signature, same packed
(total, heads, 128) layout, same int32 cu_seqlens, returns compute-dtype output.

A maintainer registers it as ``attention_mode="b200"`` (see INTEGRATION.md); unlike
the reference's dispatch there is no fallback chain: unsupported inputs raise.
"""
from __future__ import annotations

import torch
from torch import nn

from . import lib


class FlashAttentionVarlen(nn.Module):
    """Named like the reference class on purpose: ``apply_model_specific_config`` finds its attention modules by
    ``type(module).__name__ == 'FlashAttentionVarlen'`` and sets ``attention_mode`` / ``compute_dtype`` on them
    (``model_configuration.py:1206-1210``).  ``attention_mode`` is accepted and recorded but does not select a backend:
    this module has exactly one (``svr2_attn_varlen_bf16``)."""

    def __init__(self, attention_mode: str = "b200", compute_dtype: torch.dtype = torch.bfloat16):
        super().__init__()
        self.attention_mode = attention_mode
        self.compute_dtype = compute_dtype

    def forward(self, q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, **kwargs):
        if q.shape[-1] != 128:
            raise lib.Svr2Error("b200 attention supports head_dim 128 only")
        if cu_seqlens_q is not cu_seqlens_k and not torch.equal(cu_seqlens_q, cu_seqlens_k):
            raise lib.Svr2Error("b200 attention is self-attention: cu_seqlens_q must equal cu_seqlens_k")
        q, k, v = (t.to(torch.bfloat16).contiguous() for t in (q, k, v))
        cu = cu_seqlens_q.to(torch.int32)
        out = lib.attn_varlen(q, k, v, cu, int(max_seqlen_q))
        return out if self.compute_dtype in (None, torch.bfloat16) else out.to(self.compute_dtype)


B200FlashAttentionVarlen = FlashAttentionVarlen
