"""TEST INFRASTRUCTURE ONLY — the expansion of a stored weight matrix to bf16 in the engine layout
(``svr2_weight_expand_bf16``) restated in torch.

A GGUF matrix is the fp16 restatement of the reference's block functions (``gguf_oracle.dequantize_tensor``) cast to
bfloat16, an fp8_e4m3fn or fp16 matrix is torch's cast to bfloat16: what the load-time path of ``B200NaDiT`` builds.
``place`` writes the rows of one source matrix into the destination by the kernel's row map; the SwiGLU input matrix is
two of them (``swiglu_matrix``).
"""
from __future__ import annotations

import torch

from oracle import gguf_oracle as go

FMT_F16, FMT_F8_E4M3, FMT_GGML = 2, 3, 16      # the svr2_tensor_desc dtype codes of include/svr2.h


def stored_bytes(fmt: int, rows: int, cols: int) -> int:
    if fmt >= FMT_GGML:
        _, be, bb = go.TYPES[go.BY_ID[fmt - FMT_GGML]]
        return rows * cols // be * bb
    return rows * cols * (2 if fmt == FMT_F16 else 1)


def expand(fmt: int, raw: torch.Tensor, rows: int, cols: int) -> torch.Tensor:
    """raw: the matrix as stored (uint8, any device) -> [rows, cols] bfloat16."""
    raw = raw.reshape(-1)
    assert raw.dtype == torch.uint8 and raw.numel() == stored_bytes(fmt, rows, cols)
    if fmt >= FMT_GGML:
        return go.dequantize_tensor(fmt - FMT_GGML, raw, (rows, cols)).to(torch.bfloat16)
    dtype = torch.float16 if fmt == FMT_F16 else torch.float8_e4m3fn
    return raw.view(dtype).reshape(rows, cols).to(torch.bfloat16)


def row_map(rows: int, row_group: int, group_stride: int, row_offset: int) -> torch.Tensor:
    """Destination row of every source row: (r // row_group) * group_stride + row_offset + r % row_group."""
    r = torch.arange(rows)
    return (r // row_group) * group_stride + row_offset + r % row_group


def place(dst: torch.Tensor, mat: torch.Tensor, row_group: int, group_stride: int, row_offset: int) -> torch.Tensor:
    dst[row_map(mat.shape[0], row_group, group_stride, row_offset).to(dst.device)] = mat
    return dst


def swiglu_matrix(gate: torch.Tensor, proj_in: torch.Tensor) -> torch.Tensor:
    """[gate_j ; in_j] per 128 rows, by the row maps (128, 256, 0) and (128, 256, 128)."""
    dst = torch.empty(2 * gate.shape[0], gate.shape[1], dtype=gate.dtype, device=gate.device)
    place(dst, gate, 128, 256, 0)
    return place(dst, proj_in, 128, 256, 128)
