"""AWQ "GEMM" packed layers -> the GPTQ pack layout.  Host-side, pure integer tensor ops (CPU or CUDA tensors).

AutoAWQ's GEMM checkpoints store the same 4-bit weights as GPTQ (``W = s·(q − z)``, sequential groups, no ``g_idx``) in a
different place:

* ``qweight`` int32 ``[K, N/8]`` is packed along N: nibble ``i`` of word ``[k, c]`` holds column ``8c + order[i]``,
  ``order = [0, 2, 4, 6, 1, 3, 5, 7]`` (the reference inverts it in ``awq_reverse_reorder_int_tensor``,
  ``modeling/_utils.py:525-547``);
* ``qzeros`` int32 ``[G, N/8]`` is packed the same way and holds ``z`` itself;
* ``scales`` fp16 ``[G, N]`` is laid out as in GPTQ.

GPTQ packs ``qweight`` along K (nibble ``k & 7`` of word ``[k/8, n]``) and stores ``(z − 1) & 0xF``, which every kernel
reads back with the wrap rule ``(stored + 1) & 0xF`` - so each ``z`` in ``[0, 15]`` survives, 0 included.  The rewrite
is exact: the reference instead dequantises to fp16 and re-quantises column by column (``_utils.py:550-701``).
"""
from __future__ import annotations

from typing import Tuple

import torch

# AWQ nibble that holds column 8c + j of a word (the inverse of AutoAWQ's order [0, 2, 4, 6, 1, 3, 5, 7])
_AWQ_NIBBLE_OF_COLUMN = (0, 4, 1, 5, 2, 6, 3, 7)


def _check_awq_shapes(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor) -> None:
    for name, t in (("qweight", qweight), ("qzeros", qzeros)):
        if t.dtype != torch.int32 or t.dim() != 2:
            raise ValueError(f"AWQ {name} must be a 2-D int32 tensor, got {t.dtype} {tuple(t.shape)}")
    if scales.dim() != 2:
        raise ValueError(f"AWQ scales must be 2-D, got {tuple(scales.shape)}")
    K, C = qweight.shape
    G, N = scales.shape
    if N != 8 * C:
        hint = ""
        if N == C:
            hint = (" - these are the shapes of a GPTQ layer (qweight [K/8, N], packed along K): load it with "
                    "checkpoint_format='gptq'")
        raise ValueError(f"AWQ GEMM layer needs scales.shape[1] == 8 * qweight.shape[1] (qweight [K, N/8]); got qweight "
                         f"{tuple(qweight.shape)}, scales {tuple(scales.shape)}{hint}")
    if tuple(qzeros.shape) != (G, C):
        raise ValueError(f"AWQ qzeros must be [G, N/8] = {(G, C)}, got {tuple(qzeros.shape)}")
    if K % 8 != 0:
        raise ValueError(f"AWQ layer has K = {K} input features; the GPTQ layout needs a multiple of 8")


def awq_to_gptq(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """AWQ GEMM ``(qweight [K, N/8], qzeros [G, N/8])`` -> GPTQ ``(qweight [K/8, N], qzeros [G, N/8])``, bit for bit.

    ``scales`` ``[G, N]`` is only checked (both layouts share it); the sequential ``g_idx = arange(K) // group_size``
    goes with the result.  Runs on the device of the inputs.  Malformed shapes raise ``ValueError``."""
    _check_awq_shapes(qweight, qzeros, scales)
    K, C = qweight.shape
    shifts = 4 * torch.tensor(_AWQ_NIBBLE_OF_COLUMN, dtype=torch.int32, device=qweight.device)
    # word [r, c, j] of the result is column 8c + j of rows 8r..8r+7: one nibble from each of the eight AWQ rows
    rows = qweight.reshape(K // 8, 8, C)
    out = torch.zeros((K // 8, C, 8), dtype=torch.int32, device=qweight.device)
    for i in range(8):
        t = rows[:, i, :, None] >> shifts                               # one temporary per row, updated in place
        t &= 0xF
        t <<= 4 * i
        out |= t
    z = (((qzeros[:, :, None] >> shifts) & 0xF) - 1) & 0xF              # [G, N/8, 8]: z - 1 of column 8c + j
    zeros = torch.zeros(qzeros.shape, dtype=torch.int32, device=qzeros.device)
    for j in range(8):
        zeros |= z[:, :, j] << (4 * j)
    return out.reshape(K // 8, 8 * C), zeros


__all__ = ["awq_to_gptq"]
