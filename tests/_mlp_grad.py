"""Float64 reference of the dense MLP backward (``FusedQuantMLP(fused_backward=True)``, ``agb200_w4a16_mlp_backward``).

A dense MLP ``down(silu(gate x) * up x)`` is the grouped experts' block with one expert, k = 1 and routing weight 1:
dy_pair = rnd(1 * dy) = dy and dx = rnd(dx_pair), so ``tests/_moe_grad.backward`` is the reference (same rounding points,
same magnitudes A and A2 for the error bound of ``tests/test_gpu_19_mlp_grad.py``).
"""
from __future__ import annotations

import numpy as np

from tests import _moe_grad as MG


def backward(x, gate, up, down, dy, dtype: str = "float16", rounded: bool = True, round_w_fwd: bool = True,
             cols=None) -> dict:
    """dx [M, H] (or its columns ``cols``), A and A2 in float64; gate / up / down are oracle layer dicts with the scales
    and bias the device uses.  ``rounded=False``: no intermediate rounding (the float64 value of the same model)."""
    M = np.asarray(x).shape[0]
    idx = np.zeros((M, 1), dtype=np.int64)
    w = np.ones((M, 1))
    return MG.backward(x, [dict(w1=gate, w3=up, w2=down)], idx, w, dy, dtype, rounded=rounded, round_w_fwd=round_w_fwd,
                       cols=cols)
