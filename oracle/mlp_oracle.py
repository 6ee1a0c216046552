"""CPU oracle of the fused gate/up of a dense MLP (``autogptq_b200.forward_gate_up``).  TEST INFRASTRUCTURE ONLY.

    h = round(round(silu(g)) * u),  g = round(x Wg + bg),  u = round(x Wu + bu)      (every round: to the activation dtype)

the reference's 16-bit ``act_fn(gate) * up`` (``auto_gptq/nn_modules/fused_llama_mlp.py:154-166``; transformers'
``LlamaMLP.forward``).  Built from ``moe_oracle``'s ``linear`` / ``silu`` / ``round_to``; a layer is a
``w4a16_oracle.random_packed`` dict.
"""
from __future__ import annotations

import numpy as np

from .moe_oracle import linear, round_to, silu


def gate_up(x, gate, up, dtype: str = "float16", weight_dtype: str | None = None) -> np.ndarray:
    """h for the rows of x as fp32 values of ``dtype``; ``weight_dtype`` as in ``moe_oracle.linear`` (None: exact
    weights, the arithmetic of the decode kernel; the dtype: weights rounded once, that of the tensor-core GEMM)."""
    g = round_to(linear(x, gate, weight_dtype), dtype)
    u = round_to(linear(x, up, weight_dtype), dtype)
    return round_to(round_to(silu(g), dtype) * u, dtype)
