"""CPU oracle of the grouped mixture-of-experts forward (``autogptq_b200.QuantExperts``).  TEST INFRASTRUCTURE ONLY.

NumPy restatement of transformers' ``MixtralExperts.forward`` (``transformers/models/mixtral/modeling_mixtral.py:74-98``)
over 4-bit GPTQ experts (``auto_gptq/modeling/mixtral.py:4-39``):

    out[t] = sum_{j < k, 0 <= e_j < E} w[t, j] * W2_{e_j}( silu(W1_{e_j} x[t]) * W3_{e_j} x[t] ),  e_j = top_k_index[t, j]

Every projection is ``w4a16_oracle.forward`` in exact fp32 (plus bias; ``weight_dtype`` rounds the dequantised weights
to the dtype instead, the arithmetic of the tensor-core path); g, u, silu(g), h and the per-pair output are
rounded to the activation dtype where the reference's 16-bit tensors round them (``act_fn(gate) * up``, the
QuantLinear outputs); the weighted sum over the slots is fp32 with no rounding (callers compare against it with a
tolerance).  An id outside ``[0, E)`` contributes nothing (the ``expert_idx == num_experts`` skip, :88).

An expert is a dict ``{"w1": layer, "w3": layer, "w2": layer}``; a layer is a ``w4a16_oracle.random_packed`` dict
(``qweight``, ``qzeros``, ``scales``, ``g_idx``, ``group_size``, ``bias`` or None).
"""
from __future__ import annotations

import numpy as np

from . import w4a16_oracle as O


def round_to(a, dtype: str) -> np.ndarray:
    """Round fp32 values to fp16 or bf16 (round to nearest even) and return them as fp32."""
    a = np.asarray(a, dtype=np.float32)
    if dtype == "float16":
        return a.astype(np.float16).astype(np.float32)
    if dtype == "bfloat16":
        u = a.view(np.uint32).astype(np.uint64)
        r = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
        return r.view(np.float32)
    raise ValueError(f"dtype must be 'float16' or 'bfloat16' (got {dtype!r})")


def linear(x, layer, weight_dtype: str | None = None) -> np.ndarray:
    """x @ dequant(layer) (+ bias) in fp32, unrounded.  ``weight_dtype=None``: exact weights; "float16" / "bfloat16":
    every weight s * (q - z) rounded once to that dtype, as the tensor-core path (and the reference's fp16
    ``reconstruct``) forms it."""
    if weight_dtype is None:
        y = O.forward(np.asarray(x, dtype=np.float32), layer["qweight"], layer["qzeros"], layer["scales"],
                      g_idx=layer["g_idx"], group_size=layer["group_size"], out_dtype=np.float32)
    else:
        W = round_to(O.dequantize(layer["qweight"], layer["qzeros"], layer["scales"], g_idx=layer["g_idx"],
                                  group_size=layer["group_size"], dtype=np.float32), weight_dtype)
        y = np.asarray(x, dtype=np.float32) @ W
    if layer.get("bias") is not None:
        y = y + np.asarray(layer["bias"], dtype=np.float32)
    return y


def silu(a):
    a = np.asarray(a, dtype=np.float32)
    return a / (np.float32(1.0) + np.exp(-a))


def expert_mlp(x, expert, dtype: str = "float16", weight_dtype: str | None = None) -> np.ndarray:
    """w2(silu(w1 x) * w3 x) for the rows of x, with the 16-bit roundings of the reference; returns the rounded output."""
    g = round_to(linear(x, expert["w1"], weight_dtype), dtype)
    u = round_to(linear(x, expert["w3"], weight_dtype), dtype)
    h = round_to(round_to(silu(g), dtype) * u, dtype)
    return round_to(linear(h, expert["w2"], weight_dtype), dtype)


def forward(x, experts, top_k_index, top_k_weights, dtype: str = "float16", weight_dtype: str | None = None,
            return_magnitude: bool = False):
    """out [T, N2] as fp32 (see the module docstring; N2 = the output width of w2, H unless w2 is a column slice).
    ``x`` holds values of ``dtype``; ``top_k_weights`` is used as given (pass the values the device sees).
    ``return_magnitude``: also return sum_j |w[t, j] * y_pair[t, j]|, the scale of the per-pair outputs that the
    reference rounds to the dtype before the weighted sum (a last-bit difference there is one ulp of that scale)."""
    x = np.asarray(x, dtype=np.float32)
    idx = np.asarray(top_k_index).astype(np.int64)
    w = np.asarray(top_k_weights, dtype=np.float32)
    T = x.shape[0]
    E = len(experts)
    N2 = np.asarray(experts[0]["w2"]["qweight"]).shape[1]
    y_pair = np.zeros(idx.shape + (N2,), dtype=np.float32)
    for e in range(E):
        tok, slot = np.nonzero(idx == e)
        if tok.size:
            y_pair[tok, slot] = expert_mlp(x[tok], experts[e], dtype, weight_dtype)
    out = np.zeros((T, N2), dtype=np.float32)
    mag = np.zeros((T, N2), dtype=np.float32)
    for j in range(idx.shape[1]):                      # slot order, fp32
        valid = (idx[:, j] >= 0) & (idx[:, j] < E)
        term = np.where(valid[:, None], w[:, j, None] * y_pair[:, j], np.float32(0))
        out += term
        mag += np.abs(term)
    return (out, mag) if return_magnitude else out


def active_bytes(top_k_index, E: int, H: int, I: int, group_size: int, desc_act: bool = False) -> int:
    """Algorithmic bytes of one call: the three layers of every hit expert by the per-layer formula
    (``w4a16_oracle.algorithmic_bytes``, M = that expert's rows) plus the routing inputs."""
    idx = np.asarray(top_k_index).astype(np.int64)
    total = idx.size * (idx.itemsize + 4)
    for e in range(E):
        m = int((idx == e).sum())
        if m:
            total += 2 * O.algorithmic_bytes(m, H, I, group_size, desc_act) + O.algorithmic_bytes(m, I, H, group_size, desc_act)
    return total
