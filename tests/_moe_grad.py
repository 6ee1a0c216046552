"""Float64 reference of the grouped experts' backward (``QuantExperts(input_grad=True)``, ``agb200_moe_backward``).

For ``out[t] = sum_j w[t, j] * W2_e(silu(W1_e x[t]) * W3_e x[t])``, e = top_k_index[t, j], with the expert weights frozen:

    quantity    definition ("rnd": rounding to the activation dtype; skipped with ``rounded=False``)
    g, u        rnd(x W1 + b1), rnd(x W3 + b3)                         (what the forward saved)
    y_pair      rnd(rnd(rnd(silu(g)) * u) W2 + b2)                      (what the forward saved)
    dw[t, j]    sum_n dy[t, n] y_pair[t*k + j, n], rounded to w's dtype when w is 16-bit; 0 for ids outside [0, E)
    dy_pair     rnd(w[t, j] * dy[t])
    dh          dy_pair W2^T, unrounded
    dg, du      rnd(dh * u * silu'(g)), rnd(dh * rnd(silu(g))),  silu'(g) = s(g) (1 + g (1 - s(g)))
    dx_pair     dg W1^T + du W3^T, unrounded
    dx[t]       rnd(sum_j dx_pair[t*k + j]) over the valid slots

W = s * (q - z) is rounded once to the dtype in the backward (the tensor-core dgrad rule) and in the forward of the GEMM
path (T > 8); the decode path's forward uses the exact weights (``round_w_fwd``).  Besides the values, ``backward``
returns the uncancelled magnitudes the error bound of ``tests/test_gpu_18_moe_grad.py`` is built from.
"""
from __future__ import annotations

import numpy as np

from oracle import w4a16_oracle as O
from tests._precision import round_dt


def dequant(layer, dtype, round_w: bool) -> np.ndarray:
    W = O.dequantize(layer["qweight"], layer["qzeros"], layer["scales"], g_idx=layer["g_idx"],
                     group_size=layer["group_size"], dtype=np.float32).astype(np.float64)
    return round_dt(W, dtype) if round_w else W


def _bias(layer, n):
    b = layer.get("bias")
    return np.zeros(n) if b is None else np.asarray(b, dtype=np.float64)


def backward(x, experts, top_k_index, top_k_weights, dy, dtype: str = "float16", rounded: bool = True,
             round_w_fwd: bool = True, w16: bool = False, cols=None) -> dict:
    """dx [T, H] (or its columns ``cols``) and dw [T, k] in float64 (see the module docstring), with
    ``A`` = sum_j (|dg| |W1|^T + |du| |W3|^T), ``A2`` = sum_j ((A_dh |u silu'(g)|) |W1|^T + (A_dh |rnd(silu(g))|) |W3|^T),
    A_dh = |dy_pair| |W2|^T, and ``A_dw`` = sum_n |dy y_pair|.  ``w16``: top_k_weights are 16-bit (dw is rounded)."""
    rnd = (lambda a: round_dt(a, dtype)) if rounded else (lambda a: a)
    x = np.asarray(x, dtype=np.float64)
    dy = np.asarray(dy, dtype=np.float64)
    idx = np.asarray(top_k_index).astype(np.int64)
    w = np.asarray(top_k_weights, dtype=np.float64)
    T, H = x.shape
    k = idx.shape[1]
    E = len(experts)
    cols = np.arange(H) if cols is None else np.asarray(cols)
    dx_pair = np.zeros((T, k, len(cols)))
    A = np.zeros((T, len(cols)))
    A2 = np.zeros((T, len(cols)))
    dw = np.zeros((T, k))
    A_dw = np.zeros((T, k))
    for e in range(E):
        tok, slot = np.nonzero(idx == e)
        if not tok.size:
            continue
        ex = experts[e]
        I = np.asarray(ex["w1"]["qweight"]).shape[1]
        W1f, W3f, W2f = (dequant(ex[n], dtype, False) for n in ("w1", "w3", "w2"))
        W1, W3, W2 = (round_dt(W, dtype) for W in (W1f, W3f, W2f))
        if round_w_fwd:
            W1f, W3f, W2f = W1, W3, W2
        xe = x[tok]
        g = rnd(xe @ W1f + _bias(ex["w1"], I))
        u = rnd(xe @ W3f + _bias(ex["w3"], I))
        sg = rnd(g / (1 + np.exp(-g)))
        y = rnd(rnd(sg * u) @ W2f + _bias(ex["w2"], H))
        dyt = dy[tok]
        dw[tok, slot] = (dyt * y).sum(axis=1)
        A_dw[tok, slot] = np.abs(dyt * y).sum(axis=1)
        dyp = rnd(w[tok, slot, None] * dyt)
        dh = dyp @ W2.T
        adh = np.abs(dyp) @ np.abs(W2).T
        sig = 1 / (1 + np.exp(-g))
        sp = sig * (1 + g * (1 - sig))
        dg = rnd(dh * u * sp)
        du = rnd(dh * sg)
        W1c, W3c = W1[cols], W3[cols]
        dx_pair[tok, slot] = dg @ W1c.T + du @ W3c.T
        np.add.at(A, tok, np.abs(dg) @ np.abs(W1c).T + np.abs(du) @ np.abs(W3c).T)
        np.add.at(A2, tok, (adh * np.abs(u * sp)) @ np.abs(W1c).T + (adh * np.abs(sg)) @ np.abs(W3c).T)
    dx = rnd(dx_pair.sum(axis=1))
    if w16:
        dw = rnd(dw)
    return dict(dx=dx, dw=dw, A=A, A2=A2, A_dw=A_dw)
