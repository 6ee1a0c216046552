"""Float64 reference of the per-row decode attention (``agb200_decode_attention_rows``): each row is the one-row problem
of ``tests/_attention.py`` over its own positions 0..pos[b]; an idle row (pos[b] = -1) has a zero output."""
from __future__ import annotations

import numpy as np

from tests import _attention as A


def rows_reference(qh, K, V, pos, scaling):
    """qh [B, H, hd] (q̂), K / V [B, n_kv, L, hd] (caches holding each row's new entry), pos [B] -> o* [B, H, hd] and,
    per row, the parts of ``A.bound`` (None for an idle row)."""
    B, H, hd = qh.shape
    o = np.zeros((B, H, hd))
    parts = []
    for b, p in enumerate(pos):
        if p < 0:
            parts.append(None)
            continue
        ob, pb, sb, qk, Vr = A.reference(qh[b:b + 1], K[b:b + 1, :, :p + 1], V[b:b + 1, :, :p + 1], scaling)
        o[b] = ob[0]
        parts.append((ob, pb, sb, qk, Vr))
    return o, parts


def check_rows(out, qh, K, V, pos, scaling, hd, dtype, what=""):
    """Every active row within the ``tests/_attention.py`` bound, every idle row exactly zero; returns the largest
    err/bound."""
    out = np.asarray(out, np.float64)
    _, parts = rows_reference(qh, K, V, pos, scaling)
    worst = 0.0
    for b, part in enumerate(parts):
        if part is None:
            assert (out[b] == 0).all(), f"{what}: idle row {b} is not zero"
            continue
        ob, pb, sb, qk, Vr = part
        bd, budget = A.bound(ob, pb, sb, qk, Vr, scaling, hd, dtype)
        w, _, _ = A.check(out[b:b + 1], ob, bd, budget, dtype, f"{what} row {b} pos {pos[b]}")
        worst = max(worst, w)
    return worst
