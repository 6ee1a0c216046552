"""The decode chain's norm stage inputs (``x_mode="rmsnorm"`` / ``"add_rmsnorm"``, ``ch_norm_prepass`` in chain.cuh):
the kernel's arithmetic restated in NumPy, and the candidate rule that checks a normalised row to the ulp.

Rounding points (transformers 5.5 LlamaDecoderLayer / LlamaRMSNorm, also Mistral's and Qwen2's):

    h  = rnd(x + x2)                         the residual add in the activation dtype
    r  = 1 / sqrt(Σh² / K + eps)             fp32
    n  = rnd(rnd(h·r)·w)                     h·r in fp32, rounded to the dtype, times the weight in the dtype

h is exact: x + x2 of two 16-bit values rounded to fp32 and then to the dtype is the correctly rounded sum (fp32 has
24 ≥ 2·11 + 2 bits, so the double rounding is innocuous), on the GPU and in torch alike.  rnd(t)·w is exact in fp32 (two
16-bit significands), so n is fully determined by t16 = rnd(h·r).

The candidates of t16
    The kernel and torch sum h² in different fp32 orders.  Σh² has no cancellation (all terms ≥ 0), so its relative
    error is bounded like the accumulation γ of ``tests/_precision.py``: λ·√(K/4 + 64)·u, u = 2⁻²⁴ (λ = 2, the
    probabilistic bound; the squares, rounded or fused, add one u).  The division by K, the addition of eps and the
    square root / reciprocal (``__frsqrt_rn``, correctly rounded; torch's rsqrt within 2 ulp) add at most 4u; r carries
    half the relative error of its argument plus its own.  The product h·r adds u.  So

        |fl(h·r) − h·r₆₄| ≤ δ·|h·r₆₄|,   δ = ½(λ·√(K/4 + 64)·u + 2u) + 4u + u

    and δ is doubled to cover second-order terms.  t16 is rnd(h·r₆₄), or its neighbour where h·r₆₄ lies within δ·|h·r₆₄|
    of a rounding midpoint; n must equal rnd(t16·w) for one of the two.
"""
from __future__ import annotations

import numpy as np

from tests import _precision as P

U = P.U


def delta(K: int) -> float:
    """Relative bound of fl32(h·r) against h·r in float64 (module docstring), doubled."""
    return 2.0 * (0.5 * (P.LAMBDA * np.sqrt(K / 4 + 64) * U + 2 * U) + 5 * U)


def add_rounded(x, x2, dtype) -> np.ndarray:
    """h = rnd(x + x2) of 16-bit operands (float64 arrays)."""
    return P.round_dt(np.asarray(x, np.float64) + np.asarray(x2, np.float64), dtype)


def r_exact(h, eps) -> np.ndarray:
    """1 / sqrt(mean(h²) + eps) per row, in float64."""
    h = np.asarray(h, np.float64)
    return 1.0 / np.sqrt(np.mean(h * h, axis=-1, keepdims=True) + eps)


def n_candidates(h, w, eps, dtype):
    """(n0, n1, amb) for rows h [M, K] (float64, representable in dtype): n0 = rnd(rnd(h·r₆₄)·w), n1 from the
    neighbour of rnd(h·r₆₄) where h·r₆₄ lies within δ·|h·r₆₄| of a rounding midpoint (``amb``), else n0."""
    h = np.asarray(h, np.float64)
    K = h.shape[-1]
    t = h * r_exact(h, eps)
    d = delta(K) * np.abs(t)
    main, lo, hi = P.round_dt(t, dtype), P.round_dt(t - d, dtype), P.round_dt(t + d, dtype)
    alt = np.where(lo != main, lo, hi)
    amb = lo != hi
    w = np.asarray(w, np.float64)
    n0 = P.round_dt((main.astype(np.float32) * w.astype(np.float32)).astype(np.float64), dtype)
    n1 = P.round_dt((alt.astype(np.float32) * w.astype(np.float32)).astype(np.float64), dtype)
    return n0, n1, amb & (n0 != n1)


def check_n(n, h, w, eps, dtype, what="") -> float:
    """Assert that every element of n is one of its candidates; returns the share that needed the neighbour."""
    n = np.asarray(n, np.float64)
    n0, n1, amb = n_candidates(h, w, eps, dtype)
    ok0 = n == n0
    ok1 = amb & (n == n1)
    bad = ~(ok0 | ok1)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {n.size} normalised elements are neither candidate "
                           f"(first at {np.argwhere(bad)[0].tolist()}: {n[bad][0]!r} vs {n0[bad][0]!r} / {n1[bad][0]!r})")
    return float((ok1 & ~ok0).sum()) / n.size


def reference_y(d, h, w, eps, dtype, cols=None) -> P.Ref:
    """The chain's reference of a normed stage's output on the host-side n0 of the h the stage read, widened by
    Σ|n1 − n0|·|W| over the elements whose n has two candidates (the digit block maximum may be n1's).  ``cols``:
    (c0, c1) or None for every column."""
    pc = P.PATHS["chain"]
    n0, n1, amb = n_candidates(h, w, eps, dtype)
    ref = P.reference(d, n0, pc, dtype, cols=cols)
    if amb.any():
        q, z, s, gi, _ = P.layer_parts(d, dtype, cols)
        W = np.abs(s[gi] * (q - z[gi]))
        extra = (np.where(amb, np.abs(n1 - n0), 0.0) @ W) * (1 + 2.0 ** -7)
        hx = np.where(amb & (np.abs(n1) > np.abs(n0)), n1, n0)
        ref.F = np.maximum(ref.F, P.reference(d, hx, pc, dtype, cols=cols).F) + extra
    return ref


def check_y(y, d, h, w, eps, dtype, cols, what):
    """A normed stage's output y [M, N] (float64) on ``cols`` against ``reference_y``; the ``P.check`` measurement."""
    c0, c1 = cols or (0, d["N"])
    return P.check(y[:, c0:c1], reference_y(d, h, w, eps, dtype, cols), P.PATHS["chain"], dtype, what=what)


def kernel_model(x, x2, w, eps, dtype, threads: int = 384):
    """NumPy restatement of ch_norm_prepass for one launch: (h, n) with the kernel's fp32 order of Σh² (each thread
    sums its k8-rows ctid, ctid + threads, ... with fused multiply-adds, then a xor-shuffle tree per warp of 32 and the
    warps in order).  ``x2`` None: x_mode="rmsnorm"."""
    x = np.asarray(x, np.float64)
    h = x if x2 is None else add_rounded(x, x2, dtype)
    M, K = h.shape
    rows = K // 8
    hf = h.astype(np.float32)
    n = np.empty_like(h)
    for m in range(M):
        per_thread = np.zeros(threads, dtype=np.float32)
        for row in range(rows):
            t = row % threads
            acc = np.float64(per_thread[t])
            for k in range(8 * row, 8 * row + 8):       # fmaf: the square is not rounded before the add
                acc = np.float64(np.float32(acc + np.float64(hf[m, k]) * np.float64(hf[m, k])))
            per_thread[t] = np.float32(acc)
        warps = per_thread.reshape(-1, 32).copy()
        for o in (16, 8, 4, 2, 1):                      # __shfl_xor_sync tree; lane 0's value
            warps = (warps + warps[:, np.arange(32) ^ o]).astype(np.float32)
        tot = np.float32(0)
        for v in warps[:, 0]:
            tot = np.float32(tot + v)
        var = np.float32(tot / np.float32(K))
        r = np.float32(1.0 / np.sqrt(np.float64(np.float32(var + np.float32(eps)))))
        t16 = P.round_dt((hf[m] * r).astype(np.float64), dtype)
        n[m] = P.round_dt((t16.astype(np.float32) * np.asarray(w, np.float32)).astype(np.float64), dtype)
    return h, n
