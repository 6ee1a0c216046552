"""Float64 reference and error bound of the prefill attention kernel (``csrc/prefill_attention.cuh``).

Reference
    Row b's T new tokens take positions start .. start + T − 1.  For token t and query head h (kv head g = h // G):
    s_τ = σ·q̂·k_τ over τ ∈ [0, start + t], p*_τ = softmax(s)_τ, o* = Σ_τ p*_τ·v_τ, in float64 on q̂ (the rotary
    embedding of ``tests/_attention.py``) and the cache rows exactly as stored (FP8: codes times scales).

Bound, per output element (the decode kernel's, ``tests/_attention.py``, with the tensor cores and the rounding of P)
    |o − o*| ≤ ulp(o*) + 2·Σ p*_τ·η_τ·|v_τ − o*| + 2·u_p·Σ p*_τ·|v_τ| + 2·φ·p*_max·Σ_τ A_τ
               + (2·TC·γ_L + 4u)·Σ p*_τ·|v_τ|

    * Scores.  s̃_τ = fp32(fp32(q̂·k_τ)·σ) (FP8: the dot product on the codes, times the row's k scale, exact).  The
      dot product accumulates hd exact products inside the tensor core, whose internal rounding is not documented: its
      γ_hd carries the factor TC = ``tests._precision.TC_GAMMA``.  So e_τ = σ·TC·γ_hd·Σ_d |q̂_d·k_τd| + 2u·|s_τ|, and
      η_τ = e_τ + (M − s_τ + e_τ)·u + 4u·(n_tiles + 1) as in the decode bound (the running max over 64-position
      tiles; a fully masked tile rescales by expf(0) = 1 exactly).
    * P.  The weights e = expf(s̃ − m) enter the P·V product rounded to the dtype (FP8: e·vs_τ/R first, R the largest
      v scale of the tiles read so far, a power of two, so the product is one fp32 rounding).  A normal rounding errs
      by u_p = 2^-11 (fp16) / 2^-8 (bf16) relative; l sums the unrounded e, so this is an error of the numerator alone:
      u_p·Σ p*|v|.  Below the dtype's normal range the rounding errs by up to φ absolute in units of e (φ = 2^-24 for
      fp16, the smallest subnormal; 2^-126 for bf16, which also covers a flush to zero), i.e. φ·A_τ/L in o, L =
      Σ exp(s − M) = 1/p*_max.  A_τ = |v_τ| for a 16-bit cache and R·|code_τ| for FP8 (R bounded by the largest v scale
      of the row's positions 0 .. start + T − 1): rows whose v scale is far below R lose their low bits here.
    * Sums.  acc is the tensor core's fp32 accumulation over the n attended positions plus one or two rescales per
      tile; l is a 16-term fp32 sum per thread and tile, two butterfly levels and one FMA per tile.  L = n + 3·n_tiles + 8
      terms, the tensor-core γ with the factor TC, plus the division and the FP8 products (4u).
    n_tiles = ceil((start + T) / 64) bounds the tiles any CTA of the row walks.

Sharpness: elements whose budget beyond ulp(o*) is at most one ulp must round to round(o*) at ``tests/_attention.py``'s
RATE.
"""
from __future__ import annotations

import numpy as np
import torch

from tests._attention import RATE, gamma
from tests._precision import TC_GAMMA, U, round_dt, ulp

TILE = 64
U_P = {"float16": 2.0 ** -11, "bfloat16": 2.0 ** -8}
FLOOR = {"float16": 2.0 ** -24, "bfloat16": 2.0 ** -126}


def reference(qh, K, V, start, scaling):
    """One row, float64 torch tensors on any device: qh [T, H, hd] (q̂ of the new tokens), K / V [n_kv, n, hd] (the cache
    rows as stored, n >= start + T) -> o* [T, H, hd] and the parts of the bound: p* [T, H, n], s [T, H, n] (−inf where
    masked), Σ_d|q̂·k| [T, H, n], the repeated V [H, n, hd]; n = start + T."""
    T, H, hd = qh.shape
    n = start + T
    G = H // K.shape[0]
    Kr = K[:, :n].repeat_interleave(G, dim=0)
    Vr = V[:, :n].repeat_interleave(G, dim=0)
    s = scaling * torch.einsum("thd,hnd->thn", qh, Kr)
    qk_abs = torch.einsum("thd,hnd->thn", qh.abs(), Kr.abs())
    pos = torch.arange(n, device=qh.device)
    mask = pos[None, None, :] > (start + torch.arange(T, device=qh.device))[:, None, None]
    s = s.masked_fill(mask, -torch.inf)
    p = torch.softmax(s, dim=-1)
    o = torch.einsum("thn,hnd->thd", p, Vr)
    return o, p, s, qk_abs, Vr


def bound(o, p, s, qk_abs, Vr, scaling, hd, dtype, A=None):
    """Per-element bound (module docstring) and its budget beyond ulp(o*), as float64 numpy arrays.  ``A`` [H, n, hd]:
    the magnitudes the P underflow term weighs (None: |V|, a 16-bit cache)."""
    T, H, n = p.shape
    n_tiles = -(-n // TILE)
    att = p > 0
    s0 = torch.where(att, s, torch.zeros_like(s))
    e = scaling * TC_GAMMA * gamma(hd) * qk_abs + 2 * U * s0.abs()
    M = s0.amax(dim=-1, keepdim=True)
    eta = torch.where(att, e + (M - s0 + e) * U + 4 * U * (n_tiles + 1), torch.zeros_like(s))
    L = n + 3 * n_tiles + 8
    pe = p * eta
    w_dev = torch.stack([2 * torch.einsum("hn,hnd->hd", pe[t], (Vr - o[t][:, None, :]).abs()) for t in range(T)])
    pv = torch.einsum("thn,hnd->thd", p, Vr.abs())
    A = Vr.abs() if A is None else A
    under = 2 * FLOOR[dtype] * p.amax(dim=-1)[..., None] * torch.einsum("thn,hnd->thd", att.double(), A)
    budget = (w_dev + 2 * U_P[dtype] * pv + under + (2 * TC_GAMMA * gamma(L) + 4 * U) * pv).cpu().numpy()
    return ulp(o.cpu().numpy(), dtype) + budget, budget


def check(out, o, b, budget, dtype, what=""):
    """Assert the bound and the mismatch-rate limit; return (largest err/bound, mismatches, elements counted)."""
    out = np.asarray(out, np.float64)
    o = o.cpu().numpy() if isinstance(o, torch.Tensor) else o
    assert np.isfinite(out).all(), f"{what}: non-finite output"
    ratio = np.abs(out - o) / b
    worst = float(ratio.max())
    assert worst <= 1.0, f"{what}: max err/bound = {worst:.3g} at {np.unravel_index(ratio.argmax(), ratio.shape)}"
    cond = budget <= ulp(o, dtype)
    mism = int(((out != round_dt(o, dtype)) & cond).sum())
    n = int(cond.sum())
    assert mism <= RATE[dtype] * max(n, 1), f"{what}: mismatch rate {mism}/{n} > {RATE[dtype]}"
    return worst, mism, n
