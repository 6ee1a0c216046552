"""Float64 reference, error bound and rotary rounding model of the decode attention kernel (``csrc/attention.cuh``).

Rotary embedding (transformers 5.5, ``LlamaRotaryEmbedding`` + ``apply_rotary_pos_emb``)
    f = fp32(inv_freq[j mod hd/2] · fp32(pos)), c = rnd(fp32(cos(f)·a)), s = rnd(fp32(sin(f)·a)) with a the
    attention_scaling, then x̂[j] = rnd(rnd(x[j]·c) + rnd(r[j]·s)), r = rotate_half(x).  Every product of two 16-bit
    values is exact in fp32, so each step is one correct rounding to the dtype.  ``rope`` restates this on given fp32
    cos(f) / sin(f); the CPU test pins it bit-equal to transformers on the CPU's cos / sin, the GPU test pins the
    kernel's cache entries bit-equal to transformers on the GPU's.

Reference
    For query head h (kv head g = h // G) at position pos: s_t = σ·q̂·k_t over t ∈ [0, pos], p*_t = softmax(s)_t,
    o* = Σ_t p*_t·v_t, all in float64 on the 16-bit q̂, cache rows and v.

Bound, per output element
    |o − o*| ≤ ulp(o*) + 2·Σ_t p*_t·η_t·|v_t − o*| + (2·γ_L + 2u)·Σ_t p*_t·|v_t|,    u = 2^-24, γ_n = n·u / (1 − n·u)

    The kernel forms o = rnd(Σ_t w_t·v_t / Σ_t w_t).  ulp(o*) covers the final rounding (half an ulp) and the room the
    other errors give it to round the other way.

    * Weights.  Position t of split i, tile j gets w_t = E(s̃_t − m_j)·Π E(m_a − m_b)·E(M_i − M): the in-tile
      exponential, the rescales of the running sums at every later tile of the split (m_a < m_b the running maxima),
      and the combine weight of the split (M_i its maximum, M the overall one).  With exact arguments and exponentials
      the product telescopes to exp(s̃_t − M), and M is common to every t, so only relative errors matter:
        - the score: s̃_t = fp32(fp32(q̂·k_t)·fp32(σ)).  The dot product is one fp32 FMA chain of hd exact products,
          |error| ≤ γ_hd·Σ_d |q̂_d·k_td|; σ rounded to fp32 and the product rounding add 2u·|s_t|.  So
          |s̃_t − s_t| ≤ e_t = σ·γ_hd·Σ_d |q̂_d·k_td| + 2u·|s_t|, and exp(s̃_t − s_t) errs by e_t relative (to first
          order; the factor 2 below absorbs the rest);
        - the arguments: each is a rounded fp32 difference, err ≤ u·|argument|, and the arguments' magnitudes along the
          chain of t sum to M − s̃_t (the maxima only grow), so together they err by (M − s_t + e_t)·u relative;
        - the exponentials: expf is accurate to 2 ulp, ≤ 4u relative on results ≤ 1, once in the tile, once per later
          tile (at most n_tiles − 1) and once in the combine: 4u·(n_tiles + 1).
      η_t = e_t + (M − s_t + e_t)·u + 4u·(n_tiles + 1) bounds the relative error of w_t / exp(s_t − M).  With
      w_t ∝ p*_t·(1 + θ_t), |θ_t| ≤ η_t ≤ 1/2: Σ w v / Σ w − o* = Σ p*_t·θ_t·(v_t − o*) / (1 + Σ p*θ), at most
      2·Σ p*_t·η_t·|v_t − o*|.
    * Sums.  acc = Σ w·v is an FMA chain over the split's positions (≤ C), with one multiplication by the rescale per
      tile, then the combine's FMA chain over the S splits; l = Σ w is a 32-lane tree per tile (5 levels), one FMA per
      tile and the combine.  Every partial sum is bounded by Σ w·|v| (Σ w), so each errs by γ_L relative to that with
      L = C + n_tiles + S + 5, which gives γ_L·Σ p*|v| for acc and γ_L·|o*| ≤ γ_L·Σ p*|v| for l; the division adds
      u·|o|.  The kernel's split count is a device property (about four CTAs per SM), so the bound takes the largest
      values the kernel allows: S = 64, C = pos + 1, n_tiles = ceil((pos + 1) / 32).

Sharpness: elements whose budget beyond ulp(o*) is at most one ulp must round to round(o*) at the rates of DESIGN
§3.12 (5 % fp16, 1 % bf16).
"""
from __future__ import annotations

import numpy as np

from tests._precision import U, round_dt, ulp

TILE = 32
MAX_SPLITS = 64
RATE = {"float16": 0.05, "bfloat16": 0.01}


def gamma(n):
    return n * U / (1 - n * U)


def rope(x, cos32, sin32, attention_scaling, dtype):
    """x [..., hd] (dtype values as float64), cos32 / sin32 [..., hd] fp32 cos(f) / sin(f) -> x̂ (float64)."""
    a = np.float32(attention_scaling)
    c = round_dt((np.asarray(cos32, np.float32) * a).astype(np.float64), dtype)
    s = round_dt((np.asarray(sin32, np.float32) * a).astype(np.float64), dtype)
    h = x.shape[-1] // 2
    r = np.concatenate([-x[..., h:], x[..., :h]], axis=-1)
    return round_dt(round_dt(x * c, dtype) + round_dt(r * s, dtype), dtype)


def freqs32(inv_freq, pos):
    """f = fp32(inv_freq · fp32(pos)), duplicated to [hd] as transformers' cat((freqs, freqs))."""
    f = np.asarray(inv_freq, np.float32) * np.float32(pos)
    return np.concatenate([f, f])


def reference(qh, K, V, scaling):
    """qh [B, H, hd] (q̂), K / V [B, n_kv, n, hd] (cache rows 0..pos with the new token) -> o* [B, H, hd] and the parts
    of the bound: p* [B, H, n], s [B, H, n], Σ_d|q̂·k| [B, H, n]."""
    B, H, hd = qh.shape
    G = H // K.shape[1]
    Kr = np.repeat(K, G, axis=1)
    Vr = np.repeat(V, G, axis=1)
    s = scaling * np.einsum("bhd,bhtd->bht", qh, Kr)
    qk_abs = np.einsum("bhd,bhtd->bht", np.abs(qh), np.abs(Kr))
    m = s.max(axis=-1, keepdims=True)
    e = np.exp(s - m)
    p = e / e.sum(axis=-1, keepdims=True)
    o = np.einsum("bht,bhtd->bhd", p, Vr)
    return o, p, s, qk_abs, Vr


def bound(o, p, s, qk_abs, Vr, scaling, hd, dtype):
    """Per-element bound (module docstring) and its budget beyond ulp(o*)."""
    n = p.shape[-1]
    n_tiles = -(-n // TILE)
    e = scaling * gamma(hd) * qk_abs + 2 * U * np.abs(s)
    M = s.max(axis=-1, keepdims=True)
    eta = e + (M - s + e) * U + 4 * U * (n_tiles + 1)
    L = n + n_tiles + MAX_SPLITS + 5
    w_dev = 2 * np.einsum("bht,bhtd->bhd", p * eta, np.abs(Vr - o[:, :, None, :]))
    w_abs = (2 * gamma(L) + 2 * U) * np.einsum("bht,bhtd->bhd", p, np.abs(Vr))
    budget = w_dev + w_abs
    return ulp(o, dtype) + budget, budget


def check(out, o, b, budget, dtype, what=""):
    """Assert the bound and the mismatch-rate limit; return (largest err/bound, mismatch rate, elements counted)."""
    out = np.asarray(out, np.float64)
    assert np.isfinite(out).all(), f"{what}: non-finite output"
    ratio = np.abs(out - o) / b
    worst = float(ratio.max())
    assert worst <= 1.0, f"{what}: max err/bound = {worst:.3g}"
    cond = budget <= ulp(o, dtype)
    mism = (out != round_dt(o, dtype)) & cond
    rate = float(mism.sum()) / max(int(cond.sum()), 1)
    assert rate <= RATE[dtype], f"{what}: mismatch rate {rate:.4f} > {RATE[dtype]} over {int(cond.sum())} elements"
    return worst, rate, int(cond.sum())
