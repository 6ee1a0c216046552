"""Stage-wise float64 references of the two fused backwards, checked on the intermediates the kernels write:
the grouped experts' ``agb200_moe_backward`` (§3.13) and the dense MLP's ``agb200_w4a16_mlp_backward`` (§3.14).

Both run dy → dy_pair → dh → [dg | du] → dx_pair → dx and keep every rounded intermediate in the caller's workspace
(layouts below), so each stage is checked exactly on the operands it read, not through one composed bound that has to
excuse every rounded operand by an ulp:

    dy_pair   rnd(fl32(w·dy)) (``moe_combine_bwd_kernel``): bit-exact.  With fp32 weights this is a double rounding
              (fp32, then the dtype), which numpy reproduces; a 16-bit weight times a 16-bit dy is exact in fp32.
    dg, du    dh = dy_pair·W2ᵀ accumulates in fp32 on wgmma (unrounded), then ``silu_mul_backward`` (moe_dgrad.cuh):
                  du = rnd(fl32(dh·s16)),  s16 = rnd(silu(g)) (one of ``_silu_mul.silu_candidates``)
                  dg = rnd(fl32(fl32(dh·u)·sp)),  sp = fl32(σ·(1 + g·(1 − σ))),  σ = 1 / (1 + __expf(−g))
              on the saved 16-bit g and u.  With dh* = dy_pair·W2ᵀ in float64 (W2 rounded once, as the dgrad kernels
              form it), A_dh = |dy_pair|·|W2|ᵀ and γ = γ_dgrad(H), |dh − dh*| ≤ γ·A_dh, so the value the kernel
              rounds lies within β of v* (below) and the element must lie in [rnd(v* − β), rnd(v* + β)].
    dx_pair   dg·W1ᵀ + du·W3ᵀ: ONE fp32 sum over n = 2I terms, on the kernel's own dg and du; A = |dg|·|W1|ᵀ + |du|·|W3|ᵀ.
              Dense: rounded once, held to ``_precision.check`` with ``PATHS["dgrad"]`` (ulp + γ·A, mismatch-rate
              limit).  Experts: left in fp32, |e| ≤ 2⁻²⁴·|dx*| + γ·A.
    dx        experts: rnd(Σ_j dx_pair) over the valid slots, fp32 from 0 in slot order (``moe_dx_combine_kernel``):
              bit-exact.

Interval half-widths (D = |dh*| + γ·A_dh ≥ |dh|, S = |sp*| + Δ ≥ |sp|, u = 2⁻²⁴):

    du:  β = |s16|·(γ·A_dh + 1.0001·u·D)                     (dh's error, the product's rounding)
    dg:  β = |u16|·(γ·A_dh·S + |dh*|·Δ + 2.0001·u·D·S)       (dh's error, silu′'s error, the two products' roundings)

each plus 2⁻¹⁴⁸ for the fp32 subnormal range.  Δ(g) bounds |sp − silu′(g)| absolutely: silu′ = σ·(1 + g·(1 − σ))
crosses 0 at g ≈ −1.28, where a relative bound cannot hold.  σ carries the relative error of ``__expf`` scaled by
1 − σ (ρ = (1 − σ)·(2⁻²² + 2u·|g|), as in ``_silu_mul.silu_delta``) and two roundings; 1 − σ, g·(1 − σ), 1 + (…) and
σ·(…) commit one rounding each, and the error of σ reaches the result once directly and once through g·(1 − σ).  To
first order, with the rounding of 1 + e and of the division no larger than 1 − σ where σ nears 1 (1 is a floating-point
neighbour), and m = 1 + |g|·(1 − σ),

    Δ(g) = σ·m·(2ρ + 96·u) + m·2⁻¹⁴⁸.

96·u covers the roundings (≤ 6u) and the term σ·|g|·min(u, 1 − σ) ≤ 17u·σ at g ≈ 16.6, with margin; m·2⁻¹⁴⁸ covers a
σ in fp32's subnormal range (g ≈ −88);
``tests/test_backward_stages_cpu.py`` holds it against an fp32 emulation over every finite fp16 and bf16 g.  Where
``__expf(−g)`` overflows (fl32(−g·log2 e) ≥ 128, g < −88.72) σ = 0, sp = −0 and s16 = −0 exactly: v* = 0 there.

A value that rounds to ±inf is accepted exactly where its interval reaches past the largest finite value (rnd of the
interval's end is then ±inf), as ``_precision.measure`` accepts an overflow.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle import w4a16_oracle as O
from tests import _precision as P
from tests import _silu_mul as S

U = P.U
TINY = 2.0 ** -148                   # two fp32 subnormal steps: the absolute floor of an fp32 rounding


# --------------------------------------------------------------------------- workspace layouts (csrc/moe.cu)
def _align(v, a=256):
    return -(-int(v) // a) * a


def bwd_tile(P_, E):
    """The experts' backward row tile: 32 / 64 / 128 by the mean rows per hit expert (``bwd_tile``)."""
    if P_ <= 0:
        return 32
    m = min(E, P_)
    avg = -(-P_ // m)
    return 32 if avg <= 32 else 64 if avg <= 64 else 128


def bwd_layout(T, k, E, H, I) -> dict:
    """``bwd_layout``: routing tables | prow int32 [P] | dy_pair 16-bit [rows, H] | [dg | du] 16-bit [rows, 2I] |
    dx_pair fp32 [rows, H], each 256-byte aligned; rows = P + min(E, P)·(mt − 1) bounds the tile-padded rows."""
    P_ = T * k
    max_tiles = (P_ + 31) // 32 + E
    mt = bwd_tile(P_, E)
    rows = P_ + min(E, P_) * (mt - 1)
    ints = E * 4 + 4 + 2 * max_tiles + P_
    prow = _align(ints * 4)
    dyp = prow + _align(P_ * 4)
    dgu = dyp + _align(rows * H * 2)
    dxp = dgu + _align(rows * 2 * I * 2)
    return dict(mt=mt, rows=rows, prow=prow, dyp=dyp, dgu=dgu, dxp=dxp, total=dxp + _align(rows * H * 4))


def mlp_bwd_layout(M, H, I) -> dict:
    """``mlp_bwd_layout``: [dg | du] 16-bit [M, 2I] at 0 (I's natural order) | dx staged for an act-order pair [M, H]."""
    dxs = _align(M * 2 * I * 2)
    return dict(dgu=0, dxs=dxs, total=dxs + _align(M * H * 2))


# --------------------------------------------------------------------------- weights
def weights(d, dtype, rows=None) -> np.ndarray:
    """s·(q − z) rounded once to the dtype (as both dgrad kernels form it), [K, N] in natural order, or only the row
    ranges ``rows`` = [(r0, r1), ...] (multiples of 8) of K."""
    ranges = rows or [(0, d["K"])]
    qw = np.asarray(d["qweight"])
    q = np.concatenate([O.unpack_qweight(qw[r0 // 8:r1 // 8]) for r0, r1 in ranges]).astype(np.int64)
    at = np.concatenate([np.arange(r0, r1) for r0, r1 in ranges])
    z = O.unpack_qzeros(np.asarray(d["qzeros"])).astype(np.int64)
    s = P.round_dt(np.asarray(d["scales"], dtype=np.float64), dtype)
    g = np.asarray(d["g_idx"]).astype(np.int64)[at]
    return P.round_dt(s[g] * (q - z[g]).astype(np.float64), dtype)


def inverse(perm):
    """argsort of an act-order permutation (sorted row j is natural row perm[j]): natural column c at inverse[c]."""
    return np.argsort(np.asarray(perm))


def sorted_perm(d):
    """The kernels' act-order permutation of a layer (sorted row j is natural row perm[j]), or None when sequential."""
    g = np.asarray(d["g_idx"])
    return None if np.array_equal(g, O.default_g_idx(d["K"], d["group_size"])) else O.make_sequential_perm(g)


# --------------------------------------------------------------------------- bit-exact stages
def same_bits(a, b) -> np.ndarray:
    """Elementwise: same value, same sign of zero, NaN for NaN."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return ((a == b) & (np.signbit(a) == np.signbit(b))) | (np.isnan(a) & np.isnan(b))


def dy_pair(dy, w, dtype) -> np.ndarray:
    """[T, k, H] rnd(fl32(w·dy)): w as the kernel reads it (fp32, or 16-bit values), dy 16-bit."""
    with np.errstate(over="ignore", invalid="ignore"):
        p = np.asarray(w, dtype=np.float32)[:, :, None] * np.asarray(dy, dtype=np.float32)[:, None, :]
    return P.round_dt(p.astype(np.float64), dtype)


def dx_combine(dxp, idx, E, dtype) -> np.ndarray:
    """[T, H] rnd(fl32 Σ_j dx_pair[t, j]) over the slots with an id in [0, E), from +0 in slot order; dxp [T, k, H] in
    x's natural column order (what a slot without a valid id holds is never read)."""
    idx = np.asarray(idx).astype(np.int64)
    valid = (idx >= 0) & (idx < E)
    dxp = np.asarray(dxp, dtype=np.float32)
    acc = np.zeros((dxp.shape[0], dxp.shape[2]), dtype=np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for j in range(idx.shape[1]):
            acc = np.where(valid[:, j, None], acc + dxp[:, j], acc)
    return P.round_dt(acc.astype(np.float64), dtype)


def check_exact(got, want, what=""):
    bad = ~same_bits(got, want)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} elements differ (first at {np.argwhere(bad)[0]})"


# --------------------------------------------------------------------------- silu'
def sigmoid(g) -> np.ndarray:
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-np.asarray(g, dtype=np.float64)))


def silu_prime(g) -> np.ndarray:
    """σ·(1 + g·(1 − σ)) in float64, and 0 where ``__expf(−g)`` overflows (the kernel's σ is 0 there)."""
    g = np.asarray(g, dtype=np.float64)
    s = sigmoid(g)
    return np.where(S.exp_overflows(g), 0.0, s * (1.0 + g * (1.0 - s)))


def silu_prime_delta(g) -> np.ndarray:
    """Absolute bound Δ(g) of |fp32 silu′ − silu′(g)| (module docstring); 0 on the overflow domain."""
    g = np.asarray(g, dtype=np.float64)
    s = sigmoid(g)
    a = np.abs(g)
    m = 1.0 + a * (1.0 - s)
    d = s * m * (2.0 * (1.0 - s) * (S.EX2_REL + 2 * U * a) + 96 * U) + m * TINY
    return np.where(S.exp_overflows(g), 0.0, d)


# --------------------------------------------------------------------------- dg, du
@dataclass
class StageResult:
    """A stage held to per-element intervals: the elements outside (must be none) among ``n`` checked, and the
    measurement as a ``_precision.Result``: worst |v − v*| / (ulp(v*) + β), mismatch rate against rnd(v*) over the
    well-conditioned elements (β with the unscaled fp32 budget √(n/4 + 64)·u·A at most an ulp), γ share."""
    outside: int
    n: int
    res: P.Result


def _stage(v, cands, chk, dtype) -> StageResult:
    """v: observed; cands: one or two (v*, β, β_plain, β_rest, a) (two: the silu candidates; β_plain: β with the
    unscaled fp32 budget in place of γ, β_rest: the part of β that is not accumulation error, a: what γ multiplies);
    chk: the elements checked."""
    v = np.asarray(v, dtype=np.float64)
    inside = np.zeros(v.shape, dtype=bool)
    worst = np.full(v.shape, np.inf)
    share = np.full(v.shape, np.inf)
    mism = np.ones(v.shape, dtype=bool)
    star0, _, bp0, _, _ = cands[0]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for star, beta, _, rest, a in cands:
            lo, hi = P.round_dt(star - beta, dtype), P.round_dt(star + beta, dtype)
            ins = (v >= lo) & (v <= hi)
            inside |= ins
            e = np.abs(v - star)
            q = P.ulp(star, dtype)
            worst = np.minimum(worst, np.where(np.isfinite(v), e / (q + beta), np.where(ins, 0.0, np.inf)))
            sh = np.maximum(e - 0.5 * q - rest, 0) / a
            share = np.minimum(share, np.where(np.isfinite(sh), sh, np.where(np.isfinite(v), 0.0, np.inf)))
            mism &= v != P.round_dt(star, dtype)
        cond = chk & (bp0 <= P.ulp(star0, dtype))
    n_cond = int(cond.sum())
    res = P.Result(float(worst[chk].max()) if chk.any() else 0.0, float((cond & mism).sum()) / max(n_cond, 1), n_cond,
                   True, float(np.where(np.isfinite(share), share, 0.0)[chk].max()) if chk.any() else 0.0)
    return StageResult(int((chk & ~inside).sum()), int(chk.sum()), res)


@dataclass
class DhRef:
    dh: np.ndarray          # float64 dy_pair·W2ᵀ [R, Ic]
    A: np.ndarray           # |dy_pair|·|W2|ᵀ
    n_terms: int            # H


def dh_reference(dyp, W2) -> DhRef:
    """dh* and A_dh for the rows dyp [R, H] and the (rows of) w2 W2 [Ic, H] in natural order."""
    dyp = np.asarray(dyp, dtype=np.float64)
    return DhRef(dyp @ W2.T, np.abs(dyp) @ np.abs(W2).T, W2.shape[1])


def measure_dgu(dg, du, ref: DhRef, g, u, dtype) -> dict:
    """{"dg": StageResult, "du": StageResult} of the kernel's dg, du [R, Ic] against the intervals of the module
    docstring, from the saved g, u [R, Ic] (all in I's natural order).  Elements whose g or u is non-finite are not
    checked; rows whose dh* is non-finite (a non-finite dy_pair) neither."""
    g, u = np.asarray(g, dtype=np.float64), np.asarray(u, dtype=np.float64)
    chk = np.isfinite(g) & np.isfinite(u) & np.isfinite(ref.dh)
    gf, uf = np.where(chk, g, 0.0), np.where(chk, u, 0.0)
    dh = np.where(chk, ref.dh, 0.0)
    A = np.where(chk, ref.A, 0.0)
    gam = P.gamma(P.PATHS["dgrad"], ref.n_terms)
    plain = P.gamma(P._PLAIN, ref.n_terms) / P.LAMBDA           # √(n/4 + 64)·u
    sp, dl = silu_prime(gf), silu_prime_delta(gf)
    Sp = np.abs(sp) + dl

    def beta_dg(gm):
        D = np.abs(dh) + gm * A
        return np.abs(uf) * (gm * A * Sp + np.abs(dh) * dl + 2.0001 * U * D * Sp) + TINY

    rest_dg = np.abs(uf) * (np.abs(dh) * dl + 2.0001 * U * (np.abs(dh) + gam * A) * Sp) + TINY
    dg_c = [(dh * uf * sp, beta_dg(gam), beta_dg(plain), rest_dg, np.abs(uf) * Sp * P.gamma(P._PLAIN, ref.n_terms) * A)]
    s0, s1, amb = S.silu_candidates(gf, dtype)
    du_c = []
    for s in ((s0,) if not amb.any() else (s0, np.where(amb, s1, s0))):
        def beta_du(gm, s=s):
            return np.abs(s) * (gm * A + 1.0001 * U * (np.abs(dh) + gm * A)) + TINY

        rest = np.abs(s) * 1.0001 * U * (np.abs(dh) + gam * A) + TINY
        du_c.append((dh * s, beta_du(gam), beta_du(plain), rest, np.abs(s) * P.gamma(P._PLAIN, ref.n_terms) * A))
    return {"dg": _stage(dg, dg_c, chk, dtype), "du": _stage(du, du_c, chk, dtype)}


def check_dgu(dg, du, ref: DhRef, g, u, dtype, what="") -> dict:
    """``measure_dgu`` with no element outside its interval and the mismatch rate within ``_precision._RATE``."""
    r = measure_dgu(dg, du, ref, g, u, dtype)
    lim = P._RATE[P.dt_name(dtype)]
    for name, st in r.items():
        assert st.outside == 0, f"{what} {name}: {st.outside} of {st.n} elements outside their interval"
        assert st.res.rate <= lim, f"{what} {name}: mismatch rate {st.res.rate:.4f} > {lim} over {st.res.n_cond}"
    return {k: v.res for k, v in r.items()}


# --------------------------------------------------------------------------- dx_pair, dx
def dx_reference(dg, du, W1, W3) -> P.Ref:
    """dx* = dg·W1ᵀ + du·W3ᵀ in float64 on the kernel's dg, du [R, I] (natural order), W1, W3 [Hc, I] the (rows of)
    gate and up in natural order; A = |dg|·|W1|ᵀ + |du|·|W3|ᵀ, one sum over n = 2I terms."""
    dg, du = np.asarray(dg, dtype=np.float64), np.asarray(du, dtype=np.float64)
    bad = ~(np.isfinite(dg).all(axis=1) & np.isfinite(du).all(axis=1))
    dg, du = np.where(np.isfinite(dg), dg, 0.0), np.where(np.isfinite(du), du, 0.0)
    ystar = dg @ W1.T + du @ W3.T
    A = np.abs(dg) @ np.abs(W1).T + np.abs(du) @ np.abs(W3).T
    return P.Ref(ystar, A, np.zeros_like(ystar), 2 * W1.shape[1], bad, A)


def measure_dx_pair(dxp, ref: P.Ref) -> P.Result:
    """fp32 dx_pair: worst |e| / (2⁻²⁴·|dx*| + γ·A) and the γ share (no output rounding to a 16-bit dtype: rate 0)."""
    y = np.asarray(dxp, dtype=np.float64).reshape(ref.ystar.shape)
    good = ~ref.bad_rows
    ok_rows = bool(np.all(~np.isfinite(y[ref.bad_rows]).any(axis=1))) if ref.bad_rows.any() else True
    ys, yg, A = ref.ystar[good], y[good], ref.A[good]
    e = np.abs(yg - ys)
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(np.isfinite(yg), e / (U * np.abs(ys) + P.gamma(P.PATHS["dgrad"], ref.n_terms) * A + TINY), np.inf)
        share = np.maximum(e - U * np.abs(ys), 0) / (P.gamma(P._PLAIN, ref.n_terms) * A)
    share = np.where(np.isfinite(share), share, 0.0)
    return P.Result(float(ratio.max()) if ratio.size else 0.0, 0.0, 0, ok_rows, float(share.max()) if share.size else 0.0)


def check_dx_pair(dxp, ref: P.Ref, what="") -> P.Result:
    r = measure_dx_pair(dxp, ref)
    assert r.ok_rows, f"{what}: a dx_pair row from non-finite dg / du is finite"
    assert r.worst <= 1.0, f"{what}: dx_pair max err/bound = {r.worst:.3g}"
    return r
