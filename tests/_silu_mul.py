"""Stage-wise precision checks of the SiLU·mul paths: the fused gate/up pair (``forward_gate_up`` / ``FusedQuantMLP``),
the grouped experts' forward (``QuantExperts``) and the decode chain's ``silu_mul`` stage input.

Every intermediate these kernels round is observable (the saving forwards keep g, u and, for the experts, y_pair), so
each stage is checked exactly on the inputs it actually read, instead of through one loose composed bound:

    g, u      rnd(x·W1 + b1), rnd(x·W3 + b3): the bound of ``tests/_precision.py`` for the path that computes them
              (decode kernel: ``decode_mma``, the skinny arithmetic with its own measured factor; wgmma GEMM: ``gemm``, weights rounded once).
    h         rnd(s16·u16) with s16 = rnd(silu(g16)) formed in fp32 (``silu_mul_elt`` in gemm_common.cuh, ``ch_silu_mul``
              in chain.cuh).  s16·u16 is exact in fp32 (two 16-bit significands), so h is fully determined by s16, and
              s16 by one of at most two candidates (below).  Checked for equality.
    y         the down projection (``y_pair`` of the experts, the chain's down output) against the float64 reference
              applied to the host-side h, with Σ|h_alt − h|·|W2| added to the bound over the elements whose s16 has two
              candidates.
    out       rnd(Σ_j w_j·y_pair_j) over the slots with a valid expert id, fp32 in slot order (``moe_combine_kernel``):
              |out − out*| ≤ ulp(out*) + (k + 1)·2⁻²⁴·Σ_j |w_j·y_pair_j|, and the rate of elements that differ from
              rnd(out*) is bounded as in ``tests/_precision.py``.

The silu candidates
    The kernel computes s = g / (1 + e) with e = ex2.approx.f32(fl(g·c)), c = fl32(−log2 e) (``__expf``; the division
    is IEEE ``div.rn.f32``), then s16 = rnd(s).  Its relative error against silu(g) = g / (1 + exp(−g)):
      * fl(g·c): one fp32 rounding (u = 2⁻²⁴) and the constant's own error (|c + log2 e| < 2⁻²⁶·log2 e) perturb the
        exponent t = −g·log2 e by at most |t|·(u + 2⁻²⁶) < 2u·|t|, which moves 2^t by a relative ln 2·2u·|t| = 2u·|g|;
      * ex2.approx.f32: the PTX ISA states a maximum error of 2 ulp of the fp32 result, a relative 2⁻²²;
      * 1 + e: one rounding, u; a relative error ρ of e moves 1 + e, and so s, by a relative σ(−g)·ρ (σ(−g) =
        e/(1 + e));
      * the division: one rounding, u.
    To first order |s − silu(g)| ≤ (σ(−g)·(2⁻²² + 2u·|g|) + 2u)·|silu(g)|; δ(g) is twice that, which covers the
    second-order terms with a wide margin (|g| < 90 wherever e is finite, so 2u·|g| < 2⁻¹⁶).  So rnd(s) is rnd(silu₆₄(g)), or its
    neighbour when silu₆₄(g) lies within δ·|silu(g)| of a rounding midpoint; both candidates are kept there and h must
    equal rnd(s16·u16) for one of them.  The rate at which only the neighbour matches is reported and bounded
    (``NEIGHBOUR_RATE``); the rate of a correctly rounded s16 away from such midpoints is 100 % by the equality check.
    fp32 overflow domain: for g < −88.72, fl(g·c) ≥ 128 and ex2 returns +inf, so s = g / inf = −0 (torch's F.silu
    gives the same −0).  The float64 value there is tiny but, in bf16, representable (silu(−89) ≈ −1.8·10⁻³⁷); the
    candidate is −0 on that domain, which is what the kernels (and torch) compute.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np

from oracle import w4a16_oracle as O
from tests import _precision as P

U = P.U
NEG_LOG2E_F32 = np.float32(-1.4426950408889634)     # the constant __expf multiplies by (0xBFB8AA3B)
EX2_REL = 2.0 ** -22                                # ex2.approx.f32: 2 ulp of the fp32 result
# Limit on the share of finite h elements that matched only the neighbour candidate, per dtype, over a whole run of
# tests/test_gpu_20_silu_mul_precision.py.  Measured on an H100 80GB HBM3 (700 W): fp16 1.2e-4 (166 of 1.38 M; at most
# 7.1e-4 in one case), bf16 0 of 1.38 M.
NEIGHBOUR_RATE = {"float16": 2e-3, "bfloat16": 2e-4}


def silu_delta(g) -> np.ndarray:
    """Relative error bound δ(g) of the kernels' fp32 silu (see the module docstring)."""
    g = np.asarray(g, dtype=np.float64)
    with np.errstate(over="ignore"):
        w = 1.0 / (1.0 + np.exp(g))                     # e / (1 + e) = σ(−g)
    return 2.0 * (w * (EX2_REL + 2 * U * np.abs(g)) + 2 * U)


def exp_overflows(g) -> np.ndarray:
    """Where ``__expf(−g)`` is +inf: fl32(g·c) ≥ 128."""
    with np.errstate(over="ignore", invalid="ignore"):
        t = np.asarray(g, dtype=np.float32) * NEG_LOG2E_F32
    return t >= 128


def silu_candidates(g, dtype):
    """(s, s_alt, amb) for 16-bit g: s = rnd(silu₆₄(g)) (−0 on the overflow domain), s_alt its neighbour where
    silu₆₄(g) lies within δ·|silu(g)| of a rounding midpoint (``amb``), else s."""
    g = np.asarray(g, dtype=np.float64)
    fin = np.isfinite(g)
    gf = np.where(fin, g, 0.0)
    with np.errstate(over="ignore"):
        s = gf / (1.0 + np.exp(-gf))
    d = silu_delta(gf) * np.abs(s)
    main, lo, hi = P.round_dt(s, dtype), P.round_dt(s - d, dtype), P.round_dt(s + d, dtype)
    alt = np.where(lo != main, lo, hi)
    amb = (lo != hi) & fin
    over = exp_overflows(gf)
    main, alt = np.where(over, -0.0, main), np.where(over, -0.0, alt)
    return main, alt, amb & ~over


def h_of(s, u, dtype) -> np.ndarray:
    """rnd(fl32(s16·u16)): the product is exact in fp32 unless it leaves fp32's normal range, where fp32 rounds first."""
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        p = np.asarray(s, dtype=np.float32) * np.asarray(u, dtype=np.float32)
    return P.round_dt(p.astype(np.float64), dtype)


def h_candidates(g, u, dtype):
    """(h, h_alt, amb) from the saved g and u: amb marks the elements where the two silu candidates give different h."""
    s, s_alt, amb = silu_candidates(g, dtype)
    h0, h1 = h_of(s, u, dtype), h_of(s_alt, u, dtype)
    return h0, h1, amb & (h0 != h1) & np.isfinite(h0) & np.isfinite(h1)


# --------------------------------------------------------------------------- h
@dataclass
class HResult:
    n: int                  # finite (g, u) elements checked
    neighbour: float        # share of them that matched only the neighbour candidate
    ambiguous: float        # share with two candidates


def measure_h(h, g, u, dtype):
    """(HResult, number of elements h gets wrong): finite (g, u) must give h = rnd(s16·u16) for one silu candidate,
    non-finite g or u a non-finite h."""
    h, g, u = (np.asarray(a, dtype=np.float64) for a in (h, g, u))
    fin = np.isfinite(g) & np.isfinite(u)
    h0, h1, amb = h_candidates(g, u, dtype)
    ok0 = h == h0
    ok1 = amb & (h == h1) & ~ok0
    wrong = (fin & ~(ok0 | ok1)) | (~fin & np.isfinite(h))
    n = int(fin.sum())
    return HResult(n, float(ok1.sum()) / max(n, 1), float(amb.sum()) / max(n, 1)), int(wrong.sum())


def check_h(h, g, u, dtype, what="") -> HResult:
    r, wrong = measure_h(h, g, u, dtype)
    assert wrong == 0, f"{what}: {wrong} of {np.size(h)} h elements are not rnd(rnd(silu(g))·u) for either silu candidate"
    return r


# --------------------------------------------------------------------------- y = h·W2 (+ b2)
def reference_down(d2, g, u, path: P.Path, dtype, cols=None) -> P.Ref:
    """Reference of the down projection on the host-side h of the saved g and u (both in the layer's natural column
    order), with Σ|h_alt − h|·|W2| added to F over the elements whose silu has two candidates."""
    h0, h1, amb = h_candidates(g, u, dtype)
    ref = P.reference(d2, h0, path, dtype, cols=cols)
    if amb.any():
        q, z, s, gi, _ = P.layer_parts(d2, dtype, cols)
        W = np.abs(s[gi] * (q - z[gi]))
        extra = (np.where(amb, np.abs(h1 - h0), 0.0) @ W) * (1 + 2.0 ** -7)     # a rounded |W| is at most 2^-8 larger
        if path.pe_max is not None:         # the digit block maximum may be h_alt's
            hx = np.where(amb & (np.abs(h1) > np.abs(h0)), h1, h0)
            ref.F = np.maximum(ref.F, P.reference(d2, hx, path, dtype, cols=cols).F)
        ref.F = ref.F + extra
    return ref


def cat_refs(refs) -> P.Ref:
    """One Ref over the rows of several (same layer shape, same n_terms)."""
    c = lambda name: np.concatenate([getattr(r, name) for r in refs])
    return P.Ref(c("ystar"), c("A"), c("F"), refs[0].n_terms, c("bad_rows"), c("A0"))


# --------------------------------------------------------------------------- combine
def measure_combine(out, y_pair, idx, w, E, dtype):
    """(Result, tokens without a valid id whose output is not exactly 0)."""
    idx = np.asarray(idx).astype(np.int64)
    T, k = idx.shape
    valid = (idx >= 0) & (idx < E)
    y = np.asarray(y_pair, dtype=np.float64).reshape(T, k, -1)
    wv = np.asarray(w, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        terms = np.where(valid[..., None], wv[..., None] * np.where(valid[..., None], y, 0.0), 0.0)
    ystar, A = terms.sum(axis=1), np.abs(terms).sum(axis=1)
    out = np.asarray(out, dtype=np.float64).reshape(ystar.shape)
    none = ~valid.any(axis=1)
    bad_zero = int((out[none] != 0).any(axis=1).sum()) if none.any() else 0
    bad = ~np.isfinite(ystar)               # elementwise: a y_pair may overflow in one column only
    ok_rows = bool(np.all(~np.isfinite(out[bad])))
    ys, yo, Ag = ystar[~bad], out[~bad], A[~bad]
    gam = (k + 1) * U
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(np.isfinite(yo), np.abs(yo - ys) / (P.ulp(ys, dtype) + gam * Ag), np.inf)
    ratio = np.where(yo == P.round_dt(ys, dtype), 0.0, ratio)      # also an overflow to inf that rounding gives
    cond = gam * Ag <= P.ulp(ys, dtype)
    mism = (yo != P.round_dt(ys, dtype)) & cond
    n = int(cond.sum())
    return P.Result(float(ratio.max()) if ratio.size else 0.0, float(mism.sum()) / max(n, 1), n, ok_rows), bad_zero


def check_combine(out, y_pair, idx, w, E, dtype, what="") -> P.Result:
    r, bad_zero = measure_combine(out, y_pair, idx, w, E, dtype)
    lim = P._RATE[P.dt_name(dtype)]
    assert bad_zero == 0, f"{what}: {bad_zero} tokens without a valid expert id have a non-zero output"
    assert r.ok_rows, f"{what}: an output whose y_pair terms are non-finite is finite"
    assert r.worst <= 1.0, f"{what}: combine max err/bound = {r.worst:.3g}"
    assert r.rate <= lim, f"{what}: combine mismatch rate {r.rate:.4f} > {lim} over {r.n_cond} elements"
    return r


# --------------------------------------------------------------------------- whole paths
def check_gate_up(d1, d3, x, g, u, h, path: str, dtype, cols=None, what="") -> dict:
    """g and u against their bound, h exactly from them; g, u, h are the observed [M, cols] columns."""
    pth = P.PATHS[path]
    rg = P.check(g, P.reference(d1, x, pth, dtype, cols=cols), pth, dtype, what=f"{what} g")
    ru = P.check(u, P.reference(d3, x, pth, dtype, cols=cols), pth, dtype, what=f"{what} u")
    rh = check_h(h, g, u, dtype, what=f"{what} h")
    return {"g": rg, "u": ru, "h": rh}


def h_order_inverse(d2):
    """Index that puts saved columns (h's column order: w2's sorted order for an act-order w2) back in natural order."""
    g2 = np.asarray(d2["g_idx"])
    if np.array_equal(g2, O.default_g_idx(d2["K"], d2["group_size"])):
        return None
    return np.argsort(O.make_sequential_perm(g2))


def check_moe(experts, x, idx, w, dtype, up_path: str, down_path: str, g_sv, u_sv, y_sv, out, cols_i=None, cols_h=None,
              what="") -> dict:
    """Every stage of a grouped experts forward from what the saving forward kept: g_sv / u_sv [T·k, I] (pair-id rows,
    h's column order), y_sv [T·k, H], out [T, H].  ``cols_i`` / ``cols_h``: check g, u on columns (i0, i1) of I and
    y_pair, out on columns (h0, h1) of H (h is formed from all of g and u)."""
    E = len(experts)
    idx = np.asarray(idx).astype(np.int64)
    T, k = idx.shape
    x = np.asarray(x, dtype=np.float64)
    g_sv, u_sv, y_sv = (np.asarray(a, dtype=np.float64) for a in (g_sv, u_sv, y_sv))
    I, H = g_sv.shape[1], y_sv.shape[1]
    i0, i1 = cols_i or (0, I)
    h0, h1 = cols_h or (0, H)
    up, down = P.PATHS[up_path], P.PATHS[down_path]
    rg, ru, ry, og, ou, oy = [], [], [], [], [], []
    flat = idx.reshape(-1)
    for e in range(E):
        pid = np.nonzero(flat == e)[0]
        if not pid.size:
            continue
        ex = experts[e]
        inv = h_order_inverse(ex["w2"])
        g, u = (g_sv[pid], u_sv[pid]) if inv is None else (g_sv[pid][:, inv], u_sv[pid][:, inv])
        xe = x[pid // k]
        rg.append(P.reference(ex["w1"], xe, up, dtype, cols=(i0, i1)))
        ru.append(P.reference(ex["w3"], xe, up, dtype, cols=(i0, i1)))
        og.append(g[:, i0:i1])
        ou.append(u[:, i0:i1])
        ry.append(reference_down(ex["w2"], g, u, down, dtype, cols=(h0, h1)))
        oy.append(y_sv[pid, h0:h1])
    res = {"g": P.check(np.concatenate(og), cat_refs(rg), up, dtype, what=f"{what} g"),
           "u": P.check(np.concatenate(ou), cat_refs(ru), up, dtype, what=f"{what} u"),
           "y_pair": P.check(np.concatenate(oy), cat_refs(ry), down, dtype, what=f"{what} y_pair")}
    res["combine"] = check_combine(np.asarray(out, dtype=np.float64)[:, h0:h1], y_sv[:, h0:h1], idx, w, E, dtype,
                                   what=f"{what} combine")
    return res


# --------------------------------------------------------------------------- generators
@functools.lru_cache(maxsize=None)
def realistic_experts(E, H, I, group_size, dtype, seed=0, act13=False, act2=False, bias=False):
    """E experts {"w1", "w3", "w2"} of ``tests/_precision.realistic_layer`` (``wide_layer`` beyond 1024 columns); w1 and
    w3 share one (act-order, with ``act13``) g_idx.  ``group_size`` −1: one group per layer.  Cached: do not mutate."""
    dt = P.dt_name(dtype)
    out = []
    for e in range(E):
        s = seed + 3 * e
        w1 = P.wide_layer(H, I, group_size, dt, seed=s, act_order=act13, bias=bias)
        w3 = P.wide_layer(H, I, group_size, dt, seed=s + 1, bias=bias, g_idx=w1["g_idx"])
        w2 = P.wide_layer(I, H, group_size, dt, seed=s + 2, act_order=act2, bias=bias)
        out.append({"w1": w1, "w3": w3, "w2": w2})
    return tuple(out)
