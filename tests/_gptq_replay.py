"""Float64 references of the GPTQ quantiser's two kernels, with per-element error bounds (tests only).

Quantiser: a teacher-forced replay
    Given Hinv, GPTQ is chaotic across columns: one different rounding changes the error feedback of every later column,
    so comparing codes with a float64 GPTQ says nothing.  But rows are independent given Hinv, and the kernel returns
    every decision it made (codes, per-group scale / zero, Q).  So the replay runs the kernel's own trajectory in float64:
    columns in processing order (act-order ``perm``, 128-column blocks), and at column i

        w_i = W0_i − Σ_{j<i} e_j·U[j,i],   e_j = (w_j − Q_j) / U[j,j]   with the KERNEL's Q_j,

    in the blocked order (in-block steps, then the trailing update ``W[:, i2:] −= E·U[i1:i2, i2:]`` as a float64
    matmul).  The group parameters are the kernel's (checked first, then forced), so its code must be
    ``clamp(rint(w_i / s) + z, 0, 15)`` unless w_i / s lies within its error bound of a rounding midpoint.  Every decision
    is forced, so a legitimate flip cannot cascade: a mismatch on a clear element is a bug.

    Bound of the kernel's fp32 value w̃_i (_precision's conventions: probabilistic fp32 accumulation, λ = 2).  With Q
    forced, the kernel's deviation δ = w̃ − w is linear in the roundings it commits: a rounding ε_k made at column k
    reaches column i as M[k, i]·ε_k: δ_i = ε_i − Σ_{j<i} (δ_j / U[j,j])·U[j,i], so M = U⁻¹·diag(U), one float64
    triangular solve.  The roundings are independent with zero mean, so

        B_i = λ·√(Σ_{k≤i} M[k,i]²·b_k²),   b_k = √(n_k + 64)·u·A_k + 2u·Σ_{j<k} |e_j·U[j,k]|
        A_k = |W0_k| + Σ_{j<k} |e_j·U[j,k]|,   n_k = 2·(k − k1) + k1 + k1 / 128   (k1: start of k's block)

    * b_k is the size of what column k commits itself (_precision's √(n + 64)·u·A), with n_k the roundings it passes
      through in ``gptq_quantize_kernel``: two per earlier column of its own block (``__fmul_rn`` then ``__fsub_rn``),
      one per column of an earlier block (one FMA into the trailing accumulator) and one per earlier block (the
      subtraction of that accumulator); 2u·|e_j·U[j,k]| is err's own two roundings (w − q, then the division by d).
    * The worst case Σ|M[k,i]|·b_k is useless here: on correlated calibration data |M| grows along the columns and the
      worst-case bound of a few hundred columns already covers half of all codes.  The propagated roundings are
      independent, so their root sum of squares is the honest size, as for _precision's sums.
    * A column whose update terms are all exactly zero (dead columns, a diagonal Hinv, block 0 before any update) is
      never rounded: B_i = 0 and the replay demands the exact fp32 arithmetic there, ties included.
    * Dynamic group parameters after the first block read the block-start values; they are checked against the bound of
      the group's final values, which carries every rounding their block-start values carry.

    What is checked (``check_quantize``): g_idx (the oracle's rule); group parameters (bit-equal to
    ``gptq_oracle.find_params`` where they see W before any update: group_size = −1, static groups, every group whose
    columns have B = 0; otherwise within the interval that the bounds of the forced block-start values allow, with
    ``zero`` exact unless −xmin / s is within its bound of a midpoint; sym: zero = 8); codes (no mismatch on clear
    elements, and every code inside its interval); Q bit-equal to fl32(s·(c − z)) in original column order, dead columns
    exactly 0; losses within the bound that B gives ½((w − Q) / d)²; qweight / qzeros / scales bit-equal to
    ``gptq_oracle.pack_codes`` of the codes recovered from Q (bf16 scales through ``_precision.round_dt``).

Hessian: ``HessianReference``
    H* = α·H* + β·XᵀX in float64 over the same batches (α = n / (n + b), β = 2 / (n + b), b the leading dimension of a
    3-D input, 1 for a 2-D one), with an element bound carried through the recurrence: the fp32 rounding of α and β,
    ``_precision.gamma`` of the mma.sync accumulation over T and the epilogue's roundings (two products and one sum).
    The tensor-core factor of that accumulation is calibrated, as _precision's are (``HESS_MMA``).  Sharpness: the share of well-conditioned elements (accumulation budget
    √(T/16)·u·β·Σ|x_i x_j|, carried through α, at most one fp32 ulp) that differ from round_f32(H*).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from oracle import gptq_oracle as GO
from tests import _precision as P

U = P.U
BLOCK = 128
MAXQ = 15
SAFE = 1.0 + 2.0 ** -30          # covers the float64 evaluation of the bounds themselves
TINY = 2.0 ** -149               # fp32's smallest subnormal: the absolute error of an underflowing product
# gptq_hessian_kernel's mma.sync accumulation over T.  Measured on an H100 80GB HBM3 (700 W power limit) over
# tests/test_gpu_26_gptq_precision.py, the largest error needed 5.9 times the fp32 γ = λ·√(T/4 + 64)·u·Σ|x_i x_j| at
# T = 4097 per call (0.16 at T <= 33): more than _precision.TC_GAMMA = 2, as sums of 2048-4097 same-sign products of
# massive channels are where the tensor core's internal alignment shows.  The factor 9 sits 1.5x above that.
HESS_MMA = P.Path("hessian_mma", tc=True, tc_gamma=9.0)


def g_idx_rule(K, group_size, perm=None, static_groups=False) -> np.ndarray:
    """g_idx as gptq_oracle.fasterquant derives it: group of the processing position, unpermuted to original order;
    static act-order groups follow the original column."""
    gs = K if group_size == -1 else group_size
    pos = np.arange(K)
    if perm is None:
        return (pos // gs).astype(np.int32)
    perm = np.asarray(perm)
    g_proc = perm // gs if (static_groups and group_size != -1) else pos // gs
    return g_proc[np.argsort(perm)].astype(np.int32)


def ulp32(a: torch.Tensor) -> torch.Tensor:
    """Spacing of fp32 numbers at |a| (float64 in, float64 out; subnormal spacing below the normal range)."""
    _, e = torch.frexp(a.abs())
    e = torch.clamp(e.to(torch.int64) - 1, min=-126) - 23
    return torch.where(a == 0, torch.full_like(a, TINY), torch.ldexp(torch.ones_like(a), e))


# --------------------------------------------------------------------------- quantiser
@dataclass
class QuantMeasure:
    elements: int
    unclear: float          # share of codes whose float64 value lies within its bound of a rounding midpoint
    flipped: float          # share of those unclear codes that differ from the float64 rounding
    worst: float            # largest err / bound over the losses and the bound-checked scales
    params_unclear: int     # zero points whose −xmin / s lies within its bound of a midpoint


def _find_params_exact(w: torch.Tensor, sym):
    s, z = GO.find_params(w.float().cpu().numpy(), sym)
    return torch.from_numpy(s).double().to(w.device), torch.from_numpy(z).double().to(w.device)


def _check_params_bounded(w, Bg, s_k, z_k, sym, what):
    """Kernel parameters s_k, z_k [R] of groups whose forced values w [R, L] are known to within Bg [R] each.  Returns
    (largest err / bound of the scales, number of unclear zero points)."""
    wmin, wmax = w.min(1).values, w.max(1).values
    mn_lo, mn_hi = torch.clamp(wmin - Bg, max=0), torch.clamp(wmin + Bg, max=0)
    mx_lo, mx_hi = torch.clamp(wmax - Bg, min=0), torch.clamp(wmax + Bg, min=0)
    mn, mx = torch.clamp(wmin, max=0), torch.clamp(wmax, min=0)
    if sym:
        m_lo, m_hi = torch.maximum(-mn_hi, mx_lo), torch.maximum(-mn_lo, mx_hi)
        r_lo, r_hi = torch.minimum(mx_lo, 2 * m_lo), 2 * m_hi
        r = torch.where(mn < 0, 2 * torch.maximum(-mn, mx), mx)
    else:
        r_lo, r_hi, r = mx_lo - mn_hi, mx_hi - mn_lo, mx - mn
    r_hi = torch.where(r_lo == 0, torch.clamp(r_hi, min=2.0), r_hi)        # an all-zero group reads as [-1, 1]
    r = torch.where(r == 0, torch.full_like(r, 2.0), r)
    s_lo, s_hi, s = r_lo / 15 * (1 - 3 * U), r_hi / 15 * (1 + 3 * U) * SAFE, r / 15
    ratio = torch.where(s_k >= s, (s_k - s) / (s_hi - s), (s - s_k) / (s - s_lo))
    bad = ~(ratio <= 1)
    assert not bad.any(), f"{what}: {int(bad.sum())} scales outside their bound (s = {s_k[bad][:4].tolist()}, " \
                          f"float64 {s[bad][:4].tolist()})"
    if sym:
        assert bool((z_k == 8).all()), f"{what}: a symmetric zero point is not 8"
        return float(ratio.max()), 0
    t_lo = -mn_hi / s_k * (1 - U)
    t_hi = torch.where(r_lo == 0, torch.clamp(-mn_lo, min=1.0), -mn_lo) / s_k * (1 + U) * SAFE
    z_lo, z_hi = torch.round(t_lo), torch.round(t_hi)
    bad = (z_k < z_lo) | (z_k > z_hi)
    assert not bad.any(), f"{what}: {int(bad.sum())} zero points outside [{z_lo[bad][:4].tolist()}, {z_hi[bad][:4].tolist()}]"
    return float(ratio.max()), int((z_lo != z_hi).sum())


def check_quantize(W0, Hinv, out, perm=None, dead=None, group_size=-1, sym=True, static_groups=False,
                   dtype=torch.float16, what="") -> QuantMeasure:
    """Replay one ``gptq_quantize_kernel`` result in float64 on W0's device and assert every check listed in the module
    docstring.  ``W0`` [N, K] fp32 original order (before the dead columns are zeroed), ``Hinv`` fp32 [K, K] processing
    order, ``perm`` processing position -> original column, ``dead`` bool [K] original order.  ``out`` holds the
    kernel's Q [N, K] (original order), scale / zero [N, G], qweight, qzeros, scales [G, N] in ``dtype``, g_idx and
    losses [N, K] (original order, or None)."""
    dev = W0.device
    N, K = W0.shape
    gs = K if group_size == -1 else group_size
    G = -(-K // gs)
    static = bool(static_groups) and group_size != -1
    dynamic = group_size != -1 and not static
    perm_np = None if perm is None else np.asarray(torch.as_tensor(perm).cpu(), dtype=np.int64)
    perm_t = torch.arange(K, device=dev) if perm is None else torch.as_tensor(perm_np, device=dev)
    dead_t = None if dead is None else torch.as_tensor(dead, device=dev).bool()
    get = lambda k: torch.as_tensor(out[k], device=dev)          # noqa: E731

    # g_idx, and the group each processing position uses
    g_idx = g_idx_rule(K, group_size, perm_np, static_groups)
    np.testing.assert_array_equal(np.asarray(torch.as_tensor(out["g_idx"]).cpu()), g_idx, err_msg=f"{what}: g_idx")
    pos_grp = torch.as_tensor(g_idx, device=dev).long()[perm_t]

    s_k, z_k = get("scale").double(), get("zero").double()
    assert s_k.shape == z_k.shape == (N, G), f"{what}: parameter shape {tuple(s_k.shape)}"
    W = W0.double().clone()
    if dead_t is not None:
        W[:, dead_t] = 0
    worst, params_unclear = 0.0, 0

    # parameters that see W before any update: bit-equal to find_params in fp32
    if group_size == -1:
        s, z = _find_params_exact(W0, sym)
        assert torch.equal(s_k[:, 0], s) and torch.equal(z_k[:, 0], z), f"{what}: group_size=-1 parameters"
    elif static:
        for g in range(G):
            s, z = _find_params_exact(W[:, g * gs:(g + 1) * gs], sym)
            assert torch.equal(s_k[:, g], s) and torch.equal(z_k[:, g], z), f"{what}: static group {g} parameters"

    Wc = W[:, perm_t].contiguous()                  # current outer W, processing order
    W0a = Wc.abs()
    U64 = torch.as_tensor(Hinv, device=dev).double()
    Ua = U64.abs()
    d = torch.diagonal(U64).clone()
    Q = get("Q").float()
    Qp = Q.double()[:, perm_t]
    Ac = torch.zeros_like(Wc)                       # Σ_j |e_j·U[j,i]|
    w_fin = torch.empty_like(Wc)
    starts = {}                                     # dynamic group -> (its block-start values, rows not yet updated)
    for i1 in range(0, K, BLOCK):
        i2 = min(i1 + BLOCK, K)
        nb = i1 // BLOCK
        if dynamic:
            for g in range(-(-i1 // gs), (i2 - 1) // gs + 1):
                if g * gs < i2:
                    cols = slice(g * gs, min(g * gs + gs, K))
                    starts[g] = (Wc[:, cols].clone(), (Ac[:, cols] == 0).all(1))
        cnt = i2 - i1
        W1, A1 = Wc[:, i1:i2].clone(), Ac[:, i1:i2].clone()
        Ub, Uab = U64[i1:i2, i1:i2], Ua[i1:i2, i1:i2]
        E = torch.zeros((N, cnt), dtype=torch.float64, device=dev)
        for i in range(cnt):
            col = i1 + i
            w = W1[:, i]
            w_fin[:, col] = w
            E[:, i] = (w - Qp[:, col]) / d[col]
            if i + 1 < cnt:
                W1[:, i + 1:] -= E[:, i:i + 1] * Ub[i, i + 1:]
                A1[:, i + 1:] += E[:, i:i + 1].abs() * Uab[i, i + 1:]
        Ac[:, i1:i2] = A1
        if i2 < K:
            Wc[:, i2:] -= E @ U64[i1:i2, i2:]
            Ac[:, i2:] += E.abs() @ Ua[i1:i2, i2:]
    del Wc, Ua
    # b_k, then B = λ·√(b² · M²) with M = U⁻¹·diag(U)
    k = torch.arange(K, device=dev, dtype=torch.float64)
    k1 = torch.div(k, BLOCK, rounding_mode="floor")
    n = 2 * (k - k1 * BLOCK) + k1 * BLOCK + k1
    b = torch.where(Ac > 0, torch.sqrt(n + 64) * U * (W0a + Ac) + 2 * U * Ac, torch.zeros_like(Ac))
    del Ac, W0a
    M = torch.linalg.solve_triangular(U64, torch.diag(d), upper=True)
    M.square_()
    B_fin = P.LAMBDA * torch.sqrt((b * b) @ M) * SAFE
    del M, b
    for g, (w, ex) in starts.items():
        Bg = B_fin[:, g * gs:g * gs + w.shape[1]].max(1).values
        if ex.any():
            s, z = _find_params_exact(w[ex], sym)
            assert torch.equal(s_k[ex, g], s) and torch.equal(z_k[ex, g], z), \
                f"{what}: group {g} parameters (before any update)"
        if (~ex).any():
            r, nu = _check_params_bounded(w[~ex], Bg[~ex], s_k[~ex, g], z_k[~ex, g], sym, f"{what}: group {g}")
            worst, params_unclear = max(worst, r), params_unclear + nu
    del starts

    # Q: fl32(s·(c − z)) of the codes it encodes, original order; dead columns exactly 0
    gi = torch.as_tensor(g_idx, device=dev).long()
    S_o, Z_o = s_k[:, gi], z_k[:, gi]
    c_o = torch.round(Q.double() / S_o) + Z_o
    assert bool(((c_o >= 0) & (c_o <= MAXQ)).all()), f"{what}: Q holds a value outside the 4-bit grid"
    Qx = (S_o * (c_o - Z_o)).float()
    bad = Qx != Q
    assert not bad.any(), f"{what}: {int(bad.sum())} elements of Q are not fl32(s·(c − z))"
    if dead_t is not None:
        assert bool((Q[:, dead_t] == 0).all()), f"{what}: a dead column does not dequantise to 0"
    del Qx, S_o, Z_o

    # codes against the replay
    C = c_o[:, perm_t]
    S, Z = s_k[:, pos_grp], z_k[:, pos_grp]
    t = w_fin / S
    exact = B_fin == 0
    t32 = t.float().double()                        # w is an fp32 value there: the correctly rounded quotient
    delta = (B_fin + U * (w_fin.abs() + B_fin)) / S * SAFE
    clamp = lambda x: torch.clamp(torch.round(x) + Z, 0, MAXQ)      # noqa: E731
    c_lo = clamp(torch.where(exact, t32, t - delta))
    c_hi = clamp(torch.where(exact, t32, t + delta))
    c_nom = clamp(torch.where(exact, t32, t))
    wrong = (C < c_lo) | (C > c_hi)
    if wrong.any():
        r, k = (int(v) for v in wrong.nonzero()[0])
        raise AssertionError(f"{what}: {int(wrong.sum())} codes outside their interval (first: row {r}, position {k}: "
                             f"code {int(C[r, k])}, float64 w/s = {float(t[r, k])!r} ± {float(delta[r, k]):.3g}, "
                             f"zero {float(Z[r, k])})")
    unclear = c_lo != c_hi
    n_unclear = int(unclear.sum())
    flipped = int(((C != c_nom) & unclear).sum())
    del t, t32, delta, c_lo, c_hi, c_nom, C, S, Z

    # losses: ½((w̃ − Q) / d)² with |w̃ − w| ≤ B, three fp32 roundings and underflow
    if out.get("losses") is not None:
        Lk = get("losses").double()[:, perm_t]
        D = (w_fin - Qp).abs()
        Dx = (D + B_fin + U * (D + B_fin)) * SAFE
        d2 = d * d
        L = 0.5 * D * D / d2
        bound = (Dx * Dx - D * D) / (2 * d2) + 4 * U * Dx * Dx / (2 * d2) + TINY * (1 / d2 + 2)
        ratio = (Lk - L).abs() / bound
        worst = max(worst, float(ratio.max()))
        bad = ~(ratio <= 1)
        assert not bad.any(), f"{what}: {int(bad.sum())} losses outside their bound (max err/bound {float(ratio.max()):.3g})"
        del Lk, D, Dx, L, bound, ratio

    # packing: the codes recovered from Q through gptq_oracle.pack_codes; bf16 scales through round_dt
    codes = c_o.to(torch.uint8).cpu().numpy()
    qw, qz, sc16 = GO.pack_codes(codes, z_k.cpu().numpy(), s_k.float().cpu().numpy())
    np.testing.assert_array_equal(np.asarray(torch.as_tensor(out["qweight"]).cpu()), qw, err_msg=f"{what}: qweight")
    np.testing.assert_array_equal(np.asarray(torch.as_tensor(out["qzeros"]).cpu()), qz, err_msg=f"{what}: qzeros")
    scales = torch.as_tensor(out["scales"]).cpu()
    if dtype == torch.bfloat16:
        ref = P.round_dt(s_k.T.cpu().numpy(), "bfloat16").astype(np.float32)
        got = scales.float().numpy()
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), f"{what}: bf16 scales"
    else:
        assert scales.dtype == torch.float16
        assert np.array_equal(scales.numpy().view(np.uint16), sc16.view(np.uint16)), f"{what}: fp16 scales"
    return QuantMeasure(N * K, n_unclear / (N * K), flipped / max(n_unclear, 1), worst, params_unclear)


# --------------------------------------------------------------------------- Hessian
@dataclass
class HessMeasure:
    worst: float            # largest |H − H*| / bound
    rate: float             # share of well-conditioned elements with H != round_f32(H*)
    n_cond: int


class HessianReference:
    """Float64 running mean of the batches given to ``GPTQ.add_batch``, with its element bound E and the
    accumulation budget C that defines the well-conditioned elements."""

    def __init__(self, K, device):
        z = lambda: torch.zeros((K, K), dtype=torch.float64, device=device)     # noqa: E731
        self.K, self.H, self.E, self.C, self.n = K, z(), z(), z(), 0

    def add(self, x: torch.Tensor):
        b = 1 if x.dim() == 2 else int(x.shape[0])
        n1 = self.n + b
        alpha, beta = (self.n / n1, 2.0 / n1) if n1 > 0 else (0.0, 0.0)
        self.n = n1
        X = x.reshape(-1, self.K).to(self.H.device, torch.float64)
        T = X.shape[0]
        gT = P.gamma(HESS_MMA, T)
        Xa = X.abs()
        Sa = Xa.T @ Xa                              # the accumulation's uncancelled magnitude
        del Xa
        # E' = (α·E + β·γ_T·Sa)(1 + 3u) + 2u·(α|H*| + β|S|) + u·|H*'| + underflow
        self.E.mul_(alpha).add_(Sa, alpha=beta * gT).mul_(1 + 3 * U)
        self.C.mul_(alpha).add_(Sa, alpha=math.sqrt(T / 16) * U * beta)
        del Sa
        self.E.add_(self.H.abs(), alpha=2 * U * alpha)
        S = X.T @ X
        del X
        self.H.mul_(alpha).add_(S, alpha=beta)
        self.E.add_(S.abs(), alpha=2 * U * beta)
        del S
        self.E.add_(self.H.abs(), alpha=U).add_(TINY * (beta * T + 2)).mul_(SAFE)

    def measure(self, H: torch.Tensor, rows=2048) -> HessMeasure:
        """err / bound and the mismatch rate of a kernel result H (fp32 [K, K]), in row chunks."""
        worst, mism, n_cond = 0.0, 0, 0
        for r0 in range(0, self.K, rows):
            h = H[r0:r0 + rows].to(self.H.device, torch.float64)
            hs = self.H[r0:r0 + rows]
            ratio = (h - hs).abs() / self.E[r0:r0 + rows]
            worst = max(worst, float(torch.nan_to_num(ratio, nan=math.inf).max()))
            cond = self.C[r0:r0 + rows] <= ulp32(hs)
            mism += int(((h != hs.float().double()) & cond).sum())
            n_cond += int(cond.sum())
        return HessMeasure(worst, mism / max(n_cond, 1), n_cond)

    def check(self, H: torch.Tensor, rate_limit, what="", min_cond=1000) -> HessMeasure:
        """Assert the bound, and the rate limit where at least ``min_cond`` elements are well-conditioned (a rate over
        a handful of elements says nothing; it is then reported as 0)."""
        r = self.measure(H)
        assert r.worst <= 1.0, f"{what}: max err/bound = {r.worst:.3g}"
        if r.n_cond < min_cond:
            return HessMeasure(r.worst, 0.0, r.n_cond)
        assert r.rate <= rate_limit, f"{what}: mismatch rate {r.rate:.4f} > {rate_limit} over {r.n_cond} elements"
        return r
