"""Ulp-level precision checker for the W4A16 kernels: a float64 reference, a per-element error bound derived from each
kernel path's arithmetic, a sharpness (mismatch-rate) check, and generators of realistic layers and activations.

Reference
    y* = x·W + b in float64, with the scales and the bias rounded to the compute dtype (the device holds them so), the
    wrap rule of the zero points and ``g_idx``.  W = s·(q − z) is exact for the exact-weight paths (GEMV, skinny, both
    IMMA forms, the decode chain) and rounded once to the dtype for the tensor-core paths (wgmma GEMM, both dgrad
    kernels), as those kernels round it.

Per-element bound
    |y − y*| ≤ ulp_dt(y*) + γ·A + F

    * ulp_dt(y*): the single output rounding (half an ulp) plus the room that the accumulated error gives it to round
      the other way (the other half).
    * A = Σ_k |x_k|·s·(q_k + z + o) + |b| is the uncancelled magnitude of what the kernel actually sums.  Every
      small-M kernel forms s·(Σ q·x − z·Σx) per group, so its partial sums are bounded by Σ|x|·s·(q + z); the bf16
      unpack reads each nibble as 128 + q, which adds o = 128 to the summed terms (``gemv.cuh`` flush, ``skinny.cuh``
      epilogue).  Near-zero outputs have a tiny ulp, so γ·A is what
      bounds them, and it is what a cancellation bug has to get past.
    * γ bounds the relative fp32 accumulation error.  Every product is exact in fp32 (two 16-bit significands, or an
      exact int32 dot product on the IMMA paths), so the error is that of an fp32 sum of n terms whose partial sums are
      all bounded by A.  Each addition commits an error of at most u·|S_i| ≤ u·A, u = 2^-24; these errors have zero
      mean and are independent enough that their sum stays below λ·√n·u·A (Higham & Mary's probabilistic bound,
      λ = 2, i.e. about 3.5 standard deviations of a sum of uniform errors).  n is the longest chain one term can
      pass through: at most K/4 (a GEMV lane accumulates 4 products per k8-row into one register when it owns every
      row of a group) plus 64 for the group flushes and the shuffle / warp / split-K / cluster reductions.  So
      γ = 2·√(K/4 + 64)·2^-24: 66·2^-24 at K = 4096, 106·2^-24 at K = 11008.
      The tensor-core paths (mma.sync on the skinny kernel, wgmma on the GEMM and dgrad) accumulate inside the tensor
      core, whose internal alignment and rounding on Hopper is not documented; their γ carries a factor ``TC_GAMMA``
      measured on an H100 (see ``PATHS``).
    * F, for the IMMA paths and the chain only, is the block-fixed-point rounding of x: per row and 128-k block the
      kernel rounds x·2^pe to an integer, |x|max·2^pe ∈ [2^21, 2^22), so each element errs by at most
      2^-(pe+1) ≤ 2^-22·|x|max (``tests/test_imma_format_cpu.py``), and the output by that times Σ|W| over the block.
      pe is clamped at 126 (IMMA) / 120 (chain); bf16 rows whose block maximum is below 2^-105 (2^-99) then keep an
      absolute error of 2^-127 (2^-121) per element instead of the relative one, and a block whose maximum is an fp32
      subnormal (e == 0) is read as zero.  F follows the clamp, so the bound states that domain exactly.

Sharpness
    The per-element bound is a worst case and lets a sub-ulp bug through.  So the fraction of elements that differ from
    round_dt(y*) is bounded as well, over the elements whose error budget √n·u·A is at most one ulp (the others are
    ill-conditioned: the fp32 formulation alone may move them to a neighbouring value).  On those elements the model
    predicts a mismatch rate of well under the budget; the limits in ``PATHS`` are a few percent for fp16 and under
    1 % for bf16 on the fp32 paths, and the measured H100 rates are recorded next to them.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle import w4a16_oracle as O

U = 2.0 ** -24                       # fp32 unit roundoff
LAMBDA = 2.0

# (mantissa bits, minimum normal exponent, largest finite value)
_FMT = {"float16": (10, -14, 65504.0), "bfloat16": (7, -126, float((2 - 2 ** -7) * 2.0 ** 127))}


def dt_name(dtype) -> str:
    s = str(dtype)
    return "bfloat16" if "bfloat16" in s else "float16"


# --------------------------------------------------------------------------- rounding
def ulp(a, dtype) -> np.ndarray:
    """Spacing of the dtype's numbers at |a| (subnormal spacing below the normal range)."""
    m, emin, _ = _FMT[dt_name(dtype)]
    a = np.abs(np.asarray(a, dtype=np.float64))
    a = np.where(np.isfinite(a), a, 1.0)
    with np.errstate(divide="ignore"):
        e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    e = np.maximum(np.where(a > 0, e, emin), emin)
    return np.ldexp(1.0, (e - m).astype(np.int64))


def round_dt(a, dtype) -> np.ndarray:
    """Correctly rounded (to nearest even) conversion of float64 values to the dtype, returned as float64."""
    _, _, vmax = _FMT[dt_name(dtype)]
    a = np.asarray(a, dtype=np.float64)
    q = ulp(a, dtype)
    with np.errstate(invalid="ignore"):
        r = np.rint(a / q) * q                         # power-of-two scaling: exact; rint rounds half to even
        r = np.where(np.abs(r) > vmax, np.copysign(np.inf, a), r)
    return np.where(np.isfinite(a), r, a)


# --------------------------------------------------------------------------- paths
@dataclass(frozen=True)
class Path:
    """How a kernel path computes: which weights it uses, what it adds to the summed terms, its accumulation γ factor,
    block-fixed-point clamp (None: no F term) and its mismatch-rate limits per dtype."""
    name: str
    round_w: bool = False
    offset: dict = None              # dtype -> o added to q in A
    tc: bool = False                 # accumulates inside the tensor core: γ times TC_GAMMA
    pe_max: int | None = None
    rate: dict = None                # dtype -> mismatch-rate limit
    tc_gamma: float | None = None    # this path's own tensor-core factor (None: TC_GAMMA)

    def o(self, dtype):
        return (self.offset or {}).get(dt_name(dtype), 0)


# Hopper's tensor-core accumulation is calibrated, not derived.  Measured on an H100 80GB HBM3 (700 W power limit) over
# the whole matrix of tests/test_gpu_17_precision.py, the largest share of the fp32 γ = λ·√n·u·A a result needed beyond
# its half-ulp output rounding was 0.40 (wgmma dgrad, fp16), 0.22 (mma.sync skinny, fp16), 0.18 (wgmma GEMM, fp16) against
# 0.22 / 0.10 for the CUDA-core dgrad / GEMV.  TC_GAMMA = 2 leaves a factor 5 above the largest.  The fused backwards'
# stages (tests/test_gpu_28_backward_stages.py) needed up to 0.60 (dense dx, n = 2I) and, on the experts' fp32 dx_pair
# that no 16-bit rounding hides, 1.01: there TC_GAMMA = 2 leaves a factor 2.
TC_GAMMA = 2.0
_BF = {"bfloat16": 128}
# Mismatch-rate limits (fraction of well-conditioned elements with y != round(y*)).  Largest rates measured on the H100
# over the same matrix: fp16 0.41 % (CUDA-core / IMMA paths), 2.5 % (mma.sync skinny); bf16 0.38 %.  The sharpness
# mutant (weights rounded to fp16 on an exact-weight path) gives about 25 %.
_RATE = {"float16": 0.05, "bfloat16": 0.01}
PATHS = {
    "gemv": Path("gemv", offset=_BF, rate=_RATE),
    "skinny": Path("skinny", offset=_BF, tc=True, rate=_RATE),
    "imma": Path("imma", pe_max=126, rate=_RATE),
    "chain": Path("chain", pe_max=120, rate=_RATE),
    "gemm": Path("gemm", round_w=True, tc=True, rate=_RATE),
    "dgrad": Path("dgrad", round_w=True, tc=True, rate=_RATE),
    "dgrad_cuda_core": Path("dgrad_cuda_core", round_w=True, rate=_RATE),
    # moe_decode_kernel (the experts' decode path and the dense gate/up pair at M <= 8): the skinny arithmetic, but on
    # fp16 activations with massive channels it needed up to 4.0 of the fp32 γ (g and u, K = 512) and 5.9 % mismatches
    # (bf16: 0.07 of γ, 1.3 %) on the H100 (tests/test_gpu_20_silu_mul_precision.py), beyond TC_GAMMA and _RATE; its
    # own factor and limits sit 1.5x / 1.7x above that (DESIGN §3.12)
    "decode_mma": Path("decode_mma", offset=_BF, tc=True, tc_gamma=6.0, rate={"float16": 0.10, "bfloat16": 0.03}),
}


_PLAIN = Path("plain")


def gamma(path: Path, n_terms: int) -> float:
    """Relative fp32 accumulation bound γ for a sum over ``n_terms`` (K for the forward, N for dgrad)."""
    g = LAMBDA * np.sqrt(n_terms / 4 + 64) * U
    return g * (path.tc_gamma or TC_GAMMA) if path.tc else g


# --------------------------------------------------------------------------- reference
@dataclass
class Ref:
    ystar: np.ndarray       # float64 [M, n]
    A: np.ndarray           # uncancelled magnitude
    F: np.ndarray           # block-fixed-point term (zeros when the path has none)
    n_terms: int
    bad_rows: np.ndarray    # rows of x that hold a non-finite value
    A0: np.ndarray = None   # A without the unpack offset o (the bound of a kernel that sums s·(q − z)·x)


def layer_parts(d, dtype, cols=None):
    """q [K, n] int, z [G, n] int (wrap rule), s [G, n] float64 rounded to dtype, g [K] int, b [n] or None."""
    n0, n1 = cols or (0, d["N"])
    q = O.unpack_qweight(np.asarray(d["qweight"])[:, n0:n1]).astype(np.int64)
    z = O.unpack_qzeros(np.asarray(d["qzeros"])[:, n0 // 8:n1 // 8]).astype(np.int64)
    s = round_dt(np.asarray(d["scales"], dtype=np.float64)[:, n0:n1], dtype)
    g = np.asarray(d["g_idx"]).astype(np.int64)
    b = None if d.get("bias") is None else round_dt(np.asarray(d["bias"], dtype=np.float64)[n0:n1], dtype)
    return q, z, s, g, b


def _weights(q, z, s, g, dtype, round_w):
    W = s[g] * (q - z[g]).astype(np.float64)
    return round_dt(W, dtype) if round_w else W


def _block_F(x, W, perm, pe_max):
    """Σ over 128-k blocks (in the kernel's k order: sorted by group for act-order layers) of
    min(2^-(pe+1), |x|max) · Σ_block |W| — the output error the digit rounding of x can cause."""
    M, K = x.shape
    xs = x if perm is None else x[:, perm]
    Ws = np.abs(W if perm is None else W[perm])
    F = np.zeros((M, W.shape[1]))
    for k0 in range(0, K, 128):
        xb = np.abs(xs[:, k0:k0 + 128])
        xmax = np.where(np.isfinite(xb), xb, 0).max(axis=1).astype(np.float32)
        e = ((xmax.view(np.uint32) >> 23) & 255).astype(np.int64)
        pe = np.where(e == 0, 0, np.minimum(148 - e, pe_max))
        step = np.minimum(np.ldexp(1.0, -(pe + 1)), xmax.astype(np.float64))
        F += step[:, None] * Ws[k0:k0 + 128].sum(axis=0)[None, :]
    return F


def reference(d, x, path: Path, dtype, cols=None) -> Ref:
    """y*, A and F of one layer on activations ``x`` (float array already representable in ``dtype``)."""
    x = np.asarray(x, dtype=np.float64).reshape(-1, d["K"])
    q, z, s, g, b = layer_parts(d, dtype, cols)
    W = _weights(q, z, s, g, dtype, path.round_w)
    bad = ~np.isfinite(x).all(axis=1)
    xf = np.where(np.isfinite(x), x, 0.0)
    ystar = xf @ W
    A0 = np.abs(xf) @ (s[g] * (q + z[g]))
    A = A0 + path.o(dtype) * (np.abs(xf) @ s[g]) if path.o(dtype) else A0
    if b is not None:
        ystar = ystar + b
        A, A0 = A + np.abs(b), A0 + np.abs(b)
    F = np.zeros_like(ystar)
    if path.pe_max is not None:
        perm = None if np.array_equal(g, np.arange(d["K"]) // d["group_size"]) else O.make_sequential_perm(g)
        F = _block_F(xf, W, perm, path.pe_max)
    return Ref(ystar, A, F, d["K"], bad, A0)


def reference_dgrad(d, dy, path: Path, dtype) -> Ref:
    """dx* = dy·Wᵀ in float64 with W rounded once to the dtype (both dgrad kernels round s·(q − z) so)."""
    dy = np.asarray(dy, dtype=np.float64).reshape(-1, d["N"])
    q, z, s, g, _ = layer_parts(d, dtype)
    W = _weights(q, z, s, g, dtype, True)
    return Ref(dy @ W.T, np.abs(dy) @ np.abs(W).T, np.zeros((dy.shape[0], d["K"])), d["N"], ~np.isfinite(dy).all(axis=1))


def without_offset(ref: Ref) -> Ref:
    """The same reference with the bound of a kernel that sums s·(q − z)·x directly (o = 0)."""
    return Ref(ref.ystar, ref.A0, ref.F, ref.n_terms, ref.bad_rows, ref.A0)


# --------------------------------------------------------------------------- the check
@dataclass
class Result:
    worst: float            # max err / bound over finite rows
    rate: float             # mismatch rate over well-conditioned elements
    n_cond: int
    ok_rows: bool           # non-finite input rows came out non-finite
    g_used: float = 0.0     # largest (err − ½ulp − F) / (λ·√n·u·A): the share of the fp32 γ the result needed

    def passed(self, rate_limit):
        return self.worst <= 1.0 and self.rate <= rate_limit and self.ok_rows


def measure(y, ref: Ref, path: Path, dtype) -> Result:
    y = np.asarray(y, dtype=np.float64).reshape(ref.ystar.shape)
    good = ~ref.bad_rows
    ok_rows = bool(np.all(~np.isfinite(y[ref.bad_rows]).any(axis=1))) if ref.bad_rows.any() else True
    ys, yg = ref.ystar[good], y[good]
    gam = gamma(path, ref.n_terms)
    bound = ulp(ys, dtype) + gam * ref.A[good] + ref.F[good]
    with np.errstate(invalid="ignore"):
        ratio = np.abs(yg - ys) / bound
    # an infinite y is the correct rounding of a result the bound allows beyond the dtype's overflow threshold
    over = np.isinf(yg) & (np.sign(yg) == np.sign(ys)) & (np.abs(ys) + bound >= _FMT[dt_name(dtype)][2] + 0.5 * ulp(
        _FMT[dt_name(dtype)][2], dtype))
    ratio = np.where(np.isfinite(yg), ratio, np.where(over, 0.0, np.inf))
    worst = float(ratio.max()) if ratio.size else 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        excess = np.maximum(np.abs(yg - ys) - 0.5 * ulp(ys, dtype) - ref.F[good], 0) / (gamma(_PLAIN, ref.n_terms) * ref.A[good])
    g_used = float(np.nanmax(np.where(np.isfinite(excess), excess, 0))) if excess.size else 0.0
    cond = (np.sqrt(ref.n_terms / 4 + 64) * U * ref.A[good] + ref.F[good]) <= ulp(ys, dtype)
    mism = (yg != round_dt(ys, dtype)) & cond
    n_cond = int(cond.sum())
    rate = float(mism.sum()) / max(n_cond, 1)
    return Result(worst, rate, n_cond, ok_rows, g_used)


def check(y, ref: Ref, path: Path, dtype, what="") -> Result:
    """Assert the per-element bound and the mismatch-rate limit; return the measurement for the summary."""
    r = measure(y, ref, path, dtype)
    lim = path.rate[dt_name(dtype)]
    assert r.ok_rows, f"{what}: a row of x with a non-finite value gave a finite output row"
    assert r.worst <= 1.0, f"{what}: max err/bound = {r.worst:.3g} (γ = {gamma(path, ref.n_terms) / U:.0f}·2^-24)"
    assert r.rate <= lim, f"{what}: mismatch rate {r.rate:.4f} > {lim} over {r.n_cond} well-conditioned elements"
    return r


# --------------------------------------------------------------------------- layer generator
def realistic_layer(K, N, group_size, dtype, seed=0, act_order=False, bias=False, wrap_groups=True, g_idx=None):
    """GPTQ-like layer: Gaussian weights whose output columns spread log-uniformly over two decades, three heavy
    columns (×10), asymmetric round-to-nearest per group (scale = range / 15, zero = round(−min / scale)), so
    (q − z) is centred near zero.  ``wrap_groups``: a few (group, column) blocks are all positive, so their zero is 0
    and is stored as the nibble 15 (the wrap rule).  bf16 layers carry a band of columns scaled by 1e-4, whose scales
    lie below fp16's normal range.  The bias follows the column's magnitude.  Scales and bias are rounded to ``dtype``; packing goes through oracle.pack_*."""
    dn = dt_name(dtype)
    rng = np.random.default_rng(seed)
    gs = K if group_size == -1 else group_size
    G = -(-K // gs)
    col = 10.0 ** rng.uniform(-1.0, 1.0, size=N)
    col[rng.choice(N, 3, replace=False)] *= 10.0
    if dn == "bfloat16":
        col[: max(8, N // 16)] *= 1e-4
    W = rng.standard_normal((K, N)) * col[None, :] * 0.02
    if g_idx is None:
        g_idx = O.default_g_idx(K, gs)
        if act_order:
            g_idx = g_idx[np.argsort(rng.permutation(K))].astype(np.int32)
    if wrap_groups:
        for _ in range(max(2, G * N // 200)):
            gi, n = int(rng.integers(G)), int(rng.integers(N))
            rows = g_idx == gi
            W[rows, n] = np.abs(W[rows, n])
    s = np.zeros((G, N))
    z = np.zeros((G, N), dtype=np.int64)
    sequential = np.array_equal(g_idx, O.default_g_idx(K, gs))
    for gi in range(G):
        blk = W[gi * gs:(gi + 1) * gs] if sequential else W[g_idx == gi]     # same rows; a view is faster
        lo, hi = np.minimum(blk.min(axis=0), 0), np.maximum(blk.max(axis=0), 0)
        s[gi] = np.maximum(hi - lo, 1e-12) / 15
        s[gi] = round_dt(s[gi], dn)
        z[gi] = np.clip(np.rint(-lo / s[gi]), 0, 15)
    q = np.clip(np.rint(W / s[g_idx] + z[g_idx]), 0, 15).astype(np.uint32)
    b = round_dt(rng.standard_normal(N) * col * 0.1, dn).astype(np.float32) if bias else None
    return dict(qweight=O.pack_rows(q), qzeros=O.pack_cols(((z - 1) & 15).astype(np.uint32)),
                scales=s.astype(np.float32), g_idx=np.asarray(g_idx, dtype=np.int32), bias=b, K=K, N=N, group_size=gs)


def wide_layer(K, N, group_size, dtype, seed=0, act_order=False, bias=False, block=1024, g_idx=None):
    """A large layer built from ``realistic_layer`` blocks of ``block`` output columns (each with its own seed, one
    shared g_idx), so 28672-wide layers are generated at a bounded memory cost.  ``g_idx``: use this one (a sibling's)."""
    if N <= block:
        return realistic_layer(K, N, group_size, dtype, seed=seed, act_order=act_order, bias=bias, g_idx=g_idx)
    first = realistic_layer(K, block, group_size, dtype, seed=seed, act_order=act_order, bias=bias, g_idx=g_idx)
    parts = [first] + [realistic_layer(K, min(block, N - n0), group_size, dtype, seed=seed + 1 + i, bias=bias,
                                       g_idx=first["g_idx"]) for i, n0 in enumerate(range(block, N, block))]
    cat = {k: np.concatenate([p[k] for p in parts], axis=-1) for k in ("qweight", "qzeros", "scales")}
    b = np.concatenate([p["bias"] for p in parts]) if bias else None
    return dict(**cat, g_idx=first["g_idx"], bias=b, K=K, N=N, group_size=first["group_size"])


# --------------------------------------------------------------------------- activation generators
ACTS = ["gauss", "offset", "student_t", "massive", "row_scale", "subnormal", "huge_tiny", "inf"]


def acts_for(dtype):
    """The activation kinds that exist in ``dtype``: fp16 subnormals for fp16, rows near 1e5 / 1e-20 for bf16."""
    skip = "huge_tiny" if dt_name(dtype) == "float16" else "subnormal"
    return [a for a in ACTS if a != skip]


def activations(kind, M, K, dtype, seed=0):
    """float32 [M, K] already rounded to ``dtype``:
      gauss      N(0, 1);
      offset     N(0, 1) + 4 on every channel, every row (a per-channel offset of 4σ of one sign: Σx ≈ Σ|x|);
      student_t  Student-t, ν = 3 (heavy tails);
      massive    N(0, 1) with three channels ×1000;
      row_scale  row m times 10^((m mod 10) − 2) (fp16: 10^((m mod 5) − 2)), so the outputs stay in range;
      subnormal  N(0, 1)·1e-6: fp16 subnormals;
      huge_tiny  bf16: rows alternately near 1e5 and near 1e-20;
      inf        N(0, 1) with one +inf in one row (the output row must be non-finite, the others exact)."""
    dn = dt_name(dtype)
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((M, K))
    if kind == "offset":
        x = x + 4.0
    elif kind == "student_t":
        x = rng.standard_t(3, size=(M, K))
    elif kind == "massive":
        x[:, rng.choice(K, 3, replace=False)] *= 1000.0
    elif kind == "row_scale":
        e = np.arange(M) % (5 if dn == "float16" else 10) - 2.0
        x = x * 10.0 ** e[:, None]
    elif kind == "subnormal":
        x = x * 1e-6
    elif kind == "huge_tiny":
        x = x * np.where(np.arange(M) % 2 == 0, 1e5, 1e-20)[:, None]
    elif kind == "inf":
        x[M // 2, int(rng.integers(K))] = np.inf
    elif kind != "gauss":
        raise ValueError(kind)
    return round_dt(x, dn).astype(np.float32)
