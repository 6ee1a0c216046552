"""The stage-wise SiLU·mul checks of tests/_silu_mul.py have teeth: the exact computation and an fp32 formulation of
the fused gate/up pair and of the grouped experts are accepted, and each bug class below, restated as a NumPy mutant on
the GPU tests' own layer, expert and activation generators, is rejected by the same check code.  Also: the silu
candidate set covers every 16-bit g under the error model of the kernels' ``__expf`` silu.  No GPU."""
import numpy as np
import pytest

from oracle import w4a16_oracle as O
from tests import _precision as P
from tests import _silu_mul as S

K, I = 512, 256
DTS = ["float16", "bfloat16"]


def _pair(dt, act=True, seed=1):
    d1 = P.realistic_layer(K, I, 64, dt, seed=seed, act_order=act, bias=True)
    return d1, P.realistic_layer(K, I, 64, dt, seed=seed + 1, bias=True, g_idx=d1["g_idx"])


def _silu(g):
    with np.errstate(over="ignore", invalid="ignore"):
        return g / (1.0 + np.exp(-g))


def _y(d, x, path, dt, drop=None):
    """Unrounded x·W + b of the path (NaN rows where x holds a non-finite value); ``drop``: k range left out."""
    x = np.asarray(x, dtype=np.float64)
    if drop is not None:
        x = x.copy()
        x[:, drop[0]:drop[1]] = 0.0
    ref = P.reference(d, x, P.PATHS[path], dt)
    y = ref.ystar.copy()
    y[ref.bad_rows] = np.nan
    return y


def _y32(d, x, path, dt):
    """fp32 evaluation: the weights the path uses (exact in fp32), one fp32 dot product per output, fp32 bias."""
    q, z, s, gi, b = P.layer_parts(d, dt)
    W = P._weights(q, z, s, gi, dt, P.PATHS[path].round_w).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        y = np.asarray(x, dtype=np.float32) @ W
    return (y + (0 if b is None else b.astype(np.float32))).astype(np.float64)


def gate_up(d1, d3, x, dt, path="decode_mma", bug=None, fp32=False):
    """(g, u, h) of the fused gate/up pair, computed exactly (or in fp32) with one optional bug switched in."""
    rnd = lambda a: P.round_dt(a, dt)
    if fp32:
        gy, uy = _y32(d1, x, path, dt), _y32(d3, x, path, dt)
    else:
        drop = (K // 2, K) if bug == "split_dropped" else None
        if bug == "bias_u_on_g":
            d1 = dict(d1, bias=d3["bias"])
        gy, uy = _y(d1, x, path, dt, drop), _y(d3, x, path, dt)
    g, u = rnd(gy), rnd(uy)
    gh, uh = g, u
    if bug == "g_unrounded":
        gh = gy
    elif bug == "u_unrounded":
        uh = uy
    elif bug == "swapped":
        g, u = u, g
        gh, uh = g, u
    if fp32:
        g32 = g.astype(np.float32)
        with np.errstate(over="ignore", invalid="ignore"):
            s = rnd((g32 / (np.float32(1) + np.exp(-g32))).astype(np.float64))
    elif bug == "exp16":
        with np.errstate(over="ignore", invalid="ignore"):
            s = rnd(gh / (1.0 + rnd(np.exp(-gh))))
    else:
        s = _silu(gh) if bug == "silu_unrounded" else S.silu_candidates(gh, dt)[0]
    with np.errstate(invalid="ignore", over="ignore"):
        h = rnd(s * uh) if bug in ("silu_unrounded", "g_unrounded", "u_unrounded") else S.h_of(s, uh, dt)
    return g, u, h


# --------------------------------------------------------------------------- gate/up: accepted and rejected
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("path", ["decode_mma", "gemm"])
@pytest.mark.parametrize("fp32", [False, True], ids=["exact", "fp32"])
def test_gate_up_exact_and_fp32_are_accepted(dt, path, fp32):
    d1, d3 = _pair(dt)
    for kind in P.acts_for(dt):
        x = P.activations(kind, 6, K, dt, seed=3)
        g, u, h = gate_up(d1, d3, x, dt, path, fp32=fp32)
        S.check_gate_up(d1, d3, x, g, u, h, path, dt, what=f"{path} {dt} {kind}")


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("bug", ["silu_unrounded", "g_unrounded", "u_unrounded", "swapped", "bias_u_on_g",
                                 "split_dropped", "exp16"])
def test_gate_up_mutant_is_rejected(dt, bug):
    d1, d3 = _pair(dt)
    x = P.activations("gauss", 6, K, dt, seed=4)
    g, u, h = gate_up(d1, d3, x, dt, bug=bug)
    with pytest.raises(AssertionError):
        S.check_gate_up(d1, d3, x, g, u, h, "decode_mma", dt, what=bug)


# --------------------------------------------------------------------------- experts
E, HID, INT = 4, 256, 256


def _experts(dt, act2=True):
    return S.realistic_experts(E, HID, INT, 64, dt, seed=5, act13=True, act2=act2, bias=True)


def _routing(T, k, seed):
    rng = np.random.default_rng(seed)
    idx = np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)
    idx[0, 1:] = E                               # token 0 runs one expert
    idx[-1, :] = -1                              # the last token none: its output is exactly 0
    w = rng.random((T, k)).astype(np.float32) + 0.1
    return idx, w / w.sum(axis=1, keepdims=True)


def moe(ex, x, idx, w, dt, decode=True, bug=None, fp32=False):
    """(g_sv, u_sv, y_sv, out) of the grouped forward as the saving kernels lay them out, exact or in fp32."""
    rnd = lambda a: P.round_dt(a, dt)
    path = "decode_mma" if decode else "gemm"
    T, k = idx.shape
    g_sv, u_sv, y_sv, y_un = (np.full((T * k, n), np.nan) for n in (INT, INT, HID, HID))
    flat = idx.reshape(-1)
    for e in range(E):
        pid = np.nonzero(flat == e)[0]
        if not pid.size:
            continue
        w1, w3, w2 = (ex[e][n] for n in ("w1", "w3", "w2"))
        xe = x[pid // k]
        g, u, h = gate_up(w1, w3, xe, dt, path, fp32=fp32)
        if fp32:
            yy = _y32(w2, h, path, dt)
        else:
            drop = None
            if bug == "down_split_dropped":          # one of two K splits of the down stage (w2's sorted k order)
                perm = O.make_sequential_perm(np.asarray(w2["g_idx"]))
                h = h.copy()
                h[:, perm[INT // 2:]] = 0.0
            yy = _y(w2, h, path, dt, drop)
        perm = O.make_sequential_perm(np.asarray(w2["g_idx"]))
        if bug != "no_h_order":
            g, u = g[:, perm], u[:, perm]
        g_sv[pid], u_sv[pid], y_sv[pid], y_un[pid] = g, u, rnd(yy), yy
    valid = ((idx >= 0) & (idx < E))[..., None]
    wv = P.round_dt(w, dt) if bug == "w_as_16bit" else w.astype(np.float64)
    y = (y_un if bug == "y_unrounded" else y_sv).reshape(T, k, HID)
    with np.errstate(invalid="ignore"):
        if fp32:
            acc = np.zeros((T, HID), dtype=np.float32)
            for j in range(k):
                acc = acc + np.where(valid[:, j], wv[:, j, None].astype(np.float32) * y[:, j].astype(np.float32), 0)
            out = rnd(acc.astype(np.float64))
        else:
            terms = np.where(valid, wv[..., None] * np.where(valid, y, 0.0), 0.0)
            if bug == "terms_rounded":
                terms = rnd(terms)
            out = rnd(terms.sum(axis=1))
    return g_sv, u_sv, y_sv, out


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("decode", [True, False], ids=["decode", "gemm"])
@pytest.mark.parametrize("fp32", [False, True], ids=["exact", "fp32"])
def test_experts_exact_and_fp32_are_accepted(dt, decode, fp32):
    ex = _experts(dt)
    T = 8 if decode else 12
    idx, w = _routing(T, 2, seed=1)
    path = "decode_mma" if decode else "gemm"
    for kind in P.acts_for(dt):
        x = P.activations(kind, T, HID, dt, seed=2)
        sv = moe(ex, x, idx, w, dt, decode, fp32=fp32)
        S.check_moe(ex, x, idx, w, dt, path, path, *sv, what=f"{dt} {kind}")


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("bug", ["no_h_order", "down_split_dropped", "y_unrounded", "terms_rounded", "w_as_16bit"])
def test_experts_mutant_is_rejected(dt, bug):
    ex = _experts(dt)
    idx, w = _routing(8, 2, seed=3)
    x = P.activations("gauss", 8, HID, dt, seed=4)
    sv = moe(ex, x, idx, w, dt, bug=bug)
    with pytest.raises(AssertionError):
        S.check_moe(ex, x, idx, w, dt, "decode_mma", "decode_mma", *sv, what=bug)


def test_experts_nonzero_output_of_a_token_without_valid_ids_is_rejected():
    dt = "float16"
    ex = _experts(dt)
    idx, w = _routing(8, 2, seed=3)
    x = P.activations("gauss", 8, HID, dt, seed=4)
    g, u, y, out = moe(ex, x, idx, w, dt)
    out[-1, 7] = 2.0 ** -24
    with pytest.raises(AssertionError, match="without a valid expert id"):
        S.check_moe(ex, x, idx, w, dt, "decode_mma", "decode_mma", g, u, y, out)


def test_chain_down_with_ambiguous_h_is_accepted_either_way():
    """A down stage fed h_alt on the ambiguous elements stays within the widened bound."""
    dt = "float16"
    d2 = P.realistic_layer(INT, 128, 128, dt, seed=9)
    rng = np.random.default_rng(0)
    g = P.round_dt(rng.standard_normal((4, INT)) * 4, dt)
    u = P.round_dt(rng.standard_normal((4, INT)), dt)
    h0, h1, amb = S.h_candidates(g, u, dt)
    for h in (h0, np.where(amb, h1, h0)):
        y = P.round_dt(P.reference(d2, h, P.PATHS["chain"], dt).ystar, dt)
        P.check(y, S.reference_down(d2, g, u, P.PATHS["chain"], dt), P.PATHS["chain"], dt, what="chain down")


# --------------------------------------------------------------------------- the silu candidates
def _all_finite(dt):
    bits = np.arange(65536, dtype=np.uint32)
    if dt == "float16":
        v = bits.astype(np.uint16).view(np.float16).astype(np.float64)
    else:
        v = (bits << 16).view(np.float32)
        v = v[np.isfinite(v)].astype(np.float64)
    return v[np.isfinite(v)]


def _kernel_silu(g, ex2_err):
    """The kernels' fp32 silu with ex2.approx's error set to ``ex2_err`` (relative) on every element."""
    g32 = g.astype(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        t = g32 * S.NEG_LOG2E_F32
        e = (np.exp2(t.astype(np.float64)) * (1 + ex2_err)).astype(np.float32)
        e = np.where(t >= 128, np.float32(np.inf), e)
        return (g32 / (np.float32(1) + e)).astype(np.float64)


@pytest.mark.parametrize("dt", DTS)
def test_silu_candidates_cover_every_16bit_g(dt):
    """Exhaustive over the dtype's finite values, with ex2's error at both ends of its stated range."""
    g = _all_finite(dt)
    s, s_alt, amb = S.silu_candidates(g, dt)
    for err in (-S.EX2_REL, 0.0, S.EX2_REL):
        k = P.round_dt(_kernel_silu(g, err), dt)
        assert np.all((k == s) | (amb & (k == s_alt))), f"{dt} ex2 error {err}"
    assert amb[np.abs(g) <= 16].mean() < 0.01            # two candidates stay rare where g lives (0.17 % / 0.78 %)


def test_silu_overflow_domain_is_minus_zero():
    g = np.array([-88.5, -88.6875, -88.75, -89.0, -95.0, -1e4])
    assert S.exp_overflows(g).tolist() == [False, False, True, True, True, True]
    s, _, amb = S.silu_candidates(g, "bfloat16")
    assert np.all(s[2:] == 0) and np.all(np.signbit(s[2:])) and not amb[2:].any()
    assert P.round_dt(-89.0 / (1 + np.exp(89.0)), "bfloat16") != 0       # the float64 value is a bf16 number
