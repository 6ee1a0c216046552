"""The float64 GPTQ replay (tests/_gptq_replay.py) is right and sharp, without a GPU.

* Valid implementations pass it exactly: the NumPy oracle (fp32, BLAS summation order in the trailing update) and a
  second fp32 loop that sums the trailing update in reverse k order with a rounding per product, on every golden case.
* A diagonal Hinv (no error feedback) leaves no room: every code must be the exact round-half-to-even of the fp32
  quotient, constructed .5 ties and the fp32 edge of an all-zero group included.
* Mutants of the loop are caught, each on at least one case.  What each check can see: a wrong value reaches a code when
  it moves w/s by more than the bound to the other side of a midpoint; it reaches a loss when it moves w by more than
  B (a few hundred u of |w| on these layers), which is what catches the mutants that change every later column a
  little.  A Hessian error of a few u lies inside γ·A by design; the mismatch rate against round_f32(H*) is what sees
  it.
"""
import numpy as np
import pytest
import torch

from autogptq_b200.gptq import running_mean_factors
from oracle import gptq_oracle as GO
from tests import _gptq_replay as R
from tests.test_gptq_cpu import golden_cases, load_case

f32 = np.float32
MUTANTS = ("params_from_W1", "err_not_divided", "skip_trailing", "wrong_block_rows", "round_half_up",
           "static_by_position", "dead_before_initial", "Q_processing_order")


def _quantize(x, scale, zero, half_up=False):
    r = np.floor(x / scale + f32(0.5)) if half_up else np.rint(x / scale)
    q = np.clip(r + zero, 0, 15).astype(f32)
    return (scale * (q - zero)).astype(f32)


def loop(W, Hinv, perm=None, dead=None, group_size=-1, sym=True, static_groups=False, reverse_trailing=False,
         mutant=None):
    """gptq_oracle.fasterquant restated with the kernel's output conventions (losses in original order) and one switch
    per mutant.  ``reverse_trailing``: the trailing update as an fp32 sum in reverse k order, one rounding per product
    and one per addition (a second valid summation order)."""
    W = np.array(W, dtype=f32)
    N, K = W.shape
    if mutant == "dead_before_initial" and dead is not None:
        W[:, dead] = 0
    scale0, zero0 = GO.find_params(W, sym)
    if dead is not None:
        W[:, dead] = 0
    gs = K if group_size == -1 else group_size
    G = -(-K // gs)
    static = static_groups and group_size != -1
    scale, zero = np.zeros((N, G), f32), np.zeros((N, G), f32)
    if group_size == -1:
        scale[:, 0], zero[:, 0] = scale0, zero0
    if static:
        for g in range(G):
            scale[:, g], zero[:, g] = GO.find_params(W[:, g * gs:(g + 1) * gs], sym)
    pos = np.arange(K) if perm is None else np.asarray(perm)
    W = W[:, pos]
    Qp, Lp = np.zeros_like(W), np.zeros_like(W)
    for i1 in range(0, K, 128):
        i2 = min(i1 + 128, K)
        W1 = W[:, i1:i2].copy()
        Err1 = np.zeros_like(W1)
        for i in range(i2 - i1):
            col = i1 + i
            if group_size != -1 and not static and col % gs == 0:
                src = W1[:, i:i + gs] if mutant == "params_from_W1" else W[:, col:col + gs]
                scale[:, col // gs], zero[:, col // gs] = GO.find_params(src, sym)
            g = 0 if group_size == -1 else (pos[col] // gs if static and mutant != "static_by_position" else col // gs)
            w, d = W1[:, i], Hinv[col, col]
            q = _quantize(w, scale[:, g], zero[:, g], half_up=mutant == "round_half_up")
            Qp[:, col] = q
            Lp[:, col] = ((w - q) ** 2 / d ** 2) / f32(2)
            err = (w - q) if mutant == "err_not_divided" else ((w - q) / d).astype(f32)
            W1[:, i:] -= np.outer(err, Hinv[col, col:i2]).astype(f32)
            Err1[:, i] = err
        if i2 < K and not (mutant == "skip_trailing" and i1 == 0):
            rows = Hinv[0:i2 - i1, i2:] if (mutant == "wrong_block_rows" and i1 > 0) else Hinv[i1:i2, i2:]
            if reverse_trailing:
                acc = np.zeros((N, K - i2), f32)
                for k in range(i2 - i1 - 1, -1, -1):
                    acc = (acc + np.outer(Err1[:, k], rows[k]).astype(f32)).astype(f32)
            else:
                acc = (Err1 @ rows).astype(f32)
            W[:, i2:] -= acc
    inv = np.argsort(pos)
    Q = Qp if mutant == "Q_processing_order" else Qp[:, inv]
    g_idx = R.g_idx_rule(K, group_size, perm, static_groups)
    codes = (np.rint(Q / scale[:, g_idx]) + zero[:, g_idx]).astype(np.uint8)
    qweight, qzeros, scales = GO.pack_codes(codes, zero, scale)
    return dict(Q=Q, scale=scale, zero=zero, g_idx=g_idx, losses=Lp[:, inv], qweight=qweight, qzeros=qzeros,
                scales=scales)


def replay(c, out, W=None, Hinv=None):
    t = lambda a: None if a is None else torch.from_numpy(np.asarray(a))    # noqa: E731
    return R.check_quantize(t(c["W"] if W is None else W), t(c["Hinv"] if Hinv is None else Hinv),
                            {k: t(v) for k, v in out.items()}, perm=t(c["perm"]), dead=t(c["dead"]),
                            group_size=c["g"], sym=c["sym"], static_groups=c["static"])


def run(c, **kw):
    return loop(c["W"], c["Hinv"], perm=c["perm"], dead=c["dead"], group_size=c["g"], sym=c["sym"],
                static_groups=c["static"], **kw)


@pytest.mark.parametrize("f,i", golden_cases())
def test_oracle_passes_the_replay(f, i):
    """The oracle's own fasterquant (BLAS order), repacked, and the loop restated here agree and both pass."""
    c = load_case(f, i)
    r = GO.fasterquant(c["W"], c["Hinv"], perm=c["perm"], dead=c["dead"], group_size=c["g"], sym=c["sym"],
                       static_groups=c["static"])
    inv = np.arange(c["K"]) if c["perm"] is None else np.argsort(c["perm"])
    qw, qz, sc = GO.pack_codes(r["codes"], r["zero"], r["scale"])
    out = dict(Q=r["Q"], scale=r["scale"], zero=r["zero"], g_idx=r["g_idx"], losses=r["losses"][:, inv],
               qweight=qw, qzeros=qz, scales=sc)
    m = replay(c, out)
    assert m.worst <= 1.0 and m.unclear < 0.1, m
    mine = run(c)
    for k in ("Q", "scale", "zero", "qweight"):
        np.testing.assert_array_equal(mine[k], out[k], err_msg=k)


@pytest.mark.parametrize("f,i", golden_cases())
def test_second_summation_order_passes(f, i):
    c = load_case(f, i)
    replay(c, run(c, reverse_trailing=True))


def _diag_case(sym, seed=0):
    """Rows of range exactly 15 (s = 1) holding every .5 tie, an all-zero group, and a diagonal Hinv."""
    rng = np.random.default_rng(seed)
    N, K = 32, 264
    W = rng.integers(-7, 8, size=(N, K)).astype(f32) + rng.choice(f32([0.0, 0.5, -0.5, 0.25]), size=(N, K))
    W = np.clip(W, -7.5, 7.5)
    W[:, 0], W[:, 1] = -7.5, 7.5                      # every 32-column group spans [-7.5, 7.5]: s = 1
    for g0 in range(0, K, 32):
        W[:, g0], W[:, g0 + 1] = -7.5, 7.5
    W[3, 64:96] = 0                                   # all-zero group: s = fl(2/15), fl(1/s) = 7.4999995, zero 7
    d = rng.uniform(0.5, 2.0, size=K).astype(f32)
    return dict(W=W, Hinv=np.diag(d), perm=None, dead=None, g=32, sym=sym, static=False, K=K)


@pytest.mark.parametrize("sym", [False, True])
def test_diagonal_hinv_is_exact_rtn_with_ties(sym):
    c = _diag_case(sym)
    out = run(c)
    assert (np.abs(c["W"] % 1) == 0.5).mean() > 0.2                     # ties are common
    m = replay(c, out)
    assert m.unclear == 0.0 and m.params_unclear == 0, m                # no room anywhere
    if not sym:
        s, z = out["scale"][3, 2], out["zero"][3, 2]
        assert s == f32(2) / f32(15) and f32(1) / s == f32(7.4999995) and z == 7
        assert out["zero"][0, 0] == 8                                    # rint(7.5) = 8 where s is exactly 1
    # float64 find_params would give zero 8 to the all-zero group: the replay rejects it
    bad = {k: v.copy() for k, v in out.items()}
    if not sym:
        bad["zero"][3, 2] = 8
        with pytest.raises(AssertionError):
            replay(c, bad)


def _mutant_cases():
    cases = [load_case(f, i) for f, i in golden_cases()]
    extreme = load_case("gptq_dead_seq", 2)           # group_size = -1 with a dead column holding every row's maximum
    extreme["W"][:, np.flatnonzero(extreme["dead"])[0]] = 4 * np.abs(extreme["W"]).max()
    return cases + [_diag_case(False), extreme]


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutants_fail_the_replay(mutant):
    caught = []
    for c in _mutant_cases():
        out = run(c, mutant=mutant)
        try:
            replay(c, out)
        except AssertionError as e:
            caught.append(str(e).split(":")[0])
    assert caught, f"mutant {mutant} passed every case"


# --------------------------------------------------------------------------- Hessian
def hessian_model(batches, K, mutant=None):
    """The kernel's arithmetic in fp32 on the CPU: per call, fp32 sums of 32-row stages in t order, then
    fl(fl(α·H) + fl(β·acc)) on the upper triangle of 128-tiles and its mirror."""
    H = torch.zeros((K, K), dtype=torch.float32)
    n = 0
    for call, x in enumerate(batches):
        alpha, beta, n1 = running_mean_factors(n, x.shape)
        if mutant == "beta_old_count":
            beta = 2.0 / n if n > 0 else beta
        n = n1
        X = x.reshape(-1, K).float()
        T = X.shape[0]
        if mutant == "drop_tail":
            T -= T % 32
        acc = torch.zeros((K, K), dtype=torch.float32)
        for t0 in range(0, T, 32):
            xs = X[t0:min(t0 + 32, T)]
            acc = acc + xs.T @ xs
        a32, b32 = torch.tensor(alpha, dtype=torch.float32), torch.tensor(beta, dtype=torch.float32)
        new = a32 * H + b32 * acc
        if mutant == "few_u":
            new = new * torch.tensor(1 + 2.0 ** -22, dtype=torch.float32)
        up = torch.triu(torch.ones(K, K, dtype=torch.bool))
        Hn = torch.where(up, new, new.T)
        if mutant == "stale_mirror" and call > 0:
            Hn[128:256, 0:128] = H[128:256, 0:128]
        H = Hn
    return H


def _batches(K, seed=0, dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    x = [torch.randn(40, K, generator=g), torch.randn(3, 5, K, generator=g), torch.randn(1, 1, K, generator=g),
         torch.randn(0, K, generator=g)]
    x[0][:, :3] *= 1000
    return [b.to(dtype) for b in x]


def _hess(batches, K):
    ref = R.HessianReference(K, "cpu")
    for b in batches:
        ref.add(b)
    return ref


# On these batches (170 well-conditioned elements) the fp32 model above mismatches round_f32(H*) on 61 % (fp16) / 49 %
# (bf16) of them, a result perturbed by 4u on 100 %; one call of T = 1 gives 0 % against 100 %, T = 8 27 % against 99.95 %.
HESS_RATE_CPU = 0.8


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_hessian_reference_passes_the_model(dtype):
    K = 256
    b = _batches(K, dtype=dtype)
    ref = _hess(b, K)
    assert ref.n == 1 + 3 + 1 + 1
    m = ref.check(hessian_model(b, K), HESS_RATE_CPU, min_cond=100)
    assert m.n_cond >= 100, m


@pytest.mark.parametrize("mutant", ["stale_mirror", "beta_old_count", "drop_tail", "few_u"])
def test_hessian_mutants_are_caught(mutant):
    K = 256
    b = _batches(K)
    ref = _hess(b, K)
    m = ref.measure(hessian_model(b, K, mutant))
    if mutant == "few_u":                       # inside the bound, outside the mismatch-rate limit
        assert m.worst <= 1.0 and m.rate > HESS_RATE_CPU, m
    else:
        assert m.worst > 1.0, m
