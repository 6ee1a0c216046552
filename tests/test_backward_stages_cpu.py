"""The stage checks of tests/_backward_stages.py are right and sharp, on the CPU:

* right: a float32 emulation of the dense MLP backward with the kernels' rounding points (but BLAS block sums in place of
  wgmma, np.exp in place of ``__expf``) passes every stage, and silu′'s error bound Δ(g) holds for every finite fp16
  and bf16 g against an fp32 emulation whose exp is off by up to ±2 ulp (ex2.approx.f32's documented maximum);
* sharp: plausible kernel bugs fail the stage they break.  Most of them pass the end-to-end bound of
  tests/test_gpu_19_mlp_grad.py, whose ε term (one 16-bit ulp per rounded operand) makes it about 100x wider than
  the error the kernels make; those tests assert that too, to document the gap the stage checks close;
* the workspace layouts restate csrc/moe.cu: hand-computed totals, and the library's own sizes over a sweep.
"""
import numpy as np
import pytest
import torch

from oracle import w4a16_oracle as O
from tests import _backward_stages as B
from tests import _mlp_grad as MLG
from tests import _precision as P
from tests import _silu_mul as S

F16, BF16 = "float16", "bfloat16"
f32 = np.float32


# --------------------------------------------------------------------------- layouts
def test_layout_totals_by_hand():
    # T=5, k=2, E=8: P = 10 pairs, 2 per hit expert -> 32-row tile, rows = 10 + 8·31 = 258, max tiles 1 + 8 = 9,
    # tables 4·8 + 4 + 2·9 + 10 = 64 ints = 256 B; prow 40 B -> 256; dy_pair 258·1024·2; [dg|du] 258·3072·2; dx_pair fp32
    b = B.bwd_layout(5, 2, 8, 1024, 1536)
    assert (b["mt"], b["rows"], b["prow"], b["dyp"]) == (32, 258, 256, 512)
    assert (b["dgu"], b["dxp"], b["total"]) == (528896, 2114048, 3170816)
    # T=300, k=2, E=8 at Mixtral's size: 75 per expert -> 128-row tile, rows = 600 + 8·127 = 1616, max tiles 19 + 8,
    # tables 32 + 4 + 54 + 600 = 690 ints = 2760 B -> 2816; prow 2400 B -> 2560
    b = B.bwd_layout(300, 2, 8, 4096, 14336)
    assert (b["mt"], b["rows"], b["prow"], b["dyp"]) == (128, 1616, 2816, 5376)
    assert (b["dgu"], b["dxp"], b["total"]) == (13243648, 105911552, 132388096)
    assert B.bwd_layout(200, 2, 8, 1024, 1536)["mt"] == 64
    # T = 0: tables only (E = 8: 52 ints -> 256 B)
    assert B.bwd_layout(0, 2, 8, 1024, 1536)["total"] == 256
    # dense: [dg|du] 5·3072·2 = 30720 B (120·256), then dx staged 5·1024·2 = 10240 B
    assert B.mlp_bwd_layout(5, 1024, 1536) == dict(dgu=0, dxs=30720, total=40960)
    assert B.mlp_bwd_layout(3, 1088, 1472) == dict(dgu=0, dxs=17664, total=24320)


def test_layout_totals_are_the_library_sizes():
    """The restated totals equal agb200_*_backward_workspace_bytes over T, k, E, H, I (every row tile) and M, H, I."""
    from autogptq_b200 import _lib

    lib = _lib.load()
    tiles = set()
    for T in (0, 1, 3, 8, 9, 64, 100, 300, 2049):
        for k in (1, 2, 4, 8):
            for E, H, I in ((8, 1024, 1536), (64, 4096, 14336), (1, 256, 512), (3, 1408, 512)):
                tiles.add(B.bwd_tile(T * k, E))
                assert lib.agb200_moe_backward_workspace_bytes(T, k, E, H, I) == B.bwd_layout(T, k, E, H, I)["total"], \
                    (T, k, E, H, I)
    assert tiles == {32, 64, 128}
    for M in (0, 1, 5, 9, 200, 2049):
        for H, I in ((1024, 2816), (1088, 1472), (4096, 11008)):
            assert lib.agb200_w4a16_mlp_backward_workspace_bytes(M, H, I) == B.mlp_bwd_layout(M, H, I)["total"]


# --------------------------------------------------------------------------- silu'
def _all_finite(dtype):
    bits = np.arange(1 << 16, dtype=np.uint32)
    v = bits.astype(np.uint16).view(np.float16) if dtype == F16 else (bits << 16).view(np.float32)
    v = v[np.isfinite(v)]
    return v.astype(np.float64)


def _sp_fp32(g, ulps=0):
    """The kernel's fp32 silu′ (``silu_mul_backward``) with ex2 off by ``ulps`` fp32 ulps; ex2.approx.ftz flushes."""
    g32 = np.asarray(g, dtype=f32)
    with np.errstate(over="ignore", invalid="ignore"):
        e = np.exp2(g32 * S.NEG_LOG2E_F32)
        for _ in range(abs(ulps)):          # an overflow (t >= 128) stays +inf
            e = np.where(np.isinf(e), e, np.nextafter(e, f32(np.inf if ulps > 0 else 0)))
        e = np.where(e < f32(2.0 ** -126), f32(0), e).astype(f32)
        sig = f32(1) / (f32(1) + e)
        return (sig * (f32(1) + g32 * (f32(1) - sig))).astype(np.float64)


@pytest.mark.parametrize("dtype", [F16, BF16])
def test_silu_prime_error_bound_holds_for_every_g(dtype):
    g = _all_finite(dtype)
    ref, dl = B.silu_prime(g), B.silu_prime_delta(g)
    worst = 0.0
    for ulps in (-2, 0, 2):
        err = np.abs(_sp_fp32(g, ulps) - ref)
        with np.errstate(invalid="ignore", divide="ignore"):
            r = np.where(err == 0, 0.0, err / dl)
        worst = max(worst, float(r.max()))
        assert (err <= dl).all(), f"{dtype} ex2 {ulps:+d} ulp: Δ exceeded at g = {g[np.argmax(r)]!r} ({r.max():.3g})"
    print(f"[stages] silu′ {dtype}: max |sp − silu′| / Δ = {worst:.3f}")
    # Δ is an ulp-scale bound, not a loose one: far below a 16-bit half-ulp of silu′'s own scale
    scale = B.sigmoid(g) * (1 + np.abs(g) * (1 - B.sigmoid(g)))
    assert (dl <= scale * 2.0 ** -14 + 1e-38).all()
    # on the overflow domain the kernel's σ is 0: silu′ and its candidate are exactly 0 there
    over = S.exp_overflows(g)
    assert over.any() and (B.silu_prime(g)[over] == 0).all() and (_sp_fp32(g)[over] == 0).all()


def test_overflow_domain_and_overflowing_values():
    """g < −88.72: the kernel writes dg = du = −0 (σ = 0, s16 = −0), accepted exactly; the float64 value there is a
    representable bf16 number, which is outside.  A value that rounds past the largest finite one is accepted as ±inf
    exactly where its interval reaches past it."""
    g, u = np.array([[-89.0]]), np.array([[1.0]])
    ref = B.DhRef(np.array([[3.0]]), np.array([[3.0]]), 1024)
    ok = B.measure_dgu(np.array([[-0.0]]), np.array([[-0.0]]), ref, g, u, BF16)
    assert ok["dg"].outside == ok["du"].outside == 0
    s = B.sigmoid(-89.0)
    bad = B.measure_dgu(P.round_dt(3.0 * s * (1 - 89.0 * (1 - s)), BF16) * np.ones((1, 1)),
                        P.round_dt(3.0 * -89.0 * s, BF16) * np.ones((1, 1)), ref, g, u, BF16)
    assert bad["dg"].outside == bad["du"].outside == 1
    # fp16: du* = 1e5·rnd(silu(1)) ≈ 73100 rounds to +inf, dg* = 1e5·silu′(1) ≈ 92760 too
    g, u = np.array([[1.0]]), np.array([[1.0]])
    big = B.DhRef(np.array([[1e5]]), np.array([[1e5]]), 1024)
    r = B.measure_dgu(np.array([[np.inf]]), np.array([[np.inf]]), big, g, u, F16)
    assert r["dg"].outside == r["du"].outside == 0
    r = B.measure_dgu(np.array([[-np.inf]]), np.array([[65504.0]]), big, g, u, F16)
    assert r["dg"].outside == r["du"].outside == 1
    # in range: an inf is outside
    small = B.DhRef(np.array([[1e4]]), np.array([[1e4]]), 1024)
    r = B.measure_dgu(np.array([[np.inf]]), np.array([[np.inf]]), small, g, u, F16)
    assert r["dg"].outside == r["du"].outside == 1


# --------------------------------------------------------------------------- the dense MLP backward, emulated
H, I, M, G = 1024, 2816, 64, 128


def _mm32(a, b, blk=64):
    """fp32 a·b: fp32 BLAS within blocks of ``blk`` terms, fp32 adds across blocks (a summation order of its own)."""
    a, b = np.asarray(a, dtype=f32), np.asarray(b, dtype=f32)
    acc = np.zeros((a.shape[0], b.shape[1]), dtype=f32)
    for k0 in range(0, a.shape[1], blk):
        acc += a[:, k0:k0 + blk] @ b[k0:k0 + blk]
    return acc


def _rnd(a, dt=F16):
    return P.round_dt(np.asarray(a, dtype=np.float64), dt)


def _emulate(x, W, dy, mutant=None, dt=F16):
    """dg, du, dx of the fused dense backward on the rounded g, u of the forward, in fp32 with the kernels' rounding
    points; ``mutant`` injects one of the bugs below."""
    W1, W3, W2 = W
    g, u = _rnd(_mm32(x, W1), dt), _rnd(_mm32(x, W3), dt)
    g32, u32 = g.astype(f32), u.astype(f32)
    with np.errstate(over="ignore"):
        e = np.exp(-g32)
    sig = f32(1) / (f32(1) + e)
    silu32 = g32 / (f32(1) + e)
    sg32 = _rnd(silu32, dt).astype(f32)
    sp = sig * (f32(1) + g32 * (f32(1) - sig))
    if mutant == "silu′ = σ":
        sp = sig
    dh = _mm32(dy, W2.T)
    if mutant == "dh rounded to 16 bits":
        dh = _rnd(dh, dt).astype(f32)
    dg = _rnd(dh * u32 * sp, dt)
    du = _rnd(dh * (silu32 if mutant == "du from unrounded silu(g)" else sg32), dt)
    dgk, duk, W1k = dg, du.copy(), W1
    if mutant == "one du column dropped":
        duk[:, 1000] = 0
    if mutant == "first 64-wide w3 block dropped":
        duk[:, :64] = 0
    if mutant == "one W1 group's scales 1.6 % off":
        W1k = W1.copy()
        W1k[128:256] = _rnd(W1[128:256] * (1 + 2.0 ** -6), dt)
    acc = _mm32(np.concatenate([dgk, duk], axis=1), np.concatenate([W1k, W3], axis=1).T)
    if mutant == "one dx tile's w3 part × (1 + 2⁻⁸)":
        acc[:, 512:640] = _mm32(dg, W1[512:640].T) + _mm32(du, W3[512:640].T) * f32(1 + 2.0 ** -8)
    return dict(g=g, u=u, dg=dg, du=du, dx=_rnd(acc, dt))


@pytest.fixture(scope="module")
def dense():
    """The issue's setting: GPTQ layers of random_packed at H = 1024, I = 2816, g = 128, fp16, M = 64, Gaussian x, dy."""
    L = []
    for j, (K, N) in enumerate(((H, I), (H, I), (I, H))):
        d = O.random_packed(K, N, G, seed=j)
        d["scales"], d["bias"] = d["scales"].astype(np.float16), None
        L.append(d)
    rng = np.random.default_rng(0)
    x, dy = _rnd(rng.standard_normal((M, H))), _rnd(rng.standard_normal((M, H)))
    W = tuple(B.weights(d, F16) for d in L)
    old = MLG.backward(x, *L, dy, F16, round_w_fwd=True)
    return dict(L=L, x=x, dy=dy, W=W, old=old, dh=B.dh_reference(dy, W[2]))


def _stages(dense, em):
    W1, W3, _ = dense["W"]
    dgu = B.measure_dgu(em["dg"], em["du"], dense["dh"], em["g"], em["u"], F16)
    dx = P.measure(em["dx"], B.dx_reference(em["dg"], em["du"], W1, W3), P.PATHS["dgrad"], F16)
    return dgu, dx


def _old_contract(dense, dx):
    """err/bound of test_gpu_19's end-to-end check: ulp(dx*) + (γ + ε)·(A + A2) against the all-float64 block."""
    r = dense["old"]
    bound = P.ulp(r["dx"], F16) + (P.gamma(P.PATHS["dgrad"], max(2 * I, H)) + 2.0 ** -10) * (r["A"] + r["A2"])
    return float((np.abs(dx - r["dx"]) / bound).max())


def test_faithful_emulation_passes_every_stage(dense):
    em = _emulate(dense["x"], dense["W"], dense["dy"])
    dgu, dx = _stages(dense, em)
    for name, st in dgu.items():
        assert st.outside == 0, name
        assert st.res.rate <= P._RATE[F16], (name, st.res.rate)
        print(f"[stages] faithful {name}: worst {st.res.worst:.3f} rate {st.res.rate:.4f} γ share {st.res.g_used:.3f}")
    assert dx.worst <= 1.0 and dx.rate <= P._RATE[F16] and dx.ok_rows, dx
    print(f"[stages] faithful dx: worst {dx.worst:.3f} rate {dx.rate:.4f} γ share {dx.g_used:.3f}; "
          f"old contract {_old_contract(dense, em['dx']):.4f}")
    assert _old_contract(dense, em["dx"]) <= 1.0


# the issue's table: (mutant, stage it breaks, what the end-to-end ε contract says: passes it or catches it)
DX_MUTANTS = ["one du column dropped", "first 64-wide w3 block dropped", "one W1 group's scales 1.6 % off",
              "one dx tile's w3 part × (1 + 2⁻⁸)"]
DGU_MUTANTS = [("dh rounded to 16 bits", "dg"), ("du from unrounded silu(g)", "du"), ("silu′ = σ", "dg")]


@pytest.mark.parametrize("mutant", DX_MUTANTS)
def test_dx_mutants_fail_the_dx_stage(dense, mutant):
    em = _emulate(dense["x"], dense["W"], dense["dy"], mutant)
    dgu, dx = _stages(dense, em)
    assert all(st.outside == 0 for st in dgu.values())            # dg and du are intact
    assert dx.worst > 10.0, f"{mutant}: dx err/bound {dx.worst:.3g}"
    old = _old_contract(dense, em["dx"])
    print(f"[stages] {mutant}: dx err/bound {dx.worst:.1f}, old contract {old:.3f}")
    if mutant == "first 64-wide w3 block dropped":
        assert old > 1.0                                          # the only one the ε contract catches
    else:
        assert old <= 1.0, f"{mutant}: the old contract catches it ({old:.3f})"


@pytest.mark.parametrize("mutant,stage", DGU_MUTANTS)
def test_dg_du_mutants_fail_their_stage(dense, mutant, stage):
    em = _emulate(dense["x"], dense["W"], dense["dy"], mutant)
    dgu, dx = _stages(dense, em)
    st = dgu[stage]
    share = st.outside / st.n
    print(f"[stages] {mutant}: {stage} {100 * share:.1f} % outside; old contract {_old_contract(dense, em['dx']):.4f}")
    assert share > 0.01, f"{mutant}: only {st.outside} of {st.n} {stage} elements outside"
    assert dx.worst <= 1.0                                        # dx is right on the dg / du it read
    if mutant != "silu′ = σ":                                    # the issue's table rows: the ε contract passes them
        assert _old_contract(dense, em["dx"]) <= 1.0


# --------------------------------------------------------------------------- the experts' bit-exact stages
def test_dy_pair_bit_exact_and_the_double_rounding_mutant():
    rng = np.random.default_rng(1)
    T, k = 64, 2
    for dt, tdt in ((F16, torch.float16), (BF16, torch.bfloat16)):
        dy = P.activations("student_t", T, H, dt, seed=2)
        w = rng.random((T, k)).astype(np.float32)
        # torch's own fp32 product and round to nearest even: the kernel's arithmetic, independently of numpy
        dyt = torch.from_numpy(dy).to(tdt).float()
        faithful = (torch.from_numpy(w)[:, :, None] * dyt[:, None, :]).to(tdt).double().numpy()
        B.check_exact(faithful, B.dy_pair(dy, w, dt), what=f"dy_pair {dt}")
        # rnd(rnd(w)·dy): w rounded to the dtype first
        mut = (torch.from_numpy(w).to(tdt).float()[:, :, None] * dyt[:, None, :]).to(tdt).double().numpy()
        assert (~B.same_bits(mut, B.dy_pair(dy, w, dt))).mean() > 0.05
        # 16-bit weights: the product is exact in fp32, so both orders agree
        w16 = P.round_dt(w, dt)
        faithful = (torch.from_numpy(w16.astype(np.float32)).to(tdt).float()[:, :, None] * dyt[:, None, :]).to(tdt)
        B.check_exact(faithful.double().numpy(), B.dy_pair(dy, w16, dt), what=f"dy_pair 16-bit w {dt}")


def _combine_torch(dxp, idx, E, tdt, order=None, invalid_adds=False):
    T, k, _ = dxp.shape
    acc = torch.zeros(T, dxp.shape[2], dtype=torch.float32)
    x = torch.from_numpy(dxp)
    for j in (order or range(k)):
        ok = torch.from_numpy(((idx[:, j] >= 0) & (idx[:, j] < E)) | invalid_adds)
        acc = torch.where(ok[:, None], acc + x[:, j], acc)
    return acc.to(tdt).double().numpy()


@pytest.mark.parametrize("dt,tdt", [(F16, torch.float16), (BF16, torch.bfloat16)])
def test_dx_combine_bit_exact_and_its_mutants(dt, tdt):
    rng = np.random.default_rng(3)
    T, E = 256, 8
    for k in (2, 4):
        idx = rng.integers(0, E, (T, k))
        idx[rng.random((T, k)) < 0.2] = E                         # invalid ids: their slot is skipped
        mag = np.array([1.0, 300.0, 1.0, 300.0])[:k]              # cancelling slots: fp32 order shows after rounding
        dxp = (rng.standard_normal((T, k, H)) * mag[None, :, None]).astype(np.float32)
        want = B.dx_combine(dxp, idx, E, dt)
        B.check_exact(_combine_torch(dxp, idx, E, tdt), want, what=f"combine k={k}")
        rev = _combine_torch(dxp, idx, E, tdt, order=list(range(k))[::-1])
        if k == 2:      # 0 + a + b and 0 + b + a are the same fp32 sum: the order cannot show at k = 2
            B.check_exact(rev, want)
        else:
            assert (~B.same_bits(rev, want)).sum() > 0, "reverse slot order at k = 4"
        assert (~B.same_bits(_combine_torch(dxp, idx, E, tdt, invalid_adds=True), want)).mean() > 0.1
