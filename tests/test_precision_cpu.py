"""The ulp-level checker of tests/_precision.py has teeth: each bug class a W4A16 kernel could have is restated as a
NumPy mutant of the exact computation, run on the GPU tests' own layer and activation generators, and the check must
reject it while it accepts the correctly rounded result and an fp32 evaluation of the kernels' Σx formulation.
No GPU."""
import numpy as np
import pytest

from oracle import w4a16_oracle as O
from tests import _precision as P
from tests.test_imma_format_cpu import to_digits

K, N, G = 1024, 128, 128


def _parts(d, dt):
    q, z, s, g, b = P.layer_parts(d, dt)
    return q.astype(np.float64), z.astype(np.float64), s, g, (0.0 if b is None else b)


def sum_x_form(x, d, dt, round_sx=False, shift_group_row=False, zero16=False, drop_row=None, scales_via_fp16=False):
    """y = Σ_groups s_g·(Σ q·x − z_g·Σx) + b in float64 (sequential layers), with one optional bug switched in."""
    q, z, s, g, b = _parts(d, dt)
    x = np.asarray(x, dtype=np.float64)
    if zero16:          # the stored nibble 15 decoded as zero 16 instead of 0
        z = np.where(z == 0, 16.0, z)
    if scales_via_fp16:
        s = P.round_dt(s, "float16")
    if drop_row is not None:
        x = x.copy()
        x[:, drop_row:drop_row + 8] = 0
    gs = d["group_size"]
    y = np.zeros((x.shape[0], q.shape[1]))
    for gi in range(d["K"] // gs):
        k0, k1 = gi * gs, (gi + 1) * gs
        if shift_group_row and gi > 0:          # the first k8-row of this group gets the previous group's scale / zero
            r = slice(k0, k0 + 8)
            y += x[:, r] @ (s[gi - 1] * (q[r] - z[gi - 1]))
            k0 += 8
        sx = x[:, k0:k1].sum(axis=1, keepdims=True)
        if round_sx:
            sx = P.round_dt(sx, dt)
        y += s[gi] * (x[:, k0:k1] @ q[k0:k1] - z[gi] * sx)
    return y + b


def _layer(dt, act_order=False, seed=3):
    return P.realistic_layer(K, N, G, dt, seed=seed, act_order=act_order, bias=True)


def _rejected(y, d, x, path, dt, what):
    ref = P.reference(d, x, path, dt)
    r = P.measure(P.round_dt(y, dt), ref, path, dt)
    assert not r.passed(path.rate[dt]), f"{what}: mutant accepted (worst {r.worst:.3g}, rate {r.rate:.4f})"
    return r


# --------------------------------------------------------------------------- the exact computations are accepted
@pytest.mark.parametrize("dt", ["float16", "bfloat16"])
@pytest.mark.parametrize("path", sorted(P.PATHS))
def test_correctly_rounded_result_is_accepted(dt, path):
    pth = P.PATHS[path]
    d = _layer(dt, act_order=True)
    for kind in P.acts_for(dt):
        x = P.activations(kind, 4, K, dt, seed=1)
        ref = P.reference(d, x, pth, dt)
        y = P.round_dt(ref.ystar, dt)
        y[ref.bad_rows] = np.nan
        r = P.check(y, ref, pth, dt, what=f"{path} {dt} {kind}")
        assert r.worst <= 0.5 and r.rate == 0.0


@pytest.mark.parametrize("dt", ["float16", "bfloat16"])
@pytest.mark.parametrize("kind", ["gauss", "offset", "massive", "row_scale"])
def test_fp32_sum_x_formulation_is_accepted(dt, kind):
    """What the GEMV computes, in fp32: per group a = Σ q·x, Σx, s·(a − z·Σx), summed over the groups in fp32."""
    d = _layer(dt)
    x = P.activations(kind, 4, K, dt, seed=2)
    q, z, s, g, b = _parts(d, dt)
    y = np.zeros((4, N), dtype=np.float32)
    x32 = x.astype(np.float32)
    for gi in range(K // G):
        r = slice(gi * G, (gi + 1) * G)
        a = x32[:, r] @ q[r].astype(np.float32)
        sx = x32[:, r].sum(axis=1, keepdims=True, dtype=np.float32)
        y = y + s[gi].astype(np.float32) * (a - z[gi].astype(np.float32) * sx)
    y = y + np.float32(b) if np.ndim(b) else y
    P.check(P.round_dt(y.astype(np.float64), dt), P.reference(d, x, P.PATHS["gemv"], dt), P.PATHS["gemv"], dt,
            what=f"fp32 Σx form {dt} {kind}")


# --------------------------------------------------------------------------- one mutant per bug class
def test_mutant_sum_x_rounded_to_dtype_is_rejected():
    dt = "float16"
    d = _layer(dt)
    x = P.activations("offset", 4, K, dt, seed=4)
    _rejected(sum_x_form(x, d, dt, round_sx=True), d, x, P.PATHS["gemv"], dt, "Σx rounded")


def test_mutant_weights_rounded_on_exact_weight_path_is_rejected():
    dt = "float16"
    d = _layer(dt)
    x = P.activations("gauss", 4, K, dt, seed=5)
    q, z, s, g, b = _parts(d, dt)
    y = x.astype(np.float64) @ P.round_dt(s[g] * (q - z[g]), dt) + b
    r = _rejected(y, d, x, P.PATHS["gemv"], dt, "weights rounded")
    assert r.rate > P.PATHS["gemv"].rate[dt]            # a sub-ulp bug: caught by the sharpness check


@pytest.mark.parametrize("row", [K // 2, K - 8])
def test_mutant_k8_row_dropped_at_split_boundary_is_rejected(row):
    dt = "float16"
    d = _layer(dt)
    x = P.activations("gauss", 4, K, dt, seed=6)
    _rejected(sum_x_form(x, d, dt, drop_row=row), d, x, P.PATHS["gemv"], dt, "dropped k8-row")


def test_mutant_previous_group_constants_on_first_row_of_group_is_rejected():
    dt = "float16"
    d = _layer(dt)
    x = P.activations("gauss", 4, K, dt, seed=7)
    _rejected(sum_x_form(x, d, dt, shift_group_row=True), d, x, P.PATHS["gemv"], dt, "group boundary off by a row")


def test_mutant_inverted_act_order_permutation_is_rejected():
    dt = "float16"
    d = _layer(dt, act_order=True)
    x = P.activations("gauss", 4, K, dt, seed=8)
    q, z, s, g, b = _parts(d, dt)
    W = s[g] * (q - z[g])
    perm = O.make_sequential_perm(d["g_idx"])
    inv = np.argsort(perm)
    y = x.astype(np.float64)[:, inv] @ W[perm] + b      # sorted row j multiplied with x[inv[j]] instead of x[perm[j]]
    _rejected(y, d, x, P.PATHS["gemv"], dt, "inverted permutation")


def test_mutant_bf16_scales_read_through_fp16_is_rejected():
    dt = "bfloat16"
    d = _layer(dt)
    assert (P.layer_parts(d, dt)[2] < 2.0 ** -14).any()        # the generator's bf16 layers hold sub-fp16-normal scales
    x = P.activations("gauss", 4, K, dt, seed=9)
    _rejected(sum_x_form(x, d, dt, scales_via_fp16=True), d, x, P.PATHS["gemv"], dt, "bf16 scales via fp16")


def _imma_digits_y(x, d, dt, pe_from_row=None):
    """IMMA arithmetic: per row and 128-k block x -> integers at scale 2^pe, exact integer dot products, back to float."""
    q, z, s, g, b = _parts(d, dt)
    W = s[g] * (q - z[g])
    M = x.shape[0]
    y = np.zeros((M, W.shape[1]))
    for k0 in range(0, K, 128):
        blk = x[:, k0:k0 + 128]
        pes = [to_digits(blk[m])[2] for m in range(M)]
        for m in range(M):
            pe = pes[m if pe_from_row is None else pe_from_row]
            xi = np.rint(blk[m].astype(np.float64) * 2.0 ** pe)
            y[m] += (xi * 2.0 ** -pe) @ W[k0:k0 + 128]
    return y + b


def test_imma_digit_arithmetic_is_accepted():
    dt = "float16"
    d = _layer(dt)
    x = P.activations("row_scale", 4, K, dt, seed=10)
    P.check(P.round_dt(_imma_digits_y(x, d, dt), dt), P.reference(d, x, P.PATHS["imma"], dt), P.PATHS["imma"], dt,
            what="imma digits")


def test_mutant_imma_block_exponent_from_another_row_is_rejected():
    """The digits keep 2^11 of headroom below the block maximum, so the wrong exponent shows on rows that lie more than
    that apart: bf16 rows 10^-2 .. 10^5, every row quantised with the exponent of the last (largest) one."""
    dt = "bfloat16"
    d = _layer(dt)
    x = P.activations("row_scale", 8, K, dt, seed=10)
    _rejected(_imma_digits_y(x, d, dt, pe_from_row=7), d, x, P.PATHS["imma"], dt, "IMMA exponent of row 7")


def test_mutant_no_wrap_rule_is_rejected():
    dt = "float16"
    d = _layer(dt)
    assert (O.unpack_qzeros(d["qzeros"]) == 0).any()         # the generator stores zero 0 as the nibble 15
    x = P.activations("gauss", 4, K, dt, seed=11)
    _rejected(sum_x_form(x, d, dt, zero16=True), d, x, P.PATHS["gemv"], dt, "no wrap rule")


# --------------------------------------------------------------------------- generators and helpers
def test_round_dt_matches_numpy_fp16_and_the_bf16_bit_rounding():
    from oracle import moe_oracle as MO
    rng = np.random.default_rng(0)
    a = (rng.standard_normal(20000) * 10.0 ** rng.uniform(-9, 4, 20000)).astype(np.float32)
    assert np.array_equal(P.round_dt(a, "float16"), a.astype(np.float16).astype(np.float64))
    b = (rng.standard_normal(20000) * 10.0 ** rng.uniform(-35, 35, 20000)).astype(np.float32)
    assert np.array_equal(P.round_dt(b, "bfloat16"), MO.round_to(b, "bfloat16").astype(np.float64))
    assert P.ulp(1.0, "float16") == 2.0 ** -10 and P.ulp(0.0, "float16") == 2.0 ** -24
    assert P.ulp(1.0, "bfloat16") == 2.0 ** -7


@pytest.mark.parametrize("dt", ["float16", "bfloat16"])
def test_layer_generator_is_gptq_like(dt):
    d = P.realistic_layer(1024, 256, 128, dt, seed=1, act_order=True)
    q, z, s, g, _ = P.layer_parts(d, dt)
    assert not np.array_equal(g, np.arange(1024) // 128) and np.bincount(g).tolist() == [128] * 8
    assert abs(float(np.mean(q - z[g]))) < 2.0                                 # (q − z) centred near zero
    colmax = s.max(axis=0)
    assert np.percentile(colmax, 95) / np.percentile(colmax, 5) > 30          # scales spread over decades
    assert (O.unpack_qzeros(d["qzeros"]) == 0).any()                          # wrap-rule groups
    assert np.array_equal(P.round_dt(s, dt), s)
    if dt == "bfloat16":
        assert (s < 2.0 ** -14).any()


@pytest.mark.parametrize("dt", ["float16", "bfloat16"])
def test_activation_generators(dt):
    for kind in P.acts_for(dt):
        x = P.activations(kind, 6, 512, dt, seed=0)
        assert np.array_equal(P.round_dt(x, dt), x.astype(np.float64)), kind
        fin = np.isfinite(x)
        assert fin.all() == (kind != "inf"), kind
    x = P.activations("offset", 6, 512, dt)
    assert x.mean() > 3.5
    if dt == "float16":
        assert (np.abs(P.activations("subnormal", 2, 512, dt)) < 2.0 ** -14).mean() > 0.99
    else:
        ht = np.abs(P.activations("huge_tiny", 2, 512, dt))
        assert ht[0].max() > 1e5 and ht[1].max() < 1e-19


# --------------------------------------------------------------------------- bf16 digit format (IMMA / chain)
def _bf16(a):
    return P.round_dt(np.asarray(a, dtype=np.float64), "bfloat16").astype(np.float32)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("decade", [-30, -10, 0, 5, 30])
def test_bf16_digits_over_the_wide_exponent_range(seed, decade):
    """bf16 blocks far beyond fp16's range (up to 1e30) and far below it: exact balanced digits, 2^-22 relative error."""
    rng = np.random.default_rng(seed)
    x = _bf16(rng.standard_normal(128) * 10.0 ** decade)
    xi, dig, pe = to_digits(x)
    assert np.abs(xi).max() < 2 ** 22
    assert np.array_equal(xi, np.rint(x.astype(np.float64) * 2.0 ** pe).astype(np.int32))
    recon = dig[:, 0].astype(np.int64) * 65536 + dig[:, 1].astype(np.int64) * 256 + dig[:, 2].astype(np.int64)
    assert np.array_equal(recon, xi.astype(np.int64))
    xmax = np.abs(x.astype(np.float64)).max()
    assert np.abs(xi * 2.0 ** -pe - x.astype(np.float64)).max() <= xmax * 2.0 ** -22


@pytest.mark.parametrize("log2max,clamped", [(-104, False), (-105, False), (-106, True), (-115, True)])
def test_bf16_pe_clamp_edge(log2max, clamped):
    """Rows with |x|max below 2^-105 reach the clamp pe = 126: their error is 2^-127 absolute, no longer relative."""
    rng = np.random.default_rng(1)
    x = _bf16(rng.uniform(-1, 1, 128) * 2.0 ** log2max)
    x[0] = np.float32(2.0 ** log2max * 1.5)
    xi, dig, pe = to_digits(x)
    xmax = np.abs(x.astype(np.float64)).max()
    assert pe == 126 if log2max <= -105 else pe < 126            # |x|max in [2^-105, 2^-104) is the last unclamped binade
    err = np.abs(xi * 2.0 ** -pe - x.astype(np.float64)).max()
    assert err <= (2.0 ** -127 if clamped else xmax * 2.0 ** -22)
    assert np.abs(xi).max() < 2 ** 22


def test_bf16_subnormal_block_reads_as_zero():
    """A block whose maximum is an fp32 (= bf16) subnormal has e == 0: pe = 0 and every digit is 0, an absolute error
    below 2^-126 per element — the documented floor of the bf16 digit domain."""
    x = _bf16(np.linspace(-1, 1, 128) * 2.0 ** -130)
    xi, dig, pe = to_digits(x)
    assert pe == 0 and not xi.any() and not dig.any()
    assert np.abs(x.astype(np.float64)).max() < 2.0 ** -126
