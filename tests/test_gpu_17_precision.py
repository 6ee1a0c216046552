"""Every W4A16 kernel path against the float64 reference of tests/_precision.py, to the ulp, in fp16 and bf16, on
GPTQ-like layers (scales over decades, heavy columns, wrap-rule zeros, act-order) and on activations where kernels go
wrong (per-channel offsets, heavy tails, massive channels, rows of very different magnitude, subnormals, inf).

Each case asserts |y − y*| ≤ ulp(y*) + γ·A + F per element and a bound on the rate of elements that differ from the
correctly rounded y*; the module prints, per path and dtype, the largest err/bound and the largest mismatch rate it
saw.  Wide layers are checked on a column slice (every output column is independent)."""
import functools

import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from tests import _precision as P
from tests._util import make_layer

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTS = [F16, BF16]
_SUMMARY: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _print_summary():
    yield
    print("\n[precision] path               dtype     cases  max err/bound  max mismatch rate  max γ share")
    for (path, dt), (n, worst, rate, gu) in sorted(_SUMMARY.items()):
        print(f"[precision] {path:<18} {dt:<9} {n:>5}  {worst:13.3f}  {rate:17.4f}  {gu:11.3f}")


def _check(y, ref, path, dtype, what):
    pth = P.PATHS[path]
    # paths that sum (o + q)·x are also measured against the o = 0 bound (recorded, not asserted)
    plain = ((path + " (o=0)", P.without_offset(ref)),) if pth.o(dtype) else ()
    for name, rf in ((path, ref),) + plain:
        r = P.measure(y, rf, pth, dtype)
        key = (name, P.dt_name(dtype))
        n, w, rt, gu = _SUMMARY.get(key, (0, 0.0, 0.0, 0.0))
        _SUMMARY[key] = (n + 1, max(w, r.worst), max(rt, r.rate), max(gu, r.g_used))
    P.check(y, ref, pth, dtype, what=what)


@functools.lru_cache(maxsize=None)
def _layer(K, N, g, dt, act=False, bias=True, seed=0):
    return P.wide_layer(K, N, g, dt, seed=seed, act_order=act, bias=bias)


def _run(d, x, dtype, kernel=_lib.KERNEL_AUTO, tune=(0, 0), cols=None):
    lin = make_layer(d, dtype=dtype)
    lin.kernel, lin.tune = kernel, tune
    y = lin(torch.from_numpy(x).to(dtype).cuda())
    torch.cuda.synchronize()
    if cols is not None:
        y = y[:, cols[0]:cols[1]]
    return y.double().cpu().numpy()


def _case(path, d, M, kind, dtype, kernel, tune=(0, 0), cols=None, seed=0, what=""):
    x = P.activations(kind, M, d["K"], dtype, seed=seed)
    y = _run(d, x, dtype, kernel, tune, cols)
    ref = P.reference(d, x, P.PATHS[path], dtype, cols=cols)
    _check(y, ref, path, dtype, f"{path} {what} {P.dt_name(dtype)} {kind} M={M}")


# --------------------------------------------------------------------------- GEMV
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("kind", P.ACTS)
@pytest.mark.parametrize("M", [1, 2, 3, 4, 11])
def test_gemv_tails_g96_act_order(dtype, kind, M):
    if kind not in P.acts_for(dtype):
        pytest.skip(f"{kind} is not a {P.dt_name(dtype)} distribution")
    d = _layer(392, 288, 96, P.dt_name(dtype), act=True)
    _case("gemv", d, M, kind, dtype, _lib.KERNEL_GEMV, seed=M, what="392x288 g96")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("ln", [8, 16, 32])
@pytest.mark.parametrize("split", [1, 2, 4, 8])
def test_gemv_ln_split(dtype, ln, split):
    d = _layer(4096, 520, 128, P.dt_name(dtype))
    _case("gemv", d, 3, "offset", dtype, _lib.KERNEL_GEMV, tune=(ln, split), what=f"ln={ln} split={split}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("kind", ["gauss", "offset"])
def test_gemv_one_long_group(dtype, kind):
    d = _layer(11008, 256, -1, P.dt_name(dtype))
    _case("gemv", d, 2, kind, dtype, _lib.KERNEL_GEMV, what="11008x256 g=-1")


# --------------------------------------------------------------------------- IMMA (tile form tune0 1 / 4, persistent 2)
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("form", [1, 4, 2])
@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 6, 7, 8])
def test_imma_forms(dtype, form, M):
    d = _layer(2048, 392, 128, P.dt_name(dtype), act=True)
    kind = P.acts_for(dtype)[M % len(P.acts_for(dtype))]
    _case("imma", d, M, kind, dtype, _lib.KERNEL_IMMA, tune=(form, 0), seed=M, what=f"form {form}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("kind", P.ACTS)
def test_imma_activations(dtype, kind):
    if kind not in P.acts_for(dtype):
        pytest.skip(f"{kind} is not a {P.dt_name(dtype)} distribution")
    d = _layer(4096, 520, 128, P.dt_name(dtype))
    _case("imma", d, 4, kind, dtype, _lib.KERNEL_IMMA, what="4096x520")


def test_imma_bf16_rows_at_the_clamp_edge():
    """bf16 rows whose block maximum is just above, at and below 2^-105 (the pe clamp): the bound follows the clamp."""
    d = _layer(1024, 256, 128, "bfloat16", bias=False)
    x = P.activations("gauss", 4, 1024, BF16, seed=3)
    x = P.round_dt(x / np.abs(x).max(axis=1, keepdims=True) * 2.0 ** np.array([-100.0, -104.5, -105.5, -112.0])[:, None],
                   "bfloat16").astype(np.float32)
    for form in (1, 2):
        y = _run(d, x, BF16, _lib.KERNEL_IMMA, (form, 0))
        _check(y, P.reference(d, x, P.PATHS["imma"], BF16), "imma", BF16, f"imma clamp edge form {form}")


# --------------------------------------------------------------------------- skinny (mma.sync)
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("split", [0, 1, 2, 4])
@pytest.mark.parametrize("M", [1, 5, 8])
def test_skinny_splits(dtype, split, M):
    d = _layer(2048, 392 + 8, 64, P.dt_name(dtype), act=True)
    kind = ["offset", "massive", "row_scale"][M % 3]
    _case("skinny", d, M, kind, dtype, _lib.KERNEL_SKINNY, tune=(0, split), seed=M, what=f"split {split}")


# --------------------------------------------------------------------------- wgmma GEMM
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("mt", [32, 64, 128])
@pytest.mark.parametrize("split", [1, 2, 4])
def test_gemm_tiles_and_splits(dtype, mt, split):
    d = _layer(2048, 512, 128, P.dt_name(dtype), act=True)
    _case("gemm", d, 96, "offset" if split != 2 else "student_t", dtype, _lib.KERNEL_GEMM, tune=(mt, split),
          seed=mt + split, what=f"mt={mt} split={split}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_gemm_tile128_ragged_m(dtype):
    d = _layer(1024, 512, 128, P.dt_name(dtype))
    _case("gemm", d, 300, "massive", dtype, _lib.KERNEL_GEMM, tune=(128, 1), what="mt=128 split=1")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("kind", P.ACTS)
def test_gemm_activations(dtype, kind):
    if kind not in P.acts_for(dtype):
        pytest.skip(f"{kind} is not a {P.dt_name(dtype)} distribution")
    d = _layer(4096, 512, 128, P.dt_name(dtype))
    _case("gemm", d, 40, kind, dtype, _lib.KERNEL_GEMM, what="4096x512")


# --------------------------------------------------------------------------- AUTO on full-size layers
def _auto_path(M, K, N, g):
    """The path AUTO takes (abi.cu dispatch) for an act-order-free layer with 128-k groups and N % 32 == 0."""
    huge = K * N >= 1e8
    if M == 1:
        return "gemv"
    if M <= 4 or (M == 5 and huge):
        return "imma"
    if M <= 8 and not huge:
        return "skinny"
    return "gemm"


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 6, 7, 8, 9, 64, 300])
def test_auto_4096x11008(dtype, M):
    K, N = 4096, 11008
    d = _layer(K, N, 128, P.dt_name(dtype), act=True)
    cols = (N - 512, N - 256) if M % 2 else (1024, 1280)
    path = _auto_path(M, K, N, 128)
    _case(path, d, M, ["offset", "gauss", "massive", "student_t"][M % 4], dtype, _lib.KERNEL_AUTO, cols=cols, seed=M,
          what="auto 4096x11008")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 5, 6, 7, 8])
def test_auto_28672x8192_large_layer_branch(dtype, M):
    """K·N ≥ 1e8: AUTO takes the IMMA kernel at M = 5 and the 32-row wgmma tile at 6..8."""
    K, N = 28672, 8192
    d = _layer(K, N, 128, P.dt_name(dtype))
    _case(_auto_path(M, K, N, 128), d, M, "offset" if M % 2 else "gauss", dtype, _lib.KERNEL_AUTO, cols=(4096, 4352),
          seed=M, what="auto 28672x8192")


# --------------------------------------------------------------------------- forward_group
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 2, 3, 4])
def test_forward_group_shared_act_order(dtype, M):
    """q|k|v-like siblings with one act-order permutation: GEMV group at M = 1, IMMA group at 2..4."""
    from autogptq_b200 import forward_group

    dt = P.dt_name(dtype)
    K = 2048
    first = _layer(K, 512, 128, dt, act=True, seed=1)
    ds = [first] + [P.realistic_layer(K, n, 128, dt, seed=2 + i, bias=(i == 0), g_idx=first["g_idx"])
                    for i, n in enumerate((264, 384))]
    lins = [make_layer(d, dtype=dtype) for d in ds]
    x = P.activations(["offset", "massive", "student_t", "row_scale"][M - 1], M, K, dtype, seed=M)
    ys = forward_group(lins, torch.from_numpy(x).to(dtype).cuda())
    torch.cuda.synchronize()
    path = "gemv" if M == 1 else "imma"
    for i, (d, y) in enumerate(zip(ds, ys)):
        _check(y.double().cpu().numpy(), P.reference(d, x, P.PATHS[path], dtype), path, dtype, f"group layer {i} M={M}")


# --------------------------------------------------------------------------- DecodeChain
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 2])
def test_decode_chain_plain_stages(dtype, M):
    """x -> [A, B] -> C(A's output): each stage checked on the input it actually read."""
    from autogptq_b200.chain import DecodeChain

    dt = P.dt_name(dtype)
    dA, dB = _layer(2048, 1024, 128, dt, seed=3), _layer(2048, 256, 128, dt, seed=4)
    dC = _layer(1024, 640, 128, dt, seed=5)
    A, B, C = (make_layer(d, dtype=dtype) for d in (dA, dB, dC))
    ch = DecodeChain(M=M, dtype=dtype)
    xin = ch.input(2048)
    ya, yb = ch.stage([A, B], xin)
    (yc,) = ch.stage([C], ya)
    ch.build()
    for kind in ("offset", "massive", "row_scale"):
        x = P.activations(kind, M, 2048, dtype, seed=7)
        xin.copy_(torch.from_numpy(x).to(dtype).cuda())
        ch.run()
        torch.cuda.synchronize()
        xs = xin.double().cpu().numpy()
        for d, xi, y, what in ((dA, xs, ya, "A"), (dB, xs, yb, "B"), (dC, ya.double().cpu().numpy(), yc, "C")):
            _check(y.double().cpu().numpy(), P.reference(d, xi, P.PATHS["chain"], dtype), "chain", dtype,
                   f"chain {kind} stage {what} M={M}")


# --------------------------------------------------------------------------- dgrad
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("kernel,M", [(_lib.DGRAD_CUDA_CORE, 3), (_lib.DGRAD_CUDA_CORE, 16), (_lib.DGRAD_WGMMA, 64),
                                      (_lib.DGRAD_WGMMA, 300)])
@pytest.mark.parametrize("kind", ["gauss", "offset", "massive"])
def test_dgrad_kernels(dtype, kernel, M, kind):
    d = _layer(2048, 1024, 128, P.dt_name(dtype), act=True)
    lin = make_layer(d, dtype=dtype)
    dy = P.activations(kind, M, d["N"], dtype, seed=M)
    dx = lin.input_grad(torch.from_numpy(dy).to(dtype).cuda(), kernel=kernel)
    torch.cuda.synchronize()
    path = "dgrad" if kernel == _lib.DGRAD_WGMMA else "dgrad_cuda_core"
    _check(dx.double().cpu().numpy(), P.reference_dgrad(d, dy, P.PATHS[path], dtype), path, dtype, f"{path} {kind} M={M}")


# --------------------------------------------------------------------------- unaligned x
def _offset_view(x):
    """A contiguous copy of x whose storage starts 2 bytes past a 16-byte boundary (buf[1:1 + n].view(...))."""
    buf = torch.empty(x.numel() + 8, dtype=x.dtype, device=x.device)
    v = buf[1:1 + x.numel()].view(x.shape)
    v.copy_(x)
    assert v.is_contiguous() and v.data_ptr() % 16 != 0
    return v


@pytest.mark.parametrize("M", [1, 64])
def test_unaligned_x_through_every_entry_point(M):
    from autogptq_b200 import forward_group
    from autogptq_b200.mlp import forward_gate_up
    from autogptq_b200.moe import QuantExperts

    K = 512
    ds = [_layer(K, 256, 128, "float16", seed=s) for s in (11, 12)]
    a, b = (make_layer(d) for d in ds)
    x = torch.from_numpy(P.activations("gauss", M, K, F16, seed=M)).half().cuda()
    xv = _offset_view(x)
    assert torch.equal(a(xv), a(x))
    for yv, y in zip(forward_group([a, b], xv), forward_group([a, b], x)):
        assert torch.equal(yv, y)
    assert torch.equal(forward_gate_up(a, b, xv), forward_gate_up(a, b, x))
    # two experts: gate / up K -> 256, down 256 -> K
    w1s, w3s = [make_layer(_layer(K, 256, 128, "float16", seed=20 + e)) for e in range(2)], [a, b]
    w2s = [make_layer(_layer(256, K, 128, "float16", seed=30 + e)) for e in range(2)]
    ex = QuantExperts(w1s, w3s, w2s)
    idx = torch.from_numpy(np.random.default_rng(M).integers(0, 2, (M, 2))).cuda()
    w = torch.full((M, 2), 0.5, device="cuda")
    with torch.no_grad():
        assert torch.equal(ex(xv, idx, w), ex(x, idx, w))
