"""GPU parity: the integer tensor-core decode kernel (M <= 8, AGB200_KERNEL_IMMA) through the QuantLinear module /
C ABI vs the exact oracle.  x goes through a 24-bit block fixed point (exact for everything within 2^-11 of the
chunk maximum), products accumulate in int32: the tolerance is the same as for the fp32-accumulating GEMV."""
import numpy as np
import pytest
import torch

import autogptq_b200
from oracle import w4a16_oracle as O
from tests._util import assert_parity, make_layer, oracle_exact, rand_x

pytestmark = pytest.mark.gpu
IMMA = 6


def _run(d, x, tune=(0, 0), dtype=torch.float16, kernel=IMMA):
    lin = make_layer(d, dtype=dtype)
    lin.kernel = kernel
    lin.tune = tune
    xt = torch.from_numpy(np.asarray(x, dtype=np.float32)).to(dtype).cuda()
    y = lin(xt)
    torch.cuda.synchronize()
    return y.float().cpu().numpy(), xt.float().cpu().numpy()


@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 6, 8])
@pytest.mark.parametrize("K,N,g", [(1024, 1024, 128), (512, 264, 32), (384, 136, -1), (4096, 512, 128), (2048, 2048, 64),
                                   (1056, 72, 96), (11008, 256, 128)])
def test_imma_shapes(M, K, N, g):
    d = O.random_packed(K, N, g, seed=K + N + M, bias=(M % 2 == 0))
    y, x = _run(d, rand_x(M, K, seed=M))
    assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what=f"imma M={M} K={K} N={N} g={g}")


@pytest.mark.parametrize("split", [1, 2, 4, 8])
@pytest.mark.parametrize("wn", [1, 4])
@pytest.mark.parametrize("M", [1, 4, 7])
def test_imma_variants(split, wn, M):
    K, N, g = 4096, 520, 128
    d = O.random_packed(K, N, g, seed=11, bias=True)
    y, x = _run(d, rand_x(M, K, seed=2), tune=(wn, split))
    assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what=f"imma split={split} wn={wn} M={M}")


@pytest.mark.parametrize("M", [1, 2, 5, 8])
@pytest.mark.parametrize("K,N,g", [(4096, 4096, 128), (11008, 1024, 128), (2048, 4768, 128), (1024, 264, -1), (8192, 520, -1),
                                   (256, 40, 128), (28672, 136, 128), (8192, 4768, 256)])
def test_imma_persistent_form(M, K, N, g):
    """tune0 = 2 forces the one-CTA-per-SM register-ring form (AUTO's choice for 2 <= M <= 4 and 128-k groups); large
    K x M convert x in several K chunks."""
    d = O.random_packed(K, N, g, seed=K + N + M, bias=(M % 2 == 1))
    y, x = _run(d, rand_x(M, K, seed=M), tune=(2, 0))
    assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what=f"imma persistent M={M} K={K} N={N} g={g}")


def test_imma_persistent_is_deterministic_under_graph_replay():
    K, N, g, M = 4096, 5024, 128, 2
    d = O.random_packed(K, N, g, seed=5, bias=True)
    lin = make_layer(d)
    lin.kernel, lin.tune = IMMA, (2, 0)
    x = torch.from_numpy(rand_x(M, K, seed=9)).cuda()
    y0 = lin(x).clone()
    for _ in range(5):
        assert torch.equal(lin(x), y0)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        lin(x)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            yg = lin(x)
        for _ in range(5):
            graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, y0)
    assert_parity(y0.float().cpu().numpy(), oracle_exact(d, x.float().cpu().numpy()), atol_rms=6e-4, what="persistent")


def test_imma_persistent_act_order_and_bf16():
    K, N, g = 2048, 392, 128
    d = O.random_packed(K, N, g, seed=77, desc_act=True, zero_max=15, bias=True)
    for M in (1, 7):
        y, x = _run(d, rand_x(M, K, seed=5), tune=(2, 0))
        assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what="imma persistent act-order + wrap")
    d = O.random_packed(K, N, g, seed=78, scale_dtype=np.float32)
    d["scales"] = torch.from_numpy(d["scales"]).to(torch.bfloat16).float().numpy()
    y, x = _run(d, rand_x(3, K, seed=3, dtype=np.float32), tune=(2, 0), dtype=torch.bfloat16)
    assert_parity(y, oracle_exact(d, x), rtol=8e-3, atol_rms=4e-3, what="imma persistent bf16")


def test_imma_wrap_and_act_order():
    K, N, g = 1024, 384, 128
    d = O.random_packed(K, N, g, seed=23, desc_act=True, zero_max=15, bias=True)
    for M in (1, 8):
        y, x = _run(d, rand_x(M, K, seed=5))
        assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what="imma act-order + wrap")


def test_imma_more_than_8_rows():
    K, N, g, M = 512, 512, 128, 19            # forced: 3 passes
    d = O.random_packed(K, N, g, seed=29)
    y, x = _run(d, rand_x(M, K, seed=7))
    assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what="imma multi-pass")


@pytest.mark.parametrize("M", [1, 5])
def test_imma_bf16(M):
    K, N, g = 1024, 512, 128
    d = O.random_packed(K, N, g, seed=31, scale_dtype=np.float32)
    d["scales"] = torch.from_numpy(d["scales"]).to(torch.bfloat16).float().numpy()
    y, x = _run(d, rand_x(M, K, seed=3, dtype=np.float32), dtype=torch.bfloat16)
    assert_parity(y, oracle_exact(d, x), rtol=8e-3, atol_rms=4e-3, what="imma bf16")


def test_imma_dynamic_range_of_activations():
    """Block fixed point: large, tiny (fp16-subnormal) and outlier-dominated rows of x."""
    K, N, g = 1024, 256, 128
    d = O.random_packed(K, N, g, seed=37)
    x = rand_x(2, K, seed=9).astype(np.float32) * 100.0
    y, xr = _run(d, x.astype(np.float16))
    assert_parity(y, oracle_exact(d, xr), atol_rms=6e-4, what="large activations")
    xs = (rand_x(2, K, seed=10).astype(np.float32) * 1e-4).astype(np.float16)      # fp16-subnormal activations
    y2, xr2 = _run(d, xs)
    assert_parity(y2, oracle_exact(d, xr2), atol_rms=2e-3, what="tiny activations")
    # one massive activation (x2000) per row, as LLM down_proj inputs have: the other 1023 elements must still count.
    # Compare on the output with the outlier's own contribution removed (it would hide everything else).
    xo = rand_x(2, K, seed=12).astype(np.float32)
    xo[0, 17] = 2000.0
    xo[1, 900] = -1500.0
    xo = xo.astype(np.float16)
    y3, xr3 = _run(d, xo)
    ref = oracle_exact(d, xr3)
    assert_parity(y3, ref, atol_rms=6e-4, what="outlier activations")
    x_rest = xr3.copy()
    x_rest[0, 17] = 0.0
    x_rest[1, 900] = 0.0
    x_only = xr3 - x_rest
    rest_ref = oracle_exact(d, x_rest)
    rest_got = y3.astype(np.float64) - oracle_exact(d, x_only)            # fp16 output rounding of y3 dominates this
    err = np.abs(rest_got - rest_ref)
    ulp = np.abs(ref) * 2.0 ** -11 + 1e-3
    assert (err <= 1.01 * ulp + 2e-3 * np.sqrt(np.mean(rest_ref ** 2))).all(), float(err.max())


def test_imma_zero_and_nonfinite_activations():
    K, N, g = 512, 64, 128
    d = O.random_packed(K, N, g, seed=41)
    x = np.zeros((2, K), dtype=np.float16)
    x[1] = rand_x(1, K, seed=1)[0]
    y, xr = _run(d, x)
    assert (y[0] == 0).all()
    assert_parity(y[1:], oracle_exact(d, xr)[1:], atol_rms=6e-4, what="zero row next to a normal row")
    x[0, 5] = np.inf
    y, _ = _run(d, x)
    assert np.isnan(y[0]).all() or np.isinf(y[0]).any()       # the reference gives inf/nan there as well
    assert np.isfinite(y[1]).all()


def test_imma_agrees_with_gemv():
    K, N, g, M = 2048, 512, 128, 2
    d = O.random_packed(K, N, g, seed=21)
    x = rand_x(M, K, seed=8)
    y_i, _ = _run(d, x, kernel=IMMA)
    y_v, _ = _run(d, x, kernel=1)
    assert_parity(y_i, y_v, rtol=1e-3, atol_rms=6e-4, what="imma vs gemv")


def test_auto_picks_imma_for_decode_batches_and_falls_back():
    """AUTO: M <= 8 on 32-aligned shapes runs the integer kernel; group_size 16 / K % 32 != 0 still work (GEMV)."""
    for (K, N, g, M) in [(1024, 256, 128, 3), (1024, 256, 16, 3), (1000, 64, 40, 2)]:
        d = O.random_packed(K, N, g, seed=K + g)
        y, x = _run(d, rand_x(M, K, seed=M), kernel=0)
        assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what=f"auto K={K} g={g} M={M}")


@pytest.mark.parametrize("M", [1, 3, 8])
def test_forward_group_imma(M):
    K, g = 1024, 128
    Ns = [512, 136, 264]
    ds = [O.random_packed(K, N, g, seed=50 + i, bias=(i == 1)) for i, N in enumerate(Ns)]
    layers = [make_layer(d) for d in ds]
    x = torch.from_numpy(rand_x(M, K, seed=4)).cuda()
    ys = autogptq_b200.forward_group(layers, x)
    torch.cuda.synchronize()
    for d, yy in zip(ds, ys):
        assert_parity(yy.float().cpu().numpy(), oracle_exact(d, x.float().cpu().numpy()), atol_rms=6e-4, what=f"group M={M}")


@pytest.mark.parametrize("M", [1, 3])
def test_next_layer_prefetch_hint_does_not_change_results(M):
    """Opt-in learned next-layer L2 prefetch (agb200_w4_prefetch_hint): a pure hint - results must be bit-identical."""
    K, g = 1024, 128
    ds = [O.random_packed(K, n, g, seed=60 + i) for i, n in enumerate((1024, 1024, 1024))]
    layers = [make_layer(d) for d in ds]
    x = torch.from_numpy(rand_x(M, K, seed=4)).cuda()

    def chain():
        h = x
        outs = []
        for lin in layers * 2:                       # same order twice: the second pass runs with learned hints
            h = lin(h)
            outs.append(h.clone())
            h = (h / (h.abs().max() + 1e-3)).to(torch.float16)      # keep the chain in range
        torch.cuda.synchronize()
        return outs

    base = chain()
    autogptq_b200.set_next_layer_prefetch(True)
    try:
        chain()
        hinted = chain()
    finally:
        autogptq_b200.set_next_layer_prefetch(False)
    for a, b in zip(base, hinted):
        assert torch.isfinite(a).all() and torch.equal(a, b)
