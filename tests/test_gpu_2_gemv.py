"""GPU parity: the decode GEMV (M <= 4 per pass) through the QuantLinear module / C ABI vs the oracle."""
import numpy as np
import pytest
import torch

from oracle import w4a16_oracle as O
from tests._util import assert_parity, make_layer, oracle_exact, rand_x

pytestmark = pytest.mark.gpu


def _run(d, x, kernel=1, tune=(0, 0), dtype=torch.float16):
    lin = make_layer(d, dtype=dtype)
    lin.kernel = kernel
    lin.tune = tune
    xt = torch.from_numpy(np.asarray(x, dtype=np.float32)).to(dtype).cuda()
    y = lin(xt)
    torch.cuda.synchronize()
    return y.float().cpu().numpy(), xt.float().cpu().numpy()


@pytest.mark.parametrize("M", [1, 2, 3, 4])
@pytest.mark.parametrize("K,N,g", [(1024, 1024, 128), (512, 256, 32), (384, 136, -1), (4096, 512, 128)])
def test_gemv_auto(M, K, N, g):
    d = O.random_packed(K, N, g, seed=K + N + M, bias=(M % 2 == 0))
    y, x = _run(d, rand_x(M, K, seed=M))
    assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what=f"gemv M={M} K={K} N={N} g={g}")


@pytest.mark.parametrize("ln", [8, 16, 32])
@pytest.mark.parametrize("split", [1, 2, 4, 8])
def test_gemv_variants(ln, split):
    K, N, g, M = 2048, 520, 64, 2
    d = O.random_packed(K, N, g, seed=11, bias=True)
    y, x = _run(d, rand_x(M, K, seed=2), tune=(ln, split))
    assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what=f"gemv ln={ln} split={split}")


def test_gemv_wrap_rule():
    """stored nibble 15 -> zero 0 (every reference .cu kernel; qlinear_cuda_old.py:301-304)."""
    K, N, g = 256, 256, 64
    d = O.random_packed(K, N, g, seed=17, zero_max=15)
    assert (O.unpack_qzeros(d["qzeros"]) == 0).any()
    y, x = _run(d, rand_x(1, K))
    assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what="wrap rule")


@pytest.mark.parametrize("M", [1, 3])
def test_gemv_act_order(M):
    K, N, g = 1024, 384, 128
    d = O.random_packed(K, N, g, seed=23, desc_act=True, bias=True)
    y, x = _run(d, rand_x(M, K, seed=5))
    assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what="act-order gemv")


def test_gemv_more_rows_than_a_pass():
    K, N, g, M = 512, 512, 128, 11          # forced GEMV: 3 passes of <= 4 rows
    d = O.random_packed(K, N, g, seed=29)
    y, x = _run(d, rand_x(M, K, seed=7), kernel=1)
    assert_parity(y, oracle_exact(d, x), atol_rms=6e-4, what="gemv multi-pass")


def test_gemv_bf16():
    K, N, g, M = 1024, 512, 128, 2
    d = O.random_packed(K, N, g, seed=31, scale_dtype=np.float32)
    # bf16 scales: round the synthetic scales to bf16 first so oracle and kernel see the same numbers
    sc = torch.from_numpy(d["scales"]).to(torch.bfloat16)
    d["scales"] = sc.float().numpy()
    y, x = _run(d, rand_x(M, K, seed=3, dtype=np.float32), dtype=torch.bfloat16)
    # bf16 output rounding is 2^-8 relative
    assert_parity(y, oracle_exact(d, x), rtol=8e-3, atol_rms=4e-3, what="gemv bf16")


def test_gemv_large_activations_and_zero_input():
    K, N, g = 1024, 256, 128
    d = O.random_packed(K, N, g, seed=37)
    x = rand_x(1, K, seed=9).astype(np.float32) * 100.0          # outlier-scale activations
    y, xr = _run(d, x.astype(np.float16))
    assert_parity(y, oracle_exact(d, xr), atol_rms=6e-4, what="large activations")
    y0, _ = _run(d, np.zeros((1, K), np.float16))
    assert (y0 == 0).all()
    xs = (rand_x(1, K, seed=10).astype(np.float32) * 1e-4).astype(np.float16)   # fp16-subnormal activations
    y2, xr2 = _run(d, xs)
    assert_parity(y2, oracle_exact(d, xr2), atol_rms=2e-3, what="tiny activations")


def test_cuda_graph_capture_of_decode_chain():
    """PDL launches are capturable; a captured chain replays to the same result."""
    K = N = 1024
    d = O.random_packed(K, N, 128, seed=41)
    lin = make_layer(d)
    x = torch.from_numpy(rand_x(1, K)).cuda()
    y_eager = lin(lin(x) * 0.01)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        lin(x)
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            y_g = lin(lin(x) * 0.01)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y_g, y_eager)


@pytest.mark.parametrize("M", [1, 3, 4, 6])
@pytest.mark.parametrize("act", [False, True])
def test_forward_group_matches_individual_layers(M, act):
    """q|k|v-style siblings in one grouped launch == the three single-layer calls."""
    from autogptq_b200 import forward_group

    K, g = 1024, 128
    ds = [O.random_packed(K, N, g, seed=50 + i, desc_act=act, bias=(i == 1)) for i, N in enumerate((1024, 264, 512))]
    lins = [make_layer(d) for d in ds]
    x = torch.from_numpy(rand_x(M, K, seed=M)).cuda()
    ys = forward_group(lins, x)
    torch.cuda.synchronize()
    for d, lin, y in zip(ds, lins, ys):
        assert y.shape == (M, d["N"])
        assert_parity(y.float().cpu().numpy(), oracle_exact(d, x.float().cpu().numpy()), atol_rms=6e-4, what="group")
        # same arithmetic, possibly a different K split than the single-layer heuristics pick
        assert_parity(y.float().cpu().numpy(), lin(x).float().cpu().numpy(), rtol=1e-3, atol_rms=6e-4, what="group vs single")
