"""GPU parity: the wgmma tensor-core GEMM through the QuantLinear module / C ABI vs the oracle."""
import numpy as np
import pytest
import torch

from oracle import w4a16_oracle as O
from tests._util import assert_parity, make_layer, oracle_exact, oracle_fp16w, rand_x

pytestmark = pytest.mark.gpu


def _run(d, x, tune=(0, 0), dtype=torch.float16, kernel=2):
    lin = make_layer(d, dtype=dtype)
    lin.kernel = kernel
    lin.tune = tune
    xt = torch.from_numpy(np.asarray(x, dtype=np.float32)).to(dtype).cuda()
    y = lin(xt)
    torch.cuda.synchronize()
    return y.float().cpu().numpy(), xt.float().cpu().numpy()


def _check(d, y, x, what):
    # (a) the reference's own fp16 arithmetic: W rounded once to fp16, fp32 accumulate -> only output rounding left
    assert_parity(y, oracle_fp16w(d, x), rtol=1e-3, atol_rms=6e-4, what=what + " [fp16-W oracle]")
    # (b) exact oracle: adds the fp16 rounding of W the reference itself performs (2^-12 rms per weight)
    assert_parity(y, oracle_exact(d, x), rtol=1e-3, atol_rms=1.6e-3, what=what + " [exact oracle]")


@pytest.mark.parametrize("M", [1, 5, 16, 33, 64, 100, 128, 257, 512])
def test_gemm_m_sweep(M):
    K, N, g = 512, 256, 128
    d = O.random_packed(K, N, g, seed=100 + M, bias=(M % 2 == 1))
    y, x = _run(d, rand_x(M, K, seed=M))
    _check(d, y, x, f"gemm M={M}")


@pytest.mark.parametrize("K,N,g", [(64, 128, 32), (192, 160, 64), (1024, 1024, -1), (4096, 384, 128), (2048, 2048, 32), (320, 96, 64)])
def test_gemm_shapes(K, N, g):
    M = 48
    d = O.random_packed(K, N, g, seed=K + N, bias=True)
    y, x = _run(d, rand_x(M, K, seed=3))
    _check(d, y, x, f"gemm K={K} N={N} g={g}")


@pytest.mark.parametrize("mt", [32, 64, 128])
@pytest.mark.parametrize("split", [1, 2, 4, 8])
def test_gemm_tiles_and_splitk(mt, split):
    K, N, g, M = 1024, 256, 128, 70
    d = O.random_packed(K, N, g, seed=7, bias=True)
    y, x = _run(d, rand_x(M, K, seed=4), tune=(mt, split))
    _check(d, y, x, f"gemm mt={mt} split={split}")


def test_gemm_act_order_and_wrap():
    K, N, g, M = 1024, 256, 128, 40
    d = O.random_packed(K, N, g, seed=9, desc_act=True, zero_max=15, bias=True)
    y, x = _run(d, rand_x(M, K, seed=5))
    _check(d, y, x, "gemm act-order + wrap")


def test_gemm_bf16():
    K, N, g, M = 1024, 256, 128, 96
    d = O.random_packed(K, N, g, seed=13, scale_dtype=np.float32)
    d["scales"] = torch.from_numpy(d["scales"]).to(torch.bfloat16).float().numpy()
    y, x = _run(d, rand_x(M, K, seed=6, dtype=np.float32), dtype=torch.bfloat16)
    assert_parity(y, oracle_exact(d, x), rtol=8e-3, atol_rms=8e-3, what="gemm bf16")


def test_gemm_matches_gemv():
    """Two independent kernels (CUDA-core exact-W GEMV vs tensor-core fp16-W GEMM) agree within the band."""
    K, N, g, M = 2048, 512, 128, 4
    d = O.random_packed(K, N, g, seed=21)
    x = rand_x(M, K, seed=8)
    y_gemm, _ = _run(d, x, kernel=2)
    y_gemv, _ = _run(d, x, kernel=1)
    assert_parity(y_gemm, y_gemv, rtol=1e-3, atol_rms=2e-3, what="gemm vs gemv")


def test_gemm_tile128_ragged_m():
    """AUTO's 128-row tile without split-K at an M that leaves the last tile partly filled."""
    K, N, g, M = 1024, 512, 128, 300
    d = O.random_packed(K, N, g, seed=17, bias=True)
    y, x = _run(d, rand_x(M, K, seed=9), tune=(128, 1))
    _check(d, y, x, "gemm mt=128 split=1")


def test_gemm_rejects_unknown_tiles_and_tune1_bits():
    """Only the 32/64/128-row tiles exist; tune1 carries split-K and the debug bits, nothing else."""
    from autogptq_b200 import _lib

    d = O.random_packed(1024, 512, 128, seed=17)
    x = rand_x(300, 1024, seed=9)
    with pytest.raises(_lib.B200KernelError, match=r"code -1\): gemm: x-row tile must be 32/64/128 \(got 256\)"):
        _run(d, x, tune=(256, 1))
    with pytest.raises(_lib.B200KernelError,
                       match=r"code -1\): gemm: tune1 holds split-K in bits 0-7 and the debug bits 12-13 \(got 0x201\)"):
        _run(d, x, tune=(128, 1 | (2 << 8)))


def test_auto_handles_shapes_the_tensor_core_path_cannot():
    """outfeatures % 32 != 0 (TMA row pitch of qzeros) or group_size 16: AUTO falls back to the small-M kernels."""
    for (K, N, g) in ((512, 136, 64), (256, 264, 16)):
        d = O.random_packed(K, N, g, seed=3, bias=True)
        y, x = _run(d, rand_x(40, K, seed=2), kernel=0)
        assert_parity(y, oracle_exact(d, x), atol_rms=1.6e-3, what=f"auto K={K} N={N} g={g}")
    from autogptq_b200 import _lib
    d = O.random_packed(512, 136, 64, seed=3)
    with pytest.raises(_lib.B200KernelError):
        _run(d, rand_x(40, 512), kernel=2)
