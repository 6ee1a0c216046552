"""GPU: BASELINE.json's full layer sizes, through size-independent properties (the NumPy oracle would take
minutes here): (1) kernel output vs an independent dense matmul of the bit-exactly-verified dequantised
weights, (2) GEMV vs GEMM, (3) linearity, (4) column-slice consistency (what TP sharding relies on)."""
import numpy as np
import pytest
import torch

from oracle import w4a16_oracle as O
from tests._util import assert_parity, make_layer

pytestmark = pytest.mark.gpu

SHAPES = [(4096, 4096, 128), (4096, 11008, 128), (11008, 4096, 128), (4096, 4096, 32), (8192, 1024, -1)]


def _dense_ref(lin, x):
    from autogptq_b200 import _lib
    lib = _lib.load()
    K, N = lin.infeatures, lin.outfeatures
    W = torch.empty((K, N), dtype=torch.float16, device="cuda")
    lin.post_init()
    _lib.check(lib.agb200_w4_dequantize(lin.qweight.data_ptr(), lin.qzeros.data_ptr(), lin.scales.data_ptr(),
                                        lin.g_idx.data_ptr(), W.data_ptr(), K, N, lin.group_size, _lib.F16, None))
    y = x.float() @ W.float()
    if lin.bias is not None:
        y = y + lin.bias.float()
    return y


@pytest.mark.parametrize("K,N,g", SHAPES)
@pytest.mark.parametrize("M", [1, 2, 4, 8, 64, 512])
def test_full_size_vs_dense(K, N, g, M):
    d = O.random_packed(K, N, g, seed=K % 97 + M, bias=True)
    lin = make_layer(d)
    torch.manual_seed(M)
    x = torch.randn(M, K, dtype=torch.float16, device="cuda")
    y = lin(x)
    ref = _dense_ref(lin, x)
    torch.cuda.synchronize()
    assert_parity(y.float().cpu().numpy(), ref.cpu().numpy(), rtol=1e-3, atol_rms=1.6e-3, what=f"{K}x{N} g={g} M={M}")


@pytest.mark.parametrize("K,N", [(8192, 28672), (28672, 8192)])
@pytest.mark.parametrize("M", [1, 3, 5, 16])
def test_llama70b_layer_sizes_vs_dense(K, N, M):
    """BASELINE config 4 shapes: GEMV (M=1), persistent integer kernel incl. its K-chunked form (M=3, 5), wgmma tile (M=16)."""
    d = O.random_packed(K, N, 128, seed=K % 89 + M)
    lin = make_layer(d)
    torch.manual_seed(M)
    x = torch.randn(M, K, dtype=torch.float16, device="cuda")
    y = lin(x)
    ref = _dense_ref(lin, x)
    torch.cuda.synchronize()
    assert_parity(y.float().cpu().numpy(), ref.cpu().numpy(), rtol=1e-3, atol_rms=1.6e-3, what=f"{K}x{N} M={M}")


def test_gemv_equals_gemm_full_size():
    K, N, g = 4096, 11008, 128
    d = O.random_packed(K, N, g, seed=5, desc_act=True)
    lin = make_layer(d)
    x = torch.randn(4, K, dtype=torch.float16, device="cuda")
    lin.kernel = 1
    y1 = lin(x).float()
    lin.kernel = 2
    y2 = lin(x).float()
    torch.cuda.synchronize()
    assert_parity(y2.cpu().numpy(), y1.cpu().numpy(), rtol=1e-3, atol_rms=2e-3, what="gemm vs gemv act-order")


def test_linearity_and_column_slices():
    K, N, g = 4096, 4096, 128
    d = O.random_packed(K, N, g, seed=6)
    lin = make_layer(d)
    torch.manual_seed(1234)
    a = torch.randn(1, K, dtype=torch.float16, device="cuda")
    b = torch.randn(1, K, dtype=torch.float16, device="cuda")
    ya, yb, yab = lin(a).float(), lin(b).float(), lin((a.float() + b.float()).half()).float()
    rms = yab.pow(2).mean().sqrt()
    assert ((ya + yb - yab).abs().max() <= 4e-3 * rms + 2e-3 * yab.abs().max())
    # a column slice of the packed layer gives the same columns (up to the fp32 summation order: a narrower layer is
    # tiled differently, so an fp16 rounding boundary may flip by one ulp)
    n0, n1 = 1024, 1536
    ds = dict(d, qweight=d["qweight"][:, n0:n1], qzeros=d["qzeros"][:, n0 // 8:n1 // 8], scales=d["scales"][:, n0:n1],
              N=n1 - n0)
    ls = make_layer(ds)
    ya_full = lin(a)[:, n0:n1].float().cpu().numpy()
    assert_parity(ls(a).float().cpu().numpy(), ya_full, rtol=1e-3, atol_rms=1e-3, what="column slice")
