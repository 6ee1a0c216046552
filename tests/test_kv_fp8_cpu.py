"""CPU checks of the FP8 KV cache: ``quantize_kv`` bit-equal to the NumPy restatement of ``tests/_kv_fp8.py`` on the
format's edge cases, the exactness of the dequantised values, the two C ABI additions (declared, bound, argument errors
with their exact text, called without a device) and the decoders' refusals."""
import os
import re

import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from tests import _kv_fp8 as Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16, BF16 = torch.float16, torch.bfloat16
EINVAL, ENOSUP, EWORKSPACE = -1, -3, -4
A = 0x100000            # a 256-byte aligned fake device address (never dereferenced)


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def call(lib, name, *args):
    rc = getattr(lib, name)(*args)
    return rc, lib.agb200_last_error().decode()


def _check_bits(x):
    """quantize_kv(x) bit-equal to the restatement."""
    from autogptq_b200.attention import dequantize_kv, quantize_kv

    codes, scale = quantize_kv(x)
    assert codes.dtype == torch.float8_e4m3fn and scale.dtype == torch.float32
    assert codes.shape == x.shape and scale.shape == x.shape[:-1]
    rc, rs = Q.quantize(x.double().numpy())
    got = codes.view(torch.uint8).numpy()
    bad = np.argwhere(got != rc)
    assert bad.size == 0, f"code differs at {bad[0]}: {got[tuple(bad[0])]:#x} vs {rc[tuple(bad[0])]:#x}"
    assert np.array_equal(scale.double().numpy(), rs)
    assert np.array_equal(dequantize_kv(codes, scale).double().numpy(), Q.dequantize(rc, rs))
    return codes, scale


def _rows(dtype, hd, values):
    """Rows of hd values of dtype: each given value list padded with zeros."""
    x = torch.zeros(len(values), hd, dtype=dtype)
    for r, v in enumerate(values):
        x[r, :len(v)] = torch.tensor(v, dtype=torch.float64).to(dtype)
    return x


def test_table():
    v = Q.VALUES
    assert v[0x7E] == 448 and v[0x08] == 2.0 ** -6 and v[0x01] == 2.0 ** -9 and v[0x38] == 1.0
    assert np.isnan(v[0x7F]) and np.isnan(v[0xFF]) and v[0x80] == 0 and v[0xFE] == -448
    assert (np.diff(v[:0x7F]) > 0).all()
    t = torch.tensor(v[np.isfinite(v)], dtype=torch.float32).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    assert np.array_equal(Q.VALUES[t], v[np.isfinite(v)]), "table differs from torch's float8_e4m3fn"


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["f16", "bf16"])
def test_scale_boundaries(dtype, hd):
    # a exactly 448·2^e, and the next float of the dtype above it (which moves to e + 1)
    rows = []
    for e in (-20, -9, -3, 0, 1, 4, 7):
        if dtype == F16 and not -14 - 9 <= e <= 7:
            continue
        top = 448.0 * 2.0 ** e
        above = (torch.tensor([top], dtype=torch.float64).to(dtype).view(torch.int16) + 1).view(dtype)
        rows.append([top, -top / 3, top / 1000, 1.0 * 2.0 ** e])
        rows.append([above.item(), -top / 3, top / 1000, 1.0 * 2.0 ** e])
        rows.append([-top, top / 7])
    x = _rows(dtype, hd, rows)
    _, scale = _check_bits(x)
    for r in range(0, len(rows), 3):
        e_top = int(np.log2(scale[r].item()))
        assert scale[r + 1].item() == 2.0 ** (e_top + 1), "the next float above 448·2^e takes e + 1"
        assert scale[r + 2].item() == scale[r].item()


@pytest.mark.parametrize("dtype", [F16, BF16], ids=["f16", "bf16"])
def test_zero_rows_ties_and_subnormals(dtype):
    from autogptq_b200.attention import quantize_kv

    hd = 64
    ties = [448.0, 1.0625, 1.1875, -17.0, 19.0, 0.5 * 2.0 ** -9, 1.5 * 2.0 ** -9, -2.5 * 2.0 ** -9, 7.5 * 2.0 ** -9,
            240.0 + 8.0, 416.0 + 16.0]                      # midpoints between neighbouring E4M3 values
    sub = [448.0, 3 * 2.0 ** -9, 2.0 ** -9, -2.0 ** -10, 2.0 ** -11, -2.0 ** -12, 2.0 ** -7 + 2.0 ** -12, 1e-3, -1e-4]
    x = _rows(dtype, hd, [[], ties, sub, [0.0, -0.0]])
    x[3, 1] = -0.0
    codes, scale = _check_bits(x)
    c = codes.view(torch.uint8)
    assert scale[0].item() == 1.0 and (c[0] == 0).all() and scale[3].item() == 1.0 and (c[3] == 0).all()
    assert c[1, 1].item() == 0x38 and c[1, 2].item() == 0x3A       # 1.0625 -> 1 (even), 1.1875 -> 1.25 (even)
    assert c[1, 5].item() == 0x00 and c[1, 6].item() == 0x02       # half the smallest subnormal -> 0; 1.5 -> 2
    assert c[2, 5].item() == 0x80 and c[2, 4].item() == 0x00       # below half the smallest subnormal: ±0
    # bf16 reaches fp32 subnormals: the scale clamps at 2^-126
    if dtype == BF16:
        tiny = torch.tensor([[2.0 ** -130, -2.0 ** -133] + [0.0] * 62]).to(BF16)
        cc, s = _check_bits(tiny)
        assert s.item() == 2.0 ** -126
        assert quantize_kv(tiny)[1].item() == 2.0 ** -126


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["f16", "bf16"])
def test_random_rows_bit_equal(dtype, hd):
    g = torch.Generator().manual_seed(hd)
    mags = [2.0 ** k for k in range(-12, 14, 3)] if dtype == F16 else [2.0 ** k for k in range(-60, 60, 11)]
    x = torch.cat([(torch.randn(8, hd, generator=g, dtype=torch.float64) * m).to(dtype) for m in mags])
    x[::5, ::7] = 0
    _check_bits(x)
    _check_bits(x.view(4, -1, hd))                                 # leading dimensions are rows


@pytest.mark.parametrize("dtype", [F16, BF16], ids=["f16", "bf16"])
def test_dequantised_values_exact_in_dtype(dtype):
    from autogptq_b200.attention import dequantize_kv, quantize_kv

    g = torch.Generator().manual_seed(1)
    # bf16: any scale; fp16: a in (448·2^-16, 448·2^7]
    lo, hi = (-16, 7) if dtype == F16 else (-100, 100)
    for e in range(lo, hi + 1, 1 if dtype == F16 else 7):
        x = (torch.rand(16, 128, generator=g, dtype=torch.float64) * 2 - 1) * 448.0 * 2.0 ** e
        x[:, 0] = 448.0 * 2.0 ** e * 0.99
        x = x.to(dtype)
        a = x.abs().amax(-1).double()
        keep = (a > 448.0 * 2.0 ** -16) if dtype == F16 else torch.ones_like(a, dtype=torch.bool)
        d = dequantize_kv(*quantize_kv(x))[keep]
        assert torch.equal(d.to(dtype).float(), d), f"2^{e}: a dequantised value is not exact in {dtype}"


# --------------------------------------------------------------------------- the C ABI
def test_exports_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "autogptq_b200.h")).read()
    for name in ("agb200_decode_attention_fp8", "agb200_decode_attention_rows_fp8"):
        assert re.search(rf"\b{name}\s*\(", hdr), f"{name} is not declared"
        assert name in _lib.declared_symbols(), f"{name} is not bound"
        assert hasattr(_lib.load(), name)
    assert re.search(r"#define AGB200_ABI_VERSION 11\b", hdr)
    assert _lib.ABI_VERSION == 11 == _lib.load().agb200_abi_version()


@pytest.mark.parametrize("entry,max_b", [("decode_attention_fp8", 2), ("decode_attention_rows_fp8", 8)])
def test_fp8_entry_errors(lib, entry, max_b):
    name = "agb200_" + entry
    need = lib.agb200_decode_attention_workspace_bytes(1, 32, 8, 128, 4096)

    def attn(ks=A, vs=A, B=1, head_dim=128, ws_bytes=need, q=A):
        return call(lib, name, q, A, A, A, A, ks, vs, A, A, 1.0, 1.0, A, B, 32, 8, head_dim, 4096, _lib.F16, A,
                    ws_bytes, None)

    assert attn(ks=None) == (EINVAL, f"{entry}: null pointer argument")
    assert attn(vs=None) == (EINVAL, f"{entry}: null pointer argument")
    assert attn(q=None) == (EINVAL, f"{entry}: null pointer argument")
    assert attn(ks=A + 2) == (EINVAL, f"{entry}: k_scale and v_scale must be 4-byte aligned")
    assert attn(vs=A + 1) == (EINVAL, f"{entry}: k_scale and v_scale must be 4-byte aligned")
    assert attn(head_dim=96) == (ENOSUP, f"{entry}: head_dim 96; supported: 64, 128")
    assert attn(B=max_b + 1) == (ENOSUP, f"{entry}: batch {max_b + 1}; at most {max_b}")
    assert attn(ws_bytes=256) == (EWORKSPACE, f"{entry}: workspace needs {need} bytes (got 256)")


def test_wrapper_needs_cuda_and_scales():
    from autogptq_b200.attention import decode_attention_rows

    z = torch.zeros
    fp8 = lambda *s: z(*s, dtype=torch.float8_e4m3fn)
    args = (z(3, 256, dtype=F16), z(3, 128, dtype=F16), z(3, 128, dtype=F16), fp8(3, 1, 16, 128), fp8(3, 1, 16, 128),
            z(3, dtype=torch.int64), z(64), 1.0, 0.1, z(3, 256, dtype=F16))
    with pytest.raises(RuntimeError, match="CUDA"):
        decode_attention_rows(*args, k_scale=z(3, 1, 16), v_scale=z(3, 1, 16))


# --------------------------------------------------------------------------- decoder refusals
def _model():
    from tests.test_batch_decoder_cpu import _llama, _quantized

    return _quantized(_llama())


@pytest.mark.parametrize("bad", [torch.float8_e5m2, torch.int8, torch.float16, "fp8"])
def test_decoders_refuse_other_cache_dtypes(bad):
    from autogptq_b200 import BatchDecoder
    from autogptq_b200.decoder import ChainDecoder

    m = _model()
    with pytest.raises(NotImplementedError, match=r"^BatchDecoder: kv_cache_dtype .*; supported: None"):
        BatchDecoder(m, max_batch=2, max_length=128, kv_cache_dtype=bad)
    with pytest.raises(NotImplementedError, match=r"^ChainDecoder: kv_cache_dtype .*; supported: None"):
        ChainDecoder(m, batch=1, max_length=128, fused_attention=True, kv_cache_dtype=bad)


def test_chain_decoder_fp8_needs_fused_attention():
    from autogptq_b200.decoder import ChainDecoder

    with pytest.raises(NotImplementedError, match="needs fused_attention=True; the torch attention reads a 16-bit"):
        ChainDecoder(_model(), batch=1, max_length=128, kv_cache_dtype=torch.float8_e4m3fn)


def test_fp8_decoders_get_to_the_device_check():
    from autogptq_b200 import BatchDecoder
    from autogptq_b200.decoder import ChainDecoder

    fp8 = torch.float8_e4m3fn
    with pytest.raises(RuntimeError, match="CUDA device"):
        BatchDecoder(_model(), max_batch=8, max_length=128, kv_cache_dtype=fp8)
    with pytest.raises(RuntimeError, match="CUDA device"):
        ChainDecoder(_model(), batch=2, max_length=128, fused_attention=True, kv_cache_dtype=fp8)
