"""CPU tests of the GPTQ quantiser: the NumPy oracle against the reference's own results (tests/golden/gptq_*.npz,
written by make_golden_gptq.py), the running-mean bookkeeping of add_batch, argument errors, and the auto_gptq patch."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import gptq_oracle as GO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# settings files (each names its layer file: W, calibration batches, H, dead columns)
FILES = ("gptq_k128_seq", "gptq_k128_act", "gptq_k264_seq", "gptq_k264_act", "gptq_dead_seq")


def golden_cases():
    """(file, config index) of every stored quantisation setting."""
    out = []
    for f in FILES:
        n = int(np.load(os.path.join(GOLDEN, f + ".npz"))["n_configs"])
        out += [(f, i) for i in range(n)]
    return out


def load_case(f, i):
    z = np.load(os.path.join(GOLDEN, f + ".npz"))
    lay = np.load(os.path.join(GOLDEN, str(z["layer"]) + ".npz"))
    g, act, static, sym = (int(v) for v in z[f"c{i}_config"])
    K = lay["W"].shape[1]
    dead = np.zeros(K, dtype=bool)
    dead[lay["dead"]] = True
    H = lay["H"].copy()
    H[dead, dead] = 1
    perm = np.argsort(-np.diag(H), kind="stable") if act else None
    case = dict(W=lay["W"].astype(np.float32), H=lay["H"], Hinv=z["Hinv"], perm=perm,
                dead=dead if dead.any() else None, g=g, act=bool(act), static=bool(static), sym=bool(sym), K=K,
                x2d=lay["x2d"], x3d=lay["x3d"], nsamples=int(lay["nsamples"]))
    for k in ("scale", "zero", "g_idx", "Q", "loss_sum", "qweight", "qzeros", "scales"):
        case[k] = z[f"c{i}_{k}"]
    return case


def agreeing_elements(codes, codes_ref, scale, zero, c):
    """Elements whose code and group parameters both equal the reference's: there Q must be identical too.  (Across
    blocks a group's parameters can differ in the last bit, because they see W after trailing updates.)"""
    gi = c["g_idx"].astype(np.int64)
    same_params = (scale == c["scale"]) & (zero == c["zero"])            # [N, G]
    return (codes == codes_ref) & same_params[:, gi]


@pytest.mark.parametrize("f,i", golden_cases())
def test_oracle_matches_reference_goldens(f, i):
    c = load_case(f, i)
    r = GO.fasterquant(c["W"], c["Hinv"], perm=c["perm"], dead=c["dead"], group_size=c["g"], sym=c["sym"],
                       static_groups=c["static"])
    codes_ref = GO.unpack_codes(c["qweight"])
    agree = float((r["codes"] == codes_ref).mean())
    np.testing.assert_array_equal(r["g_idx"], c["g_idx"])
    if c["K"] <= 128:     # one block: the same float32 operations in the same order
        assert agree == 1.0
        np.testing.assert_array_equal(r["scale"], c["scale"])
        np.testing.assert_array_equal(r["zero"], c["zero"])
        np.testing.assert_array_equal(r["Q"].astype(np.float16), c["Q"])
    else:                 # the trailing update is a matmul whose summation order is the BLAS's
        assert agree >= 0.999, agree
        np.testing.assert_allclose(r["scale"], c["scale"], rtol=1e-5)
    assert abs(r["losses"].sum(dtype=np.float64) / c["loss_sum"] - 1) < 1e-3
    same = agreeing_elements(r["codes"], codes_ref, r["scale"], r["zero"], c)
    assert np.array_equal(r["Q"].astype(np.float16)[same], c["Q"][same])
    # codes straight from the loop pack to what QuantLinear.pack derives from (Q, scale, zero)
    if same.all():
        qw, qz, sc = GO.pack_codes(r["codes"], r["zero"], r["scale"])
        np.testing.assert_array_equal(qw, c["qweight"])
        np.testing.assert_array_equal(qz, c["qzeros"])
        np.testing.assert_array_equal(sc, c["scales"])


def test_oracle_hessian_matches_reference():
    c = load_case("gptq_k128_seq", 0)
    H, n = np.zeros((c["K"], c["K"]), np.float32), 0
    for x in (c["x2d"], c["x3d"]):
        H, n = GO.add_batch(H, n, x)
    assert n == c["nsamples"] == 4
    assert np.linalg.norm(H - c["H"]) / np.linalg.norm(c["H"]) < 1e-6


def test_running_mean_bookkeeping():
    from autogptq_b200.gptq import running_mean_factors

    # the leading dimension counts, not tokens: [4, 128, K] adds 4, a 2-D input adds 1
    a, b, n = running_mean_factors(0, (4, 128, 64))
    assert (a, b, n) == (0.0, 0.5, 4)
    a, b, n = running_mean_factors(n, (300, 64))
    assert n == 5 and a == 4 / 5 and b == 2 / 5
    # chaining the factors reproduces 2/n * sum of x^T x over all batches
    rng = np.random.default_rng(0)
    xs = [rng.standard_normal((2, 7, 8)), rng.standard_normal((5, 8)), rng.standard_normal((3, 4, 8))]
    H, n = np.zeros((8, 8)), 0
    for x in xs:
        a, b, n = running_mean_factors(n, x.shape)
        x2 = x.reshape(-1, 8)
        H = a * H + b * x2.T @ x2
    full = np.concatenate([x.reshape(-1, 8) for x in xs])
    assert n == 6
    np.testing.assert_allclose(H, 2 / 6 * full.T @ full, rtol=1e-12)


def test_quantizer_and_fasterquant_argument_errors():
    from autogptq_b200.gptq import GPTQ

    g = GPTQ(nn.Linear(64, 32, bias=False).half())
    assert (g.rows, g.columns, g.nsamples) == (32, 64, 0) and g.H.shape == (64, 64)
    for kw in (dict(bits=8, perchannel=True), dict(bits=4, perchannel=True, mse=True), dict(bits=4, perchannel=False),
               dict(bits=4, perchannel=True, trits=True)):
        with pytest.raises(NotImplementedError):
            g.quantizer.configure(**kw)
    with pytest.raises(NotImplementedError, match="configure"):
        g.fasterquant()
    g.quantizer.configure(4, perchannel=True, sym=False, mse=False)
    with pytest.raises(NotImplementedError, match="blocksize"):
        g.fasterquant(blocksize=64)
    with pytest.raises(NotImplementedError, match="group_size"):
        g.fasterquant(group_size=12)
    with pytest.raises(NotImplementedError):
        GPTQ(nn.Conv2d(4, 8, 3))
    with pytest.raises(RuntimeError, match="CUDA"):          # no CPU fallback
        g.add_batch(torch.zeros(3, 64, dtype=torch.float16), None)
    g32 = GPTQ(nn.Linear(64, 32))
    g32.quantizer.configure(4, perchannel=True)
    with pytest.raises(NotImplementedError, match="float16 or bfloat16"):
        g32.fasterquant()


def test_conv1d_shapes():
    from transformers.pytorch_utils import Conv1D

    from autogptq_b200.gptq import GPTQ

    layer = Conv1D(48, 64)            # nf=48 outputs, nx=64 inputs; weight [64, 48]
    g = GPTQ(layer)
    assert (g.rows, g.columns) == (48, 64)


def test_patch_auto_gptq_quantizer_rebinds_gptq(monkeypatch):
    from autogptq_b200.gptq import GPTQ, patch_auto_gptq_quantizer

    sentinel = object()
    base = types.ModuleType("auto_gptq.modeling._base")
    base.GPTQ = sentinel
    quant = types.ModuleType("auto_gptq.quantization")
    quant.GPTQ = sentinel
    for name, mod in (("auto_gptq", types.ModuleType("auto_gptq")), ("auto_gptq.modeling", types.ModuleType("auto_gptq.modeling")),
                      ("auto_gptq.modeling._base", base), ("auto_gptq.quantization", quant)):
        monkeypatch.setitem(sys.modules, name, mod)
    monkeypatch.setitem(sys.modules, "auto_gptq.quantization.gptq", None)   # not importable
    patched = patch_auto_gptq_quantizer()
    assert patched == ["auto_gptq.modeling._base", "auto_gptq.quantization"]
    assert base.GPTQ is GPTQ and quant.GPTQ is GPTQ
