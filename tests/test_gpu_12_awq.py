"""GPU tests of AWQ GEMM checkpoints: layers loaded through autogptq_b200.checkpoint (converted to the GPTQ layout while
loading) run every kernel family, the decode chain and the grouped experts, against the AWQ oracle
(oracle/awq_oracle.py: W = s·(q − z) straight from the AWQ tensors) with the tolerances of the GPTQ tests."""
import json
import os

import numpy as np
import pytest
import torch
from safetensors.torch import save_file

from autogptq_b200 import _lib, group_experts
from autogptq_b200 import checkpoint as C
from autogptq_b200.awq import awq_to_gptq
from autogptq_b200.chain import DecodeChain
from oracle import awq_oracle as A
from oracle import moe_oracle as MO
from tests._awq_util import gptq_view, write_awq_checkpoint
from tests._util import assert_parity

pytestmark = pytest.mark.gpu

DT = {torch.float16: "float16", torch.bfloat16: "bfloat16"}
# decode kernels (exact weights, fp32 accumulate) and the wgmma GEMM (weights rounded to the dtype), as in the GPTQ tests
DECODE_TOL = {torch.float16: dict(rtol=1e-3, atol_rms=6e-4), torch.bfloat16: dict(rtol=8e-3, atol_rms=4e-3)}
GEMM_TOL = {torch.float16: dict(rtol=1e-3, atol_rms=6e-4), torch.bfloat16: dict(rtol=8e-3, atol_rms=8e-3)}


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _oracle(d, x, dtype, round_w, cols=None):
    """x @ W (+ bias) in fp32 with the scales / bias the device computes with (rounded to ``dtype``); ``round_w`` rounds
    every weight to ``dtype`` (the wgmma path).  ``cols`` = (n0, n1), multiples of 8: those output columns only."""
    n0, n1 = cols or (0, d["N"])
    qw, qz = d["qweight"][:, n0 // 8:n1 // 8], d["qzeros"][:, n0 // 8:n1 // 8]
    s = MO.round_to(d["scales"][:, n0:n1].astype(np.float32), DT[dtype])
    W = A.dequantize_awq(qw, qz, s, d["group_size"])
    if round_w:
        W = MO.round_to(W, DT[dtype])
    y = np.asarray(x, dtype=np.float32) @ W
    if d.get("bias") is not None:
        y = y + MO.round_to(d["bias"][n0:n1].astype(np.float32), DT[dtype])
    return y


def _x(M, K, dtype, seed):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((M, K)).astype(np.float32)).to(dtype).cuda()


K_, N_, G_ = 2048, 1024, 128
PREFIX = "model.layers.0.mlp.up_proj"


@pytest.fixture(scope="module")
def awq_layer(tmp_path_factory):
    _need_gpu()
    path = tmp_path_factory.mktemp("awq_layer")
    d = A.random_awq(K_, N_, G_, seed=1, bias=True)
    write_awq_checkpoint(str(path), {PREFIX: d}, G_)
    return str(path), d


AUTO, GEMV, GEMM, SKINNY, IMMA = _lib.KERNEL_AUTO, _lib.KERNEL_GEMV, _lib.KERNEL_GEMM, _lib.KERNEL_SKINNY, _lib.KERNEL_IMMA
CASES = [(AUTO, 1), (AUTO, 3), (AUTO, 6), (AUTO, 64), (GEMV, 1), (IMMA, 2), (IMMA, 3), (IMMA, 4), (SKINNY, 5),
         (SKINNY, 8), (GEMM, 64), (GEMM, 512)]


@pytest.mark.parametrize("kernel,M", CASES)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_every_kernel_on_an_awq_layer(awq_layer, kernel, M, dtype):
    path, d = awq_layer
    lin = C.load_quant_linears(path, device="cuda")[PREFIX]
    lin.kernel = kernel
    x = _x(M, K_, dtype, seed=M)
    y = lin(x)
    torch.cuda.synchronize()
    assert y.dtype == dtype
    tensor_core = kernel == GEMM or (kernel == AUTO and M > 8)
    ref = _oracle(d, x.float().cpu().numpy(), dtype, round_w=tensor_core and dtype == torch.float16)
    tol = GEMM_TOL[dtype] if tensor_core else DECODE_TOL[dtype]
    assert_parity(y.float().cpu().numpy(), ref, what=f"awq kernel={kernel} M={M} {dtype}", **tol)


@pytest.fixture(scope="module")
def llama_layer(tmp_path_factory):
    _need_gpu()
    path = tmp_path_factory.mktemp("awq_llama")
    d = A.random_awq(4096, 11008, 128, seed=7)
    write_awq_checkpoint(str(path), {"model.layers.0.mlp.gate_proj": d}, 128, config="hf")
    return str(path), d


@pytest.mark.parametrize("M", [1, 4, 8, 64])
def test_llama_7b_shaped_layer(llama_layer, M):
    path, d = llama_layer
    lin = C.load_quant_linears(path, device="cuda:0")["model.layers.0.mlp.gate_proj"]
    x = _x(M, 4096, torch.float16, seed=M)
    y = lin(x)
    torch.cuda.synchronize()
    xs = x.float().cpu().numpy()
    for n0, n1 in ((0, 256), (5120, 5376), (11008 - 256, 11008)):           # column slices, the grid's edge included
        ref = _oracle(d, xs, torch.float16, round_w=M > 8, cols=(n0, n1))
        assert_parity(y[:, n0:n1].float().cpu().numpy(), ref, rtol=1e-3, atol_rms=1.6e-3, what=f"4096x11008 M={M} [{n0}:{n1}]")


def test_conversion_on_the_gpu_equals_the_cpu(llama_layer):
    _, d = llama_layer
    t = [torch.from_numpy(np.ascontiguousarray(d[k])) for k in ("qweight", "qzeros", "scales")]
    cpu = awq_to_gptq(*t)
    gpu = awq_to_gptq(*(a.cuda() for a in t))
    assert all(g.is_cuda and torch.equal(g.cpu(), c) for g, c in zip(gpu, cpu))


def test_decode_chain_mlp_from_awq(tmp_path):
    _need_gpu()
    H, I, g = 1024, 2816, 128
    names = {"gate_proj": (H, I, False), "up_proj": (H, I, False), "down_proj": (I, H, True)}
    raw = {f"model.layers.0.mlp.{n}": A.random_awq(K, N, g, seed=i, bias=b) for i, (n, (K, N, b)) in enumerate(names.items())}
    write_awq_checkpoint(str(tmp_path), raw, g, shards=2)
    layers = C.load_quant_linears(str(tmp_path), device="cuda")
    gp, up, dn = (layers[f"model.layers.0.mlp.{n}"] for n in names)
    dg, du, dd = (raw[f"model.layers.0.mlp.{n}"] for n in names)
    ch = DecodeChain(M=1)
    x = ch.input(H)
    gate, upo = ch.stage([gp, up], x)
    (y,) = ch.stage([dn], gate, x2=upo, x_mode="silu_mul")
    ch.build()
    x.copy_(_x(1, H, torch.float16, seed=3))
    ch.run()
    torch.cuda.synchronize()
    xs = x.float().cpu().numpy()
    for d, out in ((dg, gate), (du, upo)):
        assert_parity(out.float().cpu().numpy(), _oracle(d, xs, torch.float16, False), rtol=1e-3, atol_rms=6e-4, what="chain gate|up")
    a = gate.float()
    act = ((a / (1 + torch.exp(-a))).half().float() * upo.float()).half()
    # __expf in the kernel vs torch.exp: one ulp of the 16-bit intermediate at most (as in the GPTQ chain test)
    assert_parity(y.float().cpu().numpy(), _oracle(dd, act.float().cpu().numpy(), torch.float16, False), rtol=2e-3,
                  atol_rms=1.8e-3, what="chain down")


@pytest.fixture(scope="module")
def awq_mixtral(tmp_path_factory):
    _need_gpu()
    path = tmp_path_factory.mktemp("awq_mixtral")
    E, H, I, g = 4, 1024, 2816, 128
    pre = "model.layers.0.block_sparse_moe.experts"
    experts = [{n: A.random_awq(K, N, g, seed=10 * e + j) for j, (n, K, N) in enumerate((("w1", H, I), ("w3", H, I), ("w2", I, H)))}
               for e in range(E)]
    raw = {f"{pre}.{e}.{n}": d for e, ex in enumerate(experts) for n, d in ex.items()}
    raw["model.layers.0.self_attn.q_proj"] = A.random_awq(H, H, g, seed=99)
    write_awq_checkpoint(str(path), raw, g)
    grouped = group_experts(C.load_quant_linears(str(path), device="cuda"))
    return grouped[pre], [{n: gptq_view(d) for n, d in ex.items()} for ex in experts]


@pytest.mark.parametrize("T", [3, 64])
def test_mixtral_experts_from_awq(awq_mixtral, T):
    qe, ref = awq_mixtral
    E = len(ref)
    rng = np.random.default_rng(T)
    idx = np.stack([rng.permutation(E)[:2] for _ in range(T)]).astype(np.int64)
    w = rng.random((T, 2)).astype(np.float32)
    w /= w.sum(axis=1, keepdims=True)
    x = _x(T, 1024, torch.float16, seed=T)
    y = qe(x, torch.as_tensor(idx).cuda(), torch.as_tensor(w).cuda())
    torch.cuda.synchronize()
    y_ref, mag = MO.forward(x.float().cpu().numpy(), ref, idx, w, "float16", weight_dtype=None if T <= 8 else "float16",
                            return_magnitude=True)
    # one ulp of every per-pair output is excused, as in the GPTQ MoE tests (rounded before the weighted sum)
    err = y.float().cpu().numpy() - y_ref
    excused = np.sign(err) * np.maximum(np.abs(err) - 2.0 ** -10 * mag, 0)
    assert_parity(y_ref + excused, y_ref, rtol=1e-3, atol_rms=1.6e-3, what=f"awq mixtral T={T}")


def test_round_trip_through_a_gptq_checkpoint(awq_layer, tmp_path):
    path, d = awq_layer
    awq = C.load_quant_linears(path, device="cuda")
    save_file(C.packed_state_dict(awq), os.path.join(tmp_path, "model.safetensors"), metadata={"format": "pt"})
    json.dump({"bits": 4, "group_size": G_, "desc_act": False, "sym": False}, open(tmp_path / C.QUANT_CONFIG_FILENAME, "w"))
    gptq = C.load_quant_linears(str(tmp_path), device="cuda")
    a, b = awq[PREFIX], gptq[PREFIX]
    for leaf in ("qweight", "qzeros", "scales", "g_idx", "bias"):
        assert torch.equal(getattr(a, leaf), getattr(b, leaf)), leaf
    for M in (1, 3, 7, 64):
        x = _x(M, K_, torch.float16, seed=20 + M)
        assert torch.equal(a(x), b(x)), f"M={M}"
