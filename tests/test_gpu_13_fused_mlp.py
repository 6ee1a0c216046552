"""GPU tests of the fused gate/up of a dense MLP (forward_gate_up, FusedQuantMLP, inject_fused_mlp; agb200_w4a16_gate_up):
parity with the oracle on the decode kernel (M <= 8, exact weights) and the split-K wgmma GEMM (weights rounded to the
dtype), every forced kernel / tile / split, a Llama-2-7B-sized pair, determinism, CUDA-graph replay, the module against
the unfused layers, a tiny HF Llama with and without injection, an AWQ-loaded pair and the fallbacks."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import awq_oracle as A
from oracle import w4a16_oracle as O
from tests._awq_util import gptq_view, write_awq_checkpoint
from tests._mlp_util import TOL, assert_gate_up, make_pair, x_rows
from tests._util import assert_parity, make_layer

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _fgu():
    from autogptq_b200 import forward_gate_up

    return forward_gate_up


@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 8, 9, 16, 64, 200, 1024])
@pytest.mark.parametrize("g,desc_act,bias", [(128, False, False), (32, False, True), (64, True, False), (-1, False, True),
                                             (128, True, True)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_parity(M, g, desc_act, bias, dtype):
    _need_gpu()
    gate, up, gr, ur = make_pair(1024, 2816, g, desc_act=desc_act, bias=bias, dtype=dtype, seed=M % 7)
    x = x_rows(M, 1024, dtype, seed=M)
    h = _fgu()(gate, up, x)
    torch.cuda.synchronize()
    assert h.shape == (M, 2816) and h.dtype == dtype
    assert_gate_up(h, x, gr, ur, dtype, exact_w=M <= 8, what=f"M={M} g={g} act={desc_act} bias={bias} {dtype}")


def test_leading_dims_kept():
    _need_gpu()
    gate, up, gr, ur = make_pair(512, 1024, 128, dtype=torch.float16)
    x = x_rows(6, 512, torch.float16).reshape(2, 3, 512)
    h = _fgu()(gate, up, x)
    assert h.shape == (2, 3, 1024)
    assert_gate_up(h.reshape(6, 1024), x.reshape(6, 512), gr, ur, torch.float16, exact_w=True, what="3-d x")


@pytest.mark.parametrize("M", [1, 8])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_forced_decode(M, dtype):
    from autogptq_b200 import _lib

    _need_gpu()
    gate, up, gr, ur = make_pair(1024, 2816, 128, desc_act=True, bias=True, dtype=dtype, seed=3)
    x = x_rows(M, 1024, dtype, seed=M)
    h = _fgu()(gate, up, x, kernel=_lib.GATE_UP_DECODE)
    assert_gate_up(h, x, gr, ur, dtype, exact_w=True, what=f"decode M={M}")


@pytest.mark.parametrize("M", [1, 40, 300])
@pytest.mark.parametrize("tile_m", [32, 64, 128])
@pytest.mark.parametrize("split_k", [1, 2, 4, 8])
def test_forced_gemm(M, tile_m, split_k):
    from autogptq_b200 import _lib

    _need_gpu()
    dtype = torch.float16 if split_k % 4 else torch.bfloat16
    gate, up, gr, ur = make_pair(1024, 2816, 64, desc_act=M == 40, bias=True, dtype=dtype, seed=5)
    x = x_rows(M, 1024, dtype, seed=M)
    h = _fgu()(gate, up, x, kernel=_lib.GATE_UP_GEMM, tile_m=tile_m, split_k=split_k)
    assert_gate_up(h, x, gr, ur, dtype, exact_w=False, what=f"GEMM M={M} tile={tile_m} split={split_k}")


def test_partial_column_tile():
    """I % 64 == 32: the last 64-column half of the GEMM is half outside the layer."""
    _need_gpu()
    gate, up, gr, ur = make_pair(512, 1056, 32, dtype=torch.float16, seed=2)
    for M in (3, 77):
        x = x_rows(M, 512, torch.float16, seed=M)
        assert_gate_up(_fgu()(gate, up, x), x, gr, ur, torch.float16, exact_w=M <= 8, what=f"I=1056 M={M}")


@pytest.fixture(scope="module")
def llama_pair():
    _need_gpu()
    return make_pair(4096, 11008, 128, dtype=torch.float16, seed=11)


@pytest.mark.parametrize("M", [1, 8, 64, 512])
def test_llama7b_size(M, llama_pair):
    gate, up, gr, ur = llama_pair
    I = 11008
    cols = np.r_[0:256, I - 256:I]
    zcols = np.r_[0:32, I // 8 - 32:I // 8]
    sl = [dict(d, qweight=d["qweight"][:, cols], qzeros=d["qzeros"][:, zcols], scales=d["scales"][:, cols]) for d in (gr, ur)]
    x = x_rows(M, 4096, torch.float16, seed=M)
    h = _fgu()(gate, up, x)
    torch.cuda.synchronize()
    assert_gate_up(h[:, cols], x, sl[0], sl[1], torch.float16, exact_w=M <= 8, what=f"Llama-2-7B gate/up M={M}")


@pytest.mark.parametrize("M,split_k", [(3, 0), (300, 0), (100, 4)])
def test_deterministic(M, split_k):
    from autogptq_b200 import _lib

    _need_gpu()
    gate, up, _, _ = make_pair(1024, 2816, 128, desc_act=True, dtype=torch.float16, seed=4)
    x = x_rows(M, 1024, torch.float16)
    kern = _lib.GATE_UP_GEMM if split_k else _lib.GATE_UP_AUTO
    a = _fgu()(gate, up, x, kernel=kern, split_k=split_k)
    b = _fgu()(gate, up, x, kernel=kern, split_k=split_k)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


@pytest.mark.parametrize("M", [4, 100])
def test_cuda_graph_replay(M):
    _need_gpu()
    gate, up, gr, ur = make_pair(1024, 2816, 128, desc_act=True, bias=True, dtype=torch.float16, seed=6)
    x = x_rows(M, 1024, torch.float16, seed=2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _fgu()(gate, up, x)                 # warm-up: post_init, tensor-core copies, workspace, argument cache
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        h = _fgu()(gate, up, x)
    for r in range(2):
        x.copy_(x_rows(M, 1024, torch.float16, seed=10 + r))
        graph.replay()
        torch.cuda.synchronize()
        assert_gate_up(h, x, gr, ur, torch.float16, exact_w=M <= 8, what=f"replay {r}")


@pytest.mark.parametrize("M", [1, 7, 300])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_fused_module_matches_unfused_layers(M, dtype):
    from autogptq_b200 import FusedQuantMLP

    _need_gpu()
    gate, up, _, _ = make_pair(1024, 2816, 128, bias=True, dtype=dtype, seed=8)
    down = make_layer(O.random_packed(2816, 1024, 128, seed=9), device="cuda", dtype=dtype)
    mlp = FusedQuantMLP(gate, up, down)
    x = x_rows(M, 1024, dtype, seed=M).reshape(1, M, 1024)
    y = mlp(x)
    y_ref = down(F.silu(gate(x)) * up(x))
    torch.cuda.synchronize()
    assert y.shape == y_ref.shape == (1, M, 1024) and y.dtype == dtype
    tol = {k: 2 * v for k, v in TOL[dtype].items()}      # both sides round h; a flipped last bit of h moves y slightly
    assert_parity(y.float().cpu().numpy(), y_ref.float().cpu().numpy(), what=f"FusedQuantMLP M={M} {dtype}", **tol)


def test_tiny_llama_inject_logits_and_greedy_decode():
    from autogptq_b200 import FusedQuantMLP, QuantLinear, inject_fused_mlp
    from tests.test_integration_reference import _quant_names, _rtn_pack, _tiny_llama

    _need_gpu()
    dev = torch.device("cuda", 0)
    model = _tiny_llama(seed=1)
    packed, _ = _rtn_pack(model)
    qmodel = model.half()
    for n, q in packed.items():
        parent, _, child = n.rpartition(".")
        setattr(qmodel.get_submodule(parent), child, q)
    qmodel = qmodel.to(dev)
    ids = torch.randint(0, 128, (2, 12), device=dev)

    def greedy(m, start, steps=8):
        seq = start.clone()
        with torch.inference_mode():
            for _ in range(steps):
                seq = torch.cat([seq, m(seq).logits[:, -1].argmax(-1, keepdim=True)], dim=1)
        return seq

    with torch.inference_mode():
        l0 = qmodel(ids).logits.float()
    g0 = greedy(qmodel, ids[:, :4])
    assert inject_fused_mlp(qmodel) == 2
    assert all(isinstance(layer.mlp, FusedQuantMLP) for layer in qmodel.model.layers)
    assert isinstance(qmodel.model.layers[0].mlp.down_proj, QuantLinear)
    assert set(_quant_names(qmodel)) == set()          # every Linear stays a QuantLinear
    with torch.inference_mode():
        l1 = qmodel(ids).logits.float()
    g1 = greedy(qmodel, ids[:, :4])
    scale = l0.abs().max().item()
    assert torch.isfinite(l1).all() and (l1 - l0).abs().max().item() <= 1e-2 * scale, ((l1 - l0).abs().max().item(), scale)
    if not torch.equal(g0, g1):
        with torch.inference_mode():
            top2 = qmodel(g0[:, :-1]).logits.float().topk(2, -1).values
        assert (top2[..., 0] - top2[..., 1]).min().item() < 1e-2 * scale, "greedy decode diverged with a clear margin"


@pytest.mark.parametrize("M", [2, 50])
def test_awq_loaded_pair(M, tmp_path):
    from autogptq_b200 import checkpoint as C

    _need_gpu()
    raw = {f"model.layers.0.mlp.{n}": A.random_awq(512, 1024, 128, seed=j, bias=False) for j, n in enumerate(("gate_proj", "up_proj"))}
    write_awq_checkpoint(str(tmp_path), raw, 128)
    layers = C.load_quant_linears(str(tmp_path), device="cuda")
    gate, up = layers["model.layers.0.mlp.gate_proj"], layers["model.layers.0.mlp.up_proj"]
    gr, ur = (gptq_view(raw[f"model.layers.0.mlp.{n}"]) for n in ("gate_proj", "up_proj"))
    x = x_rows(M, 512, torch.float16, seed=M)
    assert_gate_up(_fgu()(gate, up, x), x, gr, ur, torch.float16, exact_w=M <= 8, what=f"AWQ M={M}")


def test_decode_turned_down_by_the_library_runs_the_gemm():
    """K = 14336: 16 * K bytes of x rows do not fit one CTA's shared memory, so the library runs the GEMM even at M <= 8
    (forward_gate_up then builds the tensor-core copies and repeats the call)."""
    _need_gpu()
    gate, up, gr, ur = make_pair(14336, 64, 128, dtype=torch.float16, seed=12)
    x = x_rows(2, 14336, torch.float16)
    h = _fgu()(gate, up, x)
    assert gate._qweight_tc is not None and up._qweight_tc is not None
    assert_gate_up(h, x, gr, ur, torch.float16, exact_w=False, what="K=14336 M=2")


@pytest.mark.parametrize("M", [3, 40])
def test_reloaded_weights_are_used(M):
    """A second post_init() after new weights are loaded in place replaces the run tensors (tensor-core copy, scales,
    permutation); the cached call arguments must follow."""
    _need_gpu()
    gate, up, _, _ = make_pair(512, 1024, 64, desc_act=True, bias=True, dtype=torch.float16, seed=20)
    x = x_rows(M, 512, torch.float16, seed=M)
    _fgu()(gate, up, x)
    g2, u2, gr, ur = make_pair(512, 1024, 64, desc_act=True, bias=True, dtype=torch.float16, seed=30)
    gate.load_state_dict(g2.state_dict())
    up.load_state_dict(u2.state_dict())
    gate.post_init()
    up.post_init()
    assert_gate_up(_fgu()(gate, up, x), x, gr, ur, torch.float16, exact_w=M <= 8, what=f"reloaded M={M}")


def test_fallbacks_run_the_unfused_expression():
    from autogptq_b200 import _lib

    _need_gpu()
    fgu = _fgu()

    def unfused(g, u, x):
        return F.silu(g(x)) * u(x)

    # different act-order permutations
    g1 = make_layer(O.random_packed(512, 1024, 64, seed=1, desc_act=True), dtype=torch.float16)
    u1 = make_layer(O.random_packed(512, 1024, 64, seed=2, desc_act=True), dtype=torch.float16)
    # I % 32 != 0
    g2 = make_layer(O.random_packed(512, 264, 128, seed=3), dtype=torch.float16)
    u2 = make_layer(O.random_packed(512, 264, 128, seed=4), dtype=torch.float16)
    # a group size the tensor-core GEMM cannot run (decode batches still fuse)
    g3 = make_layer(O.random_packed(480, 1024, 96, seed=5), dtype=torch.float16)
    u3 = make_layer(O.random_packed(480, 1024, 96, seed=6), dtype=torch.float16)
    # different group sizes
    g4 = make_layer(O.random_packed(512, 1024, 64, seed=7), dtype=torch.float16)
    u4 = make_layer(O.random_packed(512, 1024, 128, seed=8), dtype=torch.float16)
    for (g, u), M in (((g1, u1), 3), ((g1, u1), 64), ((g2, u2), 2), ((g2, u2), 64), ((g3, u3), 64), ((g4, u4), 5)):
        x = x_rows(M, g.infeatures, torch.float16, seed=M)
        assert torch.equal(fgu(g, u, x), unfused(g, u, x)), (g.group_size, u.group_size, g.outfeatures, M)
    # batches above FUSED_MAX_M rows: the unfused layers measured faster there
    from autogptq_b200.mlp import FUSED_MAX_M

    x = x_rows(FUSED_MAX_M + 1, 512, torch.float16)
    assert torch.equal(fgu(g4, g4, x), unfused(g4, g4, x))
    # fp32 activations: the unfused modules cast them
    x = x_rows(4, 512, torch.float32)
    assert torch.equal(fgu(g4, g4, x), unfused(g4, g4, x))
    # decode batches of the group-size-96 pair are fused
    gate, up, gr, ur = make_pair(480, 1024, 96, dtype=torch.float16, seed=5)
    x = x_rows(5, 480, torch.float16)
    assert_gate_up(fgu(gate, up, x), x, gr, ur, torch.float16, exact_w=True, what="g=96 decode")
    # a forced kernel never falls back
    with pytest.raises(NotImplementedError):
        fgu(g1, u1, x_rows(3, 512, torch.float16), kernel=_lib.GATE_UP_DECODE)
    with pytest.raises(_lib.B200KernelError):
        fgu(gate, up, x_rows(9, 480, torch.float16), kernel=_lib.GATE_UP_DECODE)
