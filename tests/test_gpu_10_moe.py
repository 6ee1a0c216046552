"""GPU tests of the grouped mixture-of-experts forward (QuantExperts, agb200_moe_*): parity with oracle/moe_oracle.py on
the decode path (T <= 8) and the grouped wgmma GEMM path (T > 8), skewed routing, determinism, CUDA-graph replay with
new routing, and agreement with the per-expert QuantLinear loop."""
import numpy as np
import pytest
import torch

from oracle import moe_oracle as MO
from oracle import w4a16_oracle as O
from tests._util import assert_parity, make_layer

pytestmark = pytest.mark.gpu

E = 8
TOL = {torch.float16: dict(rtol=1e-3, atol_rms=1.6e-3), torch.bfloat16: dict(rtol=8e-3, atol_rms=4e-3)}
DT = {torch.float16: "float16", torch.bfloat16: "bfloat16"}


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _build(H, I, g, desc_act, bias, dtype, seed=0, n_experts=E):
    """(QuantExperts, oracle experts with the scales / bias the device uses)."""
    from autogptq_b200 import QuantExperts

    mods = {"w1": [], "w3": [], "w2": []}
    ref = []
    for e in range(n_experts):
        ex = {}
        for j, (name, K, N) in enumerate((("w1", H, I), ("w3", H, I), ("w2", I, H))):
            d = O.random_packed(K, N, g, seed=seed + 3 * e + j, desc_act=desc_act, bias=bias)
            if name == "w3" and desc_act:
                d["g_idx"] = ex["w1"]["g_idx"]           # w1 and w3 see the same inputs: one act-order permutation
            lin = make_layer(d, device="cuda", dtype=dtype)
            mods[name].append(lin)
            d = dict(d, scales=lin.scales.float().cpu().numpy(),
                     bias=None if lin.bias is None else lin.bias.float().cpu().numpy())
            ex[name] = d
        ref.append(ex)
    return QuantExperts.from_linears(mods["w1"], mods["w3"], mods["w2"]), ref


def _routing(T, k, seed, n_experts=E):
    rng = np.random.default_rng(seed)
    idx = np.stack([rng.permutation(n_experts)[:k] for _ in range(T)]).astype(np.int64)
    w = rng.random((T, k)).astype(np.float32)
    return idx, w / w.sum(axis=1, keepdims=True)


def _x(T, H, dtype, seed=1):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((T, H)).astype(np.float32)).to(dtype).cuda()


ULP = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}     # one ulp, relative to a value's magnitude (upper bound)


def _assert_moe(y, x, ref, idx, w, dtype, what):
    """assert_parity against the oracle, with the arithmetic of the path T selects (decode: exact weights; GEMM:
    weights rounded to the dtype, as the tensor-core QuantLinear tests do), after excusing one ulp of every per-pair
    output: those are rounded to the dtype before the weighted sum (as in the reference), so a last-bit difference
    in the fp32 sum before that rounding moves the pair's output by one ulp."""
    T = x.shape[0]
    y_ref, mag = MO.forward(x.float().cpu().numpy(), ref, idx, w, DT[dtype],
                            weight_dtype=None if T <= 8 else DT[dtype], return_magnitude=True)
    y = np.asarray(y, dtype=np.float32)
    err = y - y_ref
    excused = np.sign(err) * np.maximum(np.abs(err) - ULP[dtype] * mag, 0)
    assert_parity(y_ref + excused, y_ref, what=what, **TOL[dtype])


def _check(qe, ref, x, idx, w, dtype, what):
    xi = torch.as_tensor(idx).cuda()
    wt = torch.as_tensor(w).cuda()
    y = qe(x, xi, wt)
    torch.cuda.synchronize()
    assert y.shape == x.shape and y.dtype == dtype
    y = y.float().cpu().numpy()
    _assert_moe(y, x, ref, idx, w, dtype, what)
    return y


@pytest.mark.parametrize("T", [1, 2, 5, 8, 9, 64, 333, 2048])
@pytest.mark.parametrize("k", [1, 2])
def test_parity_fp16_g128(T, k):
    _need_gpu()
    qe, ref = _build(1024, 2816, 128, desc_act=False, bias=False, dtype=torch.float16, seed=k)
    idx, w = _routing(T, k, seed=T)
    _check(qe, ref, _x(T, 1024, torch.float16, seed=T), idx, w, torch.float16, f"T={T} k={k}")


@pytest.mark.parametrize("T", [1, 5, 9, 333])
@pytest.mark.parametrize("g,desc_act,bias", [(-1, False, True), (128, True, False), (128, True, True)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_parity_configs(T, g, desc_act, bias, dtype):
    _need_gpu()
    qe, ref = _build(1024, 2816, g, desc_act=desc_act, bias=bias, dtype=dtype, seed=7)
    idx, w = _routing(T, 2, seed=100 + T)
    # routing weights in the activation dtype (MixtralSparseMoeBlock passes them in the router's dtype)
    wt = MO.round_to(w, DT[dtype])
    xi, ww = torch.as_tensor(idx).cuda(), torch.as_tensor(wt).to(dtype).cuda()
    x = _x(T, 1024, dtype, seed=T)
    y = qe(x, xi, ww)
    torch.cuda.synchronize()
    _assert_moe(y.float().cpu().numpy(), x, ref, idx, wt, dtype, f"T={T} g={g} act={desc_act} bias={bias} {dtype}")


@pytest.fixture(scope="module")
def mixtral_experts():
    _need_gpu()
    return _build(4096, 14336, 128, desc_act=False, bias=False, dtype=torch.float16, seed=11)


@pytest.mark.parametrize("T", [1, 8, 64])
def test_parity_mixtral_size(T, mixtral_experts):
    H = 4096
    qe, ref = mixtral_experts
    idx, w = _routing(T, 2, seed=T)
    cols = np.r_[0:256, H - 256:H]
    # column slices of the output: w2 of the oracle restricted to them (h needs all of I)
    sref = [dict(ex, w2=dict(ex["w2"], qweight=ex["w2"]["qweight"][:, cols], qzeros=None, scales=ex["w2"]["scales"][:, cols]))
            for ex in ref]
    for ex, full in zip(sref, ref):
        zf = O.unpack_qzeros(full["w2"]["qzeros"], wrap=False) - 1
        ex["w2"]["qzeros"] = O.pack_cols((zf[:, cols]).astype(np.uint32))
    xi, wt = torch.as_tensor(idx).cuda(), torch.as_tensor(w).cuda()
    x = _x(T, H, torch.float16, seed=T)
    y = qe(x, xi, wt)
    torch.cuda.synchronize()
    _assert_moe(y.float().cpu().numpy()[:, cols], x, sref, idx, w, torch.float16, f"Mixtral size T={T}")


@pytest.mark.parametrize("T", [1, 6, 40, 2048])
def test_skewed_routing(T):
    _need_gpu()
    qe, ref = _build(1024, 2816, 128, desc_act=False, bias=True, dtype=torch.float16, seed=3)
    x = _x(T, 1024, torch.float16, seed=T)
    rng = np.random.default_rng(T)
    w = rng.random((T, 2)).astype(np.float32)
    # every token to expert 5 (slot 0) and id E (skipped) in slot 1
    idx = np.stack([np.full(T, 5), np.full(T, E)], axis=1)
    _check(qe, ref, x, idx, w, torch.float16, f"one expert T={T}")
    # all pairs on two experts, the other six get nothing (long padded segments on the GEMM path)
    idx = np.stack([np.full(T, 2), np.full(T, 6)], axis=1)
    idx[::3] = idx[::3, ::-1]
    _check(qe, ref, x, idx, w, torch.float16, f"two experts T={T}")
    # int32 ids, a sprinkling of id E
    idx, w = _routing(T, 2, seed=T + 1)
    idx[rng.random(idx.shape) < 0.3] = E
    _check(qe, ref, x, idx.astype(np.int32), w, torch.float16, f"ids == E T={T}")


@pytest.mark.parametrize("T", [3, 300])
def test_deterministic(T):
    _need_gpu()
    qe, _ = _build(1024, 2816, 128, desc_act=True, bias=False, dtype=torch.float16, seed=4)
    idx, w = _routing(T, 2, seed=T)
    x, xi, wt = _x(T, 1024, torch.float16), torch.as_tensor(idx).cuda(), torch.as_tensor(w).cuda()
    a = qe(x, xi, wt)
    b = qe(x, xi, wt)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_empty_batch():
    _need_gpu()
    qe, _ = _build(1024, 2816, 128, desc_act=False, bias=False, dtype=torch.float16, seed=4, n_experts=2)
    y = qe(torch.zeros(0, 1024, dtype=torch.float16, device="cuda"), torch.zeros(0, 2, dtype=torch.int64, device="cuda"),
           torch.zeros(0, 2, device="cuda"))
    assert y.shape == (0, 1024)


@pytest.mark.parametrize("T", [4, 100])
def test_cuda_graph_replay_with_new_routing(T):
    _need_gpu()
    qe, ref = _build(1024, 2816, 128, desc_act=False, bias=False, dtype=torch.float16, seed=5)
    x = _x(T, 1024, torch.float16, seed=2)
    idx0, w0 = _routing(T, 2, seed=0)
    xi, wt = torch.as_tensor(idx0).cuda(), torch.as_tensor(w0).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        qe(x, xi, wt)                     # warm-up: plan, tensor-core copies, workspace
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = qe(x, xi, wt)
    for r in range(3):
        idx, w = _routing(T, 2, seed=10 + r)
        if r == 2:
            idx[:, 1] = E                 # second replay round: half the slots skipped
        xi.copy_(torch.as_tensor(idx))
        wt.copy_(torch.as_tensor(w))
        graph.replay()
        torch.cuda.synchronize()
        _assert_moe(y.float().cpu().numpy(), x, ref, idx, w, torch.float16, f"replay {r}")


@pytest.mark.parametrize("T", [2, 50])
def test_matches_per_expert_quantlinear_loop(T):
    _need_gpu()
    qe, _ = _build(1024, 2816, 128, desc_act=True, bias=True, dtype=torch.float16, seed=9)
    idx, w = _routing(T, 2, seed=T)
    x, xi, wt = _x(T, 1024, torch.float16), torch.as_tensor(idx).cuda(), torch.as_tensor(w).cuda()
    y = qe(x, xi, wt)
    # MixtralExperts.forward (modeling_mixtral.py:74-98) over the same QuantLinear modules
    final = torch.zeros(T, 1024, dtype=torch.float32, device="cuda")
    mask = torch.nn.functional.one_hot(xi, num_classes=E + 1).permute(2, 1, 0)
    for e in torch.greater(mask.sum(dim=(-1, -2)), 0).nonzero().flatten().tolist():
        if e == E:
            continue
        slot, tok = torch.where(mask[e])
        h = torch.nn.functional.silu(qe.w1[e](x[tok])) * qe.w3[e](x[tok])
        final.index_add_(0, tok, qe.w2[e](h).float() * wt[tok, slot, None])
    torch.cuda.synchronize()
    assert_parity(y.float().cpu().numpy(), final.to(torch.float16).float().cpu().numpy(), what=f"loop T={T}", **TOL[torch.float16])
