"""GPU tests of the input gradient dx = dy · Wᵀ (agb200_w4a16_dgrad): kernel parity against the fp32 oracle with the
weights rounded to the dtype (the GEMM tolerances of the AWQ tests), the reference's own gradients, determinism, the
autograd wiring of QuantLinear and the composite paths, and a small LoRA-style training run."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from autogptq_b200 import FusedQuantMLP, QuantExperts, _lib, forward_group
from oracle import w4a16_oracle as O
from tests._dgrad_util import DGRAD_GOLDENS, dgrad, load_golden
from tests._util import assert_parity, make_layer

pytestmark = pytest.mark.gpu

DT = {torch.float16: "float16", torch.bfloat16: "bfloat16"}
GEMM_TOL = {torch.float16: dict(rtol=1e-3, atol_rms=6e-4), torch.bfloat16: dict(rtol=8e-3, atol_rms=8e-3)}


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _t(a, dtype):
    return torch.from_numpy(np.asarray(a, dtype=np.float32)).to(dtype).cuda()


def _dy(M, N, dtype, seed):
    return _t(np.random.default_rng(seed).standard_normal((M, N)), dtype)


def _check(lin, d, M, dtype, seed, what, **kw):
    dy = _dy(M, d["N"], dtype, seed)
    dx = lin.input_grad(dy, **kw)
    torch.cuda.synchronize()
    assert dx.dtype == dtype and dx.shape == (M, d["K"])
    ref = dgrad(d, dy.float().cpu().numpy(), round_to=DT[dtype])
    assert_parity(dx.float().cpu().numpy(), ref, what=what, **GEMM_TOL[dtype])


_LAYERS = {}


def _layer(K, N, g, act, dtype):
    key = (K, N, g, act, dtype)
    if key not in _LAYERS:
        d = O.random_packed(K, N, g, seed=K + N + (g % 97) + 7 * act, desc_act=act, bias=True)
        _LAYERS[key] = (d, make_layer(d, device="cuda", dtype=dtype))
    return _LAYERS[key]


# K and N tails (392 = 3 * 128 + 8, 288 = 4 * 64 + 32); g = 96 leaves a partial last group
@pytest.mark.parametrize("M", [1, 3, 8, 16, 64, 200, 1024, 4096])
@pytest.mark.parametrize("g", [32, 64, 128, -1, 96])
@pytest.mark.parametrize("act", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_dgrad_parity_grid(M, g, act, dtype):
    d, lin = _layer(392, 288, g, act, dtype)
    _check(lin, d, M, dtype, seed=M, what=f"dgrad M={M} g={g} act={act} {dtype}")


@pytest.mark.parametrize("M", [1, 5, 130])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_dgrad_k264_act_order_shape(M, dtype):
    d, lin = _layer(264, 64, 128, True, dtype)
    _check(lin, d, M, dtype, seed=M, what=f"dgrad K=264 act M={M}")


# layers the tensor-core path does not take run the CUDA-core kernel; the CUDA-core kernel also takes every other layer
@pytest.mark.parametrize("K,N,g,act", [(256, 40, 32, False), (256, 96, 16, True), (200, 64, 40, False), (392, 288, 128, True)])
@pytest.mark.parametrize("M", [1, 37])
def test_dgrad_cuda_core_kernel(K, N, g, act, M):
    d, lin = _layer(K, N, g, act, torch.float16)
    _check(lin, d, M, torch.float16, seed=M, what=f"cuda-core K={K} N={N} g={g}", kernel=_lib.DGRAD_CUDA_CORE)
    if N % 32 == 0 and g % 16 == 0 and g >= 32:
        return
    with pytest.raises(_lib.B200KernelError, match="tensor-core path"):
        lin.input_grad(_dy(M, N, torch.float16, 0), kernel=_lib.DGRAD_WGMMA)
    _check(lin, d, M, torch.float16, seed=M, what=f"auto K={K} N={N} g={g}")


@pytest.mark.parametrize("tile_m,split_k", [(32, 1), (32, 8), (64, 2), (64, 4), (128, 1), (128, 2)])
def test_dgrad_forced_tiles_and_splits(tile_m, split_k):
    d, lin = _layer(392, 288, 128, True, torch.float16)
    _check(lin, d, 300, torch.float16, seed=5, what=f"tile {tile_m} split {split_k}", kernel=_lib.DGRAD_WGMMA,
           tile_m=tile_m, split_k=split_k)


@pytest.mark.parametrize("K,N", [(4096, 4096), (4096, 11008), (11008, 4096)])
def test_dgrad_llama_7b_shapes(K, N):
    d = O.random_packed(K, N, 128, seed=K // 7 + N, desc_act=False)
    lin = make_layer(d, device="cuda")
    dy = _dy(2048, N, torch.float16, seed=3)
    dx = lin.input_grad(dy)
    torch.cuda.synchronize()
    dys = dy.float().cpu().numpy()
    for k0, k1 in ((0, 256), (K // 2, K // 2 + 256), (K - 256, K)):     # column slices, the grid's edge included
        ref = dgrad(d, dys, round_to="float16", rows=(k0, k1))
        assert_parity(dx[:, k0:k1].float().cpu().numpy(), ref, rtol=1e-3, atol_rms=1.6e-3, what=f"{K}x{N} [{k0}:{k1}]")


@pytest.mark.parametrize("name", DGRAD_GOLDENS)
@pytest.mark.parametrize("M_rep", [1, 40])
def test_reference_gradients_on_gpu(name, M_rep):
    """The reference's x.grad (fp32 weights), reproduced by the fp16 kernels (the rows are repeated to reach the
    tensor-core tile sizes as well)."""
    d, z = load_golden(name)
    lin = make_layer(d, device="cuda")
    dy = np.tile(z["dy"], (M_rep, 1))
    x = _t(np.tile(z["x"], (M_rep, 1)), torch.float16).requires_grad_(True)
    lin(x).backward(_t(dy, torch.float16))
    torch.cuda.synchronize()
    assert_parity(x.grad.float().cpu().numpy(), np.tile(z["dx_new"], (M_rep, 1)), rtol=2e-3, atol_rms=1.6e-3, what=name)


def test_repeated_calls_are_bit_identical():
    d, lin = _layer(392, 288, 128, True, torch.float16)
    for M, kw in ((4096, {}), (64, dict(split_k=8)), (3, dict(kernel=_lib.DGRAD_CUDA_CORE))):
        dy = _dy(M, 288, torch.float16, seed=11)
        a, b = lin.input_grad(dy, **kw), lin.input_grad(dy, **kw)
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ autograd
@pytest.mark.parametrize("act", [False, True])
@pytest.mark.parametrize("M", [2, 96])
def test_autograd_matches_kernel_and_keeps_y(act, M):
    d, lin = _layer(392, 288, 64, act, torch.float16)
    x0 = _t(np.random.default_rng(M).standard_normal((M, 392)), torch.float16)
    y_plain = lin(x0)
    x = x0.clone().requires_grad_(True)
    y = lin(x)
    assert y.grad_fn is not None and y_plain.grad_fn is None
    assert torch.equal(y, y_plain)                               # same kernels, same bits
    dy = _dy(M, 288, torch.float16, seed=9)
    y.backward(dy)
    assert torch.equal(x.grad, lin.input_grad(dy))


def test_autograd_fp32_input_gets_fp32_grad_and_3d_shapes():
    d, lin = _layer(392, 288, 128, False, torch.float16)
    x = torch.randn(2, 5, 392, device="cuda", requires_grad=True)
    y = lin(x)
    assert y.dtype == torch.float32 and y.shape == (2, 5, 288)
    dy = torch.randn_like(y)
    y.backward(dy)
    assert x.grad.dtype == torch.float32 and x.grad.shape == x.shape
    ref = lin.input_grad(dy.half()).float()
    assert torch.equal(x.grad, ref)


def test_tensor_core_paths_on_a_fresh_host_thread():
    """A thread whose first CUDA work is a tensor-map encode (as on autograd's backward worker) binds the context."""
    import threading

    d, lin = _layer(392, 288, 128, True, torch.float16)
    dy = _dy(200, 288, torch.float16, seed=4)
    x = _t(np.random.default_rng(4).standard_normal((200, 392)), torch.float16)
    want = (lin.input_grad(dy), lin(x))
    got = []
    th = threading.Thread(target=lambda: got.append((lin.input_grad(dy), lin(x))))
    th.start()
    th.join()
    torch.cuda.synchronize()
    assert got and torch.equal(got[0][0], want[0]) and torch.equal(got[0][1], want[1])


def test_activation_checkpointing():
    from torch.utils.checkpoint import checkpoint

    d, lin = _layer(392, 288, 128, True, torch.float16)
    x = torch.randn(64, 392, device="cuda", dtype=torch.float16, requires_grad=True)
    checkpoint(lambda t: F.silu(lin(t)), x, use_reentrant=False).float().pow(2).sum().backward()
    g_ck = x.grad.clone()
    x.grad = None
    F.silu(lin(x)).float().pow(2).sum().backward()
    assert torch.equal(g_ck, x.grad)


def test_forward_backward_in_one_cuda_graph():
    d, lin = _layer(392, 288, 128, True, torch.float16)
    x = torch.randn(200, 392, device="cuda", dtype=torch.float16, requires_grad=True)
    dy = torch.randn(200, 288, device="cuda", dtype=torch.float16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                   # warm-up outside the capture (workspace, tensor-core copy)
        for _ in range(2):
            x.grad = None
            lin(x).backward(dy)
    torch.cuda.current_stream().wait_stream(s)
    x.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = lin(x)
        y.backward(dy)
    ref_x = torch.randn_like(x)
    ref_dy = torch.randn_like(dy)
    with torch.no_grad():
        x.copy_(ref_x)
    dy.copy_(ref_dy)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(x.grad, lin.input_grad(ref_dy))
    assert torch.equal(y, lin(ref_x))


# ------------------------------------------------------------------------------------------------ training
class _LoRA(torch.nn.Module):
    """y = base(x) + (x Aᵀ) Bᵀ · scale: hand-written rank-r adapter next to a frozen layer."""

    def __init__(self, base, K, N, r, dtype, seed):
        super().__init__()
        gen = torch.Generator().manual_seed(seed)
        self.base = base
        self.A = torch.nn.Parameter((torch.randn(r, K, generator=gen) / K ** 0.5).to(dtype).cuda())
        self.B = torch.nn.Parameter((torch.randn(N, r, generator=gen) * 0.05).to(dtype).cuda())

    def forward(self, x):
        return self.base(x) + (x @ self.A.t()) @ self.B.t()


def _dense(d, dtype):
    """fp32 twin of a QuantLinear: the dequantised weights (scales rounded to the compute dtype) and bias."""
    s = O.dequantize(d["qweight"], d["qzeros"], _round(d["scales"], dtype), g_idx=d["g_idx"])
    W = torch.from_numpy(s).cuda()                                 # [K, N]
    b = torch.from_numpy(_round(d["bias"], dtype)).cuda()
    return lambda x: x @ W + b


def _round(a, dtype):
    return torch.from_numpy(np.asarray(a, dtype=np.float32)).to(dtype).float().numpy()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_lora_adapter_gradients_and_training(dtype):
    K1, N1, N2, r, M = 512, 768, 384, 16, 256
    d1 = O.random_packed(K1, N1, 128, seed=61, bias=True)
    d2 = O.random_packed(N1, N2, 64, seed=62, desc_act=True, bias=True)
    q1, q2 = make_layer(d1, device="cuda", dtype=dtype), make_layer(d2, device="cuda", dtype=dtype)
    l1, l2 = _LoRA(q1, K1, N1, r, dtype, 1), _LoRA(q2, N1, N2, r, dtype, 2)
    f1, f2 = _LoRA(_dense(d1, dtype), K1, N1, r, torch.float32, 1), _LoRA(_dense(d2, dtype), N1, N2, r, torch.float32, 2)
    with torch.no_grad():
        for a, b in ((l1, f1), (l2, f2)):
            b.A.copy_(a.A.float())
            b.B.copy_(a.B.float())
    x = torch.randn(M, K1, device="cuda")
    target = torch.randn(M, N2, device="cuda")

    def loss_of(m1, m2, xx):
        return (m2(F.silu(m1(xx))).float() - target).pow(2).mean()

    loss_q = loss_of(l1, l2, x.to(dtype))
    loss_q.backward()
    loss_f = loss_of(f1, f2, x)
    loss_f.backward()
    # bounds: 16-bit activations and weights through two layers; fp16 keeps ~3 decimal digits, bf16 ~2
    rel_max, cos_min = (0.03, 0.999) if dtype == torch.float16 else (0.12, 0.99)
    for name, p, q in (("A1", l1.A, f1.A), ("B1", l1.B, f1.B), ("A2", l2.A, f2.A), ("B2", l2.B, f2.B)):
        g, ref = p.grad.float().flatten(), q.grad.flatten()
        rel = float((g - ref).norm() / ref.norm())
        cos = float(F.cosine_similarity(g, ref, dim=0))
        assert rel < rel_max and cos > cos_min, f"{name}: rel {rel:.4f} cos {cos:.5f}"
    opt = torch.optim.SGD([l1.A, l1.B, l2.A, l2.B], lr=0.5)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        loss = loss_of(l1, l2, x.to(dtype))
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < losses[0], losses


# ------------------------------------------------------------------------------------------------ composites
def test_fused_mlp_and_forward_group_in_grad_mode_match_unfused():
    K, I = 512, 768
    dg, du, dd = (O.random_packed(K, I, 128, seed=71), O.random_packed(K, I, 128, seed=72),
                  O.random_packed(I, K, 128, seed=73))
    g, u, dn = (make_layer(d, device="cuda") for d in (dg, du, dd))
    mlp = FusedQuantMLP(g, u, dn)
    x = torch.randn(4, 3, K, device="cuda", dtype=torch.float16, requires_grad=True)
    y = mlp(x)
    dy = torch.randn_like(y)
    y.backward(dy)
    gx = x.grad.clone()
    x.grad = None
    y2 = dn(F.silu(g(x)) * u(x))
    y2.backward(dy)
    assert torch.equal(y, y2) and torch.equal(gx, x.grad)
    x.grad = None
    outs = forward_group([g, u], x[:1, :1])                       # one row: the grouped decode kernel when not recording
    sum(o.float().sum() for o in outs).backward()
    gx = x.grad.clone()
    x.grad = None
    (g(x[:1, :1]).float().sum() + u(x[:1, :1]).float().sum()).backward()
    assert torch.equal(gx, x.grad)


def test_quant_experts_refuses_grad_mode():
    H, I, E = 256, 256, 2
    ds = [O.random_packed(k, n, 128, seed=80 + i) for i, (k, n) in enumerate([(H, I), (H, I), (I, H)] * E)]
    ls = [make_layer(d, device="cuda") for d in ds]
    ex = QuantExperts(ls[0::3], ls[1::3], ls[2::3])
    x = torch.randn(4, H, device="cuda", dtype=torch.float16, requires_grad=True)
    idx = torch.zeros(4, 1, dtype=torch.int64, device="cuda")
    w = torch.ones(4, 1, dtype=torch.float16, device="cuda")
    with pytest.raises(NotImplementedError, match="inference-only"):
        ex(x, idx, w)
    with torch.no_grad():
        assert ex(x, idx, w).shape == (4, H)
