"""GPU tests of the fused dense MLP backward (``FusedQuantMLP(fused_backward=True)``, ``agb200_w4a16_gate_up_saving``,
``agb200_w4a16_mlp_backward``).

Error bound of dx against the float64 reference of ``tests/_mlp_grad.py`` (the MoE-backward row of DESIGN §3.12 with
one expert, k = 1, w = 1):

    |dx − dx*| ≤ ulp(dx*) + (γ + ε)·(A + A2)

A, A2, γ (n = max(2·I, H)) and ε are those of ``tests/test_gpu_18_moe_grad.py``.  The largest err/bound and mismatch
rate (share of dx elements that differ from round(dx*)) are printed by ``test_report`` and recorded in DESIGN §3.12."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import w4a16_oracle as O
from tests import _mlp_grad as MLG
from tests._mlp_util import MAX_MISMATCH
from tests._precision import PATHS, gamma, ulp
from tests._util import make_layer

pytestmark = pytest.mark.gpu

DT = {torch.float16: "float16", torch.bfloat16: "bfloat16"}
EPS = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}
REPORT = {}


@pytest.fixture(autouse=True)
def _need_gpu(monkeypatch):
    """Skips without a device.  The fused backward runs at every M here (the kernels take any M); which M it takes by
    default is a speed choice, tested in test_default_cut_over."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import autogptq_b200.mlp as mlp_mod

    monkeypatch.setattr(mlp_mod, "FUSED_BACKWARD_MAX_M", 1 << 30)


def test_default_cut_over(monkeypatch):
    """Above FUSED_BACKWARD_MAX_M rows fused_backward=True gives the default path's output and gradient, bit for bit."""
    import autogptq_b200.mlp as mlp_mod

    monkeypatch.undo()
    cut = mlp_mod.FUSED_BACKWARD_MAX_M
    mlp, _ = _build(1024, 1536, 128, torch.float16, act13=True, seed=8)
    for M in (cut, cut + 1):
        x, dy = _rand(M, 1024, torch.float16, 1), _rand(M, 1024, torch.float16, 2)
        with torch.no_grad():
            y_nograd = mlp(x)
        mlp.fused_backward = True
        y_a, dx_a = _grad(mlp, x, dy)
        mlp.fused_backward = False
        y_b, dx_b = _grad(mlp, x, dy)
        if M == cut:        # the fused path: the no-grad forward's output, dx rounded once
            assert torch.equal(y_a, y_nograd) and not torch.equal(dx_a, dx_b)
        else:               # the default path, bit for bit
            assert torch.equal(y_a, y_b) and torch.equal(dx_a, dx_b)


def _build(H, I, g, dtype, act13=False, act2=False, bias=False, seed=0, fused=True):
    """(FusedQuantMLP, reference layer dicts gate / up / down with the scales and bias the device uses)."""
    from autogptq_b200 import FusedQuantMLP

    refs, mods = [], []
    g13 = g
    for j, (K, N, act) in enumerate(((H, I, act13), (H, I, act13), (I, H, act2))):
        d = O.random_packed(K, N, g13 if g != -1 else K, seed=seed + j, desc_act=act, bias=bias)
        if j == 1 and act:
            d["g_idx"] = refs[0]["g_idx"]          # gate and up are quantised on the same input: one permutation
        lin = make_layer(d, device="cuda", dtype=dtype)
        mods.append(lin)
        refs.append(dict(d, scales=lin.scales.float().cpu().numpy(),
                         bias=None if lin.bias is None else lin.bias.float().cpu().numpy()))
    return FusedQuantMLP(*mods, fused_backward=fused), refs


def _rand(M, K, dtype, seed):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((M, K)).astype(np.float32)).to(dtype).cuda()


def _grad(mlp, x, dy):
    xg = x.clone().requires_grad_(True)
    y = mlp(xg)
    y.backward(dy)
    torch.cuda.synchronize()
    return y.detach(), xg.grad


def _check(mlp, refs, x, dy, dtype, what, cols=None):
    y, dx = _grad(mlp, x, dy)
    assert dx.dtype == dtype and y.grad_fn is None
    M = x.shape[0]
    r = MLG.backward(x.float().cpu().numpy(), *refs, dy.float().cpu().numpy(), DT[dtype], round_w_fwd=M > 8, cols=cols)
    H, I = mlp.gate_proj.infeatures, mlp.gate_proj.outfeatures
    dxv = dx.float().cpu().numpy()
    if cols is not None:
        dxv = dxv[:, cols]
    err = np.abs(dxv - r["dx"])
    bound = ulp(r["dx"], DT[dtype]) + (gamma(PATHS["dgrad"], max(2 * I, H)) + EPS[dtype]) * (r["A"] + r["A2"])
    worst = float((err / bound).max())
    rate = float((dxv != r["dx"]).mean())
    REPORT[what] = (worst, rate)
    print(f"[mlp-grad] {what}: dx err/bound {worst:.3f} mismatch {100 * rate:.2f} %")
    assert np.isfinite(dxv).all()
    assert worst <= 1.0, f"{what}: dx err/bound {worst:.3f}"
    return r, dxv


# ------------------------------------------------------------------------------------------------ saving forward
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("act,bias", [(False, True), (True, False)])
@pytest.mark.parametrize("M,kernel,split", [(1, 0, 0), (3, 0, 0), (8, 0, 0), (64, 2, 1), (64, 2, 4), (200, 0, 0),
                                            (2049, 0, 0)])
def test_saving_forward_is_the_no_grad_forward(dtype, act, bias, M, kernel, split):
    from autogptq_b200 import _lib, forward_gate_up
    from autogptq_b200.mlp import FUSED_MAX_M

    assert 2049 == FUSED_MAX_M + 1
    mlp, _ = _build(1024, 1536, 128, dtype, act13=act, act2=act, bias=bias, seed=3)
    x = _rand(M, 1024, dtype, M)
    with torch.no_grad():
        y_ref = mlp(x)
        h_ref = forward_gate_up(mlp.gate_proj, mlp.up_proj, x, kernel=kernel, split_k=split) if kernel else \
            forward_gate_up(mlp.gate_proj, mlp.up_proj, x)
        y, h, g, u = mlp._forward_saving(x, kernel=kernel, split_k=split)
    assert torch.equal(h, h_ref), "h"
    if not kernel:
        assert torch.equal(y, y_ref), "y"
        xg = x.clone().requires_grad_(True)
        assert torch.equal(mlp(xg).detach(), y_ref), "y through autograd"
    # the saved g, u are what silu * mul consumed: h = rnd(rnd(silu(g)) u).  The kernels form silu with __expf, torch
    # with expf, so a rounding of silu(g) may fall the other way where the two differ (as tests/_mlp_util allows); the
    # unfused path (M > FUSED_MAX_M) is torch's own expression and matches bit for bit.
    h2 = F.silu(g) * u
    rate = float((h2 != h).float().mean())
    if M > FUSED_MAX_M:
        assert rate == 0.0
    else:
        assert rate <= MAX_MISMATCH / 10, rate
        assert torch.allclose(h2.float(), h.float(), rtol=4 * EPS[dtype], atol=0)
    assert g.shape == u.shape == (M, 1536) and g.dtype == u.dtype == dtype


# ------------------------------------------------------------------------------------------------ dx bound
@pytest.mark.parametrize("M", [1, 5, 8, 9, 64, 200, 2048, 2049])
def test_dx_bound_over_m(M):
    mlp, refs = _build(1024, 2816, 128, torch.float16, act13=True, act2=True, bias=True, seed=M)
    _check(mlp, refs, _rand(M, 1024, torch.float16, M), _rand(M, 1024, torch.float16, M + 1), torch.float16,
           f"M={M} g128 act both bias float16")


@pytest.mark.parametrize("M", [5, 200])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("H,I,g,act13,act2,bias", [(1024, 1536, 32, True, False, False), (1024, 1536, 64, False, True, True),
                                                   (1152, 2304, 96, False, False, True), (1024, 1536, 128, True, True, False),
                                                   (1024, 1536, -1, False, False, True)])
def test_dx_bound_configs(M, dtype, H, I, g, act13, act2, bias):
    mlp, refs = _build(H, I, g, dtype, act13=act13, act2=act2, bias=bias, seed=7)
    _check(mlp, refs, _rand(M, H, dtype, M), _rand(M, H, dtype, M + 9), dtype,
           f"M={M} g={g} act={act13}/{act2} bias={bias} {DT[dtype]}")


@pytest.mark.parametrize("M", [8, 300])
def test_dx_bound_llama2_7b_size(M):
    mlp, refs = _build(4096, 11008, 128, torch.float16, seed=11)
    cols = np.r_[0:256, 4096 - 256:4096]
    _check(mlp, refs, _rand(M, 4096, torch.float16, M), _rand(M, 4096, torch.float16, M + 3), torch.float16,
           f"Llama-2-7B size M={M} float16", cols=cols)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M", [5, 200])
def test_rms_error_not_above_the_unfused_path(dtype, M):
    """The fused path rounds dx once; autograd through the unfused layers rounds dh, silu(g), the two layer gradients and
    their sum as well.  Its RMS error against float64 must not be larger (10 % slack)."""
    mlp, refs = _build(1024, 2816, 128, dtype, act13=True, bias=True, seed=21)
    x, dy = _rand(M, 1024, dtype, 1), _rand(M, 1024, dtype, 2)
    r, fused = _check(mlp, refs, x, dy, dtype, f"rms M={M} g128 act13 bias {DT[dtype]}")
    mlp.fused_backward = False
    _, dx = _grad(mlp, x, dy)
    exact = MLG.backward(x.float().cpu().numpy(), *refs, dy.float().cpu().numpy(), DT[dtype], rounded=False,
                         round_w_fwd=M > 8)["dx"]
    rms = lambda a: float(np.sqrt(np.mean((a - exact) ** 2)))      # noqa: E731
    e_fused, e_default = rms(fused), rms(dx.float().cpu().numpy())
    print(f"[mlp-grad] rms vs float64 M={M} {DT[dtype]}: fused {e_fused:.3e} unfused {e_default:.3e}")
    assert e_fused <= 1.1 * e_default


# ------------------------------------------------------------------------------------------------ properties
@pytest.mark.parametrize("M", [3, 300])
def test_backward_deterministic_and_empty(M):
    mlp, _ = _build(1024, 2816, 128, torch.float16, act13=True, act2=True, seed=4)
    x, dy = _rand(M, 1024, torch.float16, 1), _rand(M, 1024, torch.float16, 2)
    _, dx1 = _grad(mlp, x, dy)
    _, dx2 = _grad(mlp, x, dy)
    assert torch.equal(dx1, dx2)
    x0 = torch.zeros(0, 1024, dtype=torch.float16, device="cuda", requires_grad=True)
    mlp(x0).sum().backward()
    assert x0.grad.shape == (0, 1024)
    x3 = _rand(2 * 3 * 4, 1024, torch.float16, 5).reshape(2, 3, 4, 1024).requires_grad_(True)   # leading dims kept
    y3 = mlp(x3)
    assert y3.shape == (2, 3, 4, 1024)
    y3.backward(torch.ones_like(y3))
    assert x3.grad.shape == x3.shape


class _Wrap(torch.nn.Module):
    def __init__(self, inner):
        super().__init__()
        self.inner = inner

    def forward(self, x):
        return self.inner(x)


@pytest.mark.parametrize("case", ["I=800", "fp32 x", "wrapped down_proj", "different perms", "forced kernel"])
def test_fallbacks_equal_the_default_path(case):
    from autogptq_b200 import FusedQuantMLP, _lib

    H, I, dtype = 1024, (800 if case == "I=800" else 1536), torch.float16
    mlp, _ = _build(H, I, 32, dtype, act13=case == "different perms", seed=30)
    g, u, d = mlp.gate_proj, mlp.up_proj, mlp.down_proj
    if case == "different perms":
        other = O.random_packed(H, I, 32, seed=99, desc_act=True)
        u = make_layer(other, device="cuda", dtype=dtype)
    if case == "wrapped down_proj":
        d = _Wrap(d)
    if case == "forced kernel":
        g.kernel = _lib.KERNEL_GEMM
    x = _rand(64, H, torch.float32 if case == "fp32 x" else dtype, 5)
    dy = _rand(64, H, x.dtype, 6)
    a, b = FusedQuantMLP(g, u, d, fused_backward=True), FusedQuantMLP(g, u, d)
    ya, dxa = _grad(a, x, dy)
    yb, dxb = _grad(b, x, dy)
    assert torch.equal(ya, yb) and torch.equal(dxa, dxb)


@pytest.mark.parametrize("M", [4, 100])
def test_cuda_graph_forward_backward_and_checkpoint(M):
    mlp, _ = _build(1024, 2816, 128, torch.float16, act13=True, bias=True, seed=5)
    x = _rand(M, 1024, torch.float16, 2).requires_grad_(True)
    dy = _rand(M, 1024, torch.float16, 8)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):                    # warm-up: tensor-core copies, descriptors, workspaces
            x.grad = None
            mlp(x).backward(dy)
    torch.cuda.current_stream().wait_stream(s)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = mlp(x)
        y.backward(dy)
    dx = x.grad
    for r in range(2):
        nx, ndy = _rand(M, 1024, torch.float16, 40 + r), _rand(M, 1024, torch.float16, 50 + r)
        with torch.no_grad():
            x.copy_(nx)
        dy.copy_(ndy)
        graph.replay()
        torch.cuda.synchronize()
        y_e, dx_e = _grad(mlp, nx, ndy)
        assert torch.equal(y, y_e) and torch.equal(dx, dx_e), f"replay {r}"
    # activation checkpointing: the recomputed forward and the backward run on autograd's worker thread
    from torch.utils.checkpoint import checkpoint

    xc = nx.clone().requires_grad_(True)
    checkpoint(mlp, xc, use_reentrant=False).backward(ndy)
    torch.cuda.synchronize()
    assert torch.equal(xc.grad, dx_e)


# ------------------------------------------------------------------------------------------------ training
class _LoRA(torch.nn.Module):
    def __init__(self, base, r, dtype, seed):
        super().__init__()
        gen = torch.Generator().manual_seed(seed)
        self.base = base
        K, N = base.in_features, base.out_features
        self.A = torch.nn.Parameter((torch.randn(r, K, generator=gen) / K ** 0.5).to(dtype).cuda())
        self.B = torch.nn.Parameter((torch.randn(N, r, generator=gen) * 0.05).to(dtype).cuda())

    def forward(self, x):
        return self.base(x) + (x @ self.A.t()) @ self.B.t()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_tiny_llama_lora_training(dtype):
    from transformers import LlamaConfig, LlamaForCausalLM

    from autogptq_b200 import FusedQuantMLP, inject_fused_mlp

    H, I, L = 256, 512, 2
    cfg = LlamaConfig(vocab_size=128, hidden_size=H, intermediate_size=I, num_hidden_layers=L, num_attention_heads=4,
                      num_key_value_heads=2, max_position_embeddings=64)
    torch.manual_seed(0)
    model = LlamaForCausalLM(cfg).to(dtype).cuda()
    model.requires_grad_(False)
    seed = 200
    for layer in model.model.layers:          # frozen 4-bit MLPs, rank-8 adapters on the attention's q and v
        for n in ("gate_proj", "up_proj", "down_proj"):
            lin = getattr(layer.mlp, n)
            seed += 1
            d = O.random_packed(lin.in_features, lin.out_features, 64, seed=seed, desc_act=n == "down_proj")
            setattr(layer.mlp, n, make_layer(d, device="cuda", dtype=dtype))
        for n in ("q_proj", "v_proj"):
            seed += 1
            setattr(layer.self_attn, n, _LoRA(getattr(layer.self_attn, n), 8, dtype, seed))
    assert inject_fused_mlp(model, fused_backward=True) == L
    mlps = [m for m in model.modules() if isinstance(m, FusedQuantMLP)]
    params = [p for p in model.parameters() if p.requires_grad]
    assert len(params) == 4 * L
    ids = torch.from_numpy(np.random.default_rng(1).integers(0, 128, (2, 32))).cuda()

    def grads(fused):
        for m in mlps:
            m.fused_backward = fused
        for p in params:
            p.grad = None
        model(input_ids=ids, labels=ids).loss.backward()
        return [p.grad.float().flatten() for p in params]

    fused, default = grads(True), grads(False)
    rel_max, cos_min = (0.03, 0.999) if dtype == torch.float16 else (0.12, 0.99)
    for i, (a, b) in enumerate(zip(fused, default)):
        assert torch.isfinite(a).all() and a.abs().max() > 0
        rel = float((a - b).norm() / b.norm())
        cos = float(F.cosine_similarity(a, b, dim=0))
        assert rel < rel_max and cos > cos_min, f"adapter param {i}: rel {rel:.4f} cos {cos:.5f}"
    for m in mlps:
        m.fused_backward = True
    opt = torch.optim.SGD(params, lr=0.5)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        loss = model(input_ids=ids, labels=ids).loss
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < losses[0], losses


def test_report():
    """Largest err/bound and mismatch rate over this module's bound checks (the DESIGN §3.12 row)."""
    if not REPORT:
        pytest.skip("no bound check ran")
    for dt in ("float16", "bfloat16"):
        rows = {k: v for k, v in REPORT.items() if ("bfloat16" in k) == (dt == "bfloat16")}
        if rows:
            print(f"[mlp-grad] {dt}: max dx err/bound {max(v[0] for v in rows.values()):.3f}, max mismatch "
                  f"{100 * max(v[1] for v in rows.values()):.2f} %")
