"""GPU tests of the grouped experts' backward (``QuantExperts(input_grad=True)``, ``agb200_moe_backward``).

Error bound of dx and dw against the float64 reference of ``tests/_moe_grad.py`` (same rounding points, weights rounded
once to the dtype as the tensor-core dgrad forms them):

    |dx − dx*| ≤ ulp(dx*) + (γ + ε)·(A + A2)          |dw − dw*| ≤ ulp_w(dw*) + γ·A_dw

* ulp(dx*): the final rounding of the slot sum (half an ulp) plus the room the accumulated error gives it to round the
  other way (``tests/_precision.py``).
* A = Σ_j Σ_i |dg_i|·|W1[c, i]| + |du_i|·|W3[c, i]| is the uncancelled magnitude of the gate/up reduction (one fp32 sum
  over 2·I terms, then k slot terms).  A2 = Σ_j Σ_i (A_dh,i·|u_i·silu′(g_i)|)·|W1[c, i]| + (A_dh,i·|silu(g_i)|)·|W3[c, i]|,
  A_dh = |dy_pair|·|W2|ᵀ, carries the accumulation error of the unrounded dh through dg and du into dx.
* γ = TC_GAMMA·λ·√(n/4 + 64)·2⁻²⁴ with n = max(2·I, H): the probabilistic fp32 accumulation bound of the tensor-core paths
  (``tests/_precision.py``; both reductions run on wgmma).
* ε = one 16-bit ulp relative to a value (2⁻¹⁰ fp16, 2⁻⁷ bf16).  Every dy_pair, dg and du is a rounded operand whose last
  bit can legitimately differ from the reference's: its inputs (the unrounded dh, and g, u, y_pair saved by a forward
  whose sums ran in a different order) carry their own fp32 error, so a rounding may fall the other way.  One ulp of
  every such operand moves dx by at most ε·(A + A2).
* dw: dw* = Σ_n dy·y_pair over the y_pair the saving forward kept (a second saving forward on the same inputs: the
  forward is deterministic), so no operand rounding is excused; A_dw = Σ_n |dy·y_pair|, the sum is fp32 over H terms
  (γ·A_dw); ulp_w is the rounding to w's dtype (fp32: 2⁻²³ relative).

Besides the bound, the mismatch rate (share of dx elements that differ from round(dx*)) is reported; the largest
err/bound and rate measured on the H100 are recorded in DESIGN §3.12."""
import numpy as np
import pytest
import torch

from oracle import w4a16_oracle as O
from tests import _moe_grad as MG
from tests._precision import PATHS, gamma, ulp
from tests._util import assert_parity, make_layer

pytestmark = pytest.mark.gpu

E = 8
DT = {torch.float16: "float16", torch.bfloat16: "bfloat16"}
EPS = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}
TOL = {torch.float16: dict(rtol=1e-3, atol_rms=1.6e-3), torch.bfloat16: dict(rtol=8e-3, atol_rms=4e-3)}
REPORT = {}


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _build(H, I, g, dtype, act13=False, act2=False, bias=False, seed=0, n_experts=E):
    """(QuantExperts(input_grad=True), reference experts with the scales / bias the device uses)."""
    from autogptq_b200 import QuantExperts

    mods = {"w1": [], "w3": [], "w2": []}
    ref = []
    for e in range(n_experts):
        ex = {}
        for j, (name, K, N) in enumerate((("w1", H, I), ("w3", H, I), ("w2", I, H))):
            act = act2 if name == "w2" else act13
            d = O.random_packed(K, N, g, seed=seed + 3 * e + j, desc_act=act, bias=bias)
            if name == "w3" and act:
                d["g_idx"] = ex["w1"]["g_idx"]
            lin = make_layer(d, device="cuda", dtype=dtype)
            mods[name].append(lin)
            ex[name] = dict(d, scales=lin.scales.float().cpu().numpy(),
                            bias=None if lin.bias is None else lin.bias.float().cpu().numpy())
        ref.append(ex)
    return QuantExperts.from_linears(mods["w1"], mods["w3"], mods["w2"], input_grad=True), ref


def _routing(T, k, seed, n_experts=E):
    rng = np.random.default_rng(seed)
    idx = np.stack([rng.permutation(n_experts)[:k] for _ in range(T)]).astype(np.int64)
    w = rng.random((T, k)).astype(np.float32)
    return idx, w / w.sum(axis=1, keepdims=True)


def _rand(T, H, dtype, seed):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((T, H)).astype(np.float32)).to(dtype).cuda()


def _run(qe, x, idx, w, dy, w_dtype=torch.float32):
    """(out, dx, dw) of one forward + backward through autograd."""
    xg = x.clone().requires_grad_(True)
    wg = torch.as_tensor(w).to(w_dtype).cuda().requires_grad_(True)
    out = qe(xg, torch.as_tensor(idx).cuda(), wg)
    out.backward(dy)
    torch.cuda.synchronize()
    return out.detach(), xg.grad, wg.grad


def _dw_from_saved(qe, x, idx, w, w_dtype, dy):
    """dw* = Σ_n dy·y_pair and A_dw = Σ_n |dy·y_pair| in float64, from the y_pair a saving forward on the same inputs
    keeps (the backward reads exactly those; the forward is deterministic), 0 for ids outside [0, E)."""
    T, k = np.asarray(idx).shape
    H, E = qe.hidden_size, qe.num_experts
    with torch.no_grad():
        _, saved = qe._forward(x.contiguous(), torch.as_tensor(idx).cuda(), torch.as_tensor(w).to(w_dtype).cuda(),
                               save=True)
    gu = -(-T * k * qe.intermediate_size * 2 // 256) * 256
    y = saved[2 * gu:2 * gu + T * k * H * 2].view(x.dtype).view(T, k, H).double().cpu().numpy()
    valid = (np.asarray(idx) >= 0) & (np.asarray(idx) < E)
    with np.errstate(invalid="ignore", over="ignore"):
        terms = np.where(valid[..., None], y, 0.0) * dy.double().cpu().numpy()[:, None, :]
    return terms.sum(axis=2), np.abs(terms).sum(axis=2)


def _check(qe, ref, x, idx, w, dy, dtype, what, w_dtype=torch.float32, cols=None):
    out, dx, dw = _run(qe, x, idx, w, dy, w_dtype)
    assert dx.dtype == dtype and dw.dtype == w_dtype
    T = x.shape[0]
    wv = torch.as_tensor(w).to(w_dtype).float().numpy()
    r = MG.backward(x.float().cpu().numpy(), ref, idx, wv, dy.float().cpu().numpy(), DT[dtype], round_w_fwd=T > 8,
                    w16=w_dtype != torch.float32, cols=cols)
    I, H = qe.intermediate_size, qe.hidden_size
    gam = gamma(PATHS["dgrad"], max(2 * I, H))
    dxv = dx.float().cpu().numpy()
    if cols is not None:
        dxv = dxv[:, cols]
    err = np.abs(dxv - r["dx"])
    bound = ulp(r["dx"], DT[dtype]) + (gam + EPS[dtype]) * (r["A"] + r["A2"])
    worst = float((err / bound).max())
    rate = float((dxv != r["dx"]).mean())
    dwv = dw.float().cpu().numpy()
    dw_ref, A_dw = _dw_from_saved(qe, x, idx, w, w_dtype, dy)
    ulp_w = np.abs(dw_ref) * 2.0 ** -23 if w_dtype == torch.float32 else ulp(dw_ref, DT[dtype])
    werr = np.abs(dwv - dw_ref)
    wbound = ulp_w + gamma(PATHS["dgrad"], H) * A_dw + 1e-30
    wworst = float((werr / wbound).max())
    REPORT[what] = (worst, rate, wworst)
    print(f"[moe-grad] {what}: dx err/bound {worst:.3f} mismatch {100 * rate:.2f} %  dw err/bound {wworst:.3f}")
    assert np.isfinite(dxv).all() and np.isfinite(dwv).all()
    assert worst <= 1.0, f"{what}: dx err/bound {worst:.3f}"
    assert wworst <= 1.0, f"{what}: dw err/bound {wworst:.3f}"
    assert not dwv[np.asarray(idx) >= E].any()


@pytest.mark.parametrize("T", [1, 5, 8, 9, 333, 2048])
@pytest.mark.parametrize("k", [1, 2])
def test_grad_parity_fp16_g128(T, k):
    _need_gpu()
    qe, ref = _build(1024, 2816, 128, torch.float16, seed=k)
    idx, w = _routing(T, k, seed=T)
    _check(qe, ref, _rand(T, 1024, torch.float16, T), idx, w, _rand(T, 1024, torch.float16, T + 50), torch.float16,
           f"T={T} k={k}")


@pytest.mark.parametrize("T", [5, 333])
@pytest.mark.parametrize("g,act13,act2,bias", [(-1, False, False, True), (32, True, False, False), (128, True, True, True),
                                               (128, False, True, False)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("w16", [False, True])
def test_grad_parity_configs(T, g, act13, act2, bias, dtype, w16):
    _need_gpu()
    qe, ref = _build(1024, 1536, g, dtype, act13=act13, act2=act2, bias=bias, seed=7)
    idx, w = _routing(T, 2, seed=100 + T)
    _check(qe, ref, _rand(T, 1024, dtype, T), idx, w, _rand(T, 1024, dtype, T + 9), dtype,
           f"T={T} g={g} act={act13}/{act2} bias={bias} {DT[dtype]} w16={w16}", w_dtype=dtype if w16 else torch.float32)


@pytest.mark.parametrize("T", [6, 300])
def test_grad_skewed_routing(T):
    _need_gpu()
    qe, ref = _build(1024, 2816, 128, torch.float16, bias=True, seed=3)
    x, dy = _rand(T, 1024, torch.float16, T), _rand(T, 1024, torch.float16, T + 1)
    rng = np.random.default_rng(T)
    w = rng.random((T, 2)).astype(np.float32)
    idx = np.stack([np.full(T, 5), np.full(T, E)], axis=1)            # one expert, slot 1 skipped
    _check(qe, ref, x, idx, w, dy, torch.float16, f"one expert T={T}")
    idx, w = _routing(T, 2, seed=T + 1)
    idx[rng.random(idx.shape) < 0.3] = E                             # a sprinkling of id E
    _check(qe, ref, x, idx.astype(np.int32), w, dy, torch.float16, f"ids == E T={T}")


@pytest.fixture(scope="module")
def mixtral_experts():
    _need_gpu()
    return _build(4096, 14336, 128, torch.float16, seed=11)


@pytest.mark.parametrize("T", [8, 64])
def test_grad_parity_mixtral_size(T, mixtral_experts):
    qe, ref = mixtral_experts
    idx, w = _routing(T, 2, seed=T)
    cols = np.r_[0:256, 4096 - 256:4096]
    _check(qe, ref, _rand(T, 4096, torch.float16, T), idx, w, _rand(T, 4096, torch.float16, T + 3), torch.float16,
           f"Mixtral size T={T}", cols=cols)


@pytest.mark.parametrize("T", [5, 300])
def test_grad_mode_forward_is_bit_identical(T):
    _need_gpu()
    qe, _ = _build(1024, 2816, 128, torch.float16, act13=True, act2=True, bias=True, seed=4)
    idx, w = _routing(T, 2, seed=T)
    x, xi, wt = _rand(T, 1024, torch.float16, 1), torch.as_tensor(idx).cuda(), torch.as_tensor(w).cuda()
    with torch.no_grad():
        a = qe(x, xi, wt)
    b = qe(x.clone().requires_grad_(True), xi, wt.clone().requires_grad_(True))
    assert b.grad_fn is not None
    assert torch.equal(a, b.detach())
    # only the routing weights need a gradient: same output, dx not computed
    c = qe(x, xi, wt.clone().requires_grad_(True))
    assert torch.equal(a, c.detach())


@pytest.mark.parametrize("T", [3, 300])
def test_backward_deterministic(T):
    _need_gpu()
    qe, _ = _build(1024, 2816, 128, torch.float16, act13=True, seed=4)
    idx, w = _routing(T, 2, seed=T)
    x, dy = _rand(T, 1024, torch.float16, 1), _rand(T, 1024, torch.float16, 2)
    _, dx1, dw1 = _run(qe, x, idx, w, dy)
    _, dx2, dw2 = _run(qe, x, idx, w, dy)
    assert torch.equal(dx1, dx2) and torch.equal(dw1, dw2)
    # dw alone (x without grad) gives the same dw
    wg = torch.as_tensor(w).cuda().requires_grad_(True)
    qe(x, torch.as_tensor(idx).cuda(), wg).backward(dy)
    assert torch.equal(wg.grad, dw1)


def test_fp32_inputs_get_fp32_gradients_and_empty_batch():
    _need_gpu()
    qe, _ = _build(1024, 2816, 128, torch.float16, seed=6, n_experts=4)
    idx, w = _routing(7, 2, seed=1, n_experts=4)
    x = _rand(7, 1024, torch.float32, 3).requires_grad_(True)
    wt = torch.as_tensor(w).cuda().requires_grad_(True)
    qe(x, torch.as_tensor(idx).cuda(), wt).sum().backward()
    assert x.grad.dtype == torch.float32 and wt.grad.dtype == torch.float32
    x0 = torch.zeros(0, 1024, dtype=torch.float16, device="cuda", requires_grad=True)
    w0 = torch.zeros(0, 2, device="cuda", requires_grad=True)
    y0 = qe(x0, torch.zeros(0, 2, dtype=torch.int64, device="cuda"), w0)
    y0.sum().backward()
    assert x0.grad.shape == (0, 1024) and w0.grad.shape == (0, 2)


def _loop(qe, x, xi, wt):
    """MixtralExperts.forward (modeling_mixtral.py) over the same QuantLinear modules, which backpropagate themselves."""
    T, H = x.shape
    final = torch.zeros(T, H, dtype=torch.float32, device="cuda")
    mask = torch.nn.functional.one_hot(xi, num_classes=qe.num_experts + 1).permute(2, 1, 0)
    for e in torch.greater(mask.sum(dim=(-1, -2)), 0).nonzero().flatten().tolist():
        if e == qe.num_experts:
            continue
        slot, tok = torch.where(mask[e])
        h = torch.nn.functional.silu(qe.w1[e](x[tok])) * qe.w3[e](x[tok])
        final = final.index_add(0, tok, qe.w2[e](h).float() * wt[tok, slot, None])
    return final.to(x.dtype)


@pytest.mark.parametrize("T", [2, 50])
def test_matches_per_expert_quantlinear_loop_backward(T):
    _need_gpu()
    qe, _ = _build(1024, 2816, 128, torch.float16, act13=True, bias=True, seed=9)
    idx, w = _routing(T, 2, seed=T)
    x, dy, xi = _rand(T, 1024, torch.float16, 1), _rand(T, 1024, torch.float16, 5), torch.as_tensor(idx).cuda()
    grads = []
    for fn in (qe, lambda a, b, c: _loop(qe, a, b, c)):
        xg = x.clone().requires_grad_(True)
        wg = torch.as_tensor(w).cuda().requires_grad_(True)
        fn(xg, xi, wg).backward(dy)
        grads.append((xg.grad.float().cpu().numpy(), wg.grad.float().cpu().numpy()))
    torch.cuda.synchronize()
    # the loop rounds dh, the w1 and w3 input gradients of every slot and their running sum to fp16 where the grouped
    # backward keeps one fp32 sum: one ulp of each of those 2k + 1 partials is excused before the MoE tolerance (as
    # _assert_moe of test_gpu_10_moe does for y_pair).  A partial is bounded by |dx| plus the spread that cancels in the
    # sum, taken as rms(dx) per partial.
    ref = grads[1][0]
    mag = np.abs(ref) + (2 * 2 + 1) * np.sqrt(np.mean(ref.astype(np.float64) ** 2))
    err = grads[0][0] - ref
    excused = np.sign(err) * np.maximum(np.abs(err) - 2.0 ** -10 * mag, 0)
    assert_parity(grads[1][0] + excused, grads[1][0], what=f"dx vs loop T={T}", **TOL[torch.float16])
    assert_parity(grads[0][1], grads[1][1], what=f"dw vs loop T={T}", **TOL[torch.float16])


@pytest.mark.parametrize("T", [4, 100])
def test_cuda_graph_forward_backward_replay(T):
    _need_gpu()
    qe, ref = _build(1024, 2816, 128, torch.float16, seed=5)
    x = _rand(T, 1024, torch.float16, 2).requires_grad_(True)
    dy = _rand(T, 1024, torch.float16, 8)
    idx0, w0 = _routing(T, 2, seed=0)
    xi, wt = torch.as_tensor(idx0).cuda(), torch.as_tensor(w0).cuda().requires_grad_(True)

    def step():
        x.grad, wt.grad = None, None
        qe(x, xi, wt).backward(dy)
        return x.grad, wt.grad

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                            # warm-up: plans, tensor-core copies, grad plan, workspaces
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    x.grad, wt.grad = None, None
    with torch.cuda.graph(graph):
        dx, dw = step()
    for r in range(3):
        idx, w = _routing(T, 2, seed=10 + r)
        if r == 2:
            idx[:, 1] = E                 # half the slots skipped
        xi.copy_(torch.as_tensor(idx))
        with torch.no_grad():
            wt.copy_(torch.as_tensor(w))
        graph.replay()
        torch.cuda.synchronize()
        want = MG.backward(x.detach().float().cpu().numpy(), ref, idx, w, dy.float().cpu().numpy(), "float16",
                           round_w_fwd=T > 8)
        assert_parity(dx.float().cpu().numpy(), want["dx"], what=f"graph replay {r} dx", **TOL[torch.float16])
        assert_parity(dw.float().cpu().numpy(), want["dw"], what=f"graph replay {r} dw", **TOL[torch.float16])


class _LoopExperts(torch.nn.Module):
    def __init__(self, qe):
        super().__init__()
        self.qe = qe

    def forward(self, hidden_states, top_k_index, top_k_weights):
        return _loop(self.qe, hidden_states, top_k_index, top_k_weights)


class _LoRA(torch.nn.Module):
    def __init__(self, base, r=8, seed=0):
        super().__init__()
        self.base = base
        g = torch.Generator().manual_seed(seed)
        self.A = torch.nn.Parameter(torch.randn(r, base.in_features, generator=g) * 0.02)
        self.B = torch.nn.Parameter(torch.randn(base.out_features, r, generator=g) * 0.02)

    def forward(self, x):
        return self.base(x) + (x @ self.A.to(x.dtype).t()) @ self.B.to(x.dtype).t()


def test_tiny_mixtral_lora_backward():
    _need_gpu()
    from transformers import MixtralConfig, MixtralForCausalLM
    from transformers.models.mixtral.modeling_mixtral import MixtralSparseMoeBlock

    H, I, L = 256, 512, 2
    cfg = MixtralConfig(vocab_size=128, hidden_size=H, intermediate_size=I, num_hidden_layers=L, num_attention_heads=4,
                        num_key_value_heads=2, num_local_experts=4, num_experts_per_tok=2, max_position_embeddings=64)
    torch.manual_seed(0)
    grads = []
    for use_grouped in (True, False):
        torch.manual_seed(0)
        model = MixtralForCausalLM(cfg).to(torch.float16).cuda()
        model.requires_grad_(False)
        blocks = [m for m in model.modules() if isinstance(m, MixtralSparseMoeBlock)]
        assert len(blocks) == L
        for b, blk in enumerate(blocks):
            qe, _ = _build(H, I, 64, torch.float16, seed=100 * b, n_experts=4)
            blk.experts = qe if use_grouped else _LoopExperts(qe)
        for i, layer in enumerate(model.model.layers):
            layer.self_attn.q_proj = _LoRA(layer.self_attn.q_proj, seed=i).cuda()
        ids = torch.from_numpy(np.random.default_rng(1).integers(0, 128, (2, 24))).cuda()
        loss = model(input_ids=ids, labels=ids).loss
        loss.backward()
        grads.append([p.grad.float().cpu().numpy() for n, p in model.named_parameters() if p.requires_grad])
    assert len(grads[0]) == 2 * L
    for a, b in zip(*grads):
        assert np.isfinite(a).all() and np.abs(a).max() > 0
        assert_parity(a, b, what="adapter gradient", rtol=2e-2, atol_rms=2e-2)


def test_report():
    """Largest err/bound and mismatch rate over this module's parity checks (the DESIGN §3.12 row)."""
    if not REPORT:
        pytest.skip("no parity check ran")
    for dt in ("float16", "bfloat16"):
        rows = {k: v for k, v in REPORT.items() if ("bfloat16" in k) == (dt == "bfloat16")}
        if rows:
            print(f"[moe-grad] {dt}: max dx err/bound {max(v[0] for v in rows.values()):.3f}, max mismatch "
                  f"{100 * max(v[1] for v in rows.values()):.2f} %, max dw err/bound {max(v[2] for v in rows.values()):.3f}")
