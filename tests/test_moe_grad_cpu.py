"""CPU tests of the grouped experts' backward: the float64 reference (tests/_moe_grad.py) against torch.autograd through
a transformers-style loop, the new C-ABI exports, and the ``input_grad`` switch of QuantExperts / group_experts."""
import numpy as np
import pytest
import torch

from autogptq_b200 import QuantExperts, QuantLinear, group_experts
from autogptq_b200 import _lib
from oracle import w4a16_oracle as O
from tests import _moe_grad as MG


def _experts(E, H, I, g, seed=0, desc_act13=False, desc_act2=False, bias=False):
    out = []
    for e in range(E):
        ex = {}
        for j, (name, K, N) in enumerate((("w1", H, I), ("w3", H, I), ("w2", I, H))):
            act = desc_act2 if name == "w2" else desc_act13
            d = O.random_packed(K, N, g, seed=seed + 3 * e + j, desc_act=act, bias=bias)
            if name == "w3" and act:
                d["g_idx"] = ex["w1"]["g_idx"]
            ex[name] = d
        out.append(ex)
    return out


def _autograd_loop(x, experts, idx, w, dy):
    """MixtralExperts.forward (modeling_mixtral.py:74-98) in float64 over the weights the backward uses (each rounded
    once to fp16, no other rounding), differentiated by torch.autograd."""
    E = len(experts)
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    wt = torch.tensor(w, dtype=torch.float64, requires_grad=True)
    it = torch.tensor(idx)
    final = torch.zeros_like(xt)
    mask = torch.nn.functional.one_hot(it, num_classes=E + 1).permute(2, 1, 0)
    for e in torch.greater(mask.sum(dim=(-1, -2)), 0).nonzero().flatten().tolist():
        if e == E:
            continue
        slot, tok = torch.where(mask[e])
        ex = experts[e]
        W1, W3, W2 = (torch.from_numpy(MG.dequant(ex[n], "float16", True)) for n in ("w1", "w3", "w2"))
        b = {n: torch.from_numpy(MG._bias(ex[n], W.shape[1])) for n, W in (("w1", W1), ("w3", W3), ("w2", W2))}
        h = torch.nn.functional.silu(xt[tok] @ W1 + b["w1"]) * (xt[tok] @ W3 + b["w3"])
        final.index_add_(0, tok, (h @ W2 + b["w2"]) * wt[tok, slot, None])
    dx, dw = torch.autograd.grad(final, (xt, wt), torch.tensor(dy, dtype=torch.float64))
    return dx.numpy(), dw.numpy()


@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("desc_act13,desc_act2,bias", [(False, False, False), (True, False, True), (False, True, False),
                                                       (True, True, True)])
def test_oracle_matches_autograd(k, desc_act13, desc_act2, bias):
    E, H, I, T = 4, 128, 256, 11
    experts = _experts(E, H, I, 64, seed=k, desc_act13=desc_act13, desc_act2=desc_act2, bias=bias)
    rng = np.random.default_rng(k)
    idx = np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)
    idx[rng.random(idx.shape) < 0.25] = E                                   # the `expert_idx == num_experts` skip
    w = rng.random((T, k))
    x = rng.standard_normal((T, H))
    dy = rng.standard_normal((T, H))
    ref = MG.backward(x, experts, idx, w, dy, rounded=False)
    dx, dw = _autograd_loop(x, experts, idx, w, dy)
    np.testing.assert_allclose(ref["dx"], dx, rtol=1e-9, atol=1e-12 * np.abs(dx).max())
    np.testing.assert_allclose(ref["dw"], dw, rtol=1e-9, atol=1e-12 * np.abs(dw).max())
    assert not ref["dw"][idx == E].any()
    # the rounded reference stays within a few fp16 ulps of the exact one (the rounding points are where stated)
    rr = MG.backward(x, experts, idx, w, dy, rounded=True)
    assert np.abs(rr["dx"] - dx).max() <= 0.02 * np.abs(dx).max()


def test_new_exports_are_bound():
    names = set(_lib.declared_symbols())
    for n in ("agb200_moe_saved_bytes", "agb200_moe_forward_saving", "agb200_moe_grad_plan_bytes", "agb200_moe_grad_attach",
              "agb200_moe_backward_workspace_bytes", "agb200_moe_backward"):
        assert n in names
    lib = _lib.load()
    E, H, I = 8, 4096, 14336
    assert lib.agb200_moe_saved_bytes(5, 2, E, H, I) == 2 * 10 * I * 2 + 10 * H * 2
    assert lib.agb200_moe_saved_bytes(0, 2, E, H, I) == 0
    assert lib.agb200_moe_grad_plan_bytes(E, H, I, 128) > 0
    assert lib.agb200_moe_backward(None, None, None, 0, None, 0, 1, 1, None, 0, None, None, None, 0, None) != 0   # bad handle


def _lin(K, N, g=64):
    return QuantLinear(4, g, K, N, False)


def test_input_grad_plumbs_through_group_experts():
    layers = {f"m.experts.{e}.{n}": _lin(*s) for e in range(2) for n, s in (("w1", (128, 256)), ("w3", (128, 256)),
                                                                             ("w2", (256, 128)))}
    assert group_experts(layers)["m.experts"].input_grad is False
    qe = group_experts(layers, input_grad=True)["m.experts"]
    assert isinstance(qe, QuantExperts) and qe.input_grad is True
    assert "input_grad=True" in repr(qe)
    assert QuantExperts.from_linears([_lin(128, 256)], [_lin(128, 256)], [_lin(256, 128)], input_grad=True).input_grad


def test_default_still_refuses_grad_mode():
    qe = QuantExperts.from_linears([_lin(128, 256)], [_lin(128, 256)], [_lin(256, 128)])
    x = torch.zeros(3, 128, dtype=torch.float16, requires_grad=True)
    with pytest.raises((NotImplementedError, RuntimeError)) as ei:
        qe(x, torch.zeros(3, 1, dtype=torch.int64), torch.ones(3, 1))
    # on a CPU tensor the device check comes first; on CUDA tensors the grad-mode refusal is pinned by the GPU suite
    assert "no CPU fallback" in str(ei.value) or "inference-only" in str(ei.value)
