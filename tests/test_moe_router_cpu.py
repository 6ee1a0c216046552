"""CPU checks of the MoE router's model and host side: the float64 reference against transformers' MixtralTopKRouter,
MixtralRMSNorm against LlamaRMSNorm, ChainDecoder's refusals of MoE blocks it cannot run, and the C ABI exports."""
import os
import re

import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from oracle import w4a16_oracle as O
from tests import _moe_router as R
from tests._precision import dt_name
from tests._util import make_layer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTS = [torch.float16, torch.bfloat16]


def _mixtral_config(**kw):
    from transformers import MixtralConfig

    base = dict(vocab_size=64, hidden_size=256, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2,
                num_key_value_heads=2, num_local_experts=4, num_experts_per_tok=2, max_position_embeddings=128)
    base.update(kw)
    return MixtralConfig(**base)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("E,k", [(8, 2), (16, 4), (64, 1)])
def test_reference_matches_transformers_router(E, k, dtype):
    """MixtralTopKRouter on CPU tensors: its logits are candidates of the reference's, and its indices and weights
    pass the reference checks on those logits (softmax of the rounded logits, top-k, renormalised)."""
    from transformers.models.mixtral.modeling_mixtral import MixtralTopKRouter

    router = MixtralTopKRouter(_mixtral_config(num_local_experts=E, num_experts_per_tok=k)).to(dtype)
    g = torch.Generator().manual_seed(E + k)
    with torch.no_grad():
        router.weight.copy_(torch.randn(E, 256, generator=g) * 0.05)
    n = torch.randn(16, 256, generator=g).to(dtype)
    n[:, :3] *= 30                                            # a few massive channels
    with torch.no_grad():
        probs, w, idx = router(n)
        logits = torch.nn.functional.linear(n, router.weight)
    nd, G, l = n.double().numpy(), router.weight.detach().double().numpy(), logits.double().numpy()
    R.check_logits(l, nd, G, dt_name(dtype), "CPU F.linear")
    np.testing.assert_allclose(probs.double().numpy(), R.softmax64(l), rtol=0, atol=1e-6)
    R.check_topk(idx.numpy(), l, k, "MixtralTopKRouter")
    R.check_weights(w.numpy(), idx.numpy(), l, "MixtralTopKRouter")
    ml, _, _, mw = R.router_model(nd, G, k, dt_name(dtype))
    R.check_logits(ml, nd, G, dt_name(dtype), "model")
    R.check_weights(mw.astype(np.float32), R.topk_ref(R.softmax64(ml), k), ml, "model")


def test_weight_check_rejects_unnormalised_weights():
    """Top-k probabilities without the renormalisation (Qwen2-MoE's norm_topk_prob=False) fail the weight check."""
    l = np.array([[1.0, 0.5, -0.25, 2.0, 0.0, -1.0, 0.75, 0.125]])
    idx = R.topk_ref(R.softmax64(l), 2)
    raw = np.take_along_axis(R.softmax64(l), idx, -1)
    with pytest.raises(AssertionError):
        R.check_weights(raw.astype(np.float32), idx, l)
    R.check_weights((raw / raw.sum()).astype(np.float32), idx, l)


def test_topk_check_resolves_ties_to_the_lower_index():
    l = np.array([[0.5, 2.0, 2.0, 1.0]])
    R.check_topk(np.array([[1, 2]]), l, 2)
    R.check_topk(np.array([[1]]), l, 1)
    with pytest.raises(AssertionError):
        R.check_topk(np.array([[2, 1]]), l, 2)
    with pytest.raises(AssertionError):
        R.check_topk(np.array([[2]]), l, 1)
    with pytest.raises(AssertionError):
        R.check_topk(np.array([[1, 3]]), l, 2)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_mixtral_rmsnorm_equals_llama_rmsnorm(dtype):
    from transformers.models.llama.modeling_llama import LlamaRMSNorm
    from transformers.models.mixtral.modeling_mixtral import MixtralRMSNorm

    from autogptq_b200.decoder import _RMSNORMS, _norm_of

    g = torch.Generator().manual_seed(11)
    a, b = MixtralRMSNorm(1024, eps=1e-5).to(dtype), LlamaRMSNorm(1024, eps=1e-5).to(dtype)
    with torch.no_grad():
        w = (torch.rand(1024, generator=g) + 0.5).to(dtype)
        a.weight.copy_(w)
        b.weight.copy_(w)
        x = (torch.randn(8, 1024, generator=g) * 3).to(dtype)
        x[:, :4] *= 200
        assert torch.equal(a(x).view(torch.int16), b(x).view(torch.int16))
    assert "MixtralRMSNorm" in _RMSNORMS
    assert _norm_of(a, "n")[1] == 1e-5


# --------------------------------------------------------------------------- ChainDecoder's refusals
def _quant(K, N, seed):
    return make_layer(O.random_packed(K, N, 128, seed=seed), device="cpu", dtype=torch.float16)


def _experts(H, I, E, seed=0):
    from autogptq_b200 import QuantExperts

    return QuantExperts([_quant(H, I, seed + 3 * e) for e in range(E)], [_quant(H, I, seed + 3 * e + 1) for e in range(E)],
                        [_quant(I, H, seed + 3 * e + 2) for e in range(E)])


def _cpu_mixtral(**kw):
    """A CPU MixtralForCausalLM whose attention projections are QuantLinear and whose experts are QuantExperts."""
    from transformers import MixtralForCausalLM

    cfg = _mixtral_config(**kw)
    m = MixtralForCausalLM(cfg).half().eval()
    for i, layer in enumerate(m.model.layers):
        at = layer.self_attn
        for j, name in enumerate(("q_proj", "k_proj", "v_proj", "o_proj")):
            lin = getattr(at, name)
            setattr(at, name, _quant(lin.in_features, lin.out_features, 100 * i + j))
        layer.mlp.experts = _experts(cfg.hidden_size, cfg.intermediate_size, cfg.num_local_experts, 1000 * i)
    return m


def _plan(model, i=0):
    from autogptq_b200.decoder import _plan_layer

    return _plan_layer(i, model.model.layers[i], 1, torch.float16)


def test_plan_layer_accepts_a_mixtral_block():
    from autogptq_b200.decoder import _is_moe

    m = _cpu_mixtral()
    plans = [_plan(m, i) for i in range(2)]
    gate_w, k, experts = plans[0][4]
    assert tuple(gate_w.shape) == (4, 256) and k == 2 and experts is m.model.layers[0].mlp.experts
    assert _is_moe(plans)


def test_refuses_ungrouped_experts():
    from transformers.models.mixtral.modeling_mixtral import MixtralExperts

    m = _cpu_mixtral()
    m.model.layers[0].mlp.experts = MixtralExperts(m.config).half()
    with pytest.raises(NotImplementedError, match=r"model\.layers\.0\.mlp\.experts is MixtralExperts.*group_experts"):
        _plan(m)


def test_refuses_qwen2_moe_block():
    from transformers import Qwen2MoeConfig
    from transformers.models.qwen2_moe.modeling_qwen2_moe import Qwen2MoeSparseMoeBlock

    m = _cpu_mixtral()
    cfg = Qwen2MoeConfig(hidden_size=256, moe_intermediate_size=256, shared_expert_intermediate_size=256,
                         num_experts=4, num_experts_per_tok=2, num_attention_heads=2, num_key_value_heads=2)
    m.model.layers[0].mlp = Qwen2MoeSparseMoeBlock(cfg).half()
    with pytest.raises(NotImplementedError, match=r"model\.layers\.0\.mlp is Qwen2MoeSparseMoeBlock"):
        _plan(m)


def test_refuses_other_router():
    m = _cpu_mixtral()
    m.model.layers[0].mlp.gate = torch.nn.Linear(256, 4, bias=False).half()
    with pytest.raises(NotImplementedError, match=r"model\.layers\.0\.mlp\.gate is Linear"):
        _plan(m)


@pytest.mark.parametrize("change,match", [
    (lambda g: setattr(g, "top_k", 9), "top_k 9"),
    (lambda g: setattr(g, "weight", torch.nn.Parameter(g.weight.detach().float())), r"weight is torch\.float32"),
    (lambda g: setattr(g, "weight", torch.nn.Parameter(g.weight.detach()[:, :128].contiguous())), r"shape \(4, 128\)"),
], ids=["top_k", "dtype", "shape"])
def test_refuses_router_outside_the_kernel(change, match):
    m = _cpu_mixtral()
    change(m.model.layers[0].mlp.gate)
    with pytest.raises(NotImplementedError, match=r"model\.layers\.0\.mlp\.gate.*" + match):
        _plan(m)


def test_refuses_experts_of_another_shape():
    m = _cpu_mixtral()
    m.model.layers[0].mlp.experts = _experts(256, 256, 8)
    with pytest.raises(NotImplementedError, match=r"model\.layers\.0\.mlp\.experts has 8 experts"):
        _plan(m)


def test_refuses_mixed_dense_and_moe_layers():
    from transformers import LlamaConfig, LlamaForCausalLM

    from autogptq_b200.decoder import _is_moe

    m = _cpu_mixtral()
    llama = LlamaForCausalLM(LlamaConfig(hidden_size=256, intermediate_size=256, num_attention_heads=2,
                                         num_key_value_heads=2, num_hidden_layers=1, vocab_size=64)).half()
    dense = llama.model.layers[0]
    for j, name in enumerate(("q_proj", "k_proj", "v_proj", "o_proj")):
        setattr(dense.self_attn, name, _quant(256, 256, 500 + j))
    for j, name in enumerate(("gate_proj", "up_proj", "down_proj")):
        setattr(dense.mlp, name, _quant(256, 256, 600 + j))
    m.model.layers[1] = dense
    plans = [_plan(m, 0), _plan(m, 1)]
    with pytest.raises(NotImplementedError, match=r"model\.layers\.1\.mlp is LlamaMLP.*mixes dense"):
        _is_moe(plans)


# --------------------------------------------------------------------------- host side
def test_exports_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "autogptq_b200.h")).read()
    assert re.search(r"\bagb200_moe_router\s*\(", hdr), "agb200_moe_router is not declared"
    assert "agb200_moe_router" in _lib.declared_symbols()
    m = re.search(r"#define AGB200_MOE_ROUTER_MAX_TOP_K (\d+)", hdr)
    assert m and int(m.group(1)) == _lib.MOE_ROUTER_MAX_TOP_K == 8
    assert _lib.ABI_VERSION == 11


def test_router_validates_arguments():
    from autogptq_b200.moe import moe_router, router_supported

    f16 = torch.float16
    assert router_supported(1, 4096, 8, 2, f16) is None
    assert router_supported(8, 16384, 256, 8, torch.bfloat16) is None
    assert "rows" in router_supported(9, 4096, 8, 2, f16)
    assert "hidden size" in router_supported(1, 4000, 8, 2, f16)
    assert "hidden size" in router_supported(1, 16384 + 128, 8, 2, f16)
    assert "top_k" in router_supported(1, 4096, 16, 9, f16)
    assert "experts" in router_supported(1, 4096, 2, 4, f16)
    assert "experts" in router_supported(1, 4096, 257, 2, f16)
    assert "dtype" in router_supported(1, 4096, 8, 2, torch.float32)
    z = torch.zeros
    with pytest.raises(RuntimeError, match="CUDA"):
        moe_router(z(1, 256, dtype=f16), None, z(256, dtype=f16), 1e-5, z(8, 256, dtype=f16), 2)
