"""CPU checks of BatchDecoder over Mixtral blocks: the router entry with idle rows (``agb200_moe_router_rows``) is
declared, bound and refuses bad arguments before any launch, and BatchDecoder's refusals of MoE blocks it cannot run
name themselves; a quantised Mixtral with grouped experts gets as far as the device check."""
import os
import re

import pytest
import torch

from autogptq_b200 import _lib
from tests.test_moe_router_cpu import _cpu_mixtral, _quant

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_router_rows_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "autogptq_b200.h")).read()
    assert re.search(r"\bagb200_moe_router_rows\s*\(\s*const void\* x", hdr), "agb200_moe_router_rows is not declared"
    assert "agb200_moe_router_rows" in _lib.declared_symbols()
    assert _lib.ABI_VERSION == 11


# --------------------------------------------------------------------------- the C entry's argument checks
def _router_rows(**kw):
    """agb200_moe_router_rows on fake (never dereferenced) addresses: every argument check runs before a launch.
    Returns (status, message)."""
    lib = _lib.load()
    a = dict(x=0x1000, x2=0x2000, norm_weight=0x3000, eps=1e-5, gate_weight=0x4000, pos=0x5000, T=4, H=256, E=8, k=2,
             dtype=_lib.F16, h=0x6000, n=0x7000, idx=0x8000, w=0x9000, logits=None, stream=None)
    a.update(kw)
    rc = lib.agb200_moe_router_rows(a["x"], a["x2"], a["norm_weight"], a["eps"], a["gate_weight"], a["pos"], a["T"],
                                    a["H"], a["E"], a["k"], a["dtype"], a["h"], a["n"], a["idx"], a["w"], a["logits"],
                                    a["stream"])
    return rc, lib.agb200_last_error().decode()


EINVAL = -1


@pytest.mark.parametrize("kw,code,match", [
    (dict(pos=None), EINVAL, "null pointer"),
    (dict(pos=0x5004), EINVAL, "pos must be 8-byte aligned"),
    (dict(T=9), _lib.ENOSUP, "T=9 rows; at most 8"),
    (dict(x=None), EINVAL, "null pointer"),
    (dict(h=None), EINVAL, "h is written exactly when x2 is given"),
    (dict(T=-1), EINVAL, "need T >= 0"),
    (dict(dtype=_lib.F32), _lib.ENOSUP, "dtype"),
    (dict(H=200), _lib.ENOSUP, "multiple of 128"),
    (dict(k=9, E=16), _lib.ENOSUP, "k=9"),
    (dict(E=1), _lib.ENOSUP, "E=1 experts"),
    (dict(x=0x1008), EINVAL, "16-byte aligned"),
], ids=["null_pos", "misaligned_pos", "T9", "null_x", "h_without_x2", "negative_T", "dtype", "H", "top_k", "E",
        "misaligned_x"])
def test_router_rows_refuses(kw, code, match):
    rc, msg = _router_rows(**kw)
    assert rc == code and re.search(match, msg), (rc, msg)


def test_router_rows_zero_rows_do_nothing():
    assert _router_rows(T=0)[0] == 0


def test_router_pos_checks_its_tensor():
    from autogptq_b200.moe import moe_router

    z = torch.zeros
    with pytest.raises(RuntimeError, match="CUDA"):
        moe_router(z(2, 256, dtype=torch.half), None, z(256, dtype=torch.half), 1e-5, z(8, 256, dtype=torch.half), 2,
                   pos=z(2, dtype=torch.int64))


# --------------------------------------------------------------------------- BatchDecoder's refusals
def _batch(model, **kw):
    from autogptq_b200 import BatchDecoder

    return BatchDecoder(model, **dict(dict(max_batch=4, max_length=128), **kw))


def _refused(model, match):
    with pytest.raises(NotImplementedError, match=match) as e:
        _batch(model)
    assert str(e.value).startswith("BatchDecoder: "), str(e.value)
    return str(e.value)


def test_refuses_experts_that_are_not_grouped():
    from transformers.models.mixtral.modeling_mixtral import MixtralExperts

    m = _cpu_mixtral()
    m.model.layers[1].mlp.experts = MixtralExperts(m.config).half()
    msg = _refused(m, r"model\.layers\.1\.mlp is MixtralSparseMoeBlock whose experts are MixtralExperts")
    assert "autogptq_b200.group_experts" in msg


def test_refuses_other_router():
    m = _cpu_mixtral()
    m.model.layers[0].mlp.gate = torch.nn.Linear(256, 4, bias=False).half()
    _refused(m, r"model\.layers\.0\.mlp\.gate is Linear; only MixtralTopKRouter")


def test_refuses_router_bias():
    m = _cpu_mixtral()
    m.model.layers[0].mlp.gate.bias = torch.nn.Parameter(torch.zeros(4, dtype=torch.half))
    _refused(m, r"model\.layers\.0\.mlp\.gate has a bias")


def test_refuses_other_moe_block():
    from transformers import Qwen2MoeConfig
    from transformers.models.qwen2_moe.modeling_qwen2_moe import Qwen2MoeSparseMoeBlock

    m = _cpu_mixtral()
    cfg = Qwen2MoeConfig(hidden_size=256, moe_intermediate_size=256, shared_expert_intermediate_size=256,
                         num_experts=4, num_experts_per_tok=2, num_attention_heads=2, num_key_value_heads=2)
    m.model.layers[0].mlp = Qwen2MoeSparseMoeBlock(cfg).half()
    _refused(m, r"model\.layers\.0\.mlp is Qwen2MoeSparseMoeBlock; the only mixture-of-experts block BatchDecoder")


def test_refuses_mixed_dense_and_moe_layers():
    from transformers import LlamaConfig, LlamaForCausalLM

    m = _cpu_mixtral()
    llama = LlamaForCausalLM(LlamaConfig(hidden_size=256, intermediate_size=256, num_attention_heads=2,
                                         num_key_value_heads=2, num_hidden_layers=1, vocab_size=64)).half()
    dense = llama.model.layers[0]
    for j, name in enumerate(("q_proj", "k_proj", "v_proj", "o_proj")):
        setattr(dense.self_attn, name, _quant(256, 256, 500 + j))
    for j, name in enumerate(("gate_proj", "up_proj", "down_proj")):
        setattr(dense.mlp, name, _quant(256, 256, 600 + j))
    m.model.layers[1] = dense
    _refused(m, r"model\.layers\.1\.mlp is LlamaMLP but model\.layers\.0\.mlp is MixtralSparseMoeBlock.*mixes dense")


def test_refuses_max_batch_9_for_mixtral_too():
    with pytest.raises(NotImplementedError, match="BatchDecoder: max_batch 9"):
        _batch(_cpu_mixtral(), max_batch=9)


def test_chain_decoder_messages_keep_their_name():
    """The planning BatchDecoder now shares still names ChainDecoder in ChainDecoder's refusals."""
    from autogptq_b200.decoder import _plan_layer

    m = _cpu_mixtral()
    m.model.layers[0].mlp.gate.bias = torch.nn.Parameter(torch.zeros(4, dtype=torch.half))
    with pytest.raises(NotImplementedError, match=r"^ChainDecoder: model\.layers\.0\.mlp\.gate has a bias"):
        _plan_layer(0, m.model.layers[0], 1, torch.float16)


@pytest.mark.parametrize("kw", [{}, dict(kv_block_size=16), dict(kv_cache_dtype=torch.float8_e4m3fn)],
                         ids=["static", "paged", "fp8"])
def test_a_quantised_mixtral_gets_to_the_device_check(kw):
    with pytest.raises(RuntimeError, match="BatchDecoder needs the model on a CUDA device"):
        _batch(_cpu_mixtral(), max_batch=8, **kw)
