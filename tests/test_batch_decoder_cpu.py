"""CPU checks of BatchDecoder's host side: the two C ABI additions it uses (per-row decode attention, residual add +
RMSNorm), its refusals before any device is needed, and the float64 reference of ragged attention with idle rows against
transformers' eager attention under per-row masks."""
import os
import re

import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from tests._batch_attention import rows_reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exports_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "autogptq_b200.h")).read()
    for name in ("agb200_decode_attention_rows", "agb200_add_rmsnorm"):
        assert re.search(rf"\b{name}\s*\(", hdr), f"{name} is not declared"
        assert name in _lib.declared_symbols(), f"{name} is not bound"
    m = re.search(r"#define AGB200_ATTN_ROWS_MAX_B (\d+)", hdr)
    assert m and int(m.group(1)) == _lib.ATTN_ROWS_MAX_B == 8
    assert _lib.ABI_VERSION == 11


def test_support_checks():
    from autogptq_b200.attention import attention_rows_supported, attention_supported
    from autogptq_b200.moe import add_rmsnorm_supported

    for B in (1, 3, 8):
        assert attention_rows_supported(32, 8, 128, B, 4096, torch.float16) is None
    assert "batch 9" in attention_rows_supported(32, 8, 128, 9, 4096, torch.float16)
    assert "batch 0" in attention_rows_supported(32, 8, 128, 0, 4096, torch.float16)
    assert "head_dim" in attention_rows_supported(32, 8, 96, 4, 4096, torch.float16)
    assert "16 query heads" in attention_rows_supported(32, 2, 128, 4, 4096, torch.float16)
    assert "2^31" in attention_rows_supported(64, 8, 128, 8, 2 ** 18, torch.bfloat16)
    assert "batch" in attention_supported(32, 8, 128, 3, 4096, torch.float16)     # the lockstep entry keeps its limit
    assert add_rmsnorm_supported(8, 4096, torch.bfloat16) is None
    assert "rows" in add_rmsnorm_supported(9, 4096, torch.float16)
    assert "hidden size" in add_rmsnorm_supported(1, 4000, torch.float16)
    assert "dtype" in add_rmsnorm_supported(1, 4096, torch.float32)


def test_wrappers_need_cuda():
    from autogptq_b200.attention import decode_attention_rows
    from autogptq_b200.moe import add_rmsnorm

    z = torch.zeros
    with pytest.raises(RuntimeError, match="CUDA"):
        decode_attention_rows(z(3, 256, dtype=torch.half), z(3, 128, dtype=torch.half), z(3, 128, dtype=torch.half),
                              z(3, 1, 16, 128, dtype=torch.half), z(3, 1, 16, 128, dtype=torch.half),
                              z(3, dtype=torch.int64), z(64), 1.0, 0.1, z(3, 256, dtype=torch.half))
    with pytest.raises(RuntimeError, match="CUDA"):
        add_rmsnorm(z(2, 256, dtype=torch.half), None, z(256, dtype=torch.half), 1e-5)


# --------------------------------------------------------------------------- refusals
def _small(**kw):
    return dict(dict(hidden_size=256, intermediate_size=512, num_attention_heads=2, num_key_value_heads=2,
                     num_hidden_layers=1, vocab_size=64, max_position_embeddings=4096), **kw)


def _llama(**kw):
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(0)
    return LlamaForCausalLM(LlamaConfig(**_small(**kw))).half().eval()


def _quantized(model):
    from autogptq_b200 import QuantLinear

    for layer in model.model.layers:
        for mod, names in ((layer.self_attn, ("q_proj", "k_proj", "v_proj", "o_proj")),
                           (layer.mlp, ("gate_proj", "up_proj", "down_proj"))):
            for n in names:
                lin = getattr(mod, n)
                setattr(mod, n, QuantLinear(4, 128, lin.in_features, lin.out_features, lin.bias is not None,
                                            weight_dtype=torch.float16))
    return model


def _mistral_window():
    from transformers import MistralConfig, MistralForCausalLM

    return MistralForCausalLM(MistralConfig(**_small(sliding_window=64))).half().eval()


def _mixtral():
    from transformers import MixtralConfig, MixtralForCausalLM

    return MixtralForCausalLM(MixtralConfig(**_small(num_local_experts=4, num_experts_per_tok=2))).half().eval()


@pytest.mark.parametrize("make,kw,match", [
    (lambda: _quantized(_llama()), dict(max_batch=0), "max_batch 0"),
    (lambda: _quantized(_llama()), dict(max_batch=9), "max_batch 9"),
    (lambda: _quantized(_llama(hidden_size=192)), {}, r"model\.layers\.\*\.self_attn: head_dim 96"),
    (_mistral_window, {}, "sliding window of 64"),
    (_mixtral, {}, r"model\.layers\.0\.mlp is MixtralSparseMoeBlock"),
    (_llama, {}, r"model\.layers\.0\.self_attn\.q_proj is Linear"),
    (lambda: _quantized(_llama(rope_parameters={"rope_type": "dynamic", "factor": 2.0, "rope_theta": 10000.0})), {},
     r"model\.model\.rotary_emb is 'dynamic'"),
], ids=["max_batch_0", "max_batch_9", "head_dim_96", "sliding_window", "mixtral", "linear_projection", "dynamic_rope"])
def test_refusals_name_the_module(make, kw, match):
    from autogptq_b200 import BatchDecoder

    with pytest.raises(NotImplementedError, match=match) as e:
        BatchDecoder(make(), **dict(dict(max_batch=4, max_length=128), **kw))
    assert str(e.value).startswith("BatchDecoder: ")


def test_refuses_mlp_projection_and_norm():
    from autogptq_b200 import BatchDecoder

    m = _quantized(_llama())
    m.model.layers[0].mlp.down_proj = torch.nn.Linear(512, 256).half()
    with pytest.raises(NotImplementedError, match=r"model\.layers\.0\.mlp\.down_proj is Linear"):
        BatchDecoder(m, max_batch=2, max_length=128)
    m = _quantized(_llama())
    m.model.norm = torch.nn.LayerNorm(256).half()
    with pytest.raises(NotImplementedError, match=r"model\.norm is LayerNorm"):
        BatchDecoder(m, max_batch=2, max_length=128)


def test_a_supported_model_gets_to_the_device_check():
    from autogptq_b200 import BatchDecoder

    with pytest.raises(RuntimeError, match="CUDA device"):
        BatchDecoder(_quantized(_llama(num_key_value_heads=1)), max_batch=8, max_length=128)


# --------------------------------------------------------------------------- the reference
@pytest.mark.parametrize("n_heads,n_kv,hd", [(4, 4, 64), (8, 2, 128), (8, 1, 64)])
def test_ragged_reference_equals_transformers_eager(n_heads, n_kv, hd):
    """Rows at positions 0, 31, 32, idle, 70 of one [B, n_kv, L, hd] cache: the per-row float64 reference equals
    transformers' eager attention with an additive per-row mask (whose softmax runs in fp32, hence the 1e-5: a position
    too many or too few moves an output by about 1/n), and idle rows are zero."""
    from types import SimpleNamespace

    from transformers.models.llama.modeling_llama import eager_attention_forward

    rng = np.random.default_rng(11)
    pos = [0, 31, 32, -1, 70]
    B, L = len(pos), 80
    qh = rng.standard_normal((B, n_heads, hd))
    K = rng.standard_normal((B, n_kv, L, hd))
    V = rng.standard_normal((B, n_kv, L, hd))
    sc = hd ** -0.5
    o, parts = rows_reference(qh, K, V, pos, sc)
    mask = np.full((B, 1, 1, L), -np.inf)
    for b, p in enumerate(pos):
        mask[b, ..., :p + 1] = 0.0
    module = SimpleNamespace(num_key_value_groups=n_heads // n_kv, training=False)
    ref, _ = eager_attention_forward(module, torch.from_numpy(qh)[:, :, None], torch.from_numpy(K),
                                     torch.from_numpy(V), torch.from_numpy(mask), scaling=sc)
    ref = ref[:, 0].numpy()                          # [B, 1, H, hd] -> [B, H, hd]
    for b, p in enumerate(pos):
        if p < 0:
            assert parts[b] is None and (o[b] == 0).all()
        else:
            np.testing.assert_allclose(o[b], ref[b], rtol=1e-5, atol=1e-6)
            if p > 0:                                # the comparison is sharp enough to see one position too few
                short, _ = rows_reference(qh[b:b + 1], K[b:b + 1], V[b:b + 1], [p - 1], sc)
                assert np.abs(short[0] - ref[b]).max() > 1e-4
