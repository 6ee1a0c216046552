"""CPU checks of the model checks ChainDecoder and BatchDecoder share (``autogptq_b200._decoding``): each refusal comes
from both decoders with the decoder's prefix and the module it names, every refusal comes before the device check, the
config's attention geometry is checked against the projections, and BatchDecoder refuses a model.norm its kernel cannot
read."""
import re

import pytest
import torch

from tests.test_batch_decoder_cpu import _llama, _mistral_window, _quantized


def _chain(model, **kw):
    from autogptq_b200.decoder import ChainDecoder

    return ChainDecoder(model, **dict(dict(batch=1, max_length=128), **kw))


def _batch(model, **kw):
    from autogptq_b200 import BatchDecoder

    return BatchDecoder(model, **dict(dict(max_batch=2, max_length=128), **kw))


DECODERS = [("ChainDecoder", _chain), ("BatchDecoder", _batch)]


def _with(model, fn):
    fn(model)
    return model


def _layer_norm(m):
    m.model.layers[0].input_layernorm = torch.nn.LayerNorm(256).half()


ROPE = {"rope_type": "dynamic", "factor": 2.0, "rope_theta": 10000.0}

CASES = {
    "linear_projection": (lambda: _llama(), {},
                          r"model\.layers\.0\.self_attn\.q_proj is Linear, not autogptq_b200\.QuantLinear$"),
    "gelu_mlp": (lambda: _quantized(_llama(hidden_act="gelu")), {},
                 r"model\.layers\.0\.mlp\.act_fn is GELUActivation, not SiLU$"),
    "layer_norm": (lambda: _with(_quantized(_llama()), _layer_norm), {},
                   r"model\.layers\.0\.input_layernorm is LayerNorm; only Llama-style RMSNorm \("),
    "norm_dtype": (lambda: _with(_quantized(_llama()), lambda m: m.model.layers[0].post_attention_layernorm.float()),
                   {}, r"model\.layers\.0\.post_attention_layernorm\.weight is torch\.float32, the activations "
                       r"torch\.float16$"),
    "sliding_window": (_mistral_window, {}, r"the model attends through a sliding window of 64 tokens, below "
                                            r"max_length=128; "),
    "kv_cache_dtype": (lambda: _quantized(_llama()), dict(kv_cache_dtype=torch.int8),
                       r"kv_cache_dtype torch\.int8; supported: None \(the activation dtype\) or "
                       r"torch\.float8_e4m3fn$"),
    "not_causal_lm": (lambda: torch.nn.Linear(4, 4), {},
                      r"Linear is not a \*ForCausalLM with model\.layers and lm_head$"),
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("who,make", DECODERS, ids=[w for w, _ in DECODERS])
def test_shared_refusals(who, make, case):
    build, kw, text = CASES[case]
    with pytest.raises(NotImplementedError, match=f"^{who}: " + text):
        make(build(), **kw)


@pytest.mark.parametrize("who,make,kw", [("ChainDecoder(fused_attention=True)", _chain, dict(fused_attention=True)),
                                         ("BatchDecoder", _batch, {})], ids=["ChainDecoder", "BatchDecoder"])
def test_dynamic_rope(who, make, kw):
    with pytest.raises(NotImplementedError,
                       match="^" + re.escape(who) + r": model\.model\.rotary_emb is 'dynamic' rope"):
        make(_quantized(_llama(rope_parameters=ROPE)), **kw)


def test_both_decoders_refuse_before_the_device_check():
    """The same unsupported model on the CPU gets the same refusal from both decoders, not the device error."""
    def linear_up(m):
        m.model.layers[0].mlp.up_proj = torch.nn.Linear(256, 512).half()

    texts = []
    for who, make in DECODERS:
        with pytest.raises(NotImplementedError) as e:
            make(_with(_quantized(_llama()), linear_up))
        assert str(e.value).startswith(who + ": ")
        texts.append(str(e.value)[len(who) + 2:])
    assert texts[0] == texts[1] == "model.layers.0.mlp.up_proj is Linear, not autogptq_b200.QuantLinear"


def test_projections_must_match_the_config_geometry():
    from autogptq_b200 import QuantLinear

    def narrow_kv(m):                        # projections of 1 kv head where the config says 2
        at = m.model.layers[0].self_attn
        for n in ("k_proj", "v_proj"):
            setattr(at, n, QuantLinear(4, 128, 256, 128, False, weight_dtype=torch.float16))

    for who, make in DECODERS:
        with pytest.raises(NotImplementedError, match=f"^{who}: " + re.escape(
                "model.layers.0.self_attn.k_proj maps 256 -> 128 features; the config (hidden_size 256, 2 heads, "
                "2 kv heads, head_dim 128) needs 256 -> 256") + "$"):
            make(_with(_quantized(_llama(num_key_value_heads=2)), narrow_kv))


def test_batch_decoder_refuses_a_final_norm_in_another_dtype():
    """BatchDecoder's last add_rmsnorm reads model.norm's weight; ChainDecoder runs that norm in torch and takes it."""
    m = _with(_quantized(_llama()), lambda m: m.model.norm.float())
    with pytest.raises(NotImplementedError,
                       match=r"^BatchDecoder: model\.norm\.weight is torch\.float32, the activations torch\.float16$"):
        _batch(m)
    with pytest.raises(RuntimeError, match="^ChainDecoder needs the model on a CUDA device$"):
        _chain(m)
