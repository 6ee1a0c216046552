"""CPU checks of the decode attention's model and host side: the rotary rounding model against transformers, the
float64 reference against float64 SDPA, the C ABI exports and ChainDecoder's refusals."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from autogptq_b200 import _lib
from tests import _attention as A
from tests._precision import dt_name

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTS = [torch.float16, torch.bfloat16]


def _llama_config(**kw):
    from transformers import LlamaConfig

    base = dict(hidden_size=256, intermediate_size=512, num_attention_heads=2, num_key_value_heads=2,
                num_hidden_layers=1, vocab_size=64, max_position_embeddings=32768)
    base.update(kw)
    return LlamaConfig(**base)


ROPES = {
    "default": {},
    "linear": {"rope_type": "linear", "factor": 4.0},
    "llama3": {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
               "original_max_position_embeddings": 8192},
    "yarn": {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 8192},
}


def _rotary(kind):
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding

    params = dict(ROPES[kind], rope_theta=500000.0 if kind == "llama3" else 10000.0)
    params.setdefault("rope_type", "default")
    return LlamaRotaryEmbedding(_llama_config(rope_parameters=params))


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("kind", list(ROPES))
def test_rope_model_matches_transformers(kind, dtype):
    """Given the CPU's fp32 cos / sin, the model's rounding steps reproduce apply_rotary_pos_emb bit for bit."""
    from transformers.models.llama.modeling_llama import apply_rotary_pos_emb

    rot = _rotary(kind)
    hd = rot.inv_freq.numel() * 2
    positions = torch.tensor([0, 1, 2, 15, 16, 17, 255, 1000, 4095, 8191, 16383, 20000, 32767])
    B, H = positions.numel(), 4
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(B, H, 1, hd, generator=g) * 3).to(dtype)
    x[:, 0, 0, :8] *= 100                                   # outlier channels
    pos_ids = positions.view(B, 1)
    cos, sin = rot(x.view(B, 1, -1), pos_ids)
    ref_q, ref_k = apply_rotary_pos_emb(x, x, cos, sin)
    assert torch.equal(ref_q.view(torch.int16), ref_k.view(torch.int16))
    # the fp32 cos / sin that rotary_emb rounds, computed by the same op on the same shape
    freqs = (rot.inv_freq[None, :, None].float().expand(B, -1, 1) @ pos_ids[:, None, :].float()).transpose(1, 2)
    emb = torch.cat((freqs, freqs), dim=-1)
    f_np = np.stack([A.freqs32(rot.inv_freq.numpy(), int(p)) for p in positions])
    assert np.array_equal(emb[:, 0].numpy(), f_np), "f is not fp32(inv_freq·pos)"
    xs = x[:, :, 0].double().numpy()
    got = A.rope(xs, emb.cos().numpy()[:, None, 0], emb.sin().numpy()[:, None, 0], rot.attention_scaling,
                 dt_name(dtype))
    np.testing.assert_array_equal(got, ref_q[:, :, 0].double().numpy())


def test_rope_model_rejects_a_fused_rounding():
    """A model that skips the intermediate roundings differs somewhere: the comparison above is sharp."""
    rot = _rotary("default")
    hd = rot.inv_freq.numel() * 2
    x = (torch.randn(64, 8, hd, generator=torch.Generator().manual_seed(4)) * 3).half().double().numpy()
    f = np.stack([A.freqs32(rot.inv_freq.numpy(), p) for p in range(1000, 1064)])[:, None]
    good = A.rope(x, np.cos(f).astype(np.float32), np.sin(f).astype(np.float32), 1.0, "float16")
    c, s = A.round_dt(np.cos(f), "float16"), A.round_dt(np.sin(f), "float16")
    r = np.concatenate([-x[..., hd // 2:], x[..., :hd // 2]], axis=-1)
    fused = A.round_dt(x * c + r * s, "float16")
    assert (fused != good).any()


@pytest.mark.parametrize("n_heads,n_kv,hd", [(4, 4, 64), (8, 2, 128), (8, 1, 64)])
def test_reference_equals_float64_sdpa(n_heads, n_kv, hd):
    rng = np.random.default_rng(7)
    B, n = 2, 37
    qh = rng.standard_normal((B, n_heads, hd))
    K = rng.standard_normal((B, n_kv, n, hd))
    V = rng.standard_normal((B, n_kv, n, hd))
    sc = hd ** -0.5
    o, p, *_ = A.reference(qh, K, V, sc)
    ref = F.scaled_dot_product_attention(torch.from_numpy(qh)[:, :, None], torch.from_numpy(K), torch.from_numpy(V),
                                         scale=sc, enable_gqa=n_kv != n_heads)[:, :, 0].numpy()
    np.testing.assert_allclose(o, ref, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(p.sum(-1), 1.0, rtol=1e-12)


def test_bound_is_tight_enough_to_catch_a_dropped_position():
    """Leaving out one position (an off-by-one split boundary) breaks the bound on realistic data."""
    rng = np.random.default_rng(8)
    B, H, n, hd = 1, 4, 300, 128
    qh = A.round_dt(rng.standard_normal((B, H, hd)), "float16")
    K = A.round_dt(rng.standard_normal((B, H, n, hd)), "float16")
    V = A.round_dt(rng.standard_normal((B, H, n, hd)), "float16")
    o, p, s, qk, Vr = A.reference(qh, K, V, hd ** -0.5)
    b, budget = A.bound(o, p, s, qk, Vr, hd ** -0.5, hd, "float16")
    o_short, *_ = A.reference(qh, K[:, :, :-1], V[:, :, :-1], hd ** -0.5)
    with pytest.raises(AssertionError):
        A.check(A.round_dt(o_short, "float16"), o, b, budget, "float16")
    A.check(A.round_dt(o, "float16"), o, b, budget, "float16")


def test_exports_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "autogptq_b200.h")).read()
    for name in ("agb200_decode_attention", "agb200_decode_attention_workspace_bytes"):
        assert re.search(rf"\b{name}\s*\(", hdr), f"{name} is not declared"
        assert name in _lib.declared_symbols(), f"{name} is not bound"
    assert _lib.ABI_VERSION == 11


def _cpu_llama(**kw):
    from transformers import LlamaForCausalLM

    return LlamaForCausalLM(_llama_config(**kw)).half().eval()


@pytest.mark.parametrize("kw,match", [
    (dict(rope_parameters={"rope_type": "dynamic", "factor": 2.0, "rope_theta": 10000.0}), "dynamic"),
    (dict(hidden_size=192, num_attention_heads=2, num_key_value_heads=2), "head_dim 96"),
    (dict(num_attention_heads=32, num_key_value_heads=2, hidden_size=2048), "16 query heads per kv head"),
])
def test_chain_decoder_refuses_what_the_kernel_does_not_take(kw, match):
    from autogptq_b200.decoder import ChainDecoder

    with pytest.raises(NotImplementedError, match=match):
        ChainDecoder(_cpu_llama(**kw), batch=1, max_length=64, fused_attention=True)


def test_chain_decoder_refuses_partial_rotary():
    from autogptq_b200.decoder import ChainDecoder

    model = _cpu_llama()
    model.model.rotary_emb.inv_freq = model.model.rotary_emb.inv_freq[:32].clone()
    with pytest.raises(NotImplementedError, match="partial rotary"):
        ChainDecoder(model, batch=1, max_length=64, fused_attention=True)


def test_decode_attention_validates_arguments():
    from autogptq_b200.attention import attention_supported, decode_attention

    assert attention_supported(32, 8, 128, 2, 4096, torch.float16) is None
    assert "head_dim" in attention_supported(32, 8, 96, 1, 4096, torch.float16)
    assert "batch" in attention_supported(32, 8, 128, 3, 4096, torch.float16)
    assert "2^31" in attention_supported(64, 8, 128, 2, 2 ** 20, torch.bfloat16)
    assert "dtype" in attention_supported(32, 8, 128, 1, 4096, torch.float32)
    z = torch.zeros
    with pytest.raises(RuntimeError, match="CUDA"):
        decode_attention(z(1, 256, dtype=torch.half), z(1, 128, dtype=torch.half), z(1, 128, dtype=torch.half),
                         z(1, 1, 16, 128, dtype=torch.half), z(1, 1, 16, 128, dtype=torch.half),
                         z(1, dtype=torch.int64), z(64), 1.0, 0.1, z(1, 256, dtype=torch.half))
