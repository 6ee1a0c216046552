"""CPU checks of the prefill attention's model and host side: the float64 causal reference against the decode reference
and transformers' eager attention, the bound's sharpness, the C ABI exports, ``prefill_attention``'s argument errors
and the decoders' ``extend`` refusals (all before any device is needed)."""
import os
import re

import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from tests import _attention as A
from tests import _prefill_attention as PA

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rand(rng, *shape):
    return torch.from_numpy(A.round_dt(rng.standard_normal(shape), "float16"))


@pytest.mark.parametrize("start", [0, 5, 63, 64, 130])
def test_one_token_equals_the_decode_reference(start):
    rng = np.random.default_rng(start)
    H, n_kv, hd = 8, 2, 64
    qh, K, V = _rand(rng, 1, H, hd), _rand(rng, n_kv, start + 1, hd), _rand(rng, n_kv, start + 1, hd)
    o, p, *_ = PA.reference(qh, K, V, start, hd ** -0.5)
    od, pd, *_ = A.reference(qh.numpy(), K[None].numpy(), V[None].numpy(), hd ** -0.5)
    np.testing.assert_allclose(o.numpy(), od, rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(p.numpy(), pd, rtol=1e-13, atol=1e-15)


@pytest.mark.parametrize("n_heads,n_kv,hd,start,T", [(4, 4, 64, 0, 9), (8, 2, 128, 17, 30), (8, 1, 64, 100, 1)])
def test_reference_equals_transformers_eager_attention(n_heads, n_kv, hd, start, T):
    """Causal attention over a prefix of ``start`` cached positions, as transformers' eager attention computes it with
    an additive causal mask (float64 inputs; its softmax runs in fp32)."""
    from transformers.models.llama.modeling_llama import eager_attention_forward

    rng = np.random.default_rng(n_heads + T)
    qh, K, V = _rand(rng, T, n_heads, hd), _rand(rng, n_kv, start + T, hd), _rand(rng, n_kv, start + T, hd)
    o, *_ = PA.reference(qh, K, V, start, hd ** -0.5)
    mod = torch.nn.Module()
    mod.num_key_value_groups = n_heads // n_kv
    mask = torch.zeros(T, start + T, dtype=torch.float64)
    mask.masked_fill_(torch.arange(start + T)[None, :] > start + torch.arange(T)[:, None], -torch.inf)
    ref, _ = eager_attention_forward(mod.eval(), qh.transpose(0, 1)[None], K[None], V[None], mask[None, None],
                                     hd ** -0.5)
    np.testing.assert_allclose(o.numpy(), ref[0].numpy(), rtol=1e-5, atol=1e-6)


def test_bound_catches_a_causality_error():
    """Letting every token see one position too many (or too few) breaks the bound on realistic data; the exact
    rounding of the reference passes."""
    rng = np.random.default_rng(3)
    T, H, hd, start = 40, 4, 128, 60
    qh, K, V = _rand(rng, T, H, hd), _rand(rng, H, start + T + 1, hd), _rand(rng, H, start + T + 1, hd)
    ref = PA.reference(qh, K, V, start, hd ** -0.5)
    b, budget = PA.bound(*ref, hd ** -0.5, hd, "float16")
    o = ref[0].numpy()
    PA.check(A.round_dt(o, "float16"), o, b, budget, "float16")
    for s in (start + 1, start - 1):
        wrong = PA.reference(qh, K, V, s, hd ** -0.5)[0].numpy()
        with pytest.raises(AssertionError):
            PA.check(A.round_dt(wrong, "float16"), o, b, budget, "float16")


def test_bound_covers_rounding_p_to_the_dtype():
    """A simulated kernel (fp32 scores, P rounded to bf16, fp32 sums) stays within the bound; dropping the P term
    from the bound would not hold it."""
    rng = np.random.default_rng(4)
    T, H, hd, start = 20, 2, 64, 300
    qh, K, V = (torch.from_numpy(A.round_dt(rng.standard_normal(s) * 2, "bfloat16"))
                for s in ((T, H, hd), (H, start + T, hd), (H, start + T, hd)))
    ref = PA.reference(qh, K, V, start, hd ** -0.5)
    o, p, s = ref[0], ref[1], ref[2]
    e = torch.exp(s - s.amax(-1, keepdim=True))
    pr = torch.from_numpy(A.round_dt(e.numpy(), "bfloat16"))
    sim = (torch.einsum("thn,hnd->thd", pr, ref[4]) / e.sum(-1, keepdim=True)).numpy()
    b, budget = PA.bound(*ref, hd ** -0.5, hd, "bfloat16")
    assert (np.abs(sim - o.numpy()) <= b).all()
    pv = torch.einsum("thn,hnd->thd", p, ref[4].abs()).numpy()
    assert (np.abs(sim - o.numpy()) > b - 2 * PA.U_P["bfloat16"] * pv).any(), "the P term is not needed"


def test_exports_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "autogptq_b200.h")).read()
    for name in ("agb200_prefill_attention", "agb200_prefill_attention_fp8"):
        assert re.search(rf"\b{name}\s*\(", hdr), f"{name} is not declared"
        assert name in _lib.declared_symbols(), f"{name} is not bound"
    assert _lib.ABI_VERSION == 11
    from autogptq_b200 import attention

    assert {"prefill_attention", "prefill_attention_supported"} <= set(attention.__all__)


def test_prefill_attention_argument_errors():
    from autogptq_b200.attention import prefill_attention, prefill_attention_supported

    assert prefill_attention_supported(32, 8, 128, 8, 4096, torch.float16) is None
    assert prefill_attention_supported(32, 8, 128, 9, 4096, torch.float16) == \
        "batch 9; the kernel takes 1..8 independent rows"
    assert prefill_attention_supported(32, 8, 96, 1, 4096, torch.float16) == "head_dim 96; the kernel takes 64 or 128"
    z = torch.zeros
    h = dict(dtype=torch.half)
    cache = z(1, 1, 16, 128, **h)
    with pytest.raises(ValueError, match=r"^q must be \[B, T, n_heads·head_dim\], got \(1, 256\)$"):
        prefill_attention(z(1, 256, **h), z(1, 128, **h), z(1, 128, **h), cache, cache, z(1, dtype=torch.int64),
                          z(64), 1.0, 0.1, z(1, 256, **h))
    with pytest.raises(ValueError, match=r"^prefill_attention: T must be at least 1$"):
        prefill_attention(z(1, 0, 256, **h), z(1, 0, 128, **h), z(1, 0, 128, **h), cache, cache,
                          z(1, dtype=torch.int64), z(64), 1.0, 0.1, z(1, 0, 256, **h))
    with pytest.raises(RuntimeError, match=r"^prefill_attention needs CUDA tensors \(there is no CPU fallback\)$"):
        prefill_attention(z(1, 3, 256, **h), z(1, 3, 128, **h), z(1, 3, 128, **h), cache, cache,
                          z(1, dtype=torch.int64), z(64), 1.0, 0.1, z(1, 3, 256, **h))


# --------------------------------------------------------------------------- extend refusals
def _batch_decoder(max_batch=3, max_length=64, pos=None):
    """A BatchDecoder's host state only: extend's checks read nothing else before they pass."""
    from autogptq_b200 import BatchDecoder

    d = BatchDecoder.__new__(BatchDecoder)
    d.max_batch, d.max_length = max_batch, max_length
    d._host_pos = list(pos or [-1] * max_batch)
    return d


def _chain_decoder(batch=1, max_length=64, position=0, moe=False):
    from autogptq_b200.decoder import ChainDecoder

    d = ChainDecoder.__new__(ChainDecoder)
    d.batch, d.max_length, d._length, d.moe = batch, max_length, position, moe
    return d


def test_batch_extend_refusals():
    ids = torch.arange(5)
    with pytest.raises(ValueError, match=r"^slot 3 outside 0\.\.2$"):
        _batch_decoder().extend(3, ids)
    with pytest.raises(ValueError, match=r"^BatchDecoder\.extend: input_ids must be 1-D \[T\] \(one slot\), got "
                                         r"\(1, 5\)$"):
        _batch_decoder().extend(0, ids[None])
    with pytest.raises(ValueError, match=r"^BatchDecoder\.extend: input_ids is empty$"):
        _batch_decoder().extend(0, ids[:0])
    with pytest.raises(ValueError, match=r"^BatchDecoder\.extend: slot 1 at position 60 \+ 4 tokens must stay below "
                                         r"max_length=64$"):
        _batch_decoder(pos=[-1, 60, 3]).extend(1, ids[:4])
    with pytest.raises(ValueError, match=r"^BatchDecoder\.extend: slot 0 at position 0 \+ 64 tokens must stay below "
                                         r"max_length=64$"):
        _batch_decoder().extend(0, torch.arange(64))


def test_chain_extend_refusals():
    with pytest.raises(NotImplementedError, match=r"^ChainDecoder\.extend: mixture-of-experts blocks are not supported "
                                                  r"\(the router kernel takes at most 8 rows\); use prefill$"):
        _chain_decoder(moe=True).extend(torch.arange(5)[None])
    with pytest.raises(ValueError, match=r"^ChainDecoder\.extend: input_ids must be \[2, T\] \(sequences in lockstep\), "
                                         r"got \(1, 5\)$"):
        _chain_decoder(batch=2).extend(torch.arange(5)[None])
    with pytest.raises(ValueError, match=r"^ChainDecoder\.extend: input_ids is empty$"):
        _chain_decoder().extend(torch.zeros(1, 0, dtype=torch.int64))
    with pytest.raises(ValueError, match=r"^ChainDecoder\.extend: position 50 \+ 14 tokens must stay below "
                                         r"max_length=64$"):
        _chain_decoder(position=50).extend(torch.arange(14)[None])
