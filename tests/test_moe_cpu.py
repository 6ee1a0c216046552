"""CPU tests of the mixture-of-experts host side: the oracle against a transformers-style loop, grouping of a Mixtral
checkpoint into QuantExperts, constructor errors."""
import json
import os

import numpy as np
import pytest
import torch
from safetensors.torch import save_file

from autogptq_b200 import QuantExperts, QuantLinear, group_experts
from autogptq_b200 import checkpoint as C
from oracle import moe_oracle as MO
from oracle import w4a16_oracle as O


def _experts(E, H, I, g, seed=0, desc_act=False, bias=False):
    return [{name: O.random_packed(K, N, g, seed=seed + 3 * e + j, desc_act=desc_act, bias=bias)
             for j, (name, K, N) in enumerate((("w1", H, I), ("w3", H, I), ("w2", I, H)))} for e in range(E)]


def _routing(T, k, E, seed, invalid=0.0):
    rng = np.random.default_rng(seed)
    idx = np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)      # distinct ids per token
    if invalid:
        idx[rng.random(idx.shape) < invalid] = E                                      # the `expert_idx == num_experts` skip
    w = rng.random((T, k)).astype(np.float32)
    return idx, w / w.sum(axis=1, keepdims=True)


def _transformers_loop(x, experts, idx, w, dtype):
    """MixtralExperts.forward (modeling_mixtral.py:74-98) restated: one_hot mask, nonzero per hit expert,
    act_fn(gate) * up, down, scale by the routing weight, index_add_ (here in float64)."""
    T, H = x.shape
    E = len(experts)
    final = np.zeros((T, H), dtype=np.float64)
    mask = np.eye(E + 1, dtype=bool)[idx].transpose(2, 1, 0)       # [E + 1, k, T]
    hit = np.nonzero(mask.sum(axis=(-1, -2)) > 0)[0]
    for e in hit:
        if e == E:
            continue
        slot, tok = np.nonzero(mask[e])
        ex = experts[e]
        g = MO.round_to(MO.linear(x[tok], ex["w1"]), dtype)
        u = MO.round_to(MO.linear(x[tok], ex["w3"]), dtype)
        h = MO.round_to(MO.round_to(g / (1 + np.exp(-g)), dtype) * u, dtype)
        y = MO.round_to(MO.linear(h, ex["w2"]), dtype)
        np.add.at(final, tok, y.astype(np.float64) * w[tok, slot, None])
    return final


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("k,desc_act,bias", [(1, False, False), (2, True, True)])
def test_oracle_matches_transformers_loop(dtype, k, desc_act, bias):
    E, H, I, T = 4, 128, 256, 9
    experts = _experts(E, H, I, 64, seed=k, desc_act=desc_act, bias=bias)
    idx, w = _routing(T, k, E, seed=k, invalid=0.2)
    x = MO.round_to(np.random.default_rng(5).standard_normal((T, H)), dtype)
    got = MO.forward(x, experts, idx, w, dtype)
    ref = _transformers_loop(x, experts, idx, w, dtype)
    np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-5 * np.abs(ref).max())
    # a token whose every slot holds id E gets zeros
    idx2 = idx.copy()
    idx2[0] = E
    assert not MO.forward(x, experts, idx2, w, dtype)[0].any()


def test_round_to_bf16_is_round_to_nearest_even():
    a = np.array([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 1.0 + 2 ** -9, -2.5e-3], dtype=np.float32)
    got = MO.round_to(a, "bfloat16")
    want = torch.from_numpy(a).to(torch.bfloat16).float().numpy()
    assert np.array_equal(got, want)


def test_group_experts_on_mixtral_checkpoint(tmp_path):
    E, H, I, g = 4, 128, 256, 64
    experts = _experts(E, H, I, g, seed=3, desc_act=True)
    sd = {}
    for blk in range(2):
        pre = f"model.layers.{blk}.block_sparse_moe.experts"
        for e, ex in enumerate(experts):
            for name, d in ex.items():
                for leaf in ("qweight", "qzeros", "scales", "g_idx"):
                    sd[f"{pre}.{e}.{name}.{leaf}"] = torch.from_numpy(np.array(d[leaf]))
        # a plain quantised attention layer and the fp16 router: neither is an expert
        att = O.random_packed(H, H, g, seed=100 + blk)
        for leaf in ("qweight", "qzeros", "scales", "g_idx"):
            sd[f"model.layers.{blk}.self_attn.q_proj.{leaf}"] = torch.from_numpy(np.ascontiguousarray(att[leaf]))
        sd[f"model.layers.{blk}.block_sparse_moe.gate.weight"] = torch.zeros(E, H, dtype=torch.float16)
    save_file(sd, os.path.join(tmp_path, "model.safetensors"))
    json.dump({"bits": 4, "group_size": g, "desc_act": True, "sym": True}, open(os.path.join(tmp_path, C.QUANT_CONFIG_FILENAME), "w"))

    layers = C.load_quant_linears(str(tmp_path))
    assert len(layers) == 2 * (3 * E + 1)
    grouped = group_experts(layers)
    assert set(grouped) == {f"model.layers.{b}.self_attn.q_proj" for b in range(2)} | {
        f"model.layers.{b}.block_sparse_moe.experts" for b in range(2)}
    for b in range(2):
        assert grouped[f"model.layers.{b}.self_attn.q_proj"] is layers[f"model.layers.{b}.self_attn.q_proj"]
        qe = grouped[f"model.layers.{b}.block_sparse_moe.experts"]
        assert isinstance(qe, QuantExperts)
        assert (qe.num_experts, qe.hidden_size, qe.intermediate_size, qe.group_size) == (E, H, I, g)
        for e in range(E):
            pre = f"model.layers.{b}.block_sparse_moe.experts.{e}"
            assert qe.w1[e] is layers[f"{pre}.w1"] and qe.w3[e] is layers[f"{pre}.w3"] and qe.w2[e] is layers[f"{pre}.w2"]
            assert np.array_equal(qe.w2[e].qweight.numpy(), experts[e]["w2"]["qweight"])
    # the state dict of a QuantExperts keeps the checkpoint names below its prefix (w1.<e>.qweight, ...)
    assert "w1.0.qweight" in grouped["model.layers.0.block_sparse_moe.experts"].state_dict()


def test_group_experts_incomplete_family():
    lin = lambda K, N: QuantLinear(4, 64, K, N, False)                      # noqa: E731
    layers = {"m.experts.0.w1": lin(128, 256), "m.experts.0.w3": lin(128, 256)}
    with pytest.raises(ValueError, match="missing"):
        group_experts(layers)
    layers["m.experts.0.w2"] = lin(256, 128)
    layers["m.experts.2.w1"] = lin(128, 256)
    with pytest.raises(ValueError, match="numbered"):
        group_experts(layers)


def test_constructor_errors():
    lin = lambda K, N, g=64: QuantLinear(4, g, K, N, False)                  # noqa: E731
    ok = QuantExperts.from_linears([lin(128, 256)], [lin(128, 256)], [lin(256, 128)])
    assert ok.group_size == 64
    assert QuantExperts.from_linears([lin(128, 256, -1)], [lin(128, 256, -1)], [lin(256, 128, -1)]).group_size == -1
    with pytest.raises(NotImplementedError, match="expert 1 w3"):
        QuantExperts.from_linears([lin(128, 256)] * 2, [lin(128, 256), lin(128, 384)], [lin(256, 128)] * 2)
    with pytest.raises(NotImplementedError, match="expert 0 w2"):
        QuantExperts.from_linears([lin(128, 256)], [lin(128, 256)], [lin(128, 256)])
    with pytest.raises(NotImplementedError, match="multiples of 128"):
        QuantExperts.from_linears([lin(128, 192)], [lin(128, 192)], [lin(192, 128)])
    with pytest.raises(NotImplementedError, match="group size"):
        QuantExperts.from_linears([lin(128, 256, 64)], [lin(128, 256, 128)], [lin(256, 128)])
    with pytest.raises(NotImplementedError, match="group_size=96"):
        QuantExperts.from_linears([lin(192 * 2, 256, 96)], [lin(384, 256, 96)], [lin(256, 384, 96)])
    with pytest.raises(ValueError):
        QuantExperts.from_linears([lin(128, 256)], [], [lin(256, 128)])
    with pytest.raises(TypeError):
        QuantExperts.from_linears([torch.nn.Linear(128, 256)], [lin(128, 256)], [lin(256, 128)])


def test_forward_refuses_cpu_tensors():
    qe = QuantExperts.from_linears([QuantLinear(4, 64, 128, 256, False)], [QuantLinear(4, 64, 128, 256, False)],
                                   [QuantLinear(4, 64, 256, 128, False)])
    x = torch.zeros(3, 128, dtype=torch.float16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        qe(x, torch.zeros(3, 1, dtype=torch.int64), torch.ones(3, 1))
