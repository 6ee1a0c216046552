"""CPU checks of the decode chain's norm stage inputs (tests/_chain_norm.py) and of the argument validation of
``DecodeChain.stage`` and ``ChainDecoder``.

* The NumPy restatement of the kernel's arithmetic gives h = rnd(x + x2) bit-equal to transformers' residual add, and
  n within the candidate set of the float64 reference, as does transformers' LlamaRMSNorm / Qwen2RMSNorm itself: the
  rule accepts both fp32 summation orders.
* The candidate rule is sharp: a norm that skips the intermediate rounding, uses the wrong eps, or rounds r to the
  activation dtype is rejected.
No GPU, no library call."""
import numpy as np
import pytest
import torch

from tests import _chain_norm as N
from tests import _precision as P

DTS = [torch.float16, torch.bfloat16]


def _rows(kind, M, K, dtype, seed):
    x = P.activations(kind, M, K, dtype, seed=seed).astype(np.float64)
    r = P.activations("gauss", M, K, dtype, seed=seed + 100).astype(np.float64) * 3.0
    return x, P.round_dt(r, P.dt_name(dtype))


def _weight(K, dtype, seed):
    rng = np.random.default_rng(seed)
    return P.round_dt(rng.uniform(0.2, 2.0, size=K) * np.where(rng.random(K) < 0.5, 1, -1), P.dt_name(dtype))


def _hf_norm(cls, w, eps, dtype):
    mod = cls(w.shape[0], eps=eps)
    with torch.no_grad():
        mod.weight.copy_(torch.from_numpy(w).to(dtype))
    return mod.to(dtype)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("kind", ["gauss", "offset", "massive", "student_t", "row_scale"])
@pytest.mark.parametrize("K", [1024, 4096])
def test_kernel_model_and_transformers_within_candidates(dtype, kind, K):
    from transformers.models.llama.modeling_llama import LlamaRMSNorm
    from transformers.models.qwen2.modeling_qwen2 import Qwen2RMSNorm

    M, eps = 2, 1e-5
    x, res = _rows(kind, M, K, dtype, seed=K + len(kind))
    w = _weight(K, dtype, seed=3)
    h, n = N.kernel_model(x, res, w, eps, dtype)
    # the residual add: exactly torch's
    h_t = (torch.from_numpy(res).to(dtype) + torch.from_numpy(x).to(dtype)).double().numpy()
    assert np.array_equal(h, h_t)
    N.check_n(n, h, w, eps, dtype, what=f"kernel model {kind}")
    for cls in (LlamaRMSNorm, Qwen2RMSNorm):
        with torch.no_grad():
            out = _hf_norm(cls, w, eps, dtype)(torch.from_numpy(h).to(dtype)).double().numpy()
        N.check_n(out, h, w, eps, dtype, what=f"{cls.__name__} {kind}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_rmsnorm_without_residual(dtype):
    K, eps = 2048, 1e-6
    x, _ = _rows("massive", 1, K, dtype, seed=5)
    w = _weight(K, dtype, seed=6)
    h, n = N.kernel_model(x, None, w, eps, dtype)
    assert np.array_equal(h, x)
    N.check_n(n, x, w, eps, dtype, what="rmsnorm")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_candidate_rule_is_sharp(dtype):
    """Three wrong formulations are caught: no rounding of h·r before the weight, a wrong eps, r rounded to the dtype."""
    K, eps = 4096, 1e-5
    dt = P.dt_name(dtype)
    x, res = _rows("gauss", 2, K, dtype, seed=11)
    w = _weight(K, dtype, seed=12)
    h = N.add_rounded(x, res, dtype)
    r = N.r_exact(h, eps)
    mutants = {
        "one rounding": P.round_dt(h * r * w, dt),
        "eps 1e-2": P.round_dt(P.round_dt(h * N.r_exact(h, 1e-2 * np.mean(h * h)), dt) * w, dt),
        "r rounded": P.round_dt(P.round_dt(h * P.round_dt(r, dt), dt) * w, dt),
    }
    for name, n in mutants.items():
        with pytest.raises(AssertionError):
            N.check_n(n, h, w, eps, dtype, what=name)


def test_ambiguous_share_is_small():
    """The candidate band is narrow: at K = 4096 well under 2 % of fp16 elements and 0.3 % of bf16 ones have two."""
    for dtype, lim in ((torch.float16, 0.02), (torch.bfloat16, 0.003)):
        x, res = _rows("gauss", 2, 4096, dtype, seed=21)
        h = N.add_rounded(x, res, dtype)
        _, _, amb = N.n_candidates(h, _weight(4096, dtype, 22), 1e-5, dtype)
        assert amb.mean() < lim, (dtype, amb.mean())


# --------------------------------------------------------------------------- argument validation
def test_stage_norm_argument_errors():
    from autogptq_b200.chain import check_norm_args

    K, dt, dev = 1024, torch.float16, torch.device("cpu")
    w = torch.ones(K, dtype=dt)
    x2 = torch.zeros(1, K, dtype=dt)
    check_norm_args("rmsnorm", 1, K, dt, dev, None, w, 1e-6)
    check_norm_args("add_rmsnorm", 2, K, dt, dev, x2, w, 1e-6)
    check_norm_args("plain", 1, K, dt, dev, None, None, 1e-6)
    cases = [
        (("rmsnorm", 1, K, dt, dev, None, None, 1e-6), ValueError, "needs norm_weight"),
        (("rmsnorm", 1, K, dt, dev, None, torch.ones(K + 8, dtype=dt), 1e-6), ValueError, "shape"),
        (("rmsnorm", 1, K, dt, dev, None, torch.ones(K, dtype=torch.bfloat16), 1e-6), ValueError, "dtype"),
        (("rmsnorm", 1, K, dt, torch.device("cuda", 0), None, w, 1e-6), ValueError, "device"),
        (("rmsnorm", 1, K, dt, dev, None, torch.ones(2 * K, dtype=dt)[::2], 1e-6), ValueError, "contiguous"),
        (("rmsnorm", 1, K, dt, dev, None, w, 0.0), ValueError, "norm_eps"),
        (("add_rmsnorm", 1, K, dt, dev, None, w, 1e-6), ValueError, "residual as x2"),
        (("rmsnorm", 1, K, dt, dev, x2, w, 1e-6), ValueError, "takes no x2"),
        (("plain", 1, K, dt, dev, None, w, 1e-6), ValueError, "only used by"),
        (("rmsnorm", 1, 32768, dt, dev, None, torch.ones(32768, dtype=dt), 1e-6), NotImplementedError, "16384"),
    ]
    for args, exc, msg in cases:
        with pytest.raises(exc, match=msg):
            check_norm_args(*args)


def test_chain_mode_constants_match_the_header():
    import os
    import re

    from autogptq_b200 import _lib

    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "autogptq_b200.h")).read()
    for name, val in (("X_RMSNORM", _lib.CHAIN_X_RMSNORM), ("X_ADD_RMSNORM", _lib.CHAIN_X_ADD_RMSNORM),
                      ("NORM_MAX_K", _lib.CHAIN_NORM_MAX_K)):
        assert int(re.search(rf"#define AGB200_CHAIN_{name} (\d+)", hdr).group(1)) == val


def test_cnorm_layout_matches_the_header():
    import ctypes

    from autogptq_b200.chain import _CNorm, _CStage

    assert ctypes.sizeof(_CNorm) == 24 and _CNorm.eps.offset == 16
    assert ctypes.sizeof(_CStage) == 280           # unchanged: norm parameters travel in their own array


def _tiny_llama(**over):
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = dict(hidden_size=256, intermediate_size=512, num_attention_heads=2, num_key_value_heads=1,
               num_hidden_layers=2, vocab_size=64, max_position_embeddings=256)
    cfg.update(over)
    torch.manual_seed(0)
    return LlamaForCausalLM(LlamaConfig(**cfg))


def test_decoder_refuses_structurally_wrong_models():
    """ChainDecoder names the module and the reason before it touches a GPU."""
    from autogptq_b200.decoder import ChainDecoder, _check_window, _plan_layer

    m = _tiny_llama()
    with pytest.raises(NotImplementedError, match="batch 3"):
        ChainDecoder(m, batch=3)
    with pytest.raises(NotImplementedError, match=r"model\.layers\.0\.self_attn\.q_proj is Linear"):
        _plan_layer(0, m.model.layers[0], 1, torch.float32)
    with pytest.raises(NotImplementedError, match="sliding window of 64"):
        _check_window(type("C", (), {"sliding_window": 64})(), 128)
    _check_window(type("C", (), {"sliding_window": 64, "use_sliding_window": False})(), 128)
    _check_window(type("C", (), {"sliding_window": None})(), 128)
    with pytest.raises(NotImplementedError, match="not a \\*ForCausalLM"):
        ChainDecoder(torch.nn.Linear(4, 4))


def test_decoder_refuses_non_silu_mlp_and_other_norms():
    from autogptq_b200 import QuantLinear
    from autogptq_b200.decoder import _plan_layer

    m = _tiny_llama(hidden_act="gelu")
    layer = m.model.layers[0]
    for name in ("q_proj", "k_proj", "v_proj", "o_proj"):
        lin = getattr(layer.self_attn, name)
        setattr(layer.self_attn, name, QuantLinear(4, 128, lin.in_features, lin.out_features, False))
    with pytest.raises(NotImplementedError, match=r"mlp\.act_fn is .*not SiLU"):
        _plan_layer(0, layer, 1, torch.float32)
    m2 = _tiny_llama()
    layer = m2.model.layers[0]
    for mod, names in ((layer.self_attn, ("q_proj", "k_proj", "v_proj", "o_proj")), (layer.mlp, ("gate_proj", "up_proj", "down_proj"))):
        for name in names:
            lin = getattr(mod, name)
            setattr(mod, name, QuantLinear(4, 128, lin.in_features, lin.out_features, False))
    layer.input_layernorm = torch.nn.LayerNorm(256)
    with pytest.raises(NotImplementedError, match=r"input_layernorm is LayerNorm"):
        _plan_layer(0, layer, 1, torch.float32)
    layer.mlp.down_proj = torch.nn.Linear(512, 256)
    with pytest.raises(NotImplementedError, match=r"mlp\.down_proj is Linear"):
        _plan_layer(0, layer, 1, torch.float32)
