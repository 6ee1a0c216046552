"""CPU tests of the fused-MLP injection (inject_fused_mlp / FusedQuantMLP): which modules are replaced and which are
left alone, unchanged state-dict keys, and the usual "no CPU fallback" error of the forward."""
import logging

import pytest
import torch
import torch.nn as nn

from autogptq_b200 import FusedQuantMLP, QuantLinear, forward_gate_up, inject_fused_mlp


class _MLP(nn.Module):
    """transformers' LlamaMLP shape: gate_proj, up_proj, down_proj and act_fn."""

    def __init__(self, H, I, act=None, down_quant=True, up_group=128):
        super().__init__()
        self.gate_proj = QuantLinear(4, 128, H, I, False)
        self.up_proj = QuantLinear(4, up_group, H, I, False)
        self.down_proj = QuantLinear(4, 128, I, H, False) if down_quant else nn.Linear(I, H, bias=False)
        self.act_fn = act if act is not None else nn.SiLU()

    def forward(self, x):
        return self.down_proj(self.act_fn(self.gate_proj(x)) * self.up_proj(x))


class _Block(nn.Module):
    def __init__(self, mlp):
        super().__init__()
        self.mlp = mlp
        self.norm = nn.LayerNorm(8)


def _model():
    return nn.ModuleDict({
        "layers": nn.ModuleList([_Block(_MLP(256, 512)), _Block(_MLP(256, 512))]),
        "gelu": _Block(_MLP(256, 512, act=nn.GELU())),
        "plain_down": _Block(_MLP(256, 512, down_quant=False)),
        "odd_i": _Block(_MLP(256, 264)),
        "two_groups": _Block(_MLP(256, 512, up_group=64)),
    })


def test_inject_selects_and_skips(caplog):
    model = _model()
    keys = set(model.state_dict())
    with caplog.at_level(logging.INFO, logger="autogptq_b200.mlp"):
        n = inject_fused_mlp(model)
    assert n == 2
    assert all(isinstance(b.mlp, FusedQuantMLP) for b in model["layers"])
    for name in ("gelu", "plain_down", "odd_i", "two_groups"):
        assert type(model[name].mlp) is _MLP, name
    assert set(model.state_dict()) == keys                  # same layers under the same names
    log = caplog.text
    assert "gelu.mlp skipped" in log and "GELU" in log
    assert "plain_down.mlp skipped" in log and "odd_i.mlp skipped" in log and "two_groups.mlp skipped" in log
    assert inject_fused_mlp(model) == 0                     # already injected


def test_inject_llama_mlp():
    transformers = pytest.importorskip("transformers")
    from transformers.models.llama.modeling_llama import LlamaMLP

    cfg = transformers.LlamaConfig(hidden_size=256, intermediate_size=512)
    root = nn.Module()
    root.mlp = LlamaMLP(cfg)
    for name in ("gate_proj", "up_proj", "down_proj"):
        lin = getattr(root.mlp, name)
        setattr(root.mlp, name, QuantLinear(4, 128, lin.in_features, lin.out_features, False))
    assert inject_fused_mlp(root) == 1 and isinstance(root.mlp, FusedQuantMLP)
    plain = nn.Module()
    plain.mlp = LlamaMLP(cfg)                              # nn.Linear layers: not ours, left alone
    assert inject_fused_mlp(plain) == 0 and isinstance(plain.mlp, LlamaMLP)


def test_mismatch_guard_catches_rounding_rule_errors():
    """The GPU tests allow MAX_MISMATCH of h to differ from the oracle at all; each plausible break of the rounding rule
    (silu(g) unrounded, g / u unrounded, only the product rounded) moves far more."""
    import numpy as np

    from oracle.moe_oracle import round_to as R, silu
    from tests._mlp_util import MAX_MISMATCH

    rng = np.random.default_rng(0)
    for dt in ("float16", "bfloat16"):
        g32 = (rng.standard_normal(100000) * 0.5).astype(np.float32)
        u32 = (rng.standard_normal(100000) * 0.5).astype(np.float32)
        g, u = R(g32, dt), R(u32, dt)
        ref = R(R(silu(g), dt) * u, dt)
        for name, wrong in (("silu unrounded", R(silu(g) * u, dt)), ("g, u unrounded", R(R(silu(g32), dt) * u32, dt)),
                            ("u unrounded", R(R(silu(g), dt) * u32, dt)), ("product only", R(silu(g32) * u32, dt))):
            assert np.mean(wrong != ref) > 4 * MAX_MISMATCH, (dt, name)


def test_forward_on_cpu_raises():
    model = _model()
    inject_fused_mlp(model)
    x = torch.zeros(2, 256, dtype=torch.float16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model["layers"][0].mlp(x)
    mlp = model["layers"][1].mlp
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        forward_gate_up(mlp.gate_proj, mlp.up_proj, x)
