"""CPU tests of the fused MLP backward's plumbing (``FusedQuantMLP(fused_backward=True)``): the flag through
``inject_fused_mlp``, which MLPs the fused backward takes, the "no CPU fallback" error and the new C-ABI bindings."""
import ctypes

import pytest
import torch
import torch.nn as nn

from autogptq_b200 import FusedQuantMLP, QuantLinear, _lib, inject_fused_mlp
from autogptq_b200.mlp import _dgrad_tc_supported, _fused_backward_unfit


class _MLP(nn.Module):
    def __init__(self, H=256, I=512, g=128):
        super().__init__()
        self.gate_proj = QuantLinear(4, g, H, I, False)
        self.up_proj = QuantLinear(4, g, H, I, False)
        self.down_proj = QuantLinear(4, g, I, H, False)
        self.act_fn = nn.SiLU()


class _Wrap(nn.Module):
    def __init__(self, inner):
        super().__init__()
        self.inner = inner

    def forward(self, x):
        return self.inner(x)


def _layers(H=256, I=512, g13=128, g2=128):
    return QuantLinear(4, g13, H, I, False), QuantLinear(4, g13, H, I, False), QuantLinear(4, g2, I, H, False)


def test_default_is_off_and_inject_passes_the_flag():
    assert FusedQuantMLP(*_layers()).fused_backward is False
    assert "fused_backward=False" in repr(FusedQuantMLP(*_layers()))
    for flag in (False, True):
        root = nn.ModuleDict({"a": nn.ModuleDict({"mlp": _MLP()}), "b": nn.ModuleDict({"mlp": _MLP()})})
        assert (inject_fused_mlp(root, fused_backward=flag) if flag else inject_fused_mlp(root)) == 2
        for k in ("a", "b"):
            assert isinstance(root[k]["mlp"], FusedQuantMLP) and root[k]["mlp"].fused_backward is flag
            assert f"fused_backward={flag}" in repr(root[k]["mlp"])


def test_eligibility():
    ok = _layers()
    assert _fused_backward_unfit(*ok, torch.float16) == ""
    assert _fused_backward_unfit(*ok, torch.bfloat16) == ""
    assert "float32" in _fused_backward_unfit(*ok, torch.float32)
    assert "I % 64" in _fused_backward_unfit(*_layers(I=800, g13=32, g2=32), torch.float16)
    assert _fused_backward_unfit(*_layers(H=1152, I=2304, g13=96, g2=96), torch.float16) == ""    # 96: a tensor-core dgrad
    assert "tensor-core dgrad" in _fused_backward_unfit(*_layers(g13=128, g2=8), torch.float16)
    g, u, d = _layers()
    assert "different group sizes" in _fused_backward_unfit(g, QuantLinear(4, 64, 256, 512, False), d, torch.float16)
    assert "not a bare" in _fused_backward_unfit(g, u, _Wrap(d), torch.float16)
    assert "not a bare" in _fused_backward_unfit(g, u, nn.Linear(512, 256), torch.float16)
    assert "expected 512x256" in _fused_backward_unfit(g, u, QuantLinear(4, 128, 512, 384, False), torch.float16)
    d.kernel = _lib.KERNEL_GEMM
    assert "forced" in _fused_backward_unfit(g, u, d, torch.float16)
    g, u, d = _layers()
    g._perm = torch.arange(256, dtype=torch.int32).flip(0)
    u._perm = torch.arange(256, dtype=torch.int32)
    assert "different act-order" in _fused_backward_unfit(g, u, d, torch.float16)
    u._perm = g._perm.clone()                                   # equal permutations (compared by value) are shared
    assert _fused_backward_unfit(g, u, d, torch.float16) == ""


def test_dgrad_tc_rule_matches_the_header():
    # the C rule (csrc/dgrad_common.cuh): N % 32 == 0 and (group >= 32 and a multiple of 16, or one group)
    assert _dgrad_tc_supported(4096, 11008, 128) and _dgrad_tc_supported(11008, 4096, 11008)
    assert not _dgrad_tc_supported(4096, 11008, 8) and not _dgrad_tc_supported(4096, 11008, 40)
    assert not _dgrad_tc_supported(256, 528, 128)


def test_cpu_tensor_raises():
    mlp = FusedQuantMLP(*_layers(), fused_backward=True)
    x = torch.zeros(2, 256, dtype=torch.float16, requires_grad=True)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        mlp(x)
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU fallback"):
        mlp(x)


def test_new_exports():
    names = set(_lib.declared_symbols())
    for n in ("agb200_w4a16_gate_up_saving", "agb200_w4a16_gate_up_saving_ex", "agb200_w4a16_mlp_backward",
              "agb200_w4a16_mlp_backward_ex", "agb200_w4a16_mlp_backward_workspace_bytes"):
        assert n in names
    P, I, S = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t

    class _Rec:
        def __getattr__(self, k):
            class F:
                restype = None
                argtypes = None
            f = F()
            self.__dict__[k] = f
            return f
    rec = _Rec()
    _lib._declare(rec)
    sig = lambda n: list(rec.__dict__[n].argtypes)      # noqa: E731
    assert sig("agb200_w4a16_gate_up_saving") == [P] * 6 + [I] * 5 + [P, S, P]
    assert sig("agb200_w4a16_gate_up_saving_ex") == [P] * 6 + [I] * 5 + [P, S, P] + [I] * 3
    assert sig("agb200_w4a16_mlp_backward") == [P] * 7 + [I] * 6 + [P, S, P]
    assert sig("agb200_w4a16_mlp_backward_ex") == [P] * 7 + [I] * 6 + [P, S, P, I, I]
    assert sig("agb200_w4a16_mlp_backward_workspace_bytes") == [I] * 3
    assert rec.__dict__["agb200_w4a16_mlp_backward_workspace_bytes"].restype is S
