"""CPU tests of the input gradient: the oracle against the reference's own autograd, the v10 exports, and the
inference path taking no autograd route."""
import ctypes

import numpy as np
import pytest
import torch

from autogptq_b200 import QuantLinear, _lib
from tests._dgrad_util import DGRAD_GOLDENS, dgrad, load_golden


@pytest.mark.parametrize("name", DGRAD_GOLDENS)
def test_oracle_reproduces_reference_gradients(name):
    d, z = load_golden(name)
    dx = dgrad(d, z["dy"])
    for key in ("dx_new", "dx_old"):
        if key in z:
            np.testing.assert_allclose(dx, z[key], rtol=1e-5, atol=1e-5 * np.abs(z[key]).max(), err_msg=f"{name} {key}")


def test_library_exports_v10_dgrad():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in ("agb200_w4a16_dgrad", "agb200_w4a16_dgrad_ex", "agb200_w4a16_dgrad_workspace_bytes"):
        assert hasattr(lib, name)
    L = _lib.load()
    assert L.agb200_abi_version() == 11
    assert L.agb200_w4a16_dgrad_workspace_bytes(3, 264, 64) == 1792       # 3 * 264 * 2 rounded up to 256 bytes


def test_inference_path_takes_no_autograd_route(monkeypatch):
    from autogptq_b200 import qlinear

    lin = QuantLinear(4, 128, 256, 256, False)
    seen = []
    monkeypatch.setattr(qlinear._QuantLinearFunction, "apply", staticmethod(lambda *a: seen.append("apply")))
    monkeypatch.setattr(QuantLinear, "_forward", lambda self, x: seen.append("plain"))
    x = torch.zeros(2, 256, dtype=torch.float16, requires_grad=True)
    with torch.no_grad():
        lin(x)
    with torch.inference_mode():
        lin(torch.zeros(2, 256, dtype=torch.float16))
    lin(torch.zeros(2, 256, dtype=torch.float16))                      # x does not require grad
    assert seen == ["plain"] * 3
    lin(x)
    assert seen[-1] == "apply"


def test_trainable_flag_still_refused_and_says_gradients_flow():
    with pytest.raises(NotImplementedError, match="input gradients flow"):
        QuantLinear(4, 128, 256, 256, False, trainable=True)
