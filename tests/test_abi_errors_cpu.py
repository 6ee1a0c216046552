"""Argument errors of every C-ABI unit: return code and exact agb200_last_error() text.

Each call fails before it touches the device, so these run without a GPU.  The pointers are fake device addresses
(never dereferenced); host-side structs are real.
"""
import ctypes
import re

import pytest
import torch

from autogptq_b200 import _lib
from autogptq_b200.chain import _CLayer as _ChainLayer, _CStage
from autogptq_b200.moe import _CExpert, _CLayer as _MoeLayer

EINVAL, ECUDA, ENOSUP, EWORKSPACE = -1, -2, -3, -4
A = 0x100000            # a 256-byte aligned fake device address
MIS = A + 8             # ... and one that is only 8-byte aligned


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def call(lib, name, *args):
    rc = getattr(lib, name)(*args)
    return rc, lib.agb200_last_error().decode()


def handle_out():
    return ctypes.byref(ctypes.c_void_p())


def fwd_args(x=A, qweight=A, qzeros=A, scales=A, y=A, M=1, K=128, N=128, group_size=128, dtype=_lib.F16):
    return (x, qweight, None, qzeros, scales, None, None, y, M, K, N, group_size, dtype, None, 0, None)


def test_w4a16_forward_errors(lib):
    assert call(lib, "agb200_w4a16_forward", *fwd_args(x=None, qweight=None, qzeros=None, scales=None, y=None)) == \
        (EINVAL, "null pointer argument")
    assert call(lib, "agb200_w4a16_forward_ex", *fwd_args(dtype=7), 0, 0, 0) == \
        (EINVAL, "dtype must be AGB200_F16 or AGB200_BF16")
    assert call(lib, "agb200_w4a16_forward_ex", *fwd_args(x=MIS), 0, 0, 0) == \
        (EINVAL, "x, qweight, scales and y must be 16-byte aligned")
    assert call(lib, "agb200_w4a16_forward_ex", *fwd_args(K=12), 0, 0, 0) == \
        (EINVAL, "infeatures K=12 must be a multiple of 8 (4-bit row packing)")
    assert call(lib, "agb200_w4a16_forward_ex", *fwd_args(group_size=12), 0, 0, 0) == \
        (ENOSUP, "group_size=12 is not a multiple of 8")


def test_forward_group_errors(lib):
    assert call(lib, "agb200_w4a16_forward_group", A, 0, None, None, None, None, None, None, None, None, 1, 128, 128,
                _lib.F16, None, 0, None) == (EINVAL, "forward_group: 1 <= n_layers <= 4 (got 0)")
    assert call(lib, "agb200_w4a16_forward_group", A, 2, None, None, None, None, None, None, None, None, 1, 128, 128,
                _lib.F16, None, 0, None) == (EINVAL, "null pointer argument")


def test_dgrad_errors(lib):
    dgrad = lambda dy, dx, dtype=_lib.F16: call(lib, "agb200_w4a16_dgrad_ex", dy, A, A, A, None, dx, 1, 128, 128, 128,
                                                 dtype, None, 0, None, 0, 0, 0)
    assert dgrad(A, A) == (EINVAL, "dgrad: dy and dx must not alias")
    assert dgrad(A, A + 256, dtype=5) == (EINVAL, "dtype must be AGB200_F16 or AGB200_BF16")
    assert dgrad(None, A) == (EINVAL, "null pointer argument")


def test_gate_up_errors(lib):
    good = _MoeLayer(qweight=A, qzeros=A, scales=A)
    bad = _MoeLayer(qweight=A + 4, qzeros=A, scales=A)

    def gate_up(gate, up, K=128, dtype=_lib.F16, kernel=0):
        return call(lib, "agb200_w4a16_gate_up_ex", A, gate, up, A, 1, K, 128, 128, dtype, None, 0, None, kernel, 0, 0)

    assert gate_up(None, ctypes.byref(good)) == (EINVAL, "gate_up: null layer descriptor")
    assert gate_up(ctypes.byref(good), ctypes.byref(good), dtype=3) == \
        (EINVAL, "gate_up: dtype must be AGB200_F16 or AGB200_BF16")
    assert gate_up(ctypes.byref(good), ctypes.byref(good), kernel=9) == (EINVAL, "gate_up: unknown kernel 9")
    assert gate_up(ctypes.byref(good), ctypes.byref(bad)) == (EINVAL, "gate_up: layer buffers must be 16-byte aligned")
    assert gate_up(ctypes.byref(good), ctypes.byref(good), K=12) == \
        (ENOSUP, "gate_up: K % 8 == 0 and I % 32 == 0 (got K=12, I=128)")
    assert call(lib, "agb200_w4a16_gate_up_saving_ex", A, ctypes.byref(good), ctypes.byref(good), A, None, None, 1, 128,
                128, 128, _lib.F16, None, 0, None, 0, 0, 0) == (EINVAL, "gate_up_saving: null g or u")


def test_mlp_backward_errors(lib):
    lay = _MoeLayer(qweight=A, qzeros=A, scales=A)
    L = ctypes.byref(lay)

    def mlp_bwd(dy=A, dx=A + 256, ws_bytes=100, gate=L):
        return call(lib, "agb200_w4a16_mlp_backward_ex", dy, gate, L, L, A, A, dx, 1, 128, 128, 128, 128, _lib.F16, A,
                    ws_bytes, None, 0, 0)

    assert mlp_bwd(gate=None) == (EINVAL, "mlp_backward: null layer descriptor")
    assert mlp_bwd(dx=A) == (EINVAL, "mlp_backward: dy and dx must not alias")
    assert mlp_bwd(dy=MIS) == \
        (EINVAL, "mlp_backward: dy, g, u and dx must be 16-byte aligned, the workspace 256-byte aligned")
    need = lib.agb200_w4a16_mlp_backward_workspace_bytes(1, 128, 128)
    assert need == 768
    assert mlp_bwd() == (EWORKSPACE, "mlp_backward: workspace needs 768 bytes (got 100)")


def test_moe_errors(lib):
    experts = (_CExpert * 1)()
    assert call(lib, "agb200_moe_create", None, 1, 128, 128, 128, _lib.F16, A, 1 << 20, handle_out()) == \
        (EINVAL, "moe: null pointer argument")
    assert call(lib, "agb200_moe_create", experts, 0, 128, 128, 128, _lib.F16, A, 1 << 20, handle_out()) == \
        (ENOSUP, "moe: 1 <= E <= 256 experts (got 0)")
    assert call(lib, "agb200_moe_create", experts, 1, 128, 128, 128, 9, A, 1 << 20, handle_out()) == \
        (EINVAL, "moe: dtype must be AGB200_F16 or AGB200_BF16")
    need = lib.agb200_moe_plan_bytes(1, 128, 128, 128)
    assert call(lib, "agb200_moe_create", experts, 1, 128, 128, 128, _lib.F16, A, 64, handle_out()) == \
        (EWORKSPACE, f"moe: plan buffer needs {need} bytes, 256-byte aligned (got 64)")
    fake = ctypes.create_string_buffer(256)          # host memory without the plan's magic word
    for handle in (None, ctypes.addressof(fake)):
        assert call(lib, "agb200_moe_forward", handle, A, A, 0, A, 2, 1, 2, A, A, 1 << 20, None) == \
            (EINVAL, "moe: bad handle")
    assert call(lib, "agb200_moe_backward", None, A, A, 0, A, 2, 1, 2, A, 1 << 20, A, A, A, 1 << 20, None) == \
        (EINVAL, "moe: bad handle")


def test_moe_router_errors(lib):
    def router(x=A, T=1, H=128, E=8, k=2):
        return call(lib, "agb200_moe_router", x, None, A, 1e-6, A, T, H, E, k, _lib.F16, None, A, A, A, None, None)

    assert router(x=None) == (EINVAL, "moe_router: null pointer argument")
    assert router(x=MIS) == (EINVAL, "moe_router: x, x2, norm_weight, gate_weight, h and n must be 16-byte aligned")
    assert router(T=9) == (ENOSUP, "moe_router: T=9 rows; at most 8")
    assert router(k=9) == (ENOSUP, "moe_router: k=9; at most 8")


def test_chain_errors(lib):
    stages = (_CStage * 1)()
    stages[0].K, stages[0].group_size, stages[0].n_layers, stages[0].x = 128, 128, 1, A
    stages[0].layer[0] = _ChainLayer(qweight=A, qzeros=A, scales=A, y=A, N=128)
    create = lambda st, n=1, M=1, plan_bytes=1 << 24: call(lib, "agb200_chain_create_norm", st, None, n, M, _lib.F16, A,
                                                           plan_bytes, handle_out())
    assert create(None) == (EINVAL, "chain: null pointer argument")
    assert create(stages, n=0) == (EINVAL, "chain: 1 <= n_stages <= 65535 (got 0)")
    assert create(stages, M=3) == (ENOSUP, "chain: 1 <= M <= 2 rows (got 3)")
    need = lib.agb200_chain_plan_bytes_norm(stages, None, 1, 1)
    assert create(stages, plan_bytes=256) == \
        (EWORKSPACE, f"chain: plan buffer needs {need} bytes, 256-byte aligned (got 256)")
    stages[0].n_layers = 0
    assert create(stages) == (EINVAL, "chain stage 0: 1 <= n_layers <= 4 (got 0)")
    assert call(lib, "agb200_chain_forward", None, 0, None) == (EINVAL, "chain: bad handle")
    assert call(lib, "agb200_chain_info", None, None, None, None) == (EINVAL, "chain: bad handle")


def test_gptq_errors(lib):
    assert call(lib, "agb200_gptq_hessian_update", None, A, 1, 128, _lib.F16, 1.0, 0.0, None) == \
        (EINVAL, "gptq_hessian_update: null pointer argument")
    assert call(lib, "agb200_gptq_hessian_update", A, A, 1, 12, _lib.F16, 1.0, 0.0, None) == \
        (EINVAL, "gptq_hessian_update: need T >= 0 and K > 0, K % 8 == 0 (got T=1, K=12)")
    assert call(lib, "agb200_gptq_hessian_update", MIS, A, 1, 128, _lib.F16, 1.0, 0.0, None) == \
        (EINVAL, "gptq_hessian_update: x and H must be 16-byte aligned")

    def quantize(group_size=-1, ws_bytes=16):
        return call(lib, "agb200_gptq_quantize", A, A, None, None, 8, 8, group_size, 0, 0, A, A, A, A, A, A, None,
                    _lib.F16, A, ws_bytes, None)

    assert quantize(group_size=12) == (ENOSUP, "gptq_quantize: group_size must be -1 or a positive multiple of 8 (got 12)")
    assert quantize() == (EWORKSPACE, "gptq_quantize: workspace needs 256 bytes (got 16)")


def test_decode_attention_errors(lib):
    def attn(q=A, head_dim=128, ws_bytes=256):
        return call(lib, "agb200_decode_attention", q, A, A, A, A, A, A, 1.0, 1.0, A, 1, 32, 8, head_dim, 4096,
                    _lib.F16, A, ws_bytes, None)

    assert attn(q=None) == (EINVAL, "decode_attention: null pointer argument")
    assert attn(head_dim=96) == (ENOSUP, "decode_attention: head_dim 96; supported: 64, 128")
    need = lib.agb200_decode_attention_workspace_bytes(1, 32, 8, 128, 4096)
    assert attn() == (EWORKSPACE, f"decode_attention: workspace needs {need} bytes (got 256)")


def test_decode_attention_workspace_without_device_query():
    """The size query has no error channel: without a usable device it plans for 132 SMs."""
    if torch.cuda.is_available() and torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the value below is the one for 132 SMs")
    assert _lib.load().agb200_decode_attention_workspace_bytes(1, 32, 8, 128, 4096) == 1081600


@pytest.mark.skipif(torch.cuda.is_available(), reason="needs a machine without a usable CUDA device")
def test_device_query_failure_is_ecuda(lib):
    """Valid-looking arguments reach the device query, whose failure is recorded as '<expression>: <CUDA error>'."""
    msgs = []
    rc, msg = call(lib, "agb200_gptq_hessian_update", A, A, 1, 128, _lib.F16, 1.0, 0.0, None)
    assert rc == ECUDA
    msgs.append(msg)
    rc, msg = call(lib, "agb200_w4a16_forward", *fwd_args())
    assert rc == ECUDA
    msgs.append(msg)
    for m in msgs:
        assert re.fullmatch(r"cudaGetDevice\(&dev\): \S.*", m), m
    assert msgs[0] == msgs[1]        # one recorder, one message shape for every unit
