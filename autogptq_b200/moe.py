"""Routed experts of a Mixtral-style block as ONE grouped W4A16 forward (``agb200_moe_*``).

    from autogptq_b200 import checkpoint, group_experts
    layers = group_experts(checkpoint.load_quant_linears(path, device="cuda"))
    block.experts = layers["model.layers.0.block_sparse_moe.experts"]      # a QuantExperts

``QuantExperts.forward(hidden_states, top_k_index, top_k_weights)`` has the signature and meaning of transformers'
``MixtralExperts.forward`` (``transformers/models/mixtral/modeling_mixtral.py:74-98``) for the experts the reference
quantises (``auto_gptq/modeling/mixtral.py:4-39``: every expert's w1 / w3 / w2 is a 4-bit ``QuantLinear``).  The
reference loop finds the hit experts with ``nonzero()`` (a host synchronisation) and runs three ``QuantLinear`` calls
plus a dozen small ops per hit expert; here the routing stays on the device and the block is one fixed sequence of
launches (CUDA-graph capturable, replayable with new routing).  The checkpoint tensors of the experts stay where they
are: the library reads them in place.  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes
import re
from ctypes import c_void_p
from typing import Dict, Mapping

import torch
import torch.nn as nn

from . import _lib
from .qlinear import _DTYPE_CODE, QuantLinear, _workspace

EXPERT_PATTERN = r"(.*\.experts)\.(\d+)\.(w1|w2|w3)$"


class _CLayer(ctypes.Structure):
    _fields_ = [("qweight", c_void_p), ("qweight_tc", c_void_p), ("qzeros", c_void_p), ("scales", c_void_p),
                ("perm", c_void_p), ("bias", c_void_p)]


class _CExpert(ctypes.Structure):
    _fields_ = [("w1", _CLayer), ("w3", _CLayer), ("w2", _CLayer)]


def _ptr(t):
    return t.data_ptr() if t is not None else None


class _Plan:
    """A created ``agb200_moe`` handle with its plan buffer and the tensors it points to."""

    def __init__(self, handle, plan, keep):
        self.handle, self.plan, self.keep = handle, plan, keep

    def __del__(self):
        if self.handle is not None and _lib._lib is not None:
            _lib._lib.agb200_moe_destroy(self.handle)
            self.handle = None


class QuantExperts(nn.Module):
    """E experts, each ``w2(silu(w1(x)) * w3(x))`` with 4-bit GPTQ ``QuantLinear`` layers, routed per token.

    All experts share the hidden size H (w1 / w3 in, w2 out), the intermediate size I and the group size."""

    def __init__(self, w1s, w3s, w2s):
        super().__init__()
        w1s, w3s, w2s = list(w1s), list(w3s), list(w2s)
        if not w1s or not (len(w1s) == len(w3s) == len(w2s)):
            raise ValueError(f"need the same non-zero number of w1, w3 and w2 layers (got {len(w1s)}, {len(w3s)}, {len(w2s)})")
        for lin in w1s + w3s + w2s:
            if not isinstance(lin, QuantLinear):
                raise TypeError(f"QuantExperts takes autogptq_b200.QuantLinear layers, got {type(lin).__name__}")
        E = len(w1s)
        H, I = w1s[0].infeatures, w1s[0].outfeatures
        if E > _lib.MOE_MAX_EXPERTS:
            raise NotImplementedError(f"{E} experts: the grouped kernels handle at most {_lib.MOE_MAX_EXPERTS}")
        for e in range(E):
            for name, lin, shape in (("w1", w1s[e], (H, I)), ("w3", w3s[e], (H, I)), ("w2", w2s[e], (I, H))):
                if (lin.infeatures, lin.outfeatures) != shape:
                    raise NotImplementedError(
                        f"expert {e} {name} is {lin.infeatures}x{lin.outfeatures}, expected {shape[0]}x{shape[1]}: "
                        "all experts must share the hidden and intermediate sizes of expert 0")
        if H % 128 or I % 128:
            raise NotImplementedError(f"hidden size {H} and intermediate size {I} must be multiples of 128")
        g13 = {lin.group_size for lin in w1s + w3s}
        g2 = {lin.group_size for lin in w2s}
        if len(g13) != 1 or len(g2) != 1:
            raise NotImplementedError(f"all experts must share one group size (w1/w3: {sorted(g13)}, w2: {sorted(g2)})")
        g13, g2 = g13.pop(), g2.pop()
        if g13 == g2:
            group_size = g13
        elif g13 == H and g2 == I:
            group_size = -1                       # one group per layer (group_size=-1 in the checkpoint)
        else:
            raise NotImplementedError(f"w1/w3 group size {g13} and w2 group size {g2} differ")
        if group_size != -1 and group_size != 32 and group_size % 64:
            raise NotImplementedError(f"group_size={group_size}: the grouped kernels need 32, a multiple of 64, or -1")
        self.w1, self.w3, self.w2 = nn.ModuleList(w1s), nn.ModuleList(w3s), nn.ModuleList(w2s)
        self.num_experts, self.hidden_size, self.intermediate_size = E, H, I
        self.group_size = group_size
        self._plans: Dict = {}     # (dtype, device index, with tensor-core copies) -> _Plan
        self._tc = False           # tensor-core copies built (first call with T > MOE_DECODE_MAX_T)

    @classmethod
    def from_linears(cls, w1s, w3s, w2s) -> "QuantExperts":
        return cls(w1s, w3s, w2s)

    def extra_repr(self) -> str:
        return (f"num_experts={self.num_experts}, hidden_size={self.hidden_size}, "
                f"intermediate_size={self.intermediate_size}, group_size={self.group_size}, backend=sm_90a")

    def _layers(self):
        return list(self.w1) + list(self.w3) + list(self.w2)

    def _plan(self, dtype, device) -> _Plan:
        key = (dtype, device.index, self._tc)
        plan = self._plans.get(key)
        if plan is not None:
            return plan
        lib = _lib.load()
        for lin in self._layers():
            if not lin._ready or lin._qweight_run is None or lin._qweight_run.device != device:
                lin.post_init()
            if self._tc and lin._qweight_tc is None:
                lin._prepare_tc()
        E, H, I = self.num_experts, self.hidden_size, self.intermediate_size
        arr = (_CExpert * E)()
        keep = []
        for e in range(E):
            p1, p3 = self.w1[e]._perm, self.w3[e]._perm
            if (p1 is None) != (p3 is None) or (p1 is not None and not torch.equal(p1, p3)):
                raise NotImplementedError(f"expert {e}: w1 and w3 must share one act-order permutation of x")
            for field, lin in (("w1", self.w1[e]), ("w3", self.w3[e]), ("w2", self.w2[e])):
                scales, bias = lin._run_tensors(dtype)
                perm = p1 if field in ("w1", "w3") else lin._perm
                keep.extend(t for t in (scales, bias, perm) if t is not None)
                L = getattr(arr[e], field)
                L.qweight, L.qzeros, L.scales = lin._qweight_run.data_ptr(), lin.qzeros.data_ptr(), scales.data_ptr()
                L.qweight_tc = _ptr(lin._qweight_tc) if self._tc else None
                L.perm, L.bias = _ptr(perm), _ptr(bias)
        nbytes = int(lib.agb200_moe_plan_bytes(E, H, I, self.group_size))
        buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        handle = c_void_p()
        with torch.cuda.device(device):
            rc = lib.agb200_moe_create(ctypes.cast(arr, c_void_p), E, H, I, self.group_size, _DTYPE_CODE[dtype],
                                       buf.data_ptr(), nbytes, ctypes.byref(handle))
        _lib.check(rc, "agb200_moe_create")
        plan = _Plan(handle.value, buf, keep)
        self._plans[key] = plan
        return plan

    def forward(self, hidden_states: torch.Tensor, top_k_index: torch.Tensor, top_k_weights: torch.Tensor) -> torch.Tensor:
        if hidden_states.device.type != "cuda":
            raise RuntimeError("autogptq_b200.QuantExperts.forward needs CUDA tensors (there is no CPU fallback).")
        device = hidden_states.device
        if top_k_index.device != device or top_k_weights.device != device:
            raise RuntimeError("hidden_states, top_k_index and top_k_weights must be on the same CUDA device")
        H = self.hidden_size
        if hidden_states.shape[-1] != H:
            raise RuntimeError(f"hidden_states has {hidden_states.shape[-1]} features, the experts expect {H}")
        x_dtype = hidden_states.dtype
        cdtype = x_dtype if x_dtype in _DTYPE_CODE else torch.float16
        x = hidden_states.reshape(-1, H)
        T = x.shape[0]
        out_shape = hidden_states.shape[:-1] + (H,)
        if T == 0:
            return torch.empty(out_shape, dtype=x_dtype, device=device)
        x = x.to(cdtype).contiguous()
        idx = top_k_index.reshape(T, -1)
        k = idx.shape[1]
        if idx.dtype not in (torch.int32, torch.int64):
            idx = idx.to(torch.int64)
        idx = idx.contiguous()
        w = top_k_weights.reshape(T, k)
        if w.dtype not in (torch.float32, cdtype):
            w = w.float()
        w = w.contiguous()
        if T > _lib.MOE_DECODE_MAX_T and not self._tc:
            self._tc = True                          # same lazy rule as QuantLinear: tensor-core copies on first need
        plan = self._plan(cdtype, device)
        lib = _lib.load()
        E, I = self.num_experts, self.intermediate_size
        ws_bytes = int(lib.agb200_moe_workspace_bytes(T, k, E, H, I))
        ws = _workspace(device, ws_bytes)
        out = torch.empty((T, H), dtype=cdtype, device=device)
        with torch.cuda.device(device):
            rc = lib.agb200_moe_forward(
                plan.handle, x.data_ptr(), idx.data_ptr(),
                _lib.MOE_INDEX_I64 if idx.dtype == torch.int64 else _lib.MOE_INDEX_I32, w.data_ptr(),
                _lib.MOE_WEIGHTS_F32 if w.dtype == torch.float32 else _DTYPE_CODE[cdtype], T, k, out.data_ptr(),
                ws.data_ptr(), ws.numel(), torch.cuda.current_stream(device).cuda_stream)
        _lib.check(rc, "agb200_moe_forward")
        out = out.reshape(out_shape)
        return out if x_dtype == cdtype else out.to(x_dtype)


def group_experts(layers: Mapping[str, QuantLinear], pattern: str = EXPERT_PATTERN) -> Dict[str, nn.Module]:
    """``{prefix: QuantLinear}`` (e.g. from ``checkpoint.load_quant_linears``) -> the same mapping with every
    ``<experts prefix>.<i>.w1|w2|w3`` family replaced by ONE ``QuantExperts`` under ``<experts prefix>``.

    ``pattern`` has three groups: the experts prefix, the expert number and the layer name (w1, w2 or w3).  Every
    other layer stays as it was."""
    rx = re.compile(pattern)
    out: Dict[str, nn.Module] = {}
    groups: Dict[str, Dict[int, Dict[str, QuantLinear]]] = {}
    for name, lin in layers.items():
        m = rx.match(name)
        if m is None:
            out[name] = lin
            continue
        groups.setdefault(m.group(1), {}).setdefault(int(m.group(2)), {})[m.group(3)] = lin
    for prefix, experts in groups.items():
        ids = sorted(experts)
        if ids != list(range(len(ids))):
            raise ValueError(f"{prefix}: experts {ids} are not numbered 0..{len(ids) - 1}")
        for i in ids:
            missing = {"w1", "w2", "w3"} - set(experts[i])
            if missing:
                raise ValueError(f"{prefix}.{i}: missing {sorted(missing)}")
        out[prefix] = QuantExperts.from_linears([experts[i]["w1"] for i in ids], [experts[i]["w3"] for i in ids],
                                                [experts[i]["w2"] for i in ids])
    return out


__all__ = ["QuantExperts", "group_experts", "EXPERT_PATTERN"]
