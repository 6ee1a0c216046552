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

``QuantExperts(..., input_grad=True)`` also backpropagates: ``hidden_states`` and ``top_k_weights`` get their gradients
from the grouped backward (``agb200_moe_backward``), so adapters of earlier layers and the router train on a frozen 4-bit
MoE checkpoint.  The expert weights get no gradient.
"""
from __future__ import annotations

import ctypes
import re
from ctypes import c_void_p
from typing import Dict, Mapping

import torch
import torch.nn as nn

from torch.autograd.function import once_differentiable

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
    """A created ``agb200_moe`` handle with its plan buffer and the tensors it points to (``arr``: the expert descriptors;
    ``grad``: the buffer of ``agb200_moe_grad_attach`` once attached)."""

    def __init__(self, handle, plan, keep, arr=None):
        self.handle, self.plan, self.keep, self.arr = handle, plan, keep, arr
        self.grad = None

    def __del__(self):
        if self.handle is not None and _lib._lib is not None:
            _lib._lib.agb200_moe_destroy(self.handle)
            self.handle = None


class QuantExperts(nn.Module):
    """E experts, each ``w2(silu(w1(x)) * w3(x))`` with 4-bit GPTQ ``QuantLinear`` layers, routed per token.

    All experts share the hidden size H (w1 / w3 in, w2 out), the intermediate size I and the group size.

    ``input_grad=True``: in grad mode, when ``hidden_states`` or ``top_k_weights`` requires grad, the forward keeps g, u
    and the per-pair outputs, ``(2 I + H) * T * k`` 16-bit values, until backward, which then computes both input
    gradients.  The default refuses grad mode instead, so that an inference model never holds that memory silently."""

    def __init__(self, w1s, w3s, w2s, *, input_grad: bool = False):
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
        self.input_grad = bool(input_grad)
        self._plans: Dict = {}     # (dtype, device index, with tensor-core copies) -> _Plan
        self._tc = False           # tensor-core copies built (first call with T > MOE_DECODE_MAX_T)

    @classmethod
    def from_linears(cls, w1s, w3s, w2s, *, input_grad: bool = False) -> "QuantExperts":
        return cls(w1s, w3s, w2s, input_grad=input_grad)

    def extra_repr(self) -> str:
        return (f"num_experts={self.num_experts}, hidden_size={self.hidden_size}, "
                f"intermediate_size={self.intermediate_size}, group_size={self.group_size}, input_grad={self.input_grad}, "
                "backend=sm_90a")

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
        plan = _Plan(handle.value, buf, keep, arr)
        self._plans[key] = plan
        return plan

    def _attach_grad(self, plan: _Plan, device) -> None:
        """Build the backward's per-expert data (tensor maps, inverse permutations) once per plan; synchronises."""
        if plan.grad is not None:
            return
        lib = _lib.load()
        nbytes = int(lib.agb200_moe_grad_plan_bytes(self.num_experts, self.hidden_size, self.intermediate_size,
                                                    self.group_size))
        buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            rc = lib.agb200_moe_grad_attach(plan.handle, ctypes.cast(plan.arr, c_void_p), buf.data_ptr(), nbytes)
        _lib.check(rc, "agb200_moe_grad_attach")
        plan.grad = buf

    def forward(self, hidden_states: torch.Tensor, top_k_index: torch.Tensor, top_k_weights: torch.Tensor) -> torch.Tensor:
        if hidden_states.device.type != "cuda":
            raise RuntimeError("autogptq_b200.QuantExperts.forward needs CUDA tensors (there is no CPU fallback).")
        grad = torch.is_grad_enabled() and (hidden_states.requires_grad or top_k_weights.requires_grad)
        if grad and not self.input_grad:
            raise NotImplementedError(
                "QuantExperts is inference-only unless built with input_grad=True: hidden_states and top_k_weights must "
                "not require grad (run it under torch.no_grad(), pass input_grad=True to QuantExperts / group_experts "
                "for the grouped backward, or use the experts' QuantLinear layers one by one).")
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
        if T == 0 and not grad:
            return torch.empty(out_shape, dtype=x_dtype, device=device)
        # the conversions are differentiable torch ops: gradients reach fp32 inputs in their own dtype
        x = x.to(cdtype).contiguous()
        if x.data_ptr() % 16:                        # the kernels read x in 16-byte words
            x = x.clone()
        idx = top_k_index.reshape(T, -1) if T else top_k_index.reshape(0, top_k_index.shape[-1])
        k = idx.shape[1]
        if idx.dtype not in (torch.int32, torch.int64):
            idx = idx.to(torch.int64)
        idx = idx.contiguous()
        w = top_k_weights.reshape(T, k)
        if w.dtype not in (torch.float32, cdtype):
            w = w.float()
        w = w.contiguous()
        if grad:
            out = _QuantExpertsFunction.apply(x, w, idx, self)
        else:
            out = self._forward(x, idx, w)[0]
        out = out.reshape(out_shape)
        return out if x_dtype == cdtype else out.to(x_dtype)

    def _static_buffers(self, T: int, k: int, dtype, device):
        """(plan, workspace) for ``_forward(..., out=, plan=, ws=)`` of up to T <= MOE_DECODE_MAX_T rows with k experts
        each: a caller that captures the forward in a CUDA graph owns both instead of the per-stream workspace cache."""
        if not 1 <= T <= _lib.MOE_DECODE_MAX_T:
            raise ValueError(f"static buffers are for decode rows, 1..{_lib.MOE_DECODE_MAX_T} (got {T})")
        device = torch.device(device)
        with torch.cuda.device(device):
            plan = self._plan(dtype, device)
            n = int(_lib.load().agb200_moe_workspace_bytes(T, k, self.num_experts, self.hidden_size,
                                                            self.intermediate_size))
        return plan, torch.empty(n, dtype=torch.uint8, device=device)

    def _forward(self, x: torch.Tensor, idx: torch.Tensor, w: torch.Tensor, save: bool = False, *, out=None,
                 plan: _Plan | None = None, ws: torch.Tensor | None = None):
        """(out [T, H], saved or None) of the grouped forward on prepared inputs (x [T, H] of the compute dtype,
        contiguous and 16-byte aligned; idx [T, k] int32 / int64; w [T, k] fp32 or the compute dtype).  ``save``: also
        keep what the backward reads (``agb200_moe_forward_saving``).  ``out``, ``plan`` and ``ws`` (from
        ``_static_buffers``): write into ``out`` with that plan and workspace, allocating nothing."""
        device, cdtype = x.device, x.dtype
        T, k = idx.shape
        H, E, I = self.hidden_size, self.num_experts, self.intermediate_size
        if out is None:
            out = torch.empty((T, H), dtype=cdtype, device=device)
        if T == 0:
            return out, (torch.empty(0, dtype=torch.uint8, device=device) if save else None)
        if plan is None:
            if T > _lib.MOE_DECODE_MAX_T and not self._tc:
                self._tc = True                      # same lazy rule as QuantLinear: tensor-core copies on first need
            plan = self._plan(cdtype, device)
        lib = _lib.load()
        ws_bytes = int(lib.agb200_moe_workspace_bytes(T, k, E, H, I))
        if ws is None:
            ws = _workspace(device, ws_bytes)
        elif ws.numel() < ws_bytes:
            raise ValueError(f"the workspace holds {ws.numel()} bytes, the forward needs {ws_bytes}")
        args = (plan.handle, x.data_ptr(), idx.data_ptr(),
                _lib.MOE_INDEX_I64 if idx.dtype == torch.int64 else _lib.MOE_INDEX_I32, w.data_ptr(),
                _lib.MOE_WEIGHTS_F32 if w.dtype == torch.float32 else _DTYPE_CODE[cdtype], T, k, out.data_ptr())
        saved = None
        with torch.cuda.device(device):
            if not save:
                rc = lib.agb200_moe_forward(*args, ws.data_ptr(), ws.numel(), torch.cuda.current_stream(device).cuda_stream)
            else:
                self._attach_grad(plan, device)
                nsaved = int(lib.agb200_moe_saved_bytes(T, k, E, H, I))
                saved = torch.empty(nsaved, dtype=torch.uint8, device=device)
                rc = lib.agb200_moe_forward_saving(*args, saved.data_ptr(), nsaved, ws.data_ptr(), ws.numel(),
                                                   torch.cuda.current_stream(device).cuda_stream)
        _lib.check(rc, "agb200_moe_forward_saving" if save else "agb200_moe_forward")
        return out, saved

    def _backward(self, dy: torch.Tensor, idx: torch.Tensor, w: torch.Tensor, saved: torch.Tensor, need_dx: bool,
                  need_dw: bool):
        """(dx [T, H] of the compute dtype or None, dw [T, k] of w's dtype or None) from dy [T, H] and the saved
        values of ``_forward(..., save=True)`` on the same x / idx / w."""
        T, k = idx.shape
        H, E, I = self.hidden_size, self.num_experts, self.intermediate_size
        device, cdtype = dy.device, dy.dtype
        dx = torch.empty((T, H), dtype=cdtype, device=device) if need_dx else None
        dw = torch.empty((T, k), dtype=w.dtype, device=device) if need_dw else None
        if T == 0 or not (need_dx or need_dw):
            return dx, dw
        plan = self._plan(cdtype, device)
        lib = _lib.load()
        ws_bytes = int(lib.agb200_moe_backward_workspace_bytes(T, k, E, H, I))
        ws = _workspace(device, ws_bytes)
        with torch.cuda.device(device):
            rc = lib.agb200_moe_backward(
                plan.handle, dy.data_ptr(), idx.data_ptr(),
                _lib.MOE_INDEX_I64 if idx.dtype == torch.int64 else _lib.MOE_INDEX_I32, w.data_ptr(),
                _lib.MOE_WEIGHTS_F32 if w.dtype == torch.float32 else _DTYPE_CODE[cdtype], T, k, saved.data_ptr(),
                saved.numel(), dx.data_ptr() if dx is not None else None, dw.data_ptr() if dw is not None else None,
                ws.data_ptr(), ws.numel(), torch.cuda.current_stream(device).cuda_stream)
        _lib.check(rc, "agb200_moe_backward")
        return dx, dw


class _QuantExpertsFunction(torch.autograd.Function):
    """out = QuantExperts._forward(x, idx, w) with dx and dw from ``agb200_moe_backward`` (the expert weights are frozen,
    top_k_index gets no gradient).  x and w arrive converted and contiguous; the conversions happen outside, as torch ops."""

    @staticmethod
    def forward(ctx, x, w, idx, qe):
        out, saved = qe._forward(x, idx, w, save=True)
        ctx.qe = qe
        ctx.save_for_backward(idx, w, saved)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        idx, w, saved = ctx.saved_tensors
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        dy = dy.contiguous()
        if dy.data_ptr() % 16:
            dy = dy.clone()
        dx, dw = ctx.qe._backward(dy, idx, w, saved, need_dx, need_dw)
        return dx, dw, None, None


def router_supported(T: int, H: int, E: int, k: int, dtype) -> str | None:
    """None when ``moe_router`` takes this shape, else the reason it does not."""
    if dtype not in _DTYPE_CODE:
        return f"dtype {dtype}; the router kernel computes in fp16 / bf16"
    if not 0 <= T <= _lib.MOE_DECODE_MAX_T:
        return f"{T} rows; the router kernel takes 0..{_lib.MOE_DECODE_MAX_T}"
    if H <= 0 or H % 128 or H > _lib.CHAIN_NORM_MAX_K:
        return f"hidden size {H}; the router kernel needs a multiple of 128 up to {_lib.CHAIN_NORM_MAX_K}"
    if not 1 <= k <= _lib.MOE_ROUTER_MAX_TOP_K:
        return f"top_k {k}; the router kernel takes 1..{_lib.MOE_ROUTER_MAX_TOP_K}"
    if not k <= E <= _lib.MOE_MAX_EXPERTS:
        return f"{E} experts; the router kernel takes top_k..{_lib.MOE_MAX_EXPERTS}"
    return None


def moe_router(x, x2, norm_weight, eps: float, gate_weight, k: int, *, h=None, n=None, idx=None, w=None, logits=None,
               pos=None):
    """The routing of a Mixtral-style block for decode rows in one launch (``agb200_moe_router``, DESIGN §3.17):

        h = x + x2 (skipped when x2 is None)   n = RMSNorm(h; norm_weight, eps)   logits = n · gate_weightᵀ
        p = softmax(fp32 logits)               idx = top-k of p (an exact tie to the lower expert)   w = p_idx / Σ p_idx

    with the roundings of transformers' MixtralDecoderLayer / MixtralRMSNorm / MixtralTopKRouter.  x, x2 [T, H] and
    norm_weight [H], gate_weight [E, H] of one 16-bit dtype.  Returns (h or None, n [T, H], idx int32 [T, k],
    w fp32 [T, k], logits [T, E] or None); ``h``, ``n``, ``idx`` and ``w`` are written in place when given (a decoder
    preallocates them), ``logits`` only when a buffer is given.  No host synchronisation.

    ``pos`` (int64 [T], ``agb200_moe_router_rows``): a row with pos < 0 is idle; it still gets h and n, but idx -1 and
    w 0 (so ``QuantExperts._forward`` gives it a zero row and streams no expert for it), and its logits row is not
    written.  Rows with pos >= 0 are bit-identical to a call without ``pos``."""
    if x.dim() != 2:
        raise ValueError(f"x must be [T, H], got {tuple(x.shape)}")
    T, H = x.shape
    dev, dt = x.device, x.dtype
    if dev.type != "cuda":
        raise RuntimeError("moe_router needs CUDA tensors (there is no CPU fallback)")
    if gate_weight.dim() != 2 or gate_weight.shape[1] != H:
        raise ValueError(f"gate_weight must be [E, {H}], got {tuple(gate_weight.shape)}")
    E = gate_weight.shape[0]
    why = router_supported(T, H, E, k, dt)
    if why is not None:
        raise NotImplementedError(f"moe_router: {why}")
    if h is None and x2 is not None:
        h = torch.empty((T, H), dtype=dt, device=dev)
    n = torch.empty((T, H), dtype=dt, device=dev) if n is None else n
    idx = torch.empty((T, k), dtype=torch.int32, device=dev) if idx is None else idx
    w = torch.empty((T, k), dtype=torch.float32, device=dev) if w is None else w
    checks = [("x", x, (T, H), dt), ("norm_weight", norm_weight, (H,), dt), ("gate_weight", gate_weight, (E, H), dt),
              ("n", n, (T, H), dt), ("idx", idx, (T, k), torch.int32), ("w", w, (T, k), torch.float32)]
    if x2 is not None:
        checks += [("x2", x2, (T, H), dt), ("h", h, (T, H), dt)]
    elif h is not None:
        raise ValueError("h is the residual x + x2; pass x2 or leave h out")
    if logits is not None:
        checks.append(("logits", logits, (T, E), dt))
    if pos is not None:
        checks.append(("pos", pos, (T,), torch.int64))
    for name, t, shape, tdt in checks:
        if tuple(t.shape) != shape or t.dtype != tdt:
            raise ValueError(f"{name} must be {tdt} {list(shape)}, got {t.dtype} {list(t.shape)}")
        if t.device != dev:
            raise ValueError(f"{name} is on {t.device}, x on {dev}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
        if t.dtype not in (torch.float32, torch.int32, torch.int64) and name != "logits" and t.data_ptr() % 16:
            raise ValueError(f"{name} must be 16-byte aligned")
    lib = _lib.load()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        if pos is None:
            rc = lib.agb200_moe_router(x.data_ptr(), _ptr(x2), norm_weight.data_ptr(), float(eps),
                                       gate_weight.data_ptr(), T, H, E, k, _DTYPE_CODE[dt], _ptr(h), n.data_ptr(),
                                       idx.data_ptr(), w.data_ptr(), _ptr(logits), stream)
        else:
            rc = lib.agb200_moe_router_rows(x.data_ptr(), _ptr(x2), norm_weight.data_ptr(), float(eps),
                                            gate_weight.data_ptr(), pos.data_ptr(), T, H, E, k, _DTYPE_CODE[dt],
                                            _ptr(h), n.data_ptr(), idx.data_ptr(), w.data_ptr(), _ptr(logits), stream)
    _lib.check(rc, "agb200_moe_router" if pos is None else "agb200_moe_router_rows")
    return h, n, idx, w, logits


def add_rmsnorm_supported(T: int, H: int, dtype) -> str | None:
    """None when ``add_rmsnorm`` takes this shape, else the reason it does not."""
    if dtype not in _DTYPE_CODE:
        return f"dtype {dtype}; the norm kernel computes in fp16 / bf16"
    if not 0 <= T <= _lib.MOE_DECODE_MAX_T:
        return f"{T} rows; the norm kernel takes 0..{_lib.MOE_DECODE_MAX_T}"
    if H <= 0 or H % 128 or H > _lib.CHAIN_NORM_MAX_K:
        return f"hidden size {H}; the norm kernel needs a multiple of 128 up to {_lib.CHAIN_NORM_MAX_K}"
    return None


def add_rmsnorm(x, x2, weight, eps: float, h=None, n=None):
    """The residual add and RMSNorm of decode rows in one launch (``agb200_add_rmsnorm``, DESIGN §3.18): the first
    phase of ``moe_router`` alone, so ``h`` and ``n`` are bit-equal to the router's on the same input.

        h = x + x2 (skipped when x2 is None)   n = RMSNorm(h; weight, eps)

    x, x2 [T, H] (T <= 8) and weight [H] of one 16-bit dtype.  Returns (h or None, n); ``h`` and ``n`` are written in
    place when given.  No host synchronisation."""
    if x.dim() != 2:
        raise ValueError(f"x must be [T, H], got {tuple(x.shape)}")
    T, H = x.shape
    dev, dt = x.device, x.dtype
    if dev.type != "cuda":
        raise RuntimeError("add_rmsnorm needs CUDA tensors (there is no CPU fallback)")
    why = add_rmsnorm_supported(T, H, dt)
    if why is not None:
        raise NotImplementedError(f"add_rmsnorm: {why}")
    if x2 is None and h is not None:
        raise ValueError("h is the residual x + x2; pass x2 or leave h out")
    if x2 is not None and h is None:
        h = torch.empty((T, H), dtype=dt, device=dev)
    n = torch.empty((T, H), dtype=dt, device=dev) if n is None else n
    checks = [("x", x, (T, H)), ("weight", weight, (H,)), ("n", n, (T, H))]
    if x2 is not None:
        checks += [("x2", x2, (T, H)), ("h", h, (T, H))]
    for name, t, shape in checks:
        if tuple(t.shape) != shape or t.dtype != dt:
            raise ValueError(f"{name} must be {dt} {list(shape)}, got {t.dtype} {list(t.shape)}")
        if t.device != dev:
            raise ValueError(f"{name} is on {t.device}, x on {dev}")
        if not t.is_contiguous() or t.data_ptr() % 16:
            raise ValueError(f"{name} must be contiguous and 16-byte aligned")
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.agb200_add_rmsnorm(x.data_ptr(), _ptr(x2), weight.data_ptr(), float(eps), T, H, _DTYPE_CODE[dt],
                                    _ptr(h), n.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(rc, "agb200_add_rmsnorm")
    return h, n


def group_experts(layers: Mapping[str, QuantLinear], pattern: str = EXPERT_PATTERN, *,
                  input_grad: bool = False) -> Dict[str, nn.Module]:
    """``{prefix: QuantLinear}`` (e.g. from ``checkpoint.load_quant_linears``) -> the same mapping with every
    ``<experts prefix>.<i>.w1|w2|w3`` family replaced by ONE ``QuantExperts`` under ``<experts prefix>``.

    ``pattern`` has three groups: the experts prefix, the expert number and the layer name (w1, w2 or w3).  Every
    other layer stays as it was.  ``input_grad`` is passed to every ``QuantExperts`` (see there)."""
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
                                                [experts[i]["w2"] for i in ids], input_grad=input_grad)
    return out


__all__ = ["QuantExperts", "group_experts", "EXPERT_PATTERN", "moe_router", "router_supported", "add_rmsnorm",
           "add_rmsnorm_supported"]
