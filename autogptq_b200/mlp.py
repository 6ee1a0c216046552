"""Fused gate/up of a dense Llama-style MLP (``agb200_w4a16_gate_up``) and the module that injects it into a model.

    from autogptq_b200 import inject_fused_mlp
    n = inject_fused_mlp(model)          # every LlamaMLP-shaped submodule over QuantLinear layers -> FusedQuantMLP

``inject_fused_mlp(model, fused_backward=True)`` also fuses the backward for adapter training on a frozen 4-bit base:
the forward keeps g and u only, and dx comes from two launches (``agb200_w4a16_mlp_backward``) instead of the unfused
layers' eight or so.

``forward_gate_up(gate_proj, up_proj, x)`` computes ``F.silu(gate_proj(x)) * up_proj(x)`` in one launch: both layers'
weights are streamed by the same CTAs and only ``h`` is written, where the unfused module runs gate, up, ``silu`` and
``*`` as four launches and moves ``g``, ``u``, ``silu(g)`` and ``h`` through device memory.  The roundings are the
reference's (its 16-bit ``act_fn(gate) * up``).  The reference's counterpart is ``inject_fused_mlp=True``
(``auto_gptq/nn_modules/fused_llama_mlp.py:131-245``), whose Triton kernels read the packed buffers directly; here the
checkpoint tensors of the ``QuantLinear`` layers are used in place.  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes
from ctypes import c_void_p
from logging import getLogger

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from . import _lib
from .moe import _CLayer, _ptr
from .qlinear import _DTYPE_CODE, QuantLinear, _workspace

logger = getLogger(__name__)

# Above this many rows the unfused layers are faster: at Llama-2-7B MLP shapes on one H100 80GB HBM3 (700 W) the fused
# module measured 1.06-1.09x the unfused one at M = 1024 and the fused GEMM 0.89-0.98x at M = 4096 in three runs
# (tools/mlp_bench.py; both compute-bound there)
FUSED_MAX_M = 2048

# FusedQuantMLP(fused_backward=True) runs the fused backward up to this many rows and the unfused autograd path above
# it.  At Llama-2-7B MLP shapes (g 128) on one H100 80GB HBM3 (700 W), forward + backward took 0.88-0.90x the unfused
# path's time at M = 16 and 64 and 1.04-1.19x at M = 256 ... 8192 (tools/mlp_grad_bench.py, fp16 and bf16, medians
# of 3 alternating rounds, spreads far apart); M between 64 and 256 is not measured and takes the unfused path.
FUSED_BACKWARD_MAX_M = 64


def _unfused(gate_proj, up_proj, x):
    return F.silu(gate_proj(x)) * up_proj(x)


def _shared_perm(gate_proj, up_proj):
    """The act-order permutation both layers use, None for sequential layers, or False when they differ."""
    p, q = gate_proj._perm, up_proj._perm
    if p is None and q is None:
        return None
    if p is None or q is None or p.shape != q.shape or not torch.equal(p, q):
        return False
    return p


def _pair_perm(gate_proj, up_proj):
    """``_shared_perm`` of the pair, cached: the comparison synchronises with the device, so it is made once per
    (re)initialised pair and later calls can be captured in a CUDA graph.  Cache entries hold the tensors they were made
    from and are matched by identity, so a post_init() that replaces any of them rebuilds them."""
    cache = gate_proj.__dict__.setdefault("_gate_up_cache", {})
    pent = cache.get(("perm", id(up_proj)))
    if pent is None or not _same((up_proj, gate_proj._perm, up_proj._perm), pent[0]):
        pent = ((up_proj, gate_proj._perm, up_proj._perm), _shared_perm(gate_proj, up_proj))
        cache[("perm", id(up_proj))] = pent
    return pent[1]


def _fusable(gate_proj, up_proj) -> str:
    """Why the pair cannot run through the fused kernels (empty string: it can, at least at some M)."""
    if not isinstance(gate_proj, QuantLinear) or not isinstance(up_proj, QuantLinear):
        return "gate_proj / up_proj are not autogptq_b200.QuantLinear"
    if gate_proj.infeatures != up_proj.infeatures or gate_proj.outfeatures != up_proj.outfeatures:
        return "gate_proj and up_proj have different shapes"
    if gate_proj.group_size != up_proj.group_size:
        return "gate_proj and up_proj have different group sizes"
    if gate_proj.infeatures % 8 or gate_proj.outfeatures % 32:
        return f"the fused kernels need K % 8 == 0 and I % 32 == 0 (K={gate_proj.infeatures}, I={gate_proj.outfeatures})"
    return ""


class _PairArgs:
    """ctypes layer descriptors of a (gate, up) pair for one compute dtype (built once, reused every call)."""

    def __init__(self, gate_proj, up_proj, perm, dtype, tc):
        self.keep = []
        self.gate, self.up = _CLayer(), _CLayer()
        for L, lin in ((self.gate, gate_proj), (self.up, up_proj)):
            scales, bias = lin._run_tensors(dtype)
            self.keep += [scales, bias, perm, lin._qweight_run, lin._qweight_tc]
            L.qweight, L.qzeros, L.scales = lin._qweight_run.data_ptr(), lin.qzeros.data_ptr(), scales.data_ptr()
            L.qweight_tc = _ptr(lin._qweight_tc) if tc else None
            L.perm, L.bias = _ptr(perm), _ptr(bias)
        self.p_gate, self.p_up = ctypes.addressof(self.gate), ctypes.addressof(self.up)


def forward_gate_up(gate_proj, up_proj, x: torch.Tensor, *, kernel: int = _lib.GATE_UP_AUTO, tile_m: int = 0,
                    split_k: int = 0) -> torch.Tensor:
    """``F.silu(gate_proj(x)) * up_proj(x)`` for two ``QuantLinear`` layers that read the same ``x``, in one launch.

    The shape of ``x`` is kept except for the last dimension (I = ``gate_proj.outfeatures``).  Pairs the kernels do not
    take (different shapes, group sizes or act-order permutations, I % 32 != 0, a group size the tensor-core path cannot
    run at M > 8, activations other than fp16 / bf16) run the unfused expression instead, and so do batches of more
    than ``FUSED_MAX_M`` rows, where the unfused layers measured faster.  ``kernel`` / ``tile_m`` /
    ``split_k`` force a kernel and its tuning (``agb200_w4a16_gate_up_ex``; tests and benchmarks): a forced call never
    falls back and raises what the library reports.

    When autograd records (grad mode on and ``x.requires_grad``) the unfused expression runs, through the layers'
    differentiable ``forward()``: output and gradients are then those of the unfused layers (a forced kernel raises)."""
    if x.device.type != "cuda":
        raise RuntimeError("autogptq_b200.forward_gate_up needs a CUDA tensor (no CPU fallback).")
    forced = kernel != _lib.GATE_UP_AUTO or tile_m or split_k
    if x.requires_grad and torch.is_grad_enabled():
        if forced:
            raise NotImplementedError("forward_gate_up: the fused kernels have no backward; x requires grad")
        return _unfused(gate_proj, up_proj, x)
    why = _fusable(gate_proj, up_proj)
    if not why and x.dtype not in _DTYPE_CODE:
        why = f"activations are {x.dtype}"
    if not why and (gate_proj.kernel != _lib.KERNEL_AUTO or up_proj.kernel != _lib.KERNEL_AUTO):
        why = "a kernel is forced on gate_proj / up_proj"
    if why:
        if forced:
            raise NotImplementedError(f"forward_gate_up: {why}")
        return _unfused(gate_proj, up_proj, x)
    K, I, gs = gate_proj.infeatures, gate_proj.outfeatures, gate_proj.group_size
    if x.shape[-1] != K:
        raise RuntimeError(f"input has {x.shape[-1]} features, gate_proj expects {K}")
    for lin in (gate_proj, up_proj):
        if not lin._ready or lin._qweight_run is None or lin._qweight_run.device != x.device:
            lin.post_init()
    perm = _pair_perm(gate_proj, up_proj)
    cache = gate_proj.__dict__["_gate_up_cache"]
    if perm is False:
        if forced:
            raise NotImplementedError("forward_gate_up: gate_proj and up_proj have different act-order permutations")
        return _unfused(gate_proj, up_proj, x)
    x2 = x.reshape(-1, K)
    if not x2.is_contiguous() or x2.data_ptr() % 16:        # the kernels read x in 16-byte words
        x2 = x2.clone(memory_format=torch.contiguous_format)
    M = x2.shape[0]
    out_shape = x.shape[:-1] + (I,)
    if M == 0:
        return torch.empty(out_shape, dtype=x.dtype, device=x.device)
    if M > FUSED_MAX_M and not forced:
        return _unfused(gate_proj, up_proj, x)
    gemm_gs = gs == 32 or gs % 64 == 0
    # Which kernel runs is the library's choice (the decode kernel's shared-memory need depends on the device); batches
    # of more than MOE_DECODE_MAX_T rows always need the tensor-core copies, smaller ones only when the library turns the
    # decode kernel down (AGB200_ENOSUP without them), and then the call is repeated with the copies.
    tc = kernel == _lib.GATE_UP_GEMM or (kernel == _lib.GATE_UP_AUTO and M > _lib.MOE_DECODE_MAX_T)
    if tc and not gemm_gs:
        if forced:
            raise NotImplementedError(f"forward_gate_up: group_size={gs} cannot run the tensor-core GEMM")
        return _unfused(gate_proj, up_proj, x)
    h = torch.empty((M, I), dtype=x2.dtype, device=x.device)
    rc = _call(gate_proj, up_proj, cache, perm, x2, h, tc, kernel, tile_m, split_k)
    if rc == _lib.ENOSUP and not forced and not tc and gemm_gs:
        rc = _call(gate_proj, up_proj, cache, perm, x2, h, True, kernel, tile_m, split_k)
    if rc == _lib.ENOSUP and not forced:
        logger.debug("forward_gate_up: unfused (%s)", _lib.load().agb200_last_error().decode(errors="replace"))
        return _unfused(gate_proj, up_proj, x)
    _lib.check(rc, "agb200_w4a16_gate_up")
    return h.reshape(out_shape)


def _same(a, b) -> bool:
    return len(a) == len(b) and all(p is q for p, q in zip(a, b))


def _call(gate_proj, up_proj, cache, perm, x2, h, tc, kernel, tile_m, split_k, g=None, u=None) -> int:
    """One agb200_w4a16_gate_up_ex call (agb200_w4a16_gate_up_saving_ex with the ``g`` / ``u`` outputs); builds the
    tensor-core copies first when ``tc`` (as QuantLinear does for its first M > 8 call) and the ctypes descriptors when
    any tensor they point to changed.  Returns the status code."""
    if tc:
        for lin in (gate_proj, up_proj):
            if lin._qweight_tc is None:
                lin._prepare_tc()
    dtype = x2.dtype
    tensors = (gate_proj._qweight_run, up_proj._qweight_run, gate_proj.qzeros, up_proj.qzeros,
               *gate_proj._run_tensors(dtype), *up_proj._run_tensors(dtype), perm,
               gate_proj._qweight_tc if tc else None, up_proj._qweight_tc if tc else None)
    key = (id(up_proj), dtype, tc)
    args = cache.get(key)
    if args is None or not _same(tensors, args.tensors):
        args = _PairArgs(gate_proj, up_proj, perm, dtype, tc)
        args.tensors = tensors          # also keeps them alive, so identity stays meaningful
        cache[key] = args
    lib = _lib.load()
    M, K = x2.shape
    I = h.shape[1]
    ws_ptr, ws_bytes = None, 0
    if tc and perm is not None:
        ws_bytes = int(lib.agb200_w4a16_gate_up_workspace_bytes(M, K, I))
        ws_ptr = _workspace(x2.device, ws_bytes).data_ptr()
    cur = torch.cuda.current_device()
    if cur != x2.device.index:
        torch.cuda.set_device(x2.device)
    try:
        stream = torch.cuda.current_stream(x2.device).cuda_stream
        if g is not None:
            return lib.agb200_w4a16_gate_up_saving_ex(x2.data_ptr(), args.p_gate, args.p_up, h.data_ptr(), g.data_ptr(),
                                                      u.data_ptr(), M, K, I, gate_proj.group_size, _DTYPE_CODE[dtype],
                                                      ws_ptr, ws_bytes, stream, kernel, tile_m, split_k)
        return lib.agb200_w4a16_gate_up_ex(x2.data_ptr(), args.p_gate, args.p_up, h.data_ptr(), M, K, I,
                                           gate_proj.group_size, _DTYPE_CODE[dtype], ws_ptr, ws_bytes, stream, kernel,
                                           tile_m, split_k)
    finally:
        if cur != x2.device.index:
            torch.cuda.set_device(cur)


def _dgrad_tc_supported(K: int, N: int, group_size: int) -> bool:
    """The tensor-core dgrad's condition (``dgrad_tc_supported`` of csrc/dgrad_common.cuh)."""
    return N % 32 == 0 and ((group_size % 16 == 0 and group_size >= 32) or group_size >= K)


def _fused_backward_unfit(gate_proj, up_proj, down_proj, dtype) -> str:
    """Why ``FusedQuantMLP(fused_backward=True)`` runs the unfused autograd path for activations of ``dtype`` (empty
    string: it runs the fused one).  The act-order permutations are compared as loaded (``_perm``)."""
    for name, lin in (("gate_proj", gate_proj), ("up_proj", up_proj), ("down_proj", down_proj)):
        if not isinstance(lin, QuantLinear):
            return f"{name} is {type(lin).__name__}, not a bare autogptq_b200.QuantLinear"
    why = _fusable(gate_proj, up_proj)
    if why:
        return why
    H, I = gate_proj.infeatures, gate_proj.outfeatures
    if (down_proj.infeatures, down_proj.outfeatures) != (I, H):
        return f"down_proj is {down_proj.infeatures}x{down_proj.outfeatures}, expected {I}x{H}"
    if any(lin.kernel != _lib.KERNEL_AUTO for lin in (gate_proj, up_proj, down_proj)):
        return "a kernel is forced on gate_proj / up_proj / down_proj"
    if dtype not in _DTYPE_CODE:
        return f"activations are {dtype}"
    if I % 64:
        return f"the fused backward needs I % 64 == 0 (I={I})"
    if not _dgrad_tc_supported(H, I, gate_proj.group_size) or not _dgrad_tc_supported(I, H, down_proj.group_size):
        return (f"group sizes {gate_proj.group_size} / {down_proj.group_size} (H={H}, I={I}) are outside the "
                "tensor-core dgrad")
    if _pair_perm(gate_proj, up_proj) is False:
        return "gate_proj and up_proj have different act-order permutations"
    return ""


class FusedQuantMLP(nn.Module):
    """``down_proj(silu(gate_proj(x)) * up_proj(x))`` with the gate/up half fused (``forward_gate_up``).

    Keeps the three layers under their LlamaMLP names, so state-dict keys do not change.

    ``fused_backward=True``: when autograd records (grad mode on and ``x.requires_grad``), the forward keeps only the
    rounded g and u (not x, not h) and the backward computes dx in two launches (``agb200_w4a16_mlp_backward``: dh, dg
    and du stay in registers and fp32, dx is rounded once).  That changes the rounding of dx against the unfused
    layers' autograd, so it is opt-in; the forward output is the same, bit for bit.  MLPs the fused backward does not
    take (layers other than bare ``QuantLinear``, I % 64 != 0, group sizes outside the tensor-core dgrad, activations
    other than fp16 / bf16, ...) and batches of more than ``FUSED_BACKWARD_MAX_M`` rows, where the unfused backward
    measured faster, run the default path; the reason is logged at debug level.  Default: in grad mode,
    outputs and gradients are those of the unfused layers."""

    def __init__(self, gate_proj, up_proj, down_proj, *, fused_backward: bool = False):
        super().__init__()
        self.gate_proj, self.up_proj, self.down_proj = gate_proj, up_proj, down_proj
        self.fused_backward = bool(fused_backward)
        self._bwd_args = {}         # compute dtype -> _MlpArgs

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.fused_backward and x.requires_grad and torch.is_grad_enabled():
            if x.device.type != "cuda":
                raise RuntimeError("autogptq_b200.FusedQuantMLP needs a CUDA tensor (no CPU fallback).")
            for lin in (self.gate_proj, self.up_proj, self.down_proj):
                if isinstance(lin, QuantLinear) and (not lin._ready or lin._qweight_run is None
                                                     or lin._qweight_run.device != x.device):
                    lin.post_init()
            why = _fused_backward_unfit(self.gate_proj, self.up_proj, self.down_proj, x.dtype)
            H = self.gate_proj.infeatures
            if not why and x.shape[-1] == H and x.numel() // H > FUSED_BACKWARD_MAX_M:
                why = f"M > FUSED_BACKWARD_MAX_M = {FUSED_BACKWARD_MAX_M}, where the unfused backward measured faster"
            if not why:
                if x.shape[-1] != H:
                    raise RuntimeError(f"input has {x.shape[-1]} features, gate_proj expects {H}")
                x2 = x.reshape(-1, H)
                if not x2.is_contiguous() or x2.data_ptr() % 16:    # the kernels read x in 16-byte words
                    x2 = x2.clone(memory_format=torch.contiguous_format)
                return _FusedMLPFunction.apply(x2, self).reshape(x.shape)
            logger.debug("FusedQuantMLP: unfused backward (%s)", why)
        return self.down_proj(forward_gate_up(self.gate_proj, self.up_proj, x))

    def extra_repr(self) -> str:
        return f"gate_up=fused silu*mul (sm_90a), fused_backward={self.fused_backward}"

    def _forward_saving(self, x2: torch.Tensor, *, kernel: int = _lib.GATE_UP_AUTO, tile_m: int = 0, split_k: int = 0):
        """(y, h, g, u) for x2 [M, H] (contiguous, 16-byte aligned, fp16 / bf16) of an MLP the fused backward takes.  y
        and h are those of the no-grad forward, bit for bit: the same kernel is chosen by M (decode kernel, fused GEMM up
        to FUSED_MAX_M rows, the two gate / up layers above), and the saving kernels also store g and u.  ``kernel`` /
        ``tile_m`` / ``split_k`` force the gate/up kernel as in ``forward_gate_up`` (tests)."""
        gate, up, down = self.gate_proj, self.up_proj, self.down_proj
        M, I = x2.shape[0], gate.outfeatures
        forced = kernel != _lib.GATE_UP_AUTO or tile_m or split_k
        gs = gate.group_size
        gemm_gs = gs == 32 or gs % 64 == 0
        tc = kernel == _lib.GATE_UP_GEMM or (kernel == _lib.GATE_UP_AUTO and M > _lib.MOE_DECODE_MAX_T)
        h = None
        if M > 0 and (forced or (M <= FUSED_MAX_M and (gemm_gs or not tc))):
            h, g, u = (torch.empty((M, I), dtype=x2.dtype, device=x2.device) for _ in range(3))
            perm = _pair_perm(gate, up)
            cache = gate.__dict__["_gate_up_cache"]
            rc = _call(gate, up, cache, perm, x2, h, tc, kernel, tile_m, split_k, g, u)
            if rc == _lib.ENOSUP and not forced and not tc and gemm_gs:
                rc = _call(gate, up, cache, perm, x2, h, True, kernel, tile_m, split_k, g, u)
            if rc == _lib.ENOSUP and not forced:
                logger.debug("FusedQuantMLP: unfused gate/up (%s)", _lib.load().agb200_last_error().decode(errors="replace"))
                h = None
            else:
                _lib.check(rc, "agb200_w4a16_gate_up_saving")
        if h is None:                   # the unfused expression: g and u exist anyway
            g, u = gate._forward(x2), up._forward(x2)
            h = F.silu(g) * u
        return down._forward(h), h, g, u

    def _args(self, dtype) -> "_MlpArgs":
        gate, up, down = self.gate_proj, self.up_proj, self.down_proj
        perm = _pair_perm(gate, up)
        tensors = (gate._qweight_run, up._qweight_run, down._qweight_run, gate.qzeros, up.qzeros, down.qzeros,
                   *gate._run_tensors(dtype), *up._run_tensors(dtype), *down._run_tensors(dtype), perm, down._perm)
        args = self._bwd_args.get(dtype)
        if args is None or not _same(tensors, args.tensors):
            args = _MlpArgs(gate, up, down, perm, dtype)
            args.tensors = tensors      # also keeps them alive, so identity stays meaningful
            self._bwd_args[dtype] = args
        return args

    def _backward(self, dy: torch.Tensor, g: torch.Tensor, u: torch.Tensor, *, tile_m: int = 0, split_k: int = 0):
        """dx [M, H] of dy's dtype from dy [M, H] (contiguous, 16-byte aligned) and the g, u of ``_forward_saving``."""
        gate, down = self.gate_proj, self.down_proj
        H, I = gate.infeatures, gate.outfeatures
        M = dy.shape[0]
        dx = torch.empty((M, H), dtype=dy.dtype, device=dy.device)
        if M == 0:
            return dx
        args = self._args(dy.dtype)
        lib = _lib.load()
        ws = _workspace(dy.device, int(lib.agb200_w4a16_mlp_backward_workspace_bytes(M, H, I)))
        with torch.cuda.device(dy.device):
            rc = lib.agb200_w4a16_mlp_backward_ex(
                dy.data_ptr(), args.pair.p_gate, args.pair.p_up, args.p_down, g.data_ptr(), u.data_ptr(), dx.data_ptr(),
                M, H, I, gate.group_size, down.group_size, _DTYPE_CODE[dy.dtype], ws.data_ptr(), ws.numel(),
                torch.cuda.current_stream(dy.device).cuda_stream, tile_m, split_k)
        _lib.check(rc, "agb200_w4a16_mlp_backward")
        return dx


class _MlpArgs:
    """ctypes layer descriptors of an MLP's gate, up and down layers for one compute dtype (the backward's)."""

    def __init__(self, gate, up, down, perm, dtype):
        self.pair = _PairArgs(gate, up, perm, dtype, False)
        scales, bias = down._run_tensors(dtype)
        self.keep = [scales, bias, down._perm, down._qweight_run]
        self.down = _CLayer()
        self.down.qweight, self.down.qzeros, self.down.scales = (down._qweight_run.data_ptr(), down.qzeros.data_ptr(),
                                                                 scales.data_ptr())
        self.down.qweight_tc, self.down.perm, self.down.bias = None, _ptr(down._perm), _ptr(bias)
        self.p_down = ctypes.addressof(self.down)


class _FusedMLPFunction(torch.autograd.Function):
    """y = FusedQuantMLP's forward of x2 [M, H], saving g and u only; dx from ``agb200_w4a16_mlp_backward``.  The layers
    are frozen and get no gradient; x2 arrives reshaped and aligned (those are torch ops outside, as in moe.py)."""

    @staticmethod
    def forward(ctx, x2, mlp):
        y, _, g, u = mlp._forward_saving(x2)
        ctx.mlp = mlp
        ctx.save_for_backward(g, u)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        g, u = ctx.saved_tensors
        dy = dy.contiguous()
        if dy.data_ptr() % 16:
            dy = dy.clone()
        return ctx.mlp._backward(dy, g, u), None


def _is_silu(act) -> bool:
    if act is F.silu or isinstance(act, nn.SiLU):
        return True
    return type(act).__name__ in ("SiLU", "SiLUActivation")      # transformers' ACT2FN["silu"] across versions


def inject_fused_mlp(model: nn.Module, *, fused_backward: bool = False) -> int:
    """Replace every submodule shaped like transformers' ``LlamaMLP`` (also Mistral's and Qwen2's: ``gate_proj``,
    ``up_proj``, ``down_proj`` and a SiLU ``act_fn``) whose three layers are ``autogptq_b200.QuantLinear`` by a
    ``FusedQuantMLP`` over the same layers.  Other modules are left alone; the reason is logged.  Returns the number of
    replaced modules.  ``fused_backward`` is passed to every ``FusedQuantMLP`` made (see there)."""
    found = []
    for name, mod in model.named_modules():
        if isinstance(mod, FusedQuantMLP) or not all(hasattr(mod, a) for a in ("gate_proj", "up_proj", "down_proj")):
            continue
        if name == "":
            logger.info("inject_fused_mlp: the model itself is an MLP; wrap it in FusedQuantMLP directly")
            continue
        if not _is_silu(getattr(mod, "act_fn", None)):
            logger.info("inject_fused_mlp: %s skipped: act_fn is %s, not SiLU", name,
                        type(getattr(mod, "act_fn", None)).__name__)
            continue
        if not isinstance(mod.down_proj, QuantLinear):
            logger.info("inject_fused_mlp: %s skipped: down_proj is not autogptq_b200.QuantLinear", name)
            continue
        why = _fusable(mod.gate_proj, mod.up_proj)
        if why:
            logger.info("inject_fused_mlp: %s skipped: %s", name, why)
            continue
        found.append(name)
    for name in found:
        mod = model.get_submodule(name)
        fused = FusedQuantMLP(mod.gate_proj, mod.up_proj, mod.down_proj, fused_backward=fused_backward)
        parent_name, _, child = name.rpartition(".")
        setattr(model.get_submodule(parent_name) if parent_name else model, child, fused)
    return len(found)


__all__ = ["forward_gate_up", "FusedQuantMLP", "inject_fused_mlp"]
