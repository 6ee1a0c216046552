"""Fused gate/up of a dense Llama-style MLP (``agb200_w4a16_gate_up``) and the module that injects it into a model.

    from autogptq_b200 import inject_fused_mlp
    n = inject_fused_mlp(model)          # every LlamaMLP-shaped submodule over QuantLinear layers -> FusedQuantMLP

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

from . import _lib
from .moe import _CLayer, _ptr
from .qlinear import _DTYPE_CODE, QuantLinear, _workspace

logger = getLogger(__name__)

# Above this many rows the unfused layers are faster: at Llama-2-7B MLP shapes on one H100 80GB HBM3 (700 W) the fused
# module measured 1.06-1.09x the unfused one at M = 1024 and the fused GEMM 0.89-0.98x at M = 4096 in three runs
# (tools/mlp_bench.py; both compute-bound there)
FUSED_MAX_M = 2048


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
    falls back and raises what the library reports."""
    if x.device.type != "cuda":
        raise RuntimeError("autogptq_b200.forward_gate_up needs a CUDA tensor (no CPU fallback).")
    forced = kernel != _lib.GATE_UP_AUTO or tile_m or split_k
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
    # The permutation comparison synchronises with the device: made once per (re)initialised pair, so that later calls
    # can be captured in a CUDA graph.  Cache entries hold the tensors they were made from and are matched by identity,
    # so a post_init() that replaces any of them (new permutation, tensor-core copy, converted scales) rebuilds them.
    cache = gate_proj.__dict__.setdefault("_gate_up_cache", {})
    pent = cache.get(("perm", id(up_proj)))
    if pent is None or not _same((up_proj, gate_proj._perm, up_proj._perm), pent[0]):
        pent = ((up_proj, gate_proj._perm, up_proj._perm), _shared_perm(gate_proj, up_proj))
        cache[("perm", id(up_proj))] = pent
    perm = pent[1]
    if perm is False:
        if forced:
            raise NotImplementedError("forward_gate_up: gate_proj and up_proj have different act-order permutations")
        return _unfused(gate_proj, up_proj, x)
    x2 = x.reshape(-1, K)
    if not x2.is_contiguous():
        x2 = x2.contiguous()
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


def _call(gate_proj, up_proj, cache, perm, x2, h, tc, kernel, tile_m, split_k) -> int:
    """One agb200_w4a16_gate_up_ex call; builds the tensor-core copies first when ``tc`` (as QuantLinear does for its
    first M > 8 call) and the ctypes descriptors when any tensor they point to changed.  Returns the status code."""
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
        return lib.agb200_w4a16_gate_up_ex(x2.data_ptr(), args.p_gate, args.p_up, h.data_ptr(), M, K, I,
                                           gate_proj.group_size, _DTYPE_CODE[dtype], ws_ptr, ws_bytes,
                                           torch.cuda.current_stream(x2.device).cuda_stream, kernel, tile_m, split_k)
    finally:
        if cur != x2.device.index:
            torch.cuda.set_device(cur)


class FusedQuantMLP(nn.Module):
    """``down_proj(silu(gate_proj(x)) * up_proj(x))`` with the gate/up half fused (``forward_gate_up``).

    Keeps the three layers under their LlamaMLP names, so state-dict keys do not change."""

    def __init__(self, gate_proj, up_proj, down_proj):
        super().__init__()
        self.gate_proj, self.up_proj, self.down_proj = gate_proj, up_proj, down_proj

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.down_proj(forward_gate_up(self.gate_proj, self.up_proj, x))

    def extra_repr(self) -> str:
        return "gate_up=fused silu*mul (sm_90a)"


def _is_silu(act) -> bool:
    if act is F.silu or isinstance(act, nn.SiLU):
        return True
    return type(act).__name__ in ("SiLU", "SiLUActivation")      # transformers' ACT2FN["silu"] across versions


def inject_fused_mlp(model: nn.Module) -> int:
    """Replace every submodule shaped like transformers' ``LlamaMLP`` (also Mistral's and Qwen2's: ``gate_proj``,
    ``up_proj``, ``down_proj`` and a SiLU ``act_fn``) whose three layers are ``autogptq_b200.QuantLinear`` by a
    ``FusedQuantMLP`` over the same layers.  Other modules are left alone; the reason is logged.  Returns the number of
    replaced modules."""
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
        fused = FusedQuantMLP(mod.gate_proj, mod.up_proj, mod.down_proj)
        parent_name, _, child = name.rpartition(".")
        setattr(model.get_submodule(parent_name) if parent_name else model, child, fused)
    return len(found)


__all__ = ["forward_gate_up", "FusedQuantMLP", "inject_fused_mlp"]
