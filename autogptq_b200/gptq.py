"""GPTQ quantiser on the H100: a drop-in for ``auto_gptq.quantization.GPTQ`` whose hot paths are the sm_90a kernels
behind ``agb200_gptq_hessian_update`` / ``agb200_gptq_quantize`` (include/autogptq_b200.h).

``GPTQ(layer)`` keeps the reference's interface (``auto_gptq/quantization/gptq.py:19-203``): ``add_batch(inp, out)``
accumulates the running-mean Hessian, ``fasterquant(...)`` quantises ``layer.weight`` in place and returns
``(scale, zero, g_idx)``.  It additionally leaves the packed result as a ready ``autogptq_b200.QuantLinear`` in
``.quant_linear``, with codes produced by the kernel, so ``pack()`` is not needed.

Scope: 4 bits, per-channel, no MSE grid search, blocksize 128 (the settings ``modeling/_base.py:303-345`` uses);
fp16 / bf16 layers and calibration inputs on a CUDA device.  Anything else raises ``NotImplementedError``.  The damping,
the dead-column edit of H and the Cholesky factorisations (``gptq.py:84-119``) run through torch on the device.
"""
from __future__ import annotations

import importlib
import sys
from logging import getLogger
from typing import Iterable, Tuple, Union

import torch
import torch.nn as nn

from . import _lib
from .qlinear import QuantLinear

logger = getLogger(__name__)

_DTYPE_CODE = {torch.float16: _lib.F16, torch.bfloat16: _lib.BF16}
BLOCKSIZE = 128


def _is_conv1d(layer) -> bool:
    # transformers.pytorch_utils.Conv1D stores the weight as [in, out]
    return layer.__class__.__name__ == "Conv1D"


def running_mean_factors(nsamples: int, inp_shape) -> Tuple[float, float, int]:
    """``(alpha, beta, nsamples')`` of one ``add_batch``: ``H' = alpha * H + beta * x^T x``.

    The reference counts samples along the leading dimension of the input, not tokens: a 2-D input is one sample, a
    ``[b, s, K]`` input is ``b`` (``gptq.py:38-40``).  Then ``H *= n / (n + b)`` and ``H += 2 / (n + b) * x^T x``
    (``gptq.py:55-60``)."""
    b = 1 if len(inp_shape) == 2 else int(inp_shape[0])
    n = nsamples + b
    alpha = nsamples / n if n > 0 else 0.0
    return alpha, (2.0 / n if n > 0 else 0.0), n


class Quantizer(nn.Module):
    """Settings holder with the signature of ``auto_gptq.quantization.Quantizer`` (``quantizer.py:17-43``).

    ``scale`` / ``zero`` hold the parameters of the last group after ``fasterquant``, as in the reference."""

    def __init__(self, shape=1):
        super().__init__()
        self.register_buffer("maxq", torch.tensor(0))
        self.register_buffer("scale", torch.zeros(shape))
        self.register_buffer("zero", torch.zeros(shape))
        self.bits, self.perchannel, self.sym, self.mse = None, False, True, False

    def configure(self, bits, perchannel=False, sym=True, mse=False, norm=2.4, grid=100, maxshrink=0.8, trits=False):
        if bits != 4:
            raise NotImplementedError(f"the GPU GPTQ quantiser writes 4-bit checkpoints only (bits={bits})")
        if not perchannel:
            raise NotImplementedError("the GPU GPTQ quantiser needs perchannel=True (one scale per output row and group)")
        if mse:
            raise NotImplementedError("mse=True (the grid search of quantizer.py:87-104) is not implemented")
        if trits:
            raise NotImplementedError("trits=True is not implemented")
        self.maxq = torch.tensor(2**bits - 1)
        self.bits, self.perchannel, self.sym, self.mse = bits, perchannel, sym, mse
        self.norm, self.grid, self.maxshrink = norm, grid, maxshrink

    def ready(self):
        return torch.all(self.scale != 0)


class GPTQ:
    """Drop-in for ``auto_gptq.quantization.GPTQ`` on one ``nn.Linear`` or ``transformers`` ``Conv1D`` layer."""

    def __init__(self, layer):
        if isinstance(layer, nn.Conv2d):
            raise NotImplementedError("GPTQ on nn.Conv2d layers is not implemented (Linear and Conv1D only)")
        self.layer = layer
        self.dev = layer.weight.device
        W = layer.weight.data
        if _is_conv1d(layer):
            W = W.t()
        self.rows, self.columns = W.shape[0], W.shape[1]
        self.H = torch.zeros((self.columns, self.columns), device=self.dev)
        self.nsamples = 0
        self.quantizer = Quantizer()
        self.quant_linear = None
        self.Losses = None

    def add_batch(self, inp, out):
        if inp.device.type != "cuda" or self.H.device.type != "cuda":
            raise RuntimeError("GPTQ.add_batch needs the layer and its inputs on a CUDA device (there is no CPU fallback)")
        if inp.dtype not in _DTYPE_CODE:
            raise NotImplementedError(f"calibration inputs must be float16 or bfloat16 (got {inp.dtype})")
        if inp.shape[-1] != self.columns:
            raise ValueError(f"input has {inp.shape[-1]} features, layer has {self.columns}")
        alpha, beta, self.nsamples = running_mean_factors(self.nsamples, inp.shape)
        x = inp.reshape(-1, self.columns).contiguous()
        if x.data_ptr() % 16:
            x = x.clone()
        lib = _lib.load()
        with torch.cuda.device(x.device):
            _lib.check(lib.agb200_gptq_hessian_update(x.data_ptr(), self.H.data_ptr(), x.shape[0], self.columns,
                                                      _DTYPE_CODE[x.dtype], alpha, beta,
                                                      torch.cuda.current_stream(x.device).cuda_stream),
                       "agb200_gptq_hessian_update")

    def fasterquant(self, blocksize=128, percdamp=0.01, group_size=-1, actorder=False, static_groups=False):
        if blocksize != BLOCKSIZE:
            raise NotImplementedError(f"blocksize={blocksize}: the GPU quantiser runs 128-column blocks")
        if self.quantizer.bits != 4:
            raise NotImplementedError("configure the quantizer first: quantizer.configure(4, perchannel=True, sym=...)")
        if group_size != -1 and (group_size <= 0 or group_size % 8 != 0):
            raise NotImplementedError(f"group_size={group_size}: must be -1 or a positive multiple of 8")
        dtype = self.layer.weight.dtype
        if dtype not in _DTYPE_CODE:
            raise NotImplementedError(f"the layer weight must be float16 or bfloat16 (got {dtype})")
        if self.dev.type != "cuda":
            raise RuntimeError("GPTQ.fasterquant needs the layer on a CUDA device (there is no CPU fallback)")
        N, K = self.rows, self.columns
        if N % 8 or K % 8:
            raise NotImplementedError(f"layer of {K} -> {N} features: both must be multiples of 8 for 4-bit packing")
        W = self.layer.weight.data
        if _is_conv1d(self.layer):
            W = W.t()
        W = W.float().contiguous()

        H = self.H
        del self.H
        Hinv, perm, dead = inverse_hessian_factor(H, percdamp, actorder)
        del H

        res = quantize_weight(W, Hinv, perm=perm, dead=dead if bool(dead.any()) else None, group_size=group_size,
                              sym=self.quantizer.sym, static_groups=static_groups, dtype=dtype, losses=True)
        Q = res["Q"]
        self.Losses = res["losses"]
        if _is_conv1d(self.layer):
            Q = Q.t()
        self.layer.weight.data = Q.reshape(self.layer.weight.shape).type_as(self.layer.weight.data)
        self.quantizer.scale = res["scale"][:, -1:].clone()
        self.quantizer.zero = res["zero"][:, -1:].clone()

        ql = QuantLinear(4, group_size, K, N, self.layer.bias is not None, weight_dtype=dtype)
        ql.qweight, ql.qzeros, ql.scales, ql.g_idx = res["qweight"], res["qzeros"], res["scales"], res["g_idx"]
        if self.layer.bias is not None:
            ql.bias = self.layer.bias.data.clone().to(dtype)
        self.quant_linear = ql
        return res["scale"], res["zero"], res["g_idx"]

    def free(self):
        self.H = None
        self.Losses = None
        self.Trace = None
        torch.cuda.empty_cache()


def inverse_hessian_factor(H: torch.Tensor, percdamp=0.01, actorder=False):
    """``(Hinv, perm, dead)`` for ``quantize_weight`` from the running-mean Hessian ``H`` [K, K] fp32, which is edited in
    place: dead columns (``diag H = 0``) get a unit diagonal, act-order permutes H by descending diagonal (a stable sort
    for ties), the damping adds ``percdamp`` times the mean diagonal, and three torch factorisations give the upper
    Cholesky factor of the damped inverse in processing order (``gptq.py:84-119``).  ``perm`` is None without act-order;
    ``dead`` is a bool [K] in original column order."""
    dead = torch.diag(H) == 0                                       # gptq.py:84-86
    H[dead, dead] = 1
    perm = None
    if actorder:                                                    # gptq.py:104-108
        perm = torch.argsort(torch.diag(H), descending=True, stable=True)
        H = H[perm][:, perm]
    damp = percdamp * torch.mean(torch.diag(H))                     # gptq.py:113-119
    H.diagonal().add_(damp)
    H = torch.linalg.cholesky(H)
    H = torch.cholesky_inverse(H)
    return torch.linalg.cholesky(H, upper=True).contiguous(), perm, dead


def quantize_weight(W: torch.Tensor, Hinv: torch.Tensor, perm=None, dead=None, group_size=-1, sym=True,
                    static_groups=False, dtype=torch.float16, losses=False) -> dict:
    """One ``agb200_gptq_quantize`` call.  ``W`` [N, K] fp32 (overwritten with Q, original column order), ``Hinv`` the
    upper Cholesky factor of the damped inverse in processing order, ``perm`` (act-order) processing position ->
    original column, ``dead`` bool [K] in original order.  Returns the outputs by name."""
    if W.dtype != torch.float32 or Hinv.dtype != torch.float32 or W.device.type != "cuda":
        raise ValueError("W and Hinv must be float32 CUDA tensors")
    N, K = W.shape
    W = W.contiguous()
    Hinv = Hinv.contiguous()
    dev = W.device
    gs = K if group_size == -1 else group_size
    G = -(-K // gs)
    f32 = dict(dtype=torch.float32, device=dev)
    out = {
        "scale": torch.empty((N, G), **f32), "zero": torch.empty((N, G), **f32),
        "scales": torch.empty((G, N), dtype=dtype, device=dev),
        "qweight": torch.empty((K // 8, N), dtype=torch.int32, device=dev),
        "qzeros": torch.empty((G, N // 8), dtype=torch.int32, device=dev),
        "g_idx": torch.empty((K,), dtype=torch.int32, device=dev),
        "losses": torch.empty((N, K), **f32) if losses else None,
    }
    perm32 = perm.to(device=dev, dtype=torch.int32).contiguous() if perm is not None else None
    dead8 = dead.to(device=dev, dtype=torch.uint8).contiguous() if dead is not None else None
    lib = _lib.load()
    ws_bytes = int(lib.agb200_gptq_workspace_bytes(N, K, int(perm is not None)))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    ptr = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
    with torch.cuda.device(dev):
        _lib.check(lib.agb200_gptq_quantize(
            W.data_ptr(), Hinv.data_ptr(), ptr(perm32), ptr(dead8), N, K, group_size, int(bool(sym)),
            int(bool(static_groups)), out["scale"].data_ptr(), out["zero"].data_ptr(), out["scales"].data_ptr(),
            out["qweight"].data_ptr(), out["qzeros"].data_ptr(), out["g_idx"].data_ptr(), ptr(out["losses"]),
            _DTYPE_CODE[dtype], ws.data_ptr(), ws_bytes, torch.cuda.current_stream(dev).cuda_stream), "agb200_gptq_quantize")
    out["Q"] = W
    return out


def quantize_linear(linear: nn.Module, inputs: Union[torch.Tensor, Iterable[torch.Tensor]], group_size=128,
                    desc_act=False, sym=True, static_groups=False, damp_percent=0.01) -> QuantLinear:
    """GPTQ-quantise one layer on its calibration inputs and return the packed ``QuantLinear``.

    ``inputs`` is one tensor or an iterable of tensors, each what the layer sees in one forward (``[..., K]``).
    Like the reference, ``linear.weight`` is replaced by the dequantised weights."""
    g = GPTQ(linear)
    g.quantizer.configure(4, perchannel=True, sym=sym, mse=False)
    for x in ([inputs] if isinstance(inputs, torch.Tensor) else inputs):
        g.add_batch(x, None)
    g.fasterquant(blocksize=BLOCKSIZE, percdamp=damp_percent, group_size=group_size, actorder=desc_act,
                  static_groups=static_groups)
    ql = g.quant_linear
    g.free()
    return ql


# modules of the reference that bind ``GPTQ`` by name at import time
_PATCH_TARGETS = ("auto_gptq.modeling._base", "auto_gptq.quantization", "auto_gptq.quantization.gptq")


def patch_auto_gptq_quantizer() -> list:
    """Make an importable, unmodified ``auto_gptq`` quantise with this ``GPTQ``: rebinds the name in every reference
    module that imported it (``modeling/_base.py:28`` is the one ``BaseGPTQForCausalLM.quantize`` uses).  Returns the
    patched module names.  ``patch_auto_gptq()`` (the QuantLinear patch) is separate and unchanged."""
    patched = []
    for name in _PATCH_TARGETS:
        mod = sys.modules.get(name)
        if mod is None:
            try:
                mod = importlib.import_module(name)
            except Exception as e:  # noqa: BLE001 - optional reference modules may not import
                logger.debug("not patching %s: %s", name, e)
                continue
        if hasattr(mod, "GPTQ"):
            setattr(mod, "GPTQ", GPTQ)
            patched.append(name)
    return patched


__all__ = ["GPTQ", "Quantizer", "inverse_hessian_factor", "quantize_linear", "quantize_weight",
           "patch_auto_gptq_quantizer", "running_mean_factors"]
