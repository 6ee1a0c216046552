"""Decode chain: a whole list of dependent QuantLinear stages in ONE persistent launch (``agb200_chain_*``).

    chain = DecodeChain(M=1, dtype=torch.float16, device=dev)
    x = chain.input(4096)                                   # external input buffer [M, 4096]
    q, k, v = chain.stage([blk.q, blk.k, blk.v], x)         # sibling layers: one stage
    o, = chain.stage([blk.o], q)
    gate, up = chain.stage([blk.gate, blk.up], o)
    y, = chain.stage([blk.down], gate, x2=up, x_mode="silu_mul")
    chain.build()
    x.copy_(...); chain.run(); ...y...                      # one cooperative launch, CUDA-graph capturable

The buffers returned by ``input`` / ``stage`` are ordinary tensors owned by the chain; a stage's input must be one of
them (or any CUDA tensor that is ready before the launch).  Weights are streamed by TMA across stage boundaries; only
the arithmetic of a stage waits for the stage that produced its input (see ``csrc/chain.cuh``).  The reference has no
counterpart: its fused modules (``fused_llama_attn.py:171-207``, ``fused_llama_mlp.py:131-245``) only merge sibling
layers, and every layer is its own launch (``exllamav2/cuda/q_gemm.cu:47,85``).
"""
from __future__ import annotations

import ctypes
from ctypes import c_int32, c_int64, c_void_p

import torch

from . import _lib
from .qlinear import _DTYPE_CODE, QuantLinear

_X_MODES = {"plain": _lib.CHAIN_X_PLAIN, "silu_mul": _lib.CHAIN_X_SILU_MUL, "sum_parts": _lib.CHAIN_X_SUM_PARTS}


class _CLayer(ctypes.Structure):
    _fields_ = [("qweight", c_void_p), ("qzeros", c_void_p), ("scales", c_void_p), ("bias", c_void_p), ("y", c_void_p),
                ("y_peers", c_void_p), ("N", c_int32), ("n_peers", c_int32)]


class _CStage(ctypes.Structure):
    _fields_ = [("x", c_void_p), ("x2", c_void_p), ("perm", c_void_p), ("K", c_int32), ("group_size", c_int32),
                ("n_layers", c_int32), ("x_mode", c_int32), ("x_parts", c_int32), ("reserved", c_int32),
                ("x_part_stride", c_int64), ("layer", _CLayer * 4)]


def chain_supported(layers, M: int) -> bool:
    """True when every layer can run inside a chain (otherwise callers fall back to per-layer launches)."""
    return (1 <= M <= _lib.CHAIN_MAX_M and 1 <= len(layers) <= 4 and all(
        isinstance(l, QuantLinear) and l.infeatures % 128 == 0 and l.group_size % 128 == 0 and l.outfeatures % 32 == 0
        and l.infeatures == layers[0].infeatures and l.group_size == layers[0].group_size for l in layers))


class DecodeChain:
    def __init__(self, M: int = 1, dtype: torch.dtype = torch.float16, device=None):
        if dtype not in _DTYPE_CODE:
            raise ValueError("DecodeChain computes in float16 or bfloat16")
        if not 1 <= M <= _lib.CHAIN_MAX_M:
            raise ValueError(f"DecodeChain handles 1 <= M <= {_lib.CHAIN_MAX_M} rows (got {M}); use QuantLinear.forward for larger batches")
        self.M, self.dtype = M, dtype
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("DecodeChain needs a CUDA device (there is no CPU fallback)")
        self._stages = []          # (layers, x, x2, mode, parts, stride, ys)
        self._producer = {}        # data_ptr of a chain-owned buffer -> index of the stage that writes it
        self._keep = []
        self._handle = None
        self._plan = None

    # ------------------------------------------------------------------ construction
    def input(self, features: int) -> torch.Tensor:
        """A chain-owned [M, features] buffer that the caller fills before run()."""
        t = torch.zeros((self.M, features), dtype=self.dtype, device=self.device)
        self._keep.append(t)
        return t

    def stage(self, layers, x: torch.Tensor, x2: torch.Tensor | None = None, x_mode: str = "plain", x_parts: int = 0,
              x_part_stride: int = 0, outputs=None, peer_tables=None):
        """Append a stage of sibling layers reading ``x``; returns their output buffers [M, N] (one per layer).

        ``x_mode="sum_parts"``: ``x`` is an int64 tensor of 8-byte words [x_parts, x_part_stride] that the peers fill
        (tensor parallelism, see ``autogptq_b200.tp``).  ``peer_tables``: per layer None or an int64 device tensor with the
        addresses this layer's output words are sent to instead of staying in the chain."""
        if self._handle is not None:
            raise RuntimeError("DecodeChain.build() has already been called")
        layers = list(layers)
        if not chain_supported(layers, self.M):
            raise NotImplementedError("DecodeChain needs 1..4 sibling QuantLinear layers with infeatures % 128 == 0, "
                                      "group_size % 128 == 0 (or -1) and outfeatures % 32 == 0")
        K = layers[0].infeatures
        mode = _X_MODES[x_mode]
        for t in (x, x2):
            want = torch.int64 if (mode == _lib.CHAIN_X_SUM_PARTS and t is x) else self.dtype
            if t is not None and (t.device != self.device or t.dtype != want or not t.is_contiguous()):
                raise ValueError("stage inputs must be contiguous tensors of the chain's dtype on the chain's device")
        if mode == _lib.CHAIN_X_SUM_PARTS and (x_parts < 1 or x.numel() < x_parts * x_part_stride or x_part_stride < self.M * K // 2):
            raise ValueError("x_mode='sum_parts' needs x_parts >= 1 and a words tensor of x_parts * x_part_stride entries")
        if mode != _lib.CHAIN_X_SUM_PARTS and tuple(x.shape) != (self.M, K):
            raise ValueError(f"stage input has shape {tuple(x.shape)}, expected {(self.M, K)}")
        if mode == _lib.CHAIN_X_SILU_MUL and (x2 is None or tuple(x2.shape) != (self.M, K)):
            raise ValueError("x_mode='silu_mul' needs x2 of the same shape as x")
        for lin in layers:
            if not lin._ready or lin._qweight_run is None or lin._qweight_run.device != self.device:
                lin.post_init()
        perms = [lin._perm for lin in layers]
        if any(q is not None for q in perms):
            if any(q is None for q in perms) or any(not torch.equal(q, perms[0]) for q in perms[1:]):
                raise NotImplementedError("act-order sibling layers of a stage must share one permutation of x")
        ys = outputs if outputs is not None else [torch.zeros((self.M, lin.outfeatures), dtype=self.dtype, device=self.device) for lin in layers]
        peer_tables = list(peer_tables) if peer_tables is not None else [None] * len(layers)
        idx = len(self._stages)
        self._stages.append((layers, x, x2, mode, x_parts, x_part_stride, ys, peer_tables, perms[0]))
        for y in ys:
            self._producer[y.data_ptr()] = idx
        self._keep.extend(ys)
        self._keep.extend(t for t in peer_tables if t is not None)
        self._keep.extend(t for t in (x, x2) if t is not None)
        return ys

    def build(self):
        lib = _lib.load()
        n = len(self._stages)
        if n == 0:
            raise RuntimeError("DecodeChain has no stages")
        arr = (_CStage * n)()
        for i, (layers, x, x2, mode, parts, stride, ys, peer_tables, perm) in enumerate(self._stages):
            st = arr[i]
            st.x, st.x2 = x.data_ptr(), (x2.data_ptr() if x2 is not None else None)
            st.perm = perm.data_ptr() if perm is not None else None
            st.K, st.group_size, st.n_layers = layers[0].infeatures, layers[0].group_size, len(layers)
            st.x_mode, st.x_parts, st.x_part_stride = mode, parts, stride
            for j, (lin, y, pt) in enumerate(zip(layers, ys, peer_tables)):
                scales, bias = lin._run_tensors(self.dtype)
                L = st.layer[j]
                L.qweight, L.qzeros, L.scales = lin._qweight_run.data_ptr(), lin.qzeros.data_ptr(), scales.data_ptr()
                L.bias, L.y, L.N = (bias.data_ptr() if bias is not None else None), y.data_ptr(), lin.outfeatures
                if pt is not None:
                    L.y_peers, L.n_peers = pt.data_ptr(), pt.numel()
                self._keep.extend((lin._qweight_run, lin.qzeros, scales, bias))
        nbytes = int(lib.agb200_chain_plan_bytes(arr, n, self.M))
        self._plan = torch.zeros(nbytes + 256, dtype=torch.uint8, device=self.device)
        base = (self._plan.data_ptr() + 255) // 256 * 256
        h = c_void_p()
        with torch.cuda.device(self.device):
            torch.cuda.synchronize(self.device)
            _lib.check(lib.agb200_chain_create(arr, n, self.M, _DTYPE_CODE[self.dtype], base, nbytes, ctypes.byref(h)),
                       "agb200_chain_create")
        self._handle = h
        return self

    # ------------------------------------------------------------------ execution
    def run(self, debug_flags: int = 0):
        """Enqueue the whole chain on the current stream (one cooperative launch)."""
        if self._handle is None:
            self.build()
        lib = _lib.load()
        cur = torch.cuda.current_device()
        if cur != self.device.index:
            torch.cuda.set_device(self.device)
        try:
            rc = lib.agb200_chain_forward(self._handle, debug_flags, torch.cuda.current_stream(self.device).cuda_stream)
        finally:
            if cur != self.device.index:
                torch.cuda.set_device(cur)
        _lib.check(rc, "agb200_chain_forward")

    def info(self):
        lib = _lib.load()
        a, b, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        _lib.check(lib.agb200_chain_info(self._handle, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)), "agb200_chain_info")
        la, la_max, inflight, backoff = (ctypes.c_int() for _ in range(4))
        _lib.check(lib.agb200_chain_tuning(self._handle, ctypes.byref(la), ctypes.byref(la_max), ctypes.byref(inflight),
                                           ctypes.byref(backoff)), "agb200_chain_tuning")
        return {"ring_slots": a.value, "smem_bytes": b.value, "grid": c.value, "stages": len(self._stages),
                "l2_lookahead": la.value, "l2_lookahead_max": la_max.value, "inflight": inflight.value,
                "poll_backoff": backoff.value}

    def profile(self):
        """Counters of the last run(debug_flags=8) as an int64 array [grid, 4, 8].  Rows 0..2, one warp per consumer
        group, in cycles: total, wait for x, convert x, wait for weights, unpack + MMA, flush, tile end, stage end.
        Row 3, the producer: total cycles, cycles blocked on a full ring, cycles blocked on the in-flight cap, slots
        issued, slots prefetched into L2, then three zeros.  Measurement aid."""
        import numpy as np

        lib = _lib.load()
        torch.cuda.synchronize(self.device)
        n = self.info()["grid"] * 4 * 8
        buf = (ctypes.c_longlong * n)()
        rc = lib.agb200_chain_profile(self._handle, buf, n)
        if rc < 0:
            _lib.check(rc, "agb200_chain_profile")
        return np.frombuffer(buf, dtype=np.int64).reshape(-1, 4, 8).copy()

    def __del__(self):
        try:
            if self._handle is not None:
                _lib.load().agb200_chain_destroy(self._handle)
                self._handle = None
        except Exception:
            pass


def chain_diag():
    """{site, stage, cta, warp, detail} of the first bounded wait that timed out inside a chain launch of this process
    (site 0: none).  Readable even after the CUDA context was lost (``agb200_chain_diag``)."""
    buf = (ctypes.c_int * 5)()
    _lib.check(_lib.load().agb200_chain_diag(buf), "agb200_chain_diag")
    return dict(zip(("site", "stage", "cta", "warp", "detail"), list(buf)))


__all__ = ["DecodeChain", "chain_supported", "chain_diag"]
