"""CPU oracle of AutoAWQ "GEMM" packed layers.  TEST INFRASTRUCTURE ONLY (the product never imports ``oracle/``).

NumPy restatement of the layout the reference reads when it converts AWQ checkpoints (paths relative to the AutoGPTQ
tree):

* ``qweight`` int32 ``[K, N/8]`` and ``qzeros`` int32 ``[G, N/8]`` are packed along N; nibble ``i`` (bits ``4i..4i+3``)
  of word ``[r, c]`` holds column ``8c + AWQ_ORDER[i]``.  The reference undoes the order with
  ``awq_reverse_reorder_int_tensor`` (``auto_gptq/modeling/_utils.py:525-547``: column ``8c + j`` comes from nibble
  ``[0, 4, 1, 5, 2, 6, 3, 7][j]``) after ``unpack_awq`` has split the words into nibbles (``:550-620``).
* ``qzeros`` holds ``z`` itself (``unpack_awq`` leaves out the ``+ 1`` of the GPTQ rule, ``:585``).
* ``scales`` ``[G, N]``, groups are sequential (``g = k // group_size``), ``W = s·(q − z)`` (``:605-613``).

Pinned by ``tests/test_awq_cpu.py`` against the reference's own ``unpack_awq`` / ``pack_from_tensors`` outputs
(``tests/golden/awq_*.npz``, written by ``tests/golden/make_golden_awq.py``).
"""
from __future__ import annotations

import numpy as np

from . import w4a16_oracle as O

AWQ_ORDER = np.array([0, 2, 4, 6, 1, 3, 5, 7])          # nibble i holds column 8c + AWQ_ORDER[i]
_SHIFTS = np.arange(8, dtype=np.uint32) * 4


def _pack_cols(v: np.ndarray) -> np.ndarray:
    """uint [R, N] (values 0..15) -> int32 [R, N/8] in AWQ column order."""
    v = np.asarray(v).astype(np.uint32)
    R, N = v.shape
    assert N % 8 == 0
    v = v.reshape(R, N // 8, 8)
    out = np.zeros((R, N // 8), dtype=np.uint32)
    for i in range(8):
        out |= (v[:, :, AWQ_ORDER[i]] & 0xF) << _SHIFTS[i]
    return out.view(np.int32)


def _unpack_cols(packed: np.ndarray) -> np.ndarray:
    """int32 [R, N/8] in AWQ column order -> uint8 [R, N]."""
    w = np.ascontiguousarray(packed).view(np.uint32)
    R, C = w.shape
    nib = (w[:, :, None] >> _SHIFTS[None, None, :]) & 0xF          # [R, C, nibble]
    out = np.empty((R, C, 8), dtype=np.uint8)
    out[:, :, AWQ_ORDER] = nib
    return out.reshape(R, 8 * C)


def pack_awq(intweight: np.ndarray, zeros: np.ndarray):
    """q [K, N] and z [G, N] (values 0..15) -> AWQ ``(qweight [K, N/8], qzeros [G, N/8])``."""
    return _pack_cols(intweight), _pack_cols(zeros)


def unpack_awq(qweight: np.ndarray, qzeros: np.ndarray):
    """AWQ ``(qweight, qzeros)`` -> ``(q uint8 [K, N], z int32 [G, N])`` (the integer part of ``unpack_awq``,
    ``_utils.py:572-603``)."""
    return _unpack_cols(qweight), _unpack_cols(qzeros).astype(np.int32)


def dequantize_awq(qweight, qzeros, scales, group_size: int, reference_fp16: bool = False) -> np.ndarray:
    """W [K, N].  Default: ``s·(q − z)`` in fp32, which is exact (an fp16 scale times an integer in [-15, 15]).
    ``reference_fp16=True``: the reference's own fp16 arithmetic, ``fp16(q·s) − fp16(z·s)`` rounded to fp16
    (``_utils.py:605-613``), as fp16."""
    q, z = unpack_awq(qweight, qzeros)
    K = q.shape[0]
    g = np.arange(K) // (K if group_size == -1 else group_size)
    s = np.asarray(scales)
    if reference_fp16:
        s = s.astype(np.float16)
        qs = (q.astype(np.float32) * s[g].astype(np.float32)).astype(np.float16)
        zs = (z.astype(np.float32) * s.astype(np.float32)).astype(np.float16)[g]
        return (qs.astype(np.float32) - zs.astype(np.float32)).astype(np.float16)
    s = s.astype(np.float32)
    return s[g] * (q.astype(np.int32) - z[g]).astype(np.float32)


def to_gptq(qweight: np.ndarray, qzeros: np.ndarray):
    """AWQ ``(qweight, qzeros)`` -> the GPTQ ``(qweight [K/8, N], qzeros [G, N/8])`` of the same layer, through the
    GPTQ oracle's packers (zeros stored minus one, ``pack_from_tensors``, ``_utils.py:682-683``)."""
    q, z = unpack_awq(qweight, qzeros)
    return O.pack_rows(q), O.pack_cols(((z - 1) & 0xF).astype(np.uint32))


def random_awq(K: int, N: int, group_size: int, seed: int = 0, bias: bool = False, scale_dtype=np.float16):
    """A random AWQ GEMM layer: uniform weight nibbles, zeros covering 0..15, scales ``rand·0.01 + 0.001``.
    Returns the AWQ tensors and the integers they were packed from (``intweight`` [K, N], ``zeros`` [G, N])."""
    rng = np.random.default_rng(seed)
    gs = K if group_size == -1 else group_size
    G = -(-K // gs)
    q = rng.integers(0, 16, size=(K, N), dtype=np.uint8)
    z = rng.integers(0, 16, size=(G, N), dtype=np.uint8)
    z.reshape(-1)[:16] = np.arange(16)
    qweight, qzeros = pack_awq(q, z)
    scales = (rng.random((G, N), dtype=np.float32) * 0.01 + 0.001).astype(scale_dtype)
    b = (rng.standard_normal(N).astype(np.float32) * 0.1).astype(scale_dtype) if bias else None
    return dict(qweight=qweight, qzeros=qzeros, scales=scales, bias=b, intweight=q, zeros=z, K=K, N=N, group_size=gs)
