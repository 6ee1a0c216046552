"""NumPy restatement of the FP8 KV-cache format (``autogptq_b200.attention.quantize_kv``, DESIGN §3.19).

For one cached row x of head_dim values (the 16-bit k̂ or v, as float64):
    a = max_j |x_j|; a = 0: scale 1, codes 0.
    e = the smallest integer with a <= 448·2^e, at least -126; scale = 2^e.
    code_j = the E4M3FN code nearest to x_j·2^-e, a tie going to the even code (subnormals included).
Here the codes come from a table of the values of all 256 E4M3FN codes, and e is found by search on the definition,
independently of the frexp rule the library uses.
"""
from __future__ import annotations

import numpy as np

E4M3_MAX = 448.0


def e4m3_values() -> np.ndarray:
    """Value of every E4M3FN code 0..255 (float64): sign, 4 exponent bits (bias 7), 3 mantissa bits; 0x7F and 0xFF
    are NaN, there is no infinity."""
    c = np.arange(256)
    E, m = (c >> 3) & 0xF, c & 7
    v = np.where(E == 0, m / 8.0 * 2.0 ** -6, (1 + m / 8.0) * 2.0 ** (E - 7.0))
    v = np.where(c & 0x80, -v, v)
    v[(c & 0x7F) == 0x7F] = np.nan
    return v


VALUES = e4m3_values()
_MAG = VALUES[:0x7F]                  # codes 0..126: the non-negative finite values, increasing


def e4m3_rne(y) -> np.ndarray:
    """y (float64, |y| <= 448) -> E4M3FN codes (uint8): the nearest value of the table, a tie to the even code; the
    sign bit is y's (so -0 and negative values that round to zero give 0x80)."""
    y = np.asarray(y, np.float64)
    a = np.abs(y)
    assert (a <= E4M3_MAX).all(), "outside the E4M3 range"
    hi = np.clip(np.searchsorted(_MAG, a, side="left"), 0, len(_MAG) - 1)     # first value >= a
    lo = np.maximum(hi - 1, 0)
    dl, dh = a - _MAG[lo], _MAG[hi] - a
    code = np.where(dh < dl, hi, np.where(dl < dh, lo, np.where(hi % 2 == 0, hi, lo)))
    return (code | np.where(np.signbit(y), 0x80, 0)).astype(np.uint8)


def scale_exp(a: float) -> int:
    """The smallest integer e >= -126 with a <= 448·2^e (a > 0), by search."""
    e = -126
    while a > E4M3_MAX * 2.0 ** e:
        e += 1
    return e


def quantize(x):
    """Rows x [..., hd] (float64 values of the 16-bit dtype) -> (codes uint8 [..., hd], scale float64 [...])."""
    x = np.asarray(x, np.float64)
    flat = x.reshape(-1, x.shape[-1])
    codes = np.zeros(flat.shape, np.uint8)
    scale = np.ones(flat.shape[0])
    for r, row in enumerate(flat):
        a = np.abs(row).max()
        if a == 0:
            continue
        e = scale_exp(a)
        scale[r] = 2.0 ** e
        codes[r] = e4m3_rne(row * 2.0 ** -e)
    return codes.reshape(x.shape), scale.reshape(x.shape[:-1])


def dequantize(codes, scale) -> np.ndarray:
    """codes [..., hd], scale [...] -> the cached values (float64, exact)."""
    return VALUES[np.asarray(codes)] * np.asarray(scale, np.float64)[..., None]
