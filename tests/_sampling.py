"""Float64 references of the sampling contract (include/autogptq_b200.h, agb200_sample; DESIGN §3.21): Philox4x32-10 in
numpy, the kept set K of temperature, top-k, top-p and min-p, and a replay of the Gumbel-max draw with the kernel's
fp32 error bound.  Tokens whose membership or draw lies within fp32 rounding of a boundary are named ambiguous."""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)
FIX = 2.0 ** 40                         # the kernel's unit of top-p mass


def philox4x32_10(counter, key):
    """Philox4x32-10 of counters [n, 4] (uint32) under key (k0, k1) -> [n, 4] uint32 words."""
    c = np.asarray(counter, dtype=np.uint64).reshape(-1, 4) & MASK32
    c0, c1, c2, c3 = (c[:, i].copy() for i in range(4))
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
        p0, p1 = M0 * c0, M1 * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK32
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
    return np.stack([c0, c1, c2, c3], axis=1).astype(np.uint32)


def words(V: int, seed: int, counter: int) -> np.ndarray:
    """r_j for j < V: word j & 3 of Philox at counter (j >> 2, counter lo, counter hi, 0), key (seed lo, seed hi)."""
    seed, counter = int(seed) % 2 ** 64, int(counter) % 2 ** 64
    n = (V + 3) // 4
    ctr = np.zeros((n, 4), dtype=np.uint64)
    ctr[:, 0] = np.arange(n, dtype=np.uint64)
    ctr[:, 1] = counter & 0xFFFFFFFF
    ctr[:, 2] = counter >> 32
    return philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32)).reshape(-1)[:V]


def gumbel64(r: np.ndarray) -> np.ndarray:
    """g = -log(-log(u)), u = ((r >> 9) + 0.5)·2^-23, in float64."""
    u = ((r.astype(np.uint64) >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23
    return -np.log(-np.log(u))


def scaled(logits, temperature: float) -> np.ndarray:
    """s_j = fl32(float(l_j) / temperature) (IEEE fp32 division, as the kernel and transformers)."""
    return np.asarray(logits, dtype=np.float32) / np.float32(temperature)


def kept(s: np.ndarray, top_k: int, top_p: float, min_p: float, tol: float = 2e-6):
    """(sure, ambiguous) boolean masks over the tokens of scaled logits s (fp32, finite or -inf): ``sure`` is K where
    every test is clear, ``ambiguous`` the tokens whose top-p or min-p test lies within ``tol`` (relative) of its
    boundary plus the kernel's fixed-point and fp32 exp error.  Top-k on s is exact."""
    s = np.asarray(s, dtype=np.float32)
    V = s.size
    keep = np.isfinite(s) | (s == -np.inf)
    amb = np.zeros(V, dtype=bool)
    smax = s.max()
    if 0 < top_k < V:
        kth = np.partition(s, V - top_k)[V - top_k]
        keep &= s >= kth
    x = (s - smax).astype(np.float32).astype(np.float64)        # the kernel's fp32 difference
    e = np.exp(x)
    if top_p < 1:
        ek = np.where(keep, e, 0.0)
        order = np.argsort(-s, kind="stable")
        so, eo = s[order], ek[order]
        cum = np.cumsum(eo)
        # mass strictly above each sorted element: the cumulative sum before its group of equal values
        first = np.searchsorted(-so, -so, side="left")
        above = np.where(first > 0, cum[np.maximum(first - 1, 0)], 0.0)
        C = np.empty(V)
        C[order] = above
        Z = ek.sum()
        ratio = C / Z
        band = tol * top_p + (V + 2) / FIX / Z
        keep_p = ratio < top_p
        amb |= keep & (np.abs(ratio - top_p) <= band)
        keep &= keep_p
    if min_p > 0:
        keep_m = e >= min_p
        amb |= np.abs(e - min_p) <= tol * min_p
        keep &= keep_m
    return keep & ~amb, amb


def replay(s: np.ndarray, sure: np.ndarray, amb: np.ndarray, seed: int, counter: int):
    """(token, ambiguous): the Gumbel-max draw over K in float64 and whether another token of K, or an ambiguous
    member, lies within the kernel's fp32 error bound of the winner (logf ulps and the rounding of s + g)."""
    s64 = np.asarray(s, dtype=np.float32).astype(np.float64)
    g = gumbel64(words(s64.size, seed, counter))
    v = s64 + g
    err = 2.0 ** -21 * (1 + np.abs(g)) + 2.0 ** -22 * np.abs(v)
    cand = sure | amb
    vs = np.where(sure, v, -np.inf)
    if not np.isfinite(vs).any():
        return int(np.argmax(s64)), True
    tok = int(np.argmax(vs))
    near = cand & np.isfinite(v) & (v >= v[tok] - err - err[tok])
    return tok, bool(near.sum() > 1 or (amb & near).any())


def draw(s: np.ndarray, top_k: int, top_p: float, min_p: float, seed: int, counter: int):
    """(token, ambiguous) of one row: replay over the reference K."""
    sure, amb = kept(s, top_k, top_p, min_p)
    return replay(s, sure, amb, seed, counter)


def probabilities(s: np.ndarray, keep: np.ndarray) -> np.ndarray:
    """The renormalised softmax over K in float64."""
    s64 = np.asarray(s, dtype=np.float32).astype(np.float64)
    w = np.where(keep, np.exp(s64 - s64[keep].max()), 0.0)
    return w / w.sum()
