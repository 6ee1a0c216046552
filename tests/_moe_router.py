"""The MoE router (``agb200_moe_router``, ``autogptq_b200.moe.moe_router``): a float64 reference of transformers'
MixtralTopKRouter and the bounds that check the kernel's outputs to the ulp, each on the inputs the kernel actually saw.

Rounding points (transformers 5.5, MixtralDecoderLayer / MixtralRMSNorm / MixtralTopKRouter):

    h = rnd(x + x2)        n = rnd(rnd(h·r)·w)        (the chain's norm pre-pass: ``tests/_chain_norm.py``)
    l = rnd(n·Gᵀ)          F.linear: an fp32 sum rounded once to the dtype
    p = softmax(fp32 l)    idx = top-k of p, largest first     w = p_idx / Σ p_idx   (fp32)

Logits
    The kernel sums H products, each exact in fp32, in a fixed order.  As for every fp32 sum here (``tests/_precision``)
    the error is at most γ·A with γ = λ·√(H/4 + 64)·u and A = Σ|n|·|G|; the bound is doubled.  So l must lie between
    rnd(z − bound) and rnd(z + bound), z the float64 dot product of the kernel's own n: rnd(z) or its neighbour where z
    lies within the bound of a midpoint, and a few ulps where the sum cancels.

Softmax and the top-k margin
    p is computed from the kernel's own (rounded) logits.  l − m costs at most u·|l − m| (exact for most fp16 pairs),
    expf is within 2 ulp, the sum of E terms at most E·u relative and the division u: so each fp32 p is within
    δp = u·(|l − m| + E + 4) relative of the float64 softmax of the same logits (doubled below).  Two experts whose
    float64 p differ by more than δp·(p_a + p_b) are ordered the same by any correct implementation; closer pairs may
    go either way, except an exact tie of the logits, which the kernel resolves to the lower expert index.

Weights
    w_j = p_j / Σ p: relative error at most 2·δp + (k + 1)·u against the float64 ratio of the selected p.
"""
from __future__ import annotations

import numpy as np

from tests import _precision as P

U = P.U


def logit_bound(n, G) -> np.ndarray:
    """Absolute bound of the fp32 sum behind each logit, doubled: [T, E]."""
    H = np.asarray(n).shape[-1]
    A = np.abs(np.asarray(n, np.float64)) @ np.abs(np.asarray(G, np.float64)).T
    return 2.0 * P.LAMBDA * np.sqrt(H / 4 + 64) * U * A


def logit_candidates(n, G, dtype):
    """(l0, lo, hi) for the kernel's n [T, H] and the router weight G [E, H] (float64 arrays of dtype values):
    l0 = rnd(z) and the rounded ends of z ± bound.  Where the bound is below half an ulp, [lo, hi] holds l0 and at most
    one neighbour; where the sum cancels (A ≫ |z|, small logits) it may span a few ulps."""
    z = np.asarray(n, np.float64) @ np.asarray(G, np.float64).T
    d = logit_bound(n, G)
    return P.round_dt(z, dtype), P.round_dt(z - d, dtype), P.round_dt(z + d, dtype)


def check_logits(l, n, G, dtype, what="") -> float:
    """Assert every logit lies in its candidate range; returns the share that differs from rnd(z)."""
    l = np.asarray(l, np.float64)
    l0, lo, hi = logit_candidates(n, G, dtype)
    bad = ~((lo <= l) & (l <= hi))
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {l.size} logits lie outside their candidates (first at "
                           f"{np.argwhere(bad)[0].tolist()}: {l[bad][0]!r} vs [{lo[bad][0]!r}, {hi[bad][0]!r}])")
    return float((l != l0).sum()) / l.size


def softmax64(l) -> np.ndarray:
    l = np.asarray(l, np.float64)
    e = np.exp(l - l.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def delta_p(l) -> np.ndarray:
    """Relative bound of each fp32 p against softmax64 of the same logits, doubled: [T, E]."""
    l = np.asarray(l, np.float64)
    E = l.shape[-1]
    return 2.0 * U * (np.abs(l - l.max(-1, keepdims=True)) + E + 4)


def topk_ref(p, k) -> np.ndarray:
    """Indices of the k largest p per row, largest first, an exact tie to the lower index: int64 [T, k]."""
    p = np.asarray(p, np.float64)
    E = p.shape[-1]
    order = np.lexsort((np.broadcast_to(np.arange(E), p.shape), -p), axis=-1)
    return order[:, :k]


def check_topk(idx, l, k, what="") -> int:
    """The kernel's indices against the reference on its own logits l [T, E]: for every j < k whose gap to the next
    sorted p is clear, the first j + 1 indices are the reference's as a set; and wherever two experts have bit-equal
    logits, a selected higher index implies the lower one is selected before it.  Returns the unclear gaps seen."""
    idx = np.asarray(idx, np.int64)
    l = np.asarray(l, np.float64)
    p = softmax64(l)
    dp = delta_p(l)
    ref = topk_ref(p, min(k + 1, l.shape[-1]))
    unclear = 0
    for t in range(idx.shape[0]):
        assert len(set(idx[t].tolist())) == k and ((0 <= idx[t]) & (idx[t] < l.shape[-1])).all(), \
            f"{what}: row {t} indices {idx[t].tolist()} are not k distinct experts"
        for j in range(k):
            a = ref[t, j]
            if j + 1 < ref.shape[1]:
                b = ref[t, j + 1]
                clear = p[t, a] - p[t, b] > dp[t, a] * p[t, a] + dp[t, b] * p[t, b]
            else:
                clear = True
            if clear:
                assert set(idx[t, :j + 1].tolist()) == set(ref[t, :j + 1].tolist()), \
                    f"{what}: row {t} top-{j + 1} {idx[t, :j + 1].tolist()} != reference {ref[t, :j + 1].tolist()}"
            else:
                unclear += 1
        pos = {int(e): j for j, e in enumerate(idx[t])}
        for e, j in pos.items():
            for lower in np.flatnonzero(l[t, :e] == l[t, e]):
                assert int(lower) in pos and pos[int(lower)] < j, \
                    f"{what}: row {t}: expert {e} tied with {int(lower)} but the lower index did not go first"
    return unclear


def check_weights(w, idx, l, what="") -> float:
    """w [T, k] fp32 against p_idx / Σ p_idx of float64 p on the kernel's logits; returns the largest err/bound."""
    w = np.asarray(w, np.float64)
    idx = np.asarray(idx, np.int64)
    l = np.asarray(l, np.float64)
    p = softmax64(l)
    sel = np.take_along_axis(p, idx, -1)
    ref = sel / sel.sum(-1, keepdims=True)
    k = idx.shape[-1]
    bound = (2 * np.take_along_axis(delta_p(l), idx, -1) + (k + 1) * U) * 2 * np.abs(ref) + 1e-300
    err = np.abs(w - ref)
    assert (err <= bound).all(), (f"{what}: weights off by up to {float((err / bound).max()):.3g} of the bound "
                                  f"(first {w[err > bound][0]!r} vs {ref[err > bound][0]!r})")
    s = np.asarray(w, np.float32).sum(-1, dtype=np.float64)
    assert (np.abs(s - 1) <= 2 * (k + 2) * U).all(), f"{what}: weights sum to {s.tolist()}"
    return float((err / bound).max())


def router_model(n, G, k, dtype):
    """transformers' MixtralTopKRouter restated in float64 from n (already rounded): (logits rounded to the dtype,
    p, idx, w).  Its p is the softmax of the rounded logits, as F.linear's output is 16-bit."""
    l = P.round_dt(np.asarray(n, np.float64) @ np.asarray(G, np.float64).T, dtype)
    p = softmax64(l)
    idx = topk_ref(p, k)
    sel = np.take_along_axis(p, idx, -1)
    return l, p, idx, sel / sel.sum(-1, keepdims=True)
