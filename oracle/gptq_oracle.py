"""NumPy fp32 restatement of the reference GPTQ quantiser (tests only).

Follows auto_gptq/quantization/gptq.py (add_batch :34-60, fasterquant :62-194) and quantizer.py (find_params :45-126,
quantize :10-14) operation by operation in float32, so that with the same inverse-Hessian factor it reproduces the
reference's single-block results bit for bit.  Settings: 4 bits, per-channel, no MSE search.
"""
from __future__ import annotations

import numpy as np

MAXQ = 15
f32 = np.float32


def add_batch(H, nsamples, inp):
    """One add_batch (gptq.py:38-60): the batch size is the leading dimension of a 3-D input, 1 for a 2-D input."""
    inp = np.asarray(inp)
    if inp.ndim == 2:
        inp = inp[None]
    tmp = inp.shape[0]
    x = inp.reshape(-1, inp.shape[-1]).astype(f32).T              # [K, tokens]
    H = H * f32(nsamples / (nsamples + tmp))
    nsamples += tmp
    x = f32(np.sqrt(2 / nsamples)) * x
    return (H + x @ x.T).astype(f32), nsamples


def find_params(x, sym):
    """Per-row (scale, zero) of x [rows, cols] (quantizer.py:64-85)."""
    x = np.asarray(x, dtype=f32)
    xmin = np.minimum(x.min(1), f32(0))
    xmax = np.maximum(x.max(1), f32(0))
    if sym:
        xmax = np.maximum(np.abs(xmin), xmax)
        neg = xmin < 0
        xmin = np.where(neg, -xmax, xmin)
    both = (xmin == 0) & (xmax == 0)
    xmin = np.where(both, f32(-1), xmin).astype(f32)
    xmax = np.where(both, f32(1), xmax).astype(f32)
    scale = ((xmax - xmin) / f32(MAXQ)).astype(f32)
    zero = np.full_like(scale, f32((MAXQ + 1) / 2)) if sym else np.rint(-xmin / scale).astype(f32)
    return scale, zero


def quantize(w, scale, zero):
    """(dequantised value, integer code) of a column (quantizer.py:10-14)."""
    q = np.clip(np.rint(w / scale) + zero, 0, MAXQ).astype(f32)
    return (scale * (q - zero)).astype(f32), q.astype(np.uint8)


def hinv_factor(H, percdamp=0.01, actorder=False):
    """Dead columns, act-order permutation, damping and the upper Cholesky factor of the inverse (gptq.py:84-119), in
    float64 LAPACK (the reference uses torch's float32 factorisation; tests that need bit agreement take its Hinv)."""
    H = np.array(H, dtype=f32)
    dead = np.diag(H) == 0
    H[dead, dead] = 1
    perm = None
    if actorder:
        perm = np.argsort(-np.diag(H), kind="stable")
        H = H[perm][:, perm]
    H[np.diag_indices_from(H)] += f32(percdamp) * np.mean(np.diag(H))
    L = np.linalg.cholesky(H.astype(np.float64))
    Linv = np.linalg.inv(L)
    Hi = Linv.T @ Linv
    U = np.linalg.cholesky(Hi).T
    return U.astype(f32), perm, dead


def fasterquant(W, Hinv, perm=None, dead=None, group_size=-1, sym=True, static_groups=False, blocksize=128):
    """The column loop of gptq.py:70-194 on W [N, K] (original order) with a given Hinv (processing order).

    Returns dict(Q, codes [N, K] original order, scale [N, G], zero [N, G], g_idx [K], losses [N, K] processing order)."""
    W = np.array(W, dtype=f32)
    N, K = W.shape
    scale0, zero0 = find_params(W, sym)                               # :79-80, before the dead columns are zeroed
    if dead is not None:
        W[:, dead] = 0
    scales, zeros, groups = [], [], []
    if static_groups and group_size != -1:                            # :93-102
        for i in range(0, K, group_size):
            s, z = find_params(W[:, i:i + group_size], sym)
            scales.append(s)
            zeros.append(z)
            groups.append((s, z))
    if perm is not None:
        W = W[:, perm]
    Q = np.zeros_like(W)
    codes = np.zeros(W.shape, dtype=np.uint8)
    losses = np.zeros_like(W)
    cur = (scale0, zero0)
    now_idx = 1
    for i1 in range(0, K, blocksize):
        i2 = min(i1 + blocksize, K)
        W1 = W[:, i1:i2].copy()
        Err1 = np.zeros_like(W1)
        Hinv1 = Hinv[i1:i2, i1:i2]
        for i in range(i2 - i1):
            w = W1[:, i]
            d = Hinv1[i, i]
            if group_size != -1:
                if not static_groups:
                    if (i1 + i) % group_size == 0:                    # :137-143, from the OUTER W
                        cur = find_params(W[:, i1 + i:i1 + i + group_size], sym)
                    if (i1 + i) // group_size - now_idx == -1:
                        scales.append(cur[0])
                        zeros.append(cur[1])
                        now_idx += 1
                else:
                    idx = i1 + i if perm is None else perm[i1 + i]
                    cur = groups[idx // group_size]
            q, c = quantize(w, cur[0], cur[1])
            Q[:, i1 + i] = q
            codes[:, i1 + i] = c
            losses[:, i1 + i] = ((w - q) ** 2 / d ** 2) / f32(2)
            err1 = ((w - q) / d).astype(f32)
            W1[:, i:] -= np.outer(err1, Hinv1[i, i:]).astype(f32)     # :155, product then subtraction
            Err1[:, i] = err1
        W[:, i2:] -= (Err1 @ Hinv[i1:i2, i2:]).astype(f32)
    gs = group_size if group_size != -1 else K
    if static_groups and perm is not None:
        g_idx = np.array([perm[i] // gs for i in range(K)], dtype=np.int32)
    else:
        g_idx = np.array([i // gs for i in range(K)], dtype=np.int32)
    if perm is not None:
        inv = np.argsort(perm)
        Q, codes, g_idx = Q[:, inv], codes[:, inv], g_idx[inv]
    if not scales:
        scales, zeros = [cur[0]], [cur[1]]
    return dict(Q=Q, codes=codes, scale=np.stack(scales, 1), zero=np.stack(zeros, 1), g_idx=g_idx, losses=losses)


def pack_codes(codes, zero, scale, dtype=np.float16):
    """Checkpoint tensors from codes [N, K] and parameters [N, G]: qweight [K/8, N], qzeros [G, N/8], scales [G, N]."""
    q = np.asarray(codes, dtype=np.uint32).T                          # [K, N]
    K, N = q.shape
    qw = np.zeros((K // 8, N), dtype=np.uint32)
    for j in range(8):
        qw |= (q[j::8] & 15) << np.uint32(4 * j)
    z = ((np.asarray(zero).T.astype(np.int64) - 1) & 15).astype(np.uint32)   # [G, N]
    qz = np.zeros((z.shape[0], N // 8), dtype=np.uint32)
    for j in range(8):
        qz |= z[:, j::8] << np.uint32(4 * j)
    return qw.view(np.int32), qz.view(np.int32), np.asarray(scale).T.astype(dtype)


def unpack_codes(qweight):
    """codes [N, K] of a packed qweight [K/8, N]."""
    qw = np.asarray(qweight).view(np.uint32)
    K8, N = qw.shape
    out = np.zeros((K8 * 8, N), dtype=np.uint8)
    for j in range(8):
        out[j::8] = (qw >> np.uint32(4 * j)) & 15
    return out.T.copy()
