"""Paged KV cache helpers of the tests: block tables, pools built from static caches and back, and the float64 reference
of paged attention (the static layout gathered through the table, then ``tests/_batch_attention.py::rows_reference``)."""
from __future__ import annotations

import numpy as np

from tests._batch_attention import rows_reference


def make_table(B, max_blocks, num_blocks, mode, seed=0):
    """int32 [B, max_blocks]: distinct blocks for every (row, j), 'scrambled' (a random permutation of the pool),
    'reversed' (the last blocks first) or 'ordered'."""
    ids = np.arange(num_blocks)
    if mode == "scrambled":
        ids = np.random.default_rng(seed).permutation(num_blocks)
    elif mode == "reversed":
        ids = ids[::-1]
    return np.ascontiguousarray(ids[:B * max_blocks].reshape(B, max_blocks)).astype(np.int32)


def _index(pool, table, length):
    """(block, offset) indices [B·length] of every position of every row, as the pool's array type."""
    bs = pool.shape[2]
    t = np.arange(length)
    blk = np.asarray(table, np.int64)[:, t // bs].reshape(-1)
    off = np.tile(t % bs, len(table))
    if isinstance(pool, np.ndarray):
        return blk, off
    import torch
    return torch.as_tensor(blk, device=pool.device), torch.as_tensor(off, device=pool.device)


def gather(pool, table, length):
    """A pool [num_blocks, n_kv, bs, ...] seen through the table [B, max_blocks] as the static layout
    [B, n_kv, length, ...] (numpy or torch)."""
    blk, off = _index(pool, table, length)
    rows = pool[blk, :, off]                                                # [B·length, n_kv, ...]
    rows = rows.reshape((len(table), length) + tuple(pool.shape[1:2]) + tuple(pool.shape[3:]))
    return rows.swapaxes(1, 2) if isinstance(rows, np.ndarray) else rows.transpose(1, 2).contiguous()


def scatter(pool, table, static):
    """Writes the static layout [B, n_kv, L, ...] into the pool through the table (in place; numpy or torch)."""
    B, L = static.shape[0], static.shape[2]
    blk, off = _index(pool, table, L)
    rows = static.swapaxes(1, 2) if isinstance(static, np.ndarray) else static.transpose(1, 2)
    pool[blk, :, off] = rows.reshape((B * L,) + tuple(static.shape[1:2]) + tuple(static.shape[3:]))
    return pool


def paged_reference(qh, k_pool, v_pool, table, pos, scaling):
    """float64 paged attention: qh [B, H, hd], pools [num_blocks, n_kv, bs, hd] (numpy, dequantised), table [B,
    max_blocks], pos [B] -> rows_reference on the gathered static layout."""
    L = np.asarray(table).shape[1] * k_pool.shape[2]
    K = gather(np.asarray(k_pool, np.float64), table, L)
    V = gather(np.asarray(v_pool, np.float64), table, L)
    return rows_reference(qh, K, V, pos, scaling)
