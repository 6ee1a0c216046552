"""The decoders' KV caches (DESIGN §3.18, §3.19, §3.22): where each layer's key and value rows live, how they are
stored and which attention call reads and writes them.  For the same contents both layouts give the same outputs and
cache bytes, bit for bit.  Only the attention calls need CUDA tensors."""
from __future__ import annotations

import torch

from .attention import (FP8, attention_rows_supported, decode_attention_rows, decode_attention_rows_paged,
                        paged_attention_supported, prefill_attention, prefill_attention_paged, quantize_kv)
from .paged_kv import BlockAllocator, blocks_for, worst_case_blocks


class KVCache:
    """The static cache of ``rows`` sequences of up to ``max_length`` positions: per layer ``k[i]`` / ``v[i]``
    [rows, n_kv, max_length, head_dim] in the activation ``dtype``, or with ``fp8`` E4M3 codes and fp32 scales
    ``k_scale[i]`` / ``v_scale[i]`` [rows, n_kv, max_length] (``quantize_kv``'s rule).  Every slot owns its row, so
    ``reserve`` and ``release`` have nothing to do, and it holds no blocks (``num_blocks`` 0)."""

    num_blocks = 0
    blocks_free = None

    def __init__(self, rows: int, n_kv: int, max_length: int, head_dim: int, dtype, fp8: bool):
        self.rows, self.n_kv, self.head_dim, self.dtype, self.fp8 = int(rows), n_kv, head_dim, dtype, bool(fp8)
        self.length = int(max_length)          # positions a row can address: the decode workspace's max_length
        self.shape = (self.rows, n_kv, self.length, head_dim)

    def unsupported(self, n_heads: int) -> str | None:
        """None when the per-row decode and prefill attention take this cache, else the reason they do not."""
        return attention_rows_supported(n_heads, self.n_kv, self.head_dim, self.rows, self.length, self.dtype)

    def allocate(self, layers: int, device):
        self.k = [torch.zeros(self.shape, dtype=FP8 if self.fp8 else self.dtype, device=device) for _ in range(layers)]
        self.v = [torch.zeros_like(c) for c in self.k]
        self.k_scale = self.v_scale = None
        if self.fp8:
            self.k_scale = [torch.ones(self.shape[:-1], dtype=torch.float32, device=device) for _ in range(layers)]
            self.v_scale = [torch.ones_like(s) for s in self.k_scale]

    @property
    def nbytes(self) -> int:
        """Bytes of every layer's tensors, scales included."""
        ts = self.k + self.v + (self.k_scale + self.v_scale if self.fp8 else [])
        return sum(t.numel() * t.element_size() for t in ts)

    def scales(self, i: int) -> dict:
        """Layer i's ``k_scale`` / ``v_scale`` keyword arguments of the attention calls ({} for a 16-bit cache)."""
        return dict(k_scale=self.k_scale[i], v_scale=self.v_scale[i]) if self.fp8 else {}

    def _positions(self, rows: slice, T: int):
        return rows, slice(0, T)            # the index of the slots' positions 0 .. T - 1 in [.., position, n_kv, ...]

    def store(self, i: int, rows: slice, keys, values):
        """Keys and values [len(rows), n_kv, T, head_dim] of the reserved slots ``rows`` at positions 0 .. T - 1."""
        at = self._positions(rows, keys.shape[2])
        for cache, scales, x in ((self.k[i], self.k_scale, keys), (self.v[i], self.v_scale, values)):
            if self.fp8:
                x, sc = quantize_kv(x)
                scales[i].transpose(1, 2)[at] = sc.transpose(1, 2)
                cache, x = cache.view(torch.uint8), x.view(torch.uint8)
            cache.transpose(1, 2)[at] = x.transpose(1, 2)

    def decode(self, i: int, q, k, v, pos, inv_freq, attention_scaling, scaling, out, workspace):
        """``decode_attention_rows`` of layer i over every row."""
        decode_attention_rows(q, k, v, self.k[i], self.v[i], pos, inv_freq, attention_scaling, scaling, out,
                              workspace, **self.scales(i))

    def prefill(self, i: int, rows: slice, q, k, v, start, inv_freq, attention_scaling, scaling, out):
        """``prefill_attention`` of layer i on the slots ``rows``: writes the new rows and attends causally."""
        prefill_attention(q, k, v, self.k[i][rows], self.v[i][rows], start, inv_freq, attention_scaling, scaling, out,
                          **{n: s[rows] for n, s in self.scales(i).items()})

    def fits(self, slot: int, n_tokens: int) -> bool:
        return True

    def reserve(self, need: dict):
        pass

    def release(self, slot: int):
        pass

    def worst_case_blocks(self, prompt_len: int, max_new_tokens: int, n: int) -> int:
        return 0


class PagedKVCache(KVCache):
    """The paged cache: per layer pools ``k[i]`` / ``v[i]`` [num_blocks, n_kv, block_size, head_dim] (FP8 scales
    [num_blocks, n_kv, block_size]; default num_blocks rows·ceil(max_length / block_size), the static capacity), the
    int32 device block table ``table`` [rows, max_blocks] (-1: no block) and a host ``BlockAllocator``.  Position t of
    slot s is row t % block_size of block table[s, t // block_size]."""

    def __init__(self, rows: int, n_kv: int, max_length: int, head_dim: int, dtype, fp8: bool, block_size: int,
                 num_blocks=None):
        super().__init__(rows, n_kv, max_length, head_dim, dtype, fp8)
        self.block_size = int(block_size)
        self.max_blocks = blocks_for(max_length, self.block_size)
        self.num_blocks = self.rows * self.max_blocks if num_blocks is None else int(num_blocks)
        self.length = self.max_blocks * self.block_size
        self.shape = (self.num_blocks, n_kv, self.block_size, head_dim)

    def unsupported(self, n_heads: int) -> str | None:
        return paged_attention_supported(n_heads, self.n_kv, self.head_dim, self.rows, self.block_size,
                                         self.num_blocks, self.dtype)

    def allocate(self, layers: int, device):
        super().allocate(layers, device)
        self.table = torch.full((self.rows, self.max_blocks), -1, dtype=torch.int32, device=device)
        self.allocator = BlockAllocator(self.num_blocks, self.block_size, self.rows, self.max_blocks)

    @property
    def blocks_free(self) -> int:
        return self.allocator.free

    def _positions(self, rows: slice, T: int):
        """(block, row in it) [len(rows), T] of the slots' positions 0 .. T - 1; IndexError where no block is held."""
        t = torch.arange(T)
        blk = torch.stack([torch.tensor(self.allocator.blocks[s], dtype=torch.int64)[t // self.block_size]
                           for s in range(self.rows)[rows]])
        return blk.to(self.table.device), (t % self.block_size).to(self.table.device)

    def decode(self, i: int, q, k, v, pos, inv_freq, attention_scaling, scaling, out, workspace):
        decode_attention_rows_paged(q, k, v, self.k[i], self.v[i], self.table, pos, inv_freq, attention_scaling,
                                    scaling, out, workspace, **self.scales(i))

    def prefill(self, i: int, rows: slice, q, k, v, start, inv_freq, attention_scaling, scaling, out):
        prefill_attention_paged(q, k, v, self.k[i], self.v[i], self.table[rows], start, inv_freq, attention_scaling,
                                scaling, out, **self.scales(i))

    def fits(self, slot: int, n_tokens: int) -> bool:
        """Whether the pool can hold ``n_tokens`` positions for the slot once the slot has released its blocks."""
        own = sum(self.allocator.ref[b] == 1 for b in self.allocator.blocks[slot])
        return blocks_for(n_tokens, self.block_size) <= self.allocator.free + own

    def reserve(self, need: dict):
        """Blocks for positions 0 .. need[s] - 1 of each slot s (``BlockAllocator.map``), mirrored into the table."""
        for s, j, b in self.allocator.map(need):
            self.table[s, j] = b

    def release(self, slot: int):
        """The slot drops its blocks (a block no slot holds is free) and its table row becomes -1."""
        self.allocator.release(slot)
        self.table[slot].fill_(-1)

    def fork(self, src: int, dst: int, pos: int):
        """The empty slot ``dst`` gets ``src``'s positions 0 .. pos - 1 (``BlockAllocator.fork``): its full blocks by
        reference and a copy of its partial last block in every layer, FP8 scales included."""
        blocks, copy = self.allocator.fork(src, dst, pos)
        if copy is not None:
            a, b = copy
            for ts in (self.k, self.v, self.k_scale or [], self.v_scale or []):
                for t in ts:
                    t[b].copy_(t[a])
        self.table[dst, :len(blocks)] = torch.tensor(blocks, dtype=torch.int32)

    def worst_case_blocks(self, prompt_len: int, max_new_tokens: int, n: int) -> int:
        return worst_case_blocks(prompt_len, max_new_tokens, n, self.block_size)


__all__ = ["KVCache", "PagedKVCache"]
