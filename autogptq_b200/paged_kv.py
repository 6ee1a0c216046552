"""Host-side block allocator of a paged KV cache (DESIGN §3.22): which pool blocks each slot holds, and how many slots
hold each block.

A slot's blocks are its block-table row in order: block j holds positions j·block_size .. (j+1)·block_size - 1.  A block
is free (count 0) or held by one or more slots (count = the number of slots whose list has it).  Invariant: the block
holding the position a slot writes next has count 1, so the kernels never write a block another slot reads.  Full
blocks are shared by ``fork``; the partially filled last block is never shared (``fork`` hands back a fresh block for a
copy of it).  Every method that can fail checks first and changes nothing when it raises.  Pure Python:
``kv_cache.PagedKVCache`` mirrors every change into its device block table.
"""
from __future__ import annotations


def blocks_for(n_tokens: int, block_size: int) -> int:
    """Blocks that hold positions 0 .. n_tokens - 1."""
    return -(-int(n_tokens) // block_size)


def worst_case_blocks(prompt_len: int, max_new_tokens: int, n: int, block_size: int) -> int:
    """The most blocks a prompt and its ``n`` samples ever hold at once: the prompt's full blocks once, plus for each
    sample its own blocks from the prompt's partial block up to its last written position.  A sample of
    ``max_new_tokens`` tokens writes positions up to prompt_len + max_new_tokens - 2 (its last token is never written)."""
    shared = int(prompt_len) // block_size
    written = max(int(prompt_len) + int(max_new_tokens) - 1, int(prompt_len))
    return shared + n * (blocks_for(written, block_size) - shared)


class BlockAllocator:
    """Blocks of a pool of ``num_blocks`` blocks of ``block_size`` rows for ``slots`` slots of at most ``max_blocks``
    blocks each."""

    def __init__(self, num_blocks: int, block_size: int, slots: int, max_blocks: int):
        self.num_blocks, self.block_size, self.max_blocks = int(num_blocks), int(block_size), int(max_blocks)
        self.ref = [0] * self.num_blocks
        self._free = list(range(self.num_blocks - 1, -1, -1))   # a stack: block 0 is handed out first
        self.blocks = [[] for _ in range(slots)]

    @property
    def free(self) -> int:
        """Blocks with count 0."""
        return len(self._free)

    def _take(self) -> int:
        b = self._free.pop()
        self.ref[b] = 1
        return b

    def map(self, need: dict) -> list:
        """Give every slot s of ``need`` enough blocks for positions 0 .. need[s] - 1.  Raises RuntimeError, with no
        change, when the pool cannot supply them all or a slot would pass max_blocks.  Returns the new table entries
        [(slot, j, block)]."""
        want = {s: blocks_for(n, self.block_size) - len(self.blocks[s]) for s, n in need.items()}
        for s, n in need.items():
            if blocks_for(n, self.block_size) > self.max_blocks:
                raise RuntimeError(f"slot {s}: {n} positions need more than {self.max_blocks} blocks")
        total = sum(w for w in want.values() if w > 0)
        if total > self.free:
            raise RuntimeError(f"the KV cache pool is exhausted: {total} more blocks needed, {self.free} free of "
                               f"{self.num_blocks}")
        new = []
        for s, w in want.items():
            for _ in range(max(w, 0)):
                b = self._take()
                new.append((s, len(self.blocks[s]), b))
                self.blocks[s].append(b)
        return new

    def fork(self, src: int, dst: int, n_tokens: int):
        """Give the empty slot ``dst`` slot ``src``'s first ``n_tokens`` positions: its full blocks by reference, and a
        fresh block for the partially filled one.  Returns (dst's blocks, (src block, fresh block) to copy, or None).
        Raises RuntimeError, with no change, when no block is free for the copy."""
        if self.blocks[dst]:
            raise RuntimeError(f"slot {dst} still holds blocks")
        full, part = divmod(int(n_tokens), self.block_size)
        if len(self.blocks[src]) < full + (part > 0):
            raise RuntimeError(f"slot {src} holds {len(self.blocks[src])} blocks, fewer than {n_tokens} positions need")
        if part and not self._free:
            raise RuntimeError(f"the KV cache pool is exhausted: fork needs 1 block, 0 free of {self.num_blocks}")
        shared = self.blocks[src][:full]
        for b in shared:
            self.ref[b] += 1
        copy = None
        self.blocks[dst] = list(shared)
        if part:
            copy = (self.blocks[src][full], self._take())
            self.blocks[dst].append(copy[1])
        return list(self.blocks[dst]), copy

    def release(self, slot: int):
        """Drop the slot's references; a block whose count reaches 0 is free again."""
        for b in reversed(self.blocks[slot]):
            self.ref[b] -= 1
            if self.ref[b] == 0:
                self._free.append(b)
        self.blocks[slot] = []

    def writable(self, slot: int, pos: int) -> bool:
        """Whether the slot holds the block of position ``pos`` and no other slot does."""
        j = int(pos) // self.block_size
        return j < len(self.blocks[slot]) and self.ref[self.blocks[slot][j]] == 1


__all__ = ["BlockAllocator", "blocks_for", "worst_case_blocks"]
