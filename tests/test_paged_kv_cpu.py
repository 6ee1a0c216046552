"""The paged KV cache without a GPU: the four C entries are declared and bound at ABI 11, the refusals of the Python API,
the host block allocator on its own (boundary crossings, forks, the written-block invariant, release, exhaustion,
``generate``'s admission on random workloads), and the float64 reference of paged attention against the static one."""
import os
import random
import re

import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from autogptq_b200.attention import decode_attention_rows_paged, paged_attention_supported, prefill_attention_paged
from autogptq_b200.paged_kv import BlockAllocator, blocks_for, worst_case_blocks
from tests import _paged as PG
from tests._batch_attention import rows_reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ["agb200_decode_attention_rows_paged", "agb200_decode_attention_rows_paged_fp8",
           "agb200_prefill_attention_paged", "agb200_prefill_attention_paged_fp8"]


def test_entries_declared_and_bound_at_abi_11():
    header = open(os.path.join(ROOT, "include", "autogptq_b200.h")).read()
    bound = _lib.declared_symbols()
    for name in ENTRIES:
        assert re.search(rf"\bint {name}\(", header), name
        assert name in bound, name
    assert _lib.ABI_VERSION == 11
    assert re.search(r"#define AGB200_ABI_VERSION 11\b", header)


def test_signatures_match_the_header():
    header = open(os.path.join(ROOT, "include", "autogptq_b200.h")).read()
    sigs = {}

    class Fake:
        def __getattr__(self, name):
            class F:
                pass
            f = F()
            sigs[name] = f
            return f
    _lib._declare(Fake())
    for name in ENTRIES:
        decl = re.search(rf"int {name}\(([^;]*)\);", header).group(1)
        assert len(decl.split(",")) == len(sigs[name].argtypes), name


@pytest.mark.parametrize("bs", [0, 8, 24, 48, 512])
def test_refuses_block_sizes(bs):
    why = paged_attention_supported(32, 8, 128, 8, bs, 100, torch.float16)
    assert why is not None and "block_size" in why


def test_refuses_pools_of_2_31_elements():
    # 8 kv heads · 16 rows · 128 dims = 2^14 elements per block: 2^17 blocks reach 2^31
    assert paged_attention_supported(32, 8, 128, 8, 16, 2 ** 17 - 1, torch.float16) is None
    assert "2^31" in paged_attention_supported(32, 8, 128, 8, 16, 2 ** 17, torch.float16)
    assert paged_attention_supported(32, 8, 128, 8, 64, 0, torch.float16) is not None


def _args(table, T=None):
    B = table.shape[0]
    lead = (B,) if T is None else (B, T)
    q = torch.zeros(lead + (256,), dtype=torch.float16)
    kv = torch.zeros(lead + (128,), dtype=torch.float16)
    pool = torch.zeros((10, 2, 16, 64), dtype=torch.float16)
    return q, kv, kv, pool, pool.clone(), table, torch.zeros(B, dtype=torch.int64), torch.zeros(32), 1.0, 0.125, q


@pytest.mark.parametrize("table", [torch.zeros((2, 4), dtype=torch.int64), torch.zeros((2, 4), dtype=torch.int16),
                                   torch.zeros(8, dtype=torch.int32), torch.zeros((2, 4, 1), dtype=torch.int32)])
def test_refuses_table_dtype_and_shape(table):
    with pytest.raises(ValueError, match="block_table"):
        decode_attention_rows_paged(*_args(table))
    with pytest.raises(ValueError, match="block_table"):
        prefill_attention_paged(*_args(table, T=3))


def test_refuses_table_rows_other_than_q_rows():
    args = list(_args(torch.zeros((2, 4), dtype=torch.int32)))
    args[5] = torch.zeros((3, 4), dtype=torch.int32)
    with pytest.raises(ValueError, match="rows"):
        decode_attention_rows_paged(*args)


# ---------------------------------------------------------------------- the allocator
def test_boundary_crossings_map_exactly_one_block():
    a = BlockAllocator(64, 16, 4, 16)
    assert len(a.map({0: 1})) == 1
    for n in range(2, 200):
        new = a.map({0: n})
        assert len(new) == (1 if (n - 1) % 16 == 0 else 0), n
        assert len(a.blocks[0]) == blocks_for(n, 16)
    assert a.free == 64 - blocks_for(199, 16)


def test_fork_shares_full_blocks_and_copies_the_partial_one():
    a = BlockAllocator(32, 16, 4, 8)
    a.map({0: 40})                                      # 2 full blocks and 8 rows of a third
    blocks, copy = a.fork(0, 1, 40)
    assert blocks[:2] == a.blocks[0][:2] and blocks[2] != a.blocks[0][2]
    assert copy == (a.blocks[0][2], blocks[2])
    assert [a.ref[b] for b in a.blocks[0]] == [2, 2, 1] and a.ref[blocks[2]] == 1
    blocks2, copy2 = a.fork(0, 2, 32)                  # on a block boundary: nothing to copy
    assert copy2 is None and blocks2 == a.blocks[0][:2]
    assert [a.ref[b] for b in a.blocks[0][:2]] == [3, 3]


def test_the_written_block_always_has_count_1():
    rng = random.Random(3)
    a = BlockAllocator(400, 16, 8, 32)
    pos = [-1] * 8
    for _ in range(2000):
        s = rng.randrange(8)
        op = rng.random()
        try:
            if pos[s] < 0 and op < 0.3:
                n = rng.randrange(1, 200)
                a.map({s: n})
                pos[s] = n
            elif pos[s] < 0 and op < 0.6:
                src = rng.choice([i for i in range(8) if pos[i] >= 0] or [s])
                if src != s and pos[src] >= 0:
                    a.fork(src, s, pos[src])
                    pos[s] = pos[src]
            elif pos[s] >= 0 and op < 0.1:
                a.release(s)
                pos[s] = -1
            elif pos[s] >= 0 and pos[s] < 500:
                a.map({s: pos[s] + 1})                 # the block of the position the step writes
                assert a.writable(s, pos[s])
                pos[s] += 1
        except RuntimeError:
            pass
        assert sum(a.ref) == sum(len(b) for b in a.blocks)
        assert a.free == sum(r == 0 for r in a.ref)


def test_release_frees_at_count_0():
    a = BlockAllocator(16, 16, 3, 8)
    a.map({0: 50})
    a.fork(0, 1, 50)
    held = a.free
    a.release(0)
    assert a.free == held + 1                          # only 0's partial block had count 1
    a.release(1)
    assert a.free == 16 and all(r == 0 for r in a.ref)


def test_exhaustion_raises_with_state_unchanged():
    a = BlockAllocator(5, 16, 3, 8)
    a.map({0: 40})
    before = (list(a.ref), [list(b) for b in a.blocks], a.free)
    with pytest.raises(RuntimeError, match="exhausted"):
        a.map({1: 20, 2: 20})                           # 4 blocks, 2 free
    assert (list(a.ref), [list(b) for b in a.blocks], a.free) == before
    a.map({1: 32})
    with pytest.raises(RuntimeError, match="exhausted"):
        a.fork(0, 2, 40)
    assert a.blocks[2] == [] and a.free == 0


def test_worst_case_blocks():
    # a 40-token prompt (2 full blocks of 16) and 4 samples of 30 tokens: each writes up to position 68 (5 blocks)
    assert worst_case_blocks(40, 30, 4, 16) == 2 + 4 * 3
    assert worst_case_blocks(32, 1, 2, 16) == 2
    assert worst_case_blocks(32, 2, 2, 16) == 2 + 2 * 1


@pytest.mark.parametrize("seed", range(6))
def test_generate_admission_never_over_commits(seed):
    """Replays generate's admission and decoding on the allocator with random prompt lengths, sample counts, EOS
    and pool sizes: no step ever runs out of blocks."""
    rng = random.Random(seed)
    bs, max_batch, max_new = rng.choice([16, 32, 64]), 8, rng.randrange(1, 120)
    n = rng.randrange(1, 5)
    prompts = [rng.randrange(1, 300) for _ in range(rng.randrange(1, 20))]
    worst = [worst_case_blocks(p, max_new, n, bs) for p in prompts]
    nb = rng.randrange(max(worst), 2 * max(worst) + 1)
    a = BlockAllocator(nb, bs, max_batch, blocks_for(400 + max_new, bs))
    owner, pos, left, live = [None] * max_batch, [-1] * max_batch, [0] * max_batch, {}
    queue, committed, peak = list(range(len(prompts))), 0, 0
    while True:
        while queue:
            free = [s for s in range(max_batch) if owner[s] is None]
            j = queue[0]
            if len(free) < n or committed + worst[j] > nb:
                break
            queue.pop(0)
            committed += worst[j]
            live[j] = n
            a.map({free[0]: prompts[j]})
            for s in free[1:n]:
                a.fork(free[0], s, prompts[j])
            for s in free[:n]:
                owner[s], pos[s], left[s] = j, prompts[j], max_new - 1
        for s in range(max_batch):                      # first tokens and EOS
            if owner[s] is not None and (left[s] == 0 or rng.random() < 0.02):
                j = owner[s]
                a.release(s)
                owner[s] = None
                live[j] -= 1
                if live[j] == 0:
                    committed -= worst[j]
        active = [s for s in range(max_batch) if owner[s] is not None]
        if not active and not queue:
            break
        if active:
            a.map({s: pos[s] + 1 for s in active})      # never raises
            peak = max(peak, nb - a.free)
            assert nb - a.free <= committed
            for s in active:
                pos[s] += 1
                left[s] -= 1
    assert a.free == nb and peak <= nb


# ---------------------------------------------------------------------- the float64 reference
def test_paged_reference_equals_the_static_reference():
    rng = np.random.default_rng(0)
    B, n_kv, G, hd, bs, max_blocks = 3, 2, 4, 64, 16, 6
    L = bs * max_blocks
    K, V = rng.standard_normal((2, B, n_kv, L, hd))
    qh = rng.standard_normal((B, n_kv * G, hd))
    pos = np.array([L - 1, 17, -1])
    table = PG.make_table(B, max_blocks, B * max_blocks + 5, "scrambled")
    pool_k = np.full((B * max_blocks + 5, n_kv, bs, hd), np.nan)
    pool_v = pool_k.copy()
    PG.scatter(pool_k, table, K)
    PG.scatter(pool_v, table, V)
    assert np.array_equal(PG.gather(pool_k, table, L), K)
    o, _ = PG.paged_reference(qh, pool_k, pool_v, table, pos, 0.125)
    o_static, _ = rows_reference(qh, K, V, pos, 0.125)
    assert np.array_equal(o, o_static)
