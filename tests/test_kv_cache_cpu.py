"""The two KV cache layouts of ``autogptq_b200.kv_cache`` on CPU tensors, fp16 and bf16, 16-bit and FP8: rows stored into
a paged cache and gathered through its block table equal the static cache's bit for bit (codes and scales), ``fork``
shares full blocks and copies the partial one in every layer, ``release`` frees blocks and clears the table row, a
``reserve`` the pool cannot meet changes nothing, and ``nbytes`` counts every tensor."""
import pytest
import torch

from autogptq_b200.kv_cache import KVCache, PagedKVCache
from tests import _paged as PG

FP8 = torch.float8_e4m3fn
ROWS, N_KV, MAX_LENGTH, HD, LAYERS, BS = 3, 2, 80, 64, 2, 16
DTS = pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
KVS = pytest.mark.parametrize("fp8", [False, True], ids=["16bit", "fp8"])


def _caches(dtype, fp8, num_blocks=20):
    st = KVCache(ROWS, N_KV, MAX_LENGTH, HD, dtype, fp8)
    pg = PagedKVCache(ROWS, N_KV, MAX_LENGTH, HD, dtype, fp8, BS, num_blocks)
    for c in (st, pg):
        c.allocate(LAYERS, "cpu")
    return st, pg


def _tensors(c):
    """Every layer's tensors, FP8 codes as bytes."""
    ts = [t.view(torch.uint8) if t.dtype == FP8 else t for t in c.k + c.v]
    return ts + (c.k_scale + c.v_scale if c.fp8 else [])


def _rows(c, i, slot, T):
    """Layer i's keys, values (and scales) at positions :T of the slot, static layout, FP8 codes as bytes."""
    ts = [c.k[i], c.v[i]] + ([c.k_scale[i], c.v_scale[i]] if c.fp8 else [])
    ts = [t.view(torch.uint8) if t.dtype == FP8 else t for t in ts]
    if isinstance(c, PagedKVCache):
        return [PG.gather(t, c.table[slot:slot + 1], T)[0] for t in ts]
    return [t[slot, :, :T] for t in ts]


def _store(caches, slot, T, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    for i in range(LAYERS):
        k, v = (torch.randn((1, N_KV, T, HD), generator=g).mul(3.0).to(dtype) for _ in range(2))
        k[0, 1, 5] = 0                                  # a zero row: scale 1, codes 0
        for c in caches:
            c.store(i, slice(slot, slot + 1), k, v)


@DTS
@KVS
def test_paged_store_equals_static_store(dtype, fp8):
    st, pg = _caches(dtype, fp8)
    pg.reserve({0: 10})
    pg.reserve({2: 16})
    pg.reserve({0: 37})                                 # slot 0's blocks are not contiguous: [0, 2, 3]
    assert pg.allocator.blocks[0] == [0, 2, 3] and pg.allocator.blocks[2] == [1]
    assert pg.table[0, :3].tolist() == [0, 2, 3] and pg.table[0, 3:].tolist() == [-1] * 2
    _store((st, pg), 0, 37, dtype, 1)
    _store((st, pg), 2, 16, dtype, 2)
    for i in range(LAYERS):
        for slot, T in ((0, 37), (2, 16)):
            for a, b in zip(_rows(st, i, slot, T), _rows(pg, i, slot, T)):
                assert torch.equal(a, b)
    assert all(t.abs().sum() > 0 for t in _rows(st, 0, 0, 37))


@DTS
@KVS
@pytest.mark.parametrize("n", [40, 32])
def test_fork_shares_full_blocks_and_copies_the_partial_one(dtype, fp8, n):
    _, pg = _caches(dtype, fp8)
    pg.reserve({0: n})
    _store((pg,), 0, n, dtype, 3)
    free = pg.blocks_free
    pg.fork(0, 1, n)
    src, dst = pg.allocator.blocks[0], pg.allocator.blocks[1]
    full = n // BS
    assert dst[:full] == src[:full] and len(dst) == len(src)
    assert pg.table[1].tolist() == dst + [-1] * (pg.max_blocks - len(dst))
    if n % BS:
        assert dst[full] != src[full] and pg.blocks_free == free - 1
        for t in _tensors(pg):
            assert torch.equal(t[dst[full]], t[src[full]])
    else:
        assert pg.blocks_free == free
    for i in range(LAYERS):
        for a, b in zip(_rows(pg, i, 0, n), _rows(pg, i, 1, n)):
            assert torch.equal(a, b)


@KVS
def test_release_frees_blocks_and_clears_the_table_row(fp8):
    _, pg = _caches(torch.float16, fp8)
    pg.reserve({0: 50})
    pg.fork(0, 1, 50)                                   # shares 3 blocks, copies the 4th
    held = pg.blocks_free
    pg.release(0)
    assert pg.blocks_free == held + 1                   # only 0's partial block had count 1
    assert pg.table[0].tolist() == [-1] * pg.max_blocks and pg.table[1, :4].tolist() == pg.allocator.blocks[1]
    assert pg.fits(1, 64) and not pg.fits(2, 20 * BS + 1)
    pg.release(1)
    assert pg.blocks_free == pg.num_blocks and (pg.table == -1).all()


def test_reserve_beyond_the_pool_changes_nothing():
    _, pg = _caches(torch.float16, False, num_blocks=5)
    pg.reserve({0: 40})                                 # 3 blocks of 5
    table = pg.table.clone()
    state = ([list(b) for b in pg.allocator.blocks], list(pg.allocator.ref), pg.blocks_free)
    with pytest.raises(RuntimeError, match="exhausted"):
        pg.reserve({1: 20, 2: 20})                      # 4 blocks, 2 free
    assert torch.equal(pg.table, table)
    assert ([list(b) for b in pg.allocator.blocks], list(pg.allocator.ref), pg.blocks_free) == state


@DTS
@KVS
def test_nbytes_is_the_sum_over_the_tensors(dtype, fp8):
    st, pg = _caches(dtype, fp8, num_blocks=7)
    for c in (st, pg):
        assert c.nbytes == sum(t.untyped_storage().nbytes() for t in _tensors(c))
    assert tuple(pg.k[0].shape) == (7, N_KV, BS, HD) and tuple(st.k[0].shape) == (ROWS, N_KV, MAX_LENGTH, HD)
    assert st.blocks_free is None and st.num_blocks == 0 and pg.blocks_free == 7
    assert pg.length == pg.max_blocks * BS == MAX_LENGTH and st.length == MAX_LENGTH
