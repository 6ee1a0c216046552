"""The paged KV cache on the GPU (DESIGN §3.22).

Kernels: the paged decode and prefill attention against the static kernels on the same contents, bit-equal in the
outputs and in every cache byte written (FP8 scales included), with every other pool byte unchanged (unused blocks hold
NaN, so a stray read shows): fp16 / bf16 × hd 64 / 128 × G 1 / 4 / 8 × B 1 / 3 / 8 × block size 16 / 32 / 64 / 256,
positions at tile and block edges and idle rows, block assignments scrambled, reversed and shared between rows, and
prefill fed in chunks that cross block boundaries.  A CUDA graph replays as the eager calls; an invalid table entry
gives NaN for its row only, and no write.

BatchDecoder: on the random Llama and Qwen2 of ``tests/test_gpu_21_chain_norm.py`` a paged decoder's step logits and
sampled tokens are bit-identical to the static one's over prefill, extend, steps, release and slot reuse, in both cache
dtypes; a forked slot equals a slot prefilled with the same prefix; ``generate(n=4)`` copy i equals the n=1 run with
seed + i; a small pool serves a workload whose live tokens fit and its exhaustion leaves the other slots' logits
unchanged; the pools take kv_blocks × bytes per block."""
import functools

import numpy as np
import pytest
import torch

from autogptq_b200.attention import (FP8, decode_attention_rows, decode_attention_rows_paged,
                                     decode_attention_workspace, prefill_attention, prefill_attention_paged)
from autogptq_b200.sampling import SamplingParams
from tests import _paged as PG

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
N_KV = 2


@functools.lru_cache(maxsize=None)
def _inv_freq(hd):
    return (1.0 / 10000.0 ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd)).cuda()


def _nan_like(pool):
    if pool.dtype == FP8:
        return pool.view(torch.uint8).fill_(0xff).view(FP8)
    if pool.dtype == torch.float32:
        return pool.fill_(float("nan"))
    return pool.view(torch.int16).fill_(0x7fff).view(pool.dtype)


def _bytes(t):
    return t.contiguous().view(torch.uint8)


class Case:
    """Random static caches of B rows (16-bit, or FP8 codes with power-of-two scales) and the same contents in NaN
    pools through a table (``mode``: scrambled, reversed, or shared: rows 1.. share row 0's first ``n_shared`` blocks,
    whose contents are made equal)."""

    def __init__(self, dtype, hd, G, B, bs, fp8, mode, L, n_shared=0, seed=0):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.dtype, self.hd, self.G, self.B, self.bs, self.fp8, self.L = dtype, hd, G, B, bs, fp8, L
        self.max_blocks = L // bs
        self.num_blocks = B * self.max_blocks + 3
        shape = (B, N_KV, L, hd)
        if fp8:
            codes = torch.randint(0, 0x7f, shape, generator=g, device="cuda", dtype=torch.uint8)
            codes |= torch.randint(0, 2, shape, generator=g, device="cuda", dtype=torch.uint8) << 7
            self.k, self.v = codes.view(FP8), codes.flip(-1).contiguous().view(FP8)
            e = torch.randint(-8, 0, (2, B, N_KV, L), generator=g, device="cuda").float()
            self.ks, self.vs = (2.0 ** e[0]).contiguous(), (2.0 ** e[1]).contiguous()
        else:
            self.k = torch.randn(shape, generator=g, device="cuda").to(dtype)
            self.v = torch.randn(shape, generator=g, device="cuda").to(dtype)
            self.ks = self.vs = None
        table = PG.make_table(B, self.max_blocks, self.num_blocks, "reversed" if mode == "reversed" else "scrambled",
                              seed)
        if mode == "shared" and n_shared:
            table[1:, :n_shared] = table[0, :n_shared]
            for t in [x for x in (self.k, self.v, self.ks, self.vs) if x is not None]:
                t = t.view(torch.uint8) if t.dtype == FP8 else t
                t[1:, :, :n_shared * bs] = t[:1, :, :n_shared * bs]
        self.table_np = table
        self.table = torch.from_numpy(table).cuda()
        pshape = (self.num_blocks, N_KV, bs, hd)
        self.kp = _nan_like(torch.empty(pshape, dtype=self.k.dtype, device="cuda"))
        self.vp = _nan_like(torch.empty(pshape, dtype=self.k.dtype, device="cuda"))
        self.ksp = self.vsp = None
        for pool, st in ((self.kp, self.k), (self.vp, self.v)):
            PG.scatter(pool.view(torch.uint8) if fp8 else pool, self.table_np, st.view(torch.uint8) if fp8 else st)
        if fp8:
            self.ksp = _nan_like(torch.empty(pshape[:-1], dtype=torch.float32, device="cuda"))
            self.vsp = _nan_like(torch.empty(pshape[:-1], dtype=torch.float32, device="cuda"))
            PG.scatter(self.ksp, self.table_np, self.ks)
            PG.scatter(self.vsp, self.table_np, self.vs)
        self.used = torch.zeros(self.num_blocks, dtype=torch.bool)
        self.used[torch.from_numpy(table.reshape(-1).astype(np.int64))] = True

    def static_kw(self):
        return {} if not self.fp8 else dict(k_scale=self.ks, v_scale=self.vs)

    def paged_kw(self):
        return {} if not self.fp8 else dict(k_scale=self.ksp, v_scale=self.vsp)

    def pools(self):
        return [p for p in (self.kp, self.vp, self.ksp, self.vsp) if p is not None]

    def check_pools(self, before):
        """The pools seen through the table equal the static caches; unused blocks are as before."""
        for pool, st, old in zip(self.pools(), [x for x in (self.k, self.v, self.ks, self.vs) if x is not None],
                                 before):
            got = PG.gather(pool.view(torch.uint8) if pool.dtype == FP8 else pool, self.table_np, self.L)
            want = st.view(torch.uint8) if st.dtype == FP8 else st
            assert torch.equal(_bytes(got), _bytes(want))
            unused = ~self.used.cuda()
            assert torch.equal(_bytes(pool[unused]), _bytes(old[unused]))


def _positions(B, L, bs):
    edges = [bs - 1, bs, 31, 32, 33, L - 1, bs + 1, 2 * bs - 1]
    return [(-1 if b == 1 and B > 2 else edges[b % len(edges)]) for b in range(B)]


GRID = [(dt, hd, G, B, bs) for dt in (F16, BF16) for hd in (64, 128) for G in (1, 4, 8) for B in (1, 3, 8)
        for bs in (16, 32, 64, 256)]


@pytest.mark.parametrize("fp8", [False, True], ids=["16bit", "fp8"])
@pytest.mark.parametrize("dt,hd,G,B,bs", GRID)
def test_decode_paged_equals_static(dt, hd, G, B, bs, fp8):
    L = max(512, 2 * bs)
    mode = ("scrambled", "reversed", "shared")[(hd + G + B + bs) % 3]
    pos = _positions(B, L, bs)
    n_shared = max(0, min(p for p in pos if p >= 0) // bs) if B > 1 else 0
    c = Case(dt, hd, G, B, bs, fp8, mode, L, n_shared, seed=B * 7 + G)
    g = torch.Generator(device="cuda").manual_seed(1)
    nh = N_KV * G
    q = torch.randn((B, nh * hd), generator=g, device="cuda").to(dt)
    k = torch.randn((B, N_KV * hd), generator=g, device="cuda").to(dt)
    v = torch.randn((B, N_KV * hd), generator=g, device="cuda").to(dt)
    p = torch.tensor(pos, dtype=torch.int64, device="cuda")
    before = [x.clone() for x in c.pools()]
    out_s = torch.empty((B, nh * hd), dtype=dt, device="cuda")
    out_p = torch.empty_like(out_s)
    decode_attention_rows(q, k, v, c.k, c.v, p, _inv_freq(hd), 1.0, hd ** -0.5, out_s, **c.static_kw())
    decode_attention_rows_paged(q, k, v, c.kp, c.vp, c.table, p, _inv_freq(hd), 1.0, hd ** -0.5, out_p,
                                **c.paged_kw())
    torch.cuda.synchronize()
    assert torch.equal(_bytes(out_p), _bytes(out_s))
    assert not out_s[[b for b in range(B) if pos[b] >= 0]].isnan().any()
    c.check_pools(before)


@pytest.mark.parametrize("fp8", [False, True], ids=["16bit", "fp8"])
@pytest.mark.parametrize("dt,hd,G,B,bs", GRID)
def test_prefill_paged_equals_static_in_chunks(dt, hd, G, B, bs, fp8):
    L = max(512, 8 * bs)
    mode = ("scrambled", "reversed")[(hd + G + B + bs) % 2]
    c = Case(dt, hd, G, B, bs, fp8, mode, L, seed=B * 5 + G)
    g = torch.Generator(device="cuda").manual_seed(2)
    nh = N_KV * G
    starts = [(b * (bs // 2 + 3)) % (L // 2) for b in range(B)]
    before = [x.clone() for x in c.pools()]
    for T in (bs + 5, 7, 2 * bs - 1):                   # chunks that cross block boundaries
        q = torch.randn((B, T, nh * hd), generator=g, device="cuda").to(dt)
        k = torch.randn((B, T, N_KV * hd), generator=g, device="cuda").to(dt)
        v = torch.randn((B, T, N_KV * hd), generator=g, device="cuda").to(dt)
        st = torch.tensor(starts, dtype=torch.int64, device="cuda")
        out_s = torch.empty((B, T, nh * hd), dtype=dt, device="cuda")
        out_p = torch.empty_like(out_s)
        prefill_attention(q, k, v, c.k, c.v, st, _inv_freq(hd), 1.0, hd ** -0.5, out_s, **c.static_kw())
        prefill_attention_paged(q, k, v, c.kp, c.vp, c.table, st, _inv_freq(hd), 1.0, hd ** -0.5, out_p,
                                **c.paged_kw())
        torch.cuda.synchronize()
        assert torch.equal(_bytes(out_p), _bytes(out_s)), T
        assert not out_s.isnan().any()
        starts = [s + T for s in starts]
    c.check_pools(before)


@pytest.mark.parametrize("fp8", [False, True], ids=["16bit", "fp8"])
def test_graph_replay_and_invalid_entries(fp8):
    dt, hd, G, B, bs, L = BF16, 128, 4, 8, 32, 1024
    c = Case(dt, hd, G, B, bs, fp8, "scrambled", L, seed=9)
    nh = N_KV * G
    g = torch.Generator(device="cuda").manual_seed(3)
    q = torch.randn((B, nh * hd), generator=g, device="cuda").to(dt)
    k = torch.randn((B, N_KV * hd), generator=g, device="cuda").to(dt)
    v = torch.randn((B, N_KV * hd), generator=g, device="cuda").to(dt)
    pos0 = torch.tensor([5, 31, 32, 100, -1, 700, 1022, 64], dtype=torch.int64, device="cuda")
    pos = pos0.clone()
    ws = decode_attention_workspace(B, nh, N_KV, hd, L, "cuda")
    out = torch.empty((B, nh * hd), dtype=dt, device="cuda")

    def call():
        decode_attention_rows_paged(q, k, v, c.kp, c.vp, c.table, pos, _inv_freq(hd), 1.0, hd ** -0.5, out, ws,
                                    **c.paged_kw())

    call()
    torch.cuda.synchronize()
    eager = [out.clone()]
    pos.add_(pos >= 0)
    call()
    torch.cuda.synchronize()
    eager.append(out.clone())
    pos.copy_(pos0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    for want in eager:
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bytes(out), _bytes(want))
        pos.add_(pos >= 0)
    pos.copy_(pos0)
    # an invalid entry at row 3's position: that row NaN, nothing written; every other row as before
    before = [x.clone() for x in c.pools()]
    j = int(pos[3]) // bs
    c.table[3, j] = c.num_blocks + 7
    graph.replay()
    torch.cuda.synchronize()
    assert out[3].isnan().all()
    others = [b for b in range(B) if b != 3]
    assert torch.equal(_bytes(out[others]), _bytes(eager[0][others]))
    blk = int(c.table_np[3, j])
    for p_, old in zip(c.pools(), before):
        assert torch.equal(_bytes(p_[blk]), _bytes(old[blk]))
    # an invalid entry below the position (row 5): NaN for that row only
    c.table[3, j] = int(c.table_np[3, j])
    c.table[5, 2] = -1
    graph.replay()
    torch.cuda.synchronize()
    assert out[5].isnan().all()
    others = [b for b in range(B) if b != 5]
    assert torch.equal(_bytes(out[others]), _bytes(eager[0][others]))
    # prefill: a row with an invalid entry gets NaN and writes nothing
    T = 9
    qp = torch.randn((B, T, nh * hd), generator=g, device="cuda").to(dt)
    kp = torch.randn((B, T, N_KV * hd), generator=g, device="cuda").to(dt)
    vp = torch.randn((B, T, N_KV * hd), generator=g, device="cuda").to(dt)
    st = torch.tensor([0, 10, 40, 60, 0, 100, 200, 300], dtype=torch.int64, device="cuda")
    before = [x.clone() for x in c.pools()]
    po = torch.empty((B, T, nh * hd), dtype=dt, device="cuda")
    prefill_attention_paged(qp, kp, vp, c.kp, c.vp, c.table, st, _inv_freq(hd), 1.0, hd ** -0.5, po, **c.paged_kw())
    torch.cuda.synchronize()
    assert po[5].isnan().all() and not po[[b for b in range(B) if b != 5]].isnan().any()
    for blk in sorted({int(c.table_np[5, t // bs]) for t in range(100 + T)}):
        for p_, old in zip(c.pools(), before):
            assert torch.equal(_bytes(p_[blk]), _bytes(old[blk]))


# ---------------------------------------------------------------------- BatchDecoder
@functools.lru_cache(maxsize=None)
def _model(arch, dtype):
    from tests.test_gpu_21_chain_norm import _model as m
    return m(arch, dtype)


def _decoders(arch, dtype, kv, max_batch=4, max_length=256, bs=16, kv_blocks=None):
    from autogptq_b200.batch_decoder import BatchDecoder

    model = _model(arch, dtype)
    return (BatchDecoder(model, max_batch, max_length, kv_cache_dtype=kv),
            BatchDecoder(model, max_batch, max_length, kv_cache_dtype=kv, kv_block_size=bs, kv_blocks=kv_blocks))


def _prompt(n, seed):
    return torch.randint(0, 512, (n,), generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("kv", [None, FP8], ids=["16bit", "fp8"])
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_batch_decoder_paged_equals_static(arch, dtype, kv):
    st, pg = _decoders(arch, dtype, kv)
    g = torch.Generator().manual_seed(4)
    for d in (st, pg):
        d.set_sampling(2, SamplingParams(temperature=0.9, top_k=40, seed=11))
    outs = []
    for d in (st, pg):
        log = []
        log.append(d.prefill(0, _prompt(37, 1)))
        log.append(d.extend(1, _prompt(20, 2)))
        log.append(d.extend(1, _prompt(13, 3)))           # crosses a block boundary
        log.append(d.extend(2, _prompt(16, 4)))
        for i in range(20):
            ids = torch.randint(0, 512, (4,), generator=torch.Generator().manual_seed(100 + i)).cuda()
            if i % 2:
                tok, lg = d.step_sample(ids)
                log += [tok.clone(), lg.clone()]
            else:
                log.append(d.step(ids).clone())
            if i == 8:
                d.release(0)
                log.append(d.extend(0, _prompt(40, 5)))   # slot reuse
            if i == 12:
                log.append(d.extend(1, _prompt(9, 6)))    # a new turn on an active slot
        outs.append(log)
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert pg.kv_blocks_free < pg.kv_blocks


@pytest.mark.parametrize("kv", [None, FP8], ids=["16bit", "fp8"])
@pytest.mark.parametrize("n_prefix", [32, 45])
def test_fork_equals_a_slot_prefilled_alone(kv, n_prefix):
    _, pg = _decoders("llama", BF16, kv)
    prefix = _prompt(n_prefix, 7)
    pg.prefill(0, prefix)
    free = pg.kv_blocks_free
    pg.fork(0, 1)
    assert pg.kv_blocks_free == free - (1 if n_prefix % 16 else 0)
    pg.prefill(2, prefix)
    for i in range(24):
        ids = torch.full((4,), 17 + i, dtype=torch.int64).cuda()
        lg = pg.step(ids)
        assert torch.equal(lg[1], lg[2]) and torch.equal(lg[0], lg[2])
    with pytest.raises(RuntimeError):
        pg.fork(0, 1)                                     # dst busy
    pg.release(0), pg.release(1), pg.release(2)
    assert pg.kv_blocks_free == pg.kv_blocks


def test_generate_n_samples_equal_seeded_single_runs():
    _, pg = _decoders("llama", F16, None, max_batch=8, max_length=256)
    p = _prompt(50, 8)
    sp = SamplingParams(temperature=0.8, top_k=50, seed=2 ** 64 - 2)
    many = pg.generate([p], 24, sampling=sp, n=4)
    assert len(many) == 4
    for i in range(4):
        one = pg.generate([p], 24, sampling=SamplingParams(temperature=0.8, top_k=50, seed=(2 ** 64 - 2 + i) % 2 ** 64))
        assert torch.equal(many[i], one[0])
    assert pg.kv_blocks_free == pg.kv_blocks
    many = pg.generate([p, _prompt(30, 9), _prompt(70, 10)], 20, sampling=sp, n=3)
    assert len(many) == 9 and all(m.numel() == n0 + 20 for m, n0 in zip(many, [50] * 3 + [30] * 3 + [70] * 3))


def test_static_decoder_refuses_fork_and_n():
    st, _ = _decoders("llama", F16, None)
    with pytest.raises(NotImplementedError):
        st.fork(0, 1)
    with pytest.raises(NotImplementedError):
        st.generate([_prompt(5, 1)], 3, sampling=SamplingParams(seed=1), n=2)


def test_small_pool_and_exhaustion():
    # 4 slots of max_length 256 would take 64 blocks of 16; the small pool has 20, its twin the full 64
    small = _decoders("llama", BF16, None, bs=16, kv_blocks=20)[1]
    twin = _decoders("llama", BF16, None, bs=16)[1]
    outs = []
    for d in (small, twin):
        d.prefill(0, _prompt(60, 1))                     # 4 blocks
        d.prefill(1, _prompt(100, 2))                    # 7 blocks
        d.extend(2, _prompt(111, 3))                     # 7 blocks
        log = []
        for i in range(4):                               # slot 2 crosses into its 8th block: 19 of 20
            log.append(d.step(torch.full((4,), i, dtype=torch.int64).cuda()).clone())
        d.extend(3, _prompt(16, 4))                      # the 20th block
        outs.append(log)
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert small.kv_blocks_free == 0
    pos = small.positions                                # slot 0 at 64: its next step needs a 21st block
    with pytest.raises(RuntimeError, match="exhausted"):
        small.step(torch.full((4,), 5, dtype=torch.int64).cuda())
    assert small.positions == pos and small.kv_blocks_free == 0
    for d in (small, twin):
        d.release(3)
    ids = torch.full((4,), 6, dtype=torch.int64).cuda()
    assert torch.equal(small.step(ids)[:3], twin.step(ids)[:3])


@pytest.mark.parametrize("kv", [None, FP8], ids=["16bit", "fp8"])
def test_pool_bytes(kv):
    _, pg = _decoders("qwen2", BF16, kv, bs=32, kv_blocks=37)
    hd, n_kv, layers = pg.head_dim, pg.n_kv, len(pg._plans)
    per_block = 2 * n_kv * 32 * hd * (1 if kv is FP8 else 2) + (2 * n_kv * 32 * 4 if kv is FP8 else 0)
    assert pg.kv_cache_bytes == layers * 37 * per_block
    pools = pg.k_cache + pg.v_cache + (pg.k_scale + pg.v_scale if kv is FP8 else [])
    assert sum(t.untyped_storage().nbytes() for t in pools) == layers * 37 * per_block
    assert tuple(pg.k_cache[0].shape) == (37, n_kv, 32, hd)
    with pytest.raises(RuntimeError, match="paged"):
        pg.positions = [-1] * 4
