"""The decode chain's L2 lookahead (the producer prefetches the slots after a blocked one into L2 while the ring is full).

It moves bytes into L2 earlier and nothing else, so every output must be bit-identical to the chain without it, at every
lookahead and ring size; the producer's profile row must count exactly the schedule's slots."""
import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from autogptq_b200.chain import DecodeChain, chain_diag
from oracle import w4a16_oracle as O
from tests._util import assert_parity, make_layer, oracle_exact, rand_x

pytestmark = pytest.mark.gpu

PROFILE = 8
SLOT_BYTES = 17 * 1024
# lookahead settings: "d" = library default, "max" = more than any device allows (clamped to the chain's maximum)
LOOKAHEADS = ["0", "1", "d", "max"]
SLOTS = ["d", "3", "4", "10"]


def _unit_gain(d, rng=None):
    sign = 1.0 if rng is None else rng.integers(0, 2, size=d["scales"].shape) * 2.0 - 1.0
    d["scales"] = (d["scales"].astype(np.float32) * sign * (0.9 / (6.3 * np.sqrt(d["K"]) * 0.006))).astype(np.float16)
    return d


def _llama7b_two_blocks():
    H, I, g = 4096, 11008, 128
    rng = np.random.default_rng(0)
    blocks = []
    for b in range(2):
        ds = [_unit_gain(O.random_packed(K, N, g, seed=200 * b + i), rng)
              for i, (K, N) in enumerate([(H, H)] * 4 + [(H, I)] * 2 + [(I, H)])]
        blocks.append([make_layer(d) for d in ds])

    def build(ch):
        x = ch.input(H)
        t, outs = x, []
        for q, k, v, o, gt, up, dn in blocks:
            outs += ch.stage([q, k, v], t)
            outs += ch.stage([o], outs[-3])
            outs += ch.stage([gt, up], outs[-1])
            (t,) = ch.stage([dn], outs[-2])
            outs.append(t)
        return x, outs
    stages = [(H, [H, H, H]), (H, [H]), (H, [I, I]), (I, [H])] * 2
    return 1, torch.float16, build, torch.from_numpy(rand_x(1, H, seed=1)), stages, None


def _ragged_k():
    K = 1408                                   # 176 k8-rows: the second ring slot of every tile is ragged
    dA, dB = _unit_gain(O.random_packed(K, K, 128, seed=1, bias=True)), O.random_packed(K, 96, 128, seed=2)
    dC, dD = _unit_gain(O.random_packed(K, 640, 128, seed=3)), O.random_packed(640, 64, 128, seed=4)
    A, B, C, D = (make_layer(d) for d in (dA, dB, dC, dD))

    def build(ch):
        x = ch.input(K)
        ya, yb = ch.stage([A, B], x)
        (yc,) = ch.stage([C], ya)
        (yd,) = ch.stage([D], yc)
        return x, [ya, yb, yc, yd]
    stages = [(K, [K, 96]), (K, [640]), (640, [64])]
    return 2, torch.float16, build, torch.from_numpy(rand_x(2, K, seed=5)), stages, [(dA, None, 0), (dC, 0, 2), (dD, 2, 3)]


def _silu_mul_mlp():
    H, I, g = 1024, 2816, 128
    ds = [O.random_packed(H, I, g, seed=1), O.random_packed(H, I, g, seed=2), O.random_packed(I, H, g, seed=3, bias=True)]
    for d in ds:
        d["scales"] = torch.from_numpy(d["scales"]).to(torch.bfloat16).float().numpy()
        if d["bias"] is not None:
            d["bias"] = torch.from_numpy(d["bias"]).to(torch.bfloat16).float().numpy()
    G_, U_, D_ = (make_layer(d, dtype=torch.bfloat16) for d in ds)

    def build(ch):
        x = ch.input(H)
        gate, up = ch.stage([G_, U_], x)
        (y,) = ch.stage([D_], gate, x2=up, x_mode="silu_mul")
        return x, [gate, up, y]
    stages = [(H, [I, I]), (I, [H])]
    return 2, torch.bfloat16, build, torch.from_numpy(rand_x(2, H, seed=5).astype(np.float32)).to(torch.bfloat16), stages, None


CASES = {"llama7b_two_blocks": _llama7b_two_blocks, "ragged_k1408": _ragged_k, "silu_mul_mlp": _silu_mul_mlp}


def _schedule_slots(stages):
    """Ring slots of one launch: every 32-column tile of every layer, one slot per 1024 k of the stage's K."""
    return sum(sum(N // 32 for N in Ns) * (-(-K // 1024)) for K, Ns in stages)


def _make(monkeypatch, M, dtype, build, lookahead, slots):
    for var, val in (("AGB200_CHAIN_L2_LOOKAHEAD", lookahead), ("AGB200_CHAIN_SLOTS", slots)):
        if val == "d":
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, "100000" if val == "max" else val)
    ch = DecodeChain(M=M, dtype=dtype)
    x, outs = build(ch)
    ch.build()
    return ch, x, outs


@pytest.mark.parametrize("case", sorted(CASES))
def test_chain_lookahead_is_bit_identical(case, monkeypatch):
    M, dtype, build, x_in, stages, oracle_checks = CASES[case]()
    x_in = x_in.cuda()
    ref = None
    n_slots = _schedule_slots(stages)
    for la in LOOKAHEADS:
        for sl in SLOTS:
            ch, x, outs = _make(monkeypatch, M, dtype, build, la, sl)
            info = ch.info()
            if la == "0":
                assert info["l2_lookahead"] == 0
            elif la == "max":
                assert info["l2_lookahead"] == info["l2_lookahead_max"]
            x.copy_(x_in)
            for _ in range(2):                                  # second launch: new tags
                ch.run()
            torch.cuda.synchronize()
            got = [o.clone() for o in outs]
            if ref is None:
                ref = got
                for d, xi, yi in oracle_checks or []:
                    xs = x if xi is None else outs[xi]
                    assert_parity(outs[yi].float().cpu().numpy(), oracle_exact(d, xs.float().cpu().numpy()), what=f"{case} stage")
            for i, (a, b) in enumerate(zip(ref, got)):
                assert torch.equal(a, b), f"{case}: output {i} differs at lookahead={la} slots={sl} ({info})"
            # the profiled launch computes the same outputs; its producer row counts the schedule
            ch.run(PROFILE)
            torch.cuda.synchronize()
            for i, (a, b) in enumerate(zip(ref, outs)):
                assert torch.equal(a, b), f"{case}: profiled output {i} differs at lookahead={la} slots={sl}"
            prod = ch.profile()[:, 3, :]
            assert (prod[:, 0] > 0).all()
            assert (prod[:, 1] <= prod[:, 0]).all() and (prod[:, 2] <= prod[:, 0]).all() and (prod[:, 1:3] >= 0).all()
            assert int(prod[:, 3].sum()) == n_slots, f"{case}: producer issued {int(prod[:, 3].sum())} slots, schedule has {n_slots}"
            if info["l2_lookahead"] == 0:
                assert int(prod[:, 4].sum()) == 0
            del ch
    assert chain_diag()["site"] == 0


def test_chain_lookahead_graph_replay_is_deterministic(monkeypatch):
    M, dtype, build, x_in, _, _ = _ragged_k()
    ch, x, outs = _make(monkeypatch, M, dtype, build, "max", "3")
    x.copy_(x_in.cuda())
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ch.run()
        torch.cuda.synchronize()
        first = [o.clone() for o in outs]
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            ch.run()
        for _ in range(5):
            gr.replay()
            torch.cuda.synchronize()
            for a, b in zip(first, outs):
                assert torch.equal(a, b)


def test_chain_lookahead_clamp_and_env(monkeypatch):
    props = torch.cuda.get_device_properties(0)
    want_max = props.L2_cache_size // 3 // (SLOT_BYTES * props.multi_processor_count)
    M, dtype, build, _, _, _ = _silu_mul_mlp()
    ch, _, _ = _make(monkeypatch, M, dtype, build, "d", "d")
    info = ch.info()
    assert info["l2_lookahead_max"] == want_max
    assert 0 <= info["l2_lookahead"] <= want_max
    for la, expect in (("0", 0), ("1", min(1, want_max)), ("max", want_max)):
        ch, _, _ = _make(monkeypatch, M, dtype, build, la, "d")
        assert ch.info()["l2_lookahead"] == expect
    assert ch.info()["l2_lookahead"] * SLOT_BYTES * ch.info()["grid"] <= props.L2_cache_size // 3
    monkeypatch.setenv("AGB200_CHAIN_L2_LOOKAHEAD", "-1")            # ignored: the default stays
    ch = DecodeChain(M=M, dtype=dtype)
    build(ch)
    ch.build()
    assert ch.info()["l2_lookahead"] == info["l2_lookahead"]
    assert _lib.ABI_VERSION >= 8
