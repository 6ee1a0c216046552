"""The SiLU·mul paths against the stage-wise float64 reference of tests/_silu_mul.py, to the ulp, in fp16 and bf16, on
GPTQ-like layers and experts (scales over decades, heavy columns, wrap-rule zeros, bf16 scales below fp16's range,
act-order) and every activation kind of ``tests/_precision.py``:

* the fused gate/up pair (``FusedQuantMLP._forward_saving``): decode kernel and wgmma GEMM (tiles × split-K), AUTO;
* the grouped experts (``QuantExperts._forward(save=True)``): decode (T ≤ 8) and GEMM (T > 8) paths, the combine;
* the decode chain's gate|up → silu_mul down stages.

g and u are held to the bound of the path that computed them, h to equality with rnd(rnd(silu(g))·u) for one of the
silu candidates, y_pair / the chain's down output to the reference on the host-side h, out to the combine bound; the
no-grad entry points must be bit-identical to the saving runs.  The module prints, per path, stage and dtype, the
largest err/bound, mismatch rate and γ share, the rate at which h needed the neighbour silu candidate, and the rate at
which h differs from torch's F.silu(g)·u."""
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from autogptq_b200 import _lib
from tests import _precision as P
from tests import _silu_mul as S
from tests._util import make_layer

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTS = [F16, BF16]
_SUMMARY: dict = {}
_H_TOTAL: dict = {}          # dtype -> [elements, neighbour matches]


@pytest.fixture(scope="module", autouse=True)
def _print_summary():
    yield
    print("\n[silu-mul] path / stage              dtype     cases  max err/bound  max mismatch  max γ share  "
          "max neighbour  max torch≠")
    for (name, dt), (n, worst, rate, gu, nb, tr) in sorted(_SUMMARY.items()):
        print(f"[silu-mul] {name:<28} {dt:<9} {n:>5}  {worst:13.3f}  {rate:12.4f}  {gu:11.3f}  {nb:13.5f}  {tr:10.5f}")
    for dt, (n, nb) in sorted(_H_TOTAL.items()):
        print(f"[silu-mul] h neighbour-candidate rate {dt}: {nb} of {n} = {nb / max(n, 1):.2e}")


def _record(path, dtype, res: dict, torch_rate=None):
    dt = P.dt_name(dtype)
    for stage, r in res.items():
        key = (f"{path} {stage}", dt)
        n, w, rt, gu, nb, tr = _SUMMARY.get(key, (0, 0.0, 0.0, 0.0, 0.0, 0.0))
        if isinstance(r, S.HResult):
            tot = _H_TOTAL.setdefault(dt, [0, 0])
            tot[0] += r.n
            tot[1] += int(round(r.neighbour * r.n))
            _SUMMARY[key] = (n + 1, w, rt, gu, max(nb, r.neighbour), max(tr, torch_rate or 0.0))
        else:
            _SUMMARY[key] = (n + 1, max(w, r.worst), max(rt, r.rate), max(gu, r.g_used), nb, tr)


def _np(t):
    return t.double().cpu().numpy()


def _bits_equal(a, b):
    """Bit-identical 16-bit tensors (NaN payloads included)."""
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# --------------------------------------------------------------------------- fused gate/up
@functools.lru_cache(maxsize=None)
def _pair(K, I, g, dt, act=True, seed=0):
    d1 = P.wide_layer(K, I, g, dt, seed=seed, act_order=act, bias=True)
    return d1, P.wide_layer(K, I, g, dt, seed=seed + 1, bias=True, g_idx=d1["g_idx"])


@functools.lru_cache(maxsize=None)
def _mlp(K, I, g, dtype, act=True, seed=0):
    from autogptq_b200 import FusedQuantMLP

    d1, d3 = _pair(K, I, g, P.dt_name(dtype), act, seed)
    down = P.realistic_layer(I, 128, 32, P.dt_name(dtype), seed=seed + 2)
    return FusedQuantMLP(*(make_layer(d, dtype=dtype) for d in (d1, d3, down)))


def _gate_up_case(K, I, g, dtype, M, kind, kernel=_lib.GATE_UP_AUTO, tile_m=0, split_k=0, act=True, cols=None,
                  seed=0, what=""):
    from autogptq_b200.mlp import forward_gate_up

    dt = P.dt_name(dtype)
    d1, d3 = _pair(K, I, g, dt, act)
    mlp = _mlp(K, I, g, dtype, act)
    x = P.activations(kind, M, K, dtype, seed=seed)
    xt = torch.from_numpy(x).to(dtype).cuda()
    with torch.no_grad():
        h_ng = forward_gate_up(mlp.gate_proj, mlp.up_proj, xt, kernel=kernel, tile_m=tile_m, split_k=split_k)
        _, h, gt, ut = mlp._forward_saving(xt, kernel=kernel, tile_m=tile_m, split_k=split_k)
        h_torch = F.silu(gt) * ut
    torch.cuda.synchronize()
    assert _bits_equal(h_ng, h), f"{what}: forward_gate_up differs from the saving forward"
    c0, c1 = cols or (0, I)
    fin = torch.isfinite(gt) & torch.isfinite(ut)
    torch_rate = float(((h_torch != h) & fin).sum()) / max(int(fin.sum()), 1)
    tc = kernel == _lib.GATE_UP_GEMM or (kernel == _lib.GATE_UP_AUTO and M > _lib.MOE_DECODE_MAX_T)
    path = "gemm" if tc else "decode_mma"
    res = S.check_gate_up(d1, d3, x, _np(gt[:, c0:c1]), _np(ut[:, c0:c1]), _np(h[:, c0:c1]), path, dtype, cols=cols,
                          what=f"gate/up {path} {what} {dt} {kind} M={M}")
    _record(f"gate/up {'gemm' if tc else 'decode'}", dtype, res, torch_rate)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", range(1, 9))
def test_gate_up_decode_forced(dtype, M):
    kind = P.acts_for(dtype)[M % len(P.acts_for(dtype))]
    _gate_up_case(1024, 352, 128, dtype, M, kind, kernel=_lib.GATE_UP_DECODE, seed=M, what="forced")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("tile_m", [32, 64, 128])
@pytest.mark.parametrize("split_k", [1, 2, 4, 8])
def test_gate_up_gemm_tiles_and_splits(dtype, tile_m, split_k):
    kind = ["offset", "massive", "student_t", "row_scale"][split_k.bit_length() - 1]
    _gate_up_case(2048, 352, 128, dtype, 96, kind, kernel=_lib.GATE_UP_GEMM, tile_m=tile_m, split_k=split_k,
                  seed=tile_m + split_k, what=f"mt={tile_m} split={split_k}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("kind", P.ACTS)
@pytest.mark.parametrize("M", [6, 100])
def test_gate_up_activations(dtype, kind, M):
    if kind not in P.acts_for(dtype):
        pytest.skip(f"{kind} is not a {P.dt_name(dtype)} distribution")
    _gate_up_case(1024, 352, 128, dtype, M, kind, seed=3, what="auto")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("g", [32, 64, 128, 192, -1])
@pytest.mark.parametrize("M", [5, 40])
def test_gate_up_group_sizes(dtype, g, M):
    """I = 352 (I % 64 == 32: a half column tile on the GEMM path), act-order, bias."""
    _gate_up_case(1536, 352, g, dtype, M, ["offset", "gauss", "massive"][M % 3], seed=g % 97, what=f"g={g}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 8, 9, 64, 300, 2048])
def test_gate_up_auto_llama7b(dtype, M):
    """Llama-2-7B's gate/up pair (4096 -> 11008, act-order), checked on a column slice."""
    cols = (11008 - 256, 11008) if M % 2 else (2048, 2304)
    _gate_up_case(4096, 11008, 128, dtype, M, ["offset", "gauss", "student_t", "massive"][M % 4], cols=cols, seed=M,
                  what="llama-7b")


# --------------------------------------------------------------------------- grouped experts
@functools.lru_cache(maxsize=None)
def _qe(E, H, I, g, dtype, act13, act2, bias, seed):
    from autogptq_b200 import QuantExperts

    ex = S.realistic_experts(E, H, I, g, P.dt_name(dtype), seed=seed, act13=act13, act2=act2, bias=bias)
    mods = {n: [make_layer(e[n], dtype=dtype) for e in ex] for n in ("w1", "w3", "w2")}
    return QuantExperts(mods["w1"], mods["w3"], mods["w2"]), ex


def _routing(T, k, E, seed, spread=None, invalid=None):
    """[T, k] ids and fp32 weights summing to 1.  ``spread``: draw ids from the first ``spread`` experts with repeats
    (tokens repeat an expert); ``invalid``: this id on every slot of the last token and on the last slot of token 0."""
    rng = np.random.default_rng(seed)
    if spread is not None:
        idx = rng.integers(0, spread, (T, k)).astype(np.int64)
    else:
        idx = np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)
    if invalid is not None and T >= 3:
        idx[T - 1] = invalid
        if k > 1:
            idx[0, k - 1] = invalid
    w = rng.random((T, k)).astype(np.float32) + 0.05
    return idx, w / w.sum(axis=1, keepdims=True)


def _unpack(saved, T, k, I, H, dtype):
    Pn = T * k
    gu = -(-Pn * I * 2 // 256) * 256
    part = lambda off, n: saved[off:off + Pn * n * 2].view(dtype).view(Pn, n)
    return part(0, I), part(gu, I), part(2 * gu, H)


def _moe_case(E, H, I, g, dtype, T, k, idx, w, kind, act13=True, act2=True, bias=True, seed=0, idx_dtype=torch.int64,
              w16=False, cols_i=None, cols_h=None, what=""):
    qe, ex = _qe(E, H, I, g, dtype, act13, act2, bias, seed)
    dt = P.dt_name(dtype)
    x = P.activations(kind, T, H, dtype, seed=T + k)
    xt = torch.from_numpy(x).to(dtype).cuda()
    it = torch.from_numpy(np.asarray(idx)).to(idx_dtype).cuda()
    wt = torch.from_numpy(w).to(dtype if w16 else torch.float32).cuda()
    with torch.no_grad():
        out, saved = qe._forward(xt, it, wt, save=True)
        out_ng = qe(xt, it, wt)
    torch.cuda.synchronize()
    assert _bits_equal(out, out_ng), f"{what}: QuantExperts.forward differs from the saving forward"
    gs, us, ys = _unpack(saved, T, k, I, H, dtype)
    path = "decode_mma" if T <= _lib.MOE_DECODE_MAX_T else "gemm"
    res = S.check_moe(ex, x, np.asarray(idx), wt.double().cpu().numpy(), dtype, path, path, _np(gs), _np(us), _np(ys),
                      _np(out), cols_i=cols_i, cols_h=cols_h, what=f"moe {path} {what} {dt} {kind} T={T} k={k}")
    _record(f"moe {'decode' if path == 'decode_mma' else 'gemm'}", dtype, res)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("k", [1, 2, 4, 8])
@pytest.mark.parametrize("T", [1, 3, 8])
def test_moe_decode_k_and_T(dtype, k, T):
    acts = P.acts_for(dtype)
    idx, w = _routing(T, k, 8, seed=10 * T + k, invalid=8)
    _moe_case(8, 512, 1536, 128, dtype, T, k, idx, w, acts[(T + k) % len(acts)], what="E=8")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("T", [2, 8])
def test_moe_decode_64_experts(dtype, T):
    idx, w = _routing(T, 8, 64, seed=T, invalid=64)
    _moe_case(64, 512, 512, 64, dtype, T, 8, idx, w, "offset", act2=False, what="E=64")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("spread", [1, 2])
def test_moe_decode_repeated_experts(dtype, spread):
    """Tokens repeat an expert: one or two experts take all T·k = 64 rows, so the decode kernel runs 4 or 8 row passes."""
    idx, w = _routing(8, 8, 8, seed=spread, spread=spread)
    _moe_case(8, 512, 1536, 128, dtype, 8, 8, idx, w, "row_scale", what=f"repeats over {spread}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("invalid,idx_dtype", [(8, torch.int64), (-1, torch.int32), (2 ** 31 + 7, torch.int64),
                                               (-(2 ** 40), torch.int64)], ids=["E", "m1_i32", "2e31_i64", "neg_i64"])
@pytest.mark.parametrize("w16", [False, True], ids=["w32", "w16"])
def test_moe_decode_ids_and_weights(dtype, invalid, idx_dtype, w16):
    idx, w = _routing(6, 2, 8, seed=3, invalid=invalid)
    _moe_case(8, 512, 1536, 128, dtype, 6, 2, idx, w, "student_t", idx_dtype=idx_dtype, w16=w16, what=f"id {invalid}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("I", [4224, 8320])
def test_moe_decode_down_split(dtype, I):
    """I > 4096 splits the down stage's K in 2 (I <= 8192) or 4 (agb200_moe_create: <= 64 KB of h per work item)."""
    idx, w = _routing(4, 2, 8, seed=I, invalid=8)
    _moe_case(8, 256, I, 128, dtype, 4, 2, idx, w, "massive", what=f"I={I}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_moe_decode_one_group(dtype):
    """H = 1408 with one group per layer (group_size -1: 1408 rows for w1 / w3, I for w2)."""
    idx, w = _routing(5, 2, 8, seed=5, invalid=8)
    _moe_case(8, 1408, 512, -1, dtype, 5, 2, idx, w, "offset", act13=False, act2=False, what="H=1408 g=-1")


def test_moe_plans_of_different_sizes_coexist():
    """A plan created later for smaller experts leaves an earlier plan's decode launches working.  The decode kernels'
    shared-memory attribute belongs to the kernel, not the plan; it used to be set to each new plan's own need, so a
    plan with I = 512 after one with I = 1536 made every decode forward of the larger one fail (invalid argument)."""
    from autogptq_b200 import QuantExperts

    def fresh(I):
        ex = S.realistic_experts(8, 512, I, 128, "float16", seed=60)
        return QuantExperts(*([make_layer(e[n]) for e in ex] for n in ("w1", "w3", "w2")))

    big, small = fresh(1536), fresh(512)
    idx, w = _routing(4, 2, 8, seed=1)
    x = torch.from_numpy(P.activations("gauss", 4, 512, F16, seed=1)).half().cuda()
    it, wt = torch.from_numpy(idx).cuda(), torch.from_numpy(w).cuda()
    with torch.no_grad():
        before = big(x, it, wt)
        small(x, it, wt)                                   # creates the smaller plan
        after = big(x, it, wt)
    torch.cuda.synchronize()
    assert _bits_equal(before, after)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("T,mt", [(64, 32), (200, 64), (600, 128)])
def test_moe_gemm_row_tiles(dtype, T, mt):
    """E = 8, k = 2: mean rows per expert T·k / 8 picks the 32-, 64- and 128-row tile (moe.cu)."""
    assert mt == (32 if T * 2 / 8 <= 32 else 64 if T * 2 / 8 <= 64 else 128)
    acts = P.acts_for(dtype)
    idx, w = _routing(T, 2, 8, seed=T, invalid=8)
    _moe_case(8, 512, 1536, 128, dtype, T, 2, idx, w, acts[T % len(acts)], idx_dtype=torch.int32 if mt == 64 else
              torch.int64, w16=mt == 128, what=f"mt={mt}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("kind", ["inf", "subnormal", "huge_tiny"])
def test_moe_gemm_activations(dtype, kind):
    if kind not in P.acts_for(dtype):
        pytest.skip(f"{kind} is not a {P.dt_name(dtype)} distribution")
    idx, w = _routing(40, 2, 8, seed=4, invalid=-1)
    _moe_case(8, 512, 1536, 128, dtype, 40, 2, idx, w, kind, idx_dtype=torch.int32, what="gemm")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_moe_gemm_skewed_and_one_group(dtype):
    rng = np.random.default_rng(1)
    w = rng.random((300, 2)).astype(np.float32)
    idx = np.stack([np.full(300, 5), np.full(300, 8)], axis=1)          # one expert takes every token
    _moe_case(8, 512, 1536, 128, dtype, 300, 2, idx, w, "offset", what="one expert")
    idx, w = _routing(100, 2, 8, seed=2, invalid=8)
    _moe_case(8, 1408, 512, -1, dtype, 100, 2, idx, w, "massive", act13=False, act2=False, what="H=1408 g=-1")


@pytest.mark.parametrize("T", [8, 64])
def test_moe_mixtral_size(T):
    """Mixtral-8x7B's expert shapes (H = 4096, I = 14336: the decode down stage splits K in 4), on column slices."""
    idx, w = _routing(T, 2, 8, seed=T, invalid=8)
    _moe_case(8, 4096, 14336, 128, F16, T, 2, idx, w, "offset", act13=False, act2=False, bias=False,
              cols_i=(14336 - 256, 14336), cols_h=(1024, 1280), what="mixtral")


# --------------------------------------------------------------------------- DecodeChain
@functools.lru_cache(maxsize=None)
def _chain_layers(H, I, dt, act):
    d1, d3 = _pair(H, I, 128, dt, act, seed=40)
    return d1, d3, P.wide_layer(I, H, 128, dt, seed=42, act_order=act, bias=True)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 2])
@pytest.mark.parametrize("H,I,act", [(4096, 11008, False), (1024, 2816, True)], ids=["llama7b", "act_order"])
def test_chain_silu_mul_stage(dtype, M, H, I, act):
    from autogptq_b200.chain import DecodeChain

    dt = P.dt_name(dtype)
    d1, d3, d2 = _chain_layers(H, I, dt, act)
    G_, U_, D_ = (make_layer(d, dtype=dtype) for d in (d1, d3, d2))
    ch = DecodeChain(M=M, dtype=dtype)
    xin = ch.input(H)
    gate, up = ch.stage([G_, U_], xin)
    (y,) = ch.stage([D_], gate, x2=up, x_mode="silu_mul")
    ch.build()
    ci, chh = (I - 256, I), (H - 256, H) if H > 1024 else None
    for kind in ("offset", "massive", "row_scale", "gauss"):
        x = P.activations(kind, M, H, dtype, seed=7 + M)
        xin.copy_(torch.from_numpy(x).to(dtype).cuda())
        ch.run()
        y1 = y.clone()
        ch.run()
        torch.cuda.synchronize()
        assert _bits_equal(y, y1), "two runs of the chain differ"
        xs, g, u = _np(xin), _np(gate), _np(up)
        pc = P.PATHS["chain"]
        res = {"g": P.check(g[:, ci[0]:ci[1]], P.reference(d1, xs, pc, dtype, cols=ci), pc, dtype, what=f"chain g {kind}"),
               "u": P.check(u[:, ci[0]:ci[1]], P.reference(d3, xs, pc, dtype, cols=ci), pc, dtype, what=f"chain u {kind}")}
        c0, c1 = chh or (0, H)
        res["down"] = P.check(_np(y)[:, c0:c1], S.reference_down(d2, g, u, pc, dtype, cols=chh), pc, dtype,
                              what=f"chain silu_mul down {kind} M={M}")
        _record("chain silu_mul", dtype, res)


# --------------------------------------------------------------------------- the neighbour rate over the module
def test_zz_neighbour_candidate_rate():
    """h matched only the neighbour silu candidate on a small share of its elements (S.NEIGHBOUR_RATE)."""
    if not _H_TOTAL:
        pytest.skip("no gate/up case ran")
    for dt, (n, nb) in _H_TOTAL.items():
        assert nb / max(n, 1) <= S.NEIGHBOUR_RATE[dt], f"{dt}: h took the neighbour candidate on {nb} of {n} elements"
