"""The two fused backwards stage by stage against float64 (tests/_backward_stages.py), on the intermediates they write,
in fp16 and bf16, on GPTQ-like layers and experts and the finite activation kinds of ``tests/_precision.py`` as dy:

* the dense MLP (``agb200_w4a16_mlp_backward_ex``, ``FusedQuantMLP(fused_backward=True)``): [dg | du] against their
  intervals, dx against the dgrad bound on the kernel's own dg and du, every row tile and cluster split forced;
* the grouped experts (``agb200_moe_backward``, ``QuantExperts(input_grad=True)``): prow, dy_pair bit-exact, [dg | du]
  against their intervals, dx_pair against its fp32 bound, dx bit-exact from dx_pair, every row tile.

Both entries are called directly with a workspace owned by the test and filled with 0xFF, so what a kernel did not write
shows; the dx of the same call made with the automatic tile and split equals the module's autograd dx bit for bit.
``test_report`` prints, per stage and dtype, the largest err/bound, mismatch rate and share of the fp32 γ used
(DESIGN §3.12).  tests/test_gpu_18_moe_grad.py and tests/test_gpu_19_mlp_grad.py keep the end-to-end check against
the all-float64 block."""
import functools

import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from tests import _backward_stages as B
from tests import _precision as P
from tests import _silu_mul as S
from tests._util import make_layer

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTS = [F16, BF16]
CODE = {F16: _lib.F16, BF16: _lib.BF16}
REPORT: dict = {}           # (stage, dtype name) -> [cases, worst, rate, γ share]
TILES = [(mt, sk) for sk in (1, 2, 4, 8) for mt in (32, 64, 128)]


@pytest.fixture(autouse=True)
def _need_gpu(monkeypatch):
    """Skips without a device; the fused backward runs at every M here (which M it takes by default is a speed choice)."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import autogptq_b200.mlp as mlp_mod

    monkeypatch.setattr(mlp_mod, "FUSED_BACKWARD_MAX_M", 1 << 30)


def _record(stage, dtype, r: P.Result):
    key = (stage, P.dt_name(dtype))
    n, w, rt, gu = REPORT.get(key, (0, 0.0, 0.0, 0.0))
    REPORT[key] = (n + 1, max(w, r.worst), max(rt, r.rate), max(gu, r.g_used))


def _np(t):
    return t.double().cpu().numpy()


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def _kinds(dtype):
    return [k for k in P.acts_for(dtype) if k != "inf"]


def _act(kind, M, K, dtype, seed):
    return torch.from_numpy(P.activations(kind, M, K, dtype, seed=seed)).to(dtype).cuda()


def _workspace(nbytes):
    return torch.full((max(nbytes, 256),), 0xFF, dtype=torch.uint8, device="cuda")


def _part(ws, off, shape, dtype):
    n = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
    return ws[off:off + n].view(dtype).view(*shape)


def _unwritten(t):
    """Elements still holding the workspace's 0xFF fill."""
    return int((t.view(torch.int16 if t.element_size() == 2 else torch.int32) == -1).sum())


# --------------------------------------------------------------------------- dense MLP
@functools.lru_cache(maxsize=None)
def _mlp(H, I, g, dtype, act13, act2, bias, seed):
    from autogptq_b200 import FusedQuantMLP

    dt = P.dt_name(dtype)
    d1 = P.wide_layer(H, I, g, dt, seed=seed, act_order=act13, bias=bias)
    d3 = P.wide_layer(H, I, g, dt, seed=seed + 1, bias=bias, g_idx=d1["g_idx"])
    d2 = P.wide_layer(I, H, g, dt, seed=seed + 2, act_order=act2, bias=bias)
    return FusedQuantMLP(*(make_layer(d, dtype=dtype) for d in (d1, d3, d2)), fused_backward=True), (d1, d3, d2)


def _dense_case(dtype, M, cfg, tile, dy_kind, x_kind, rows_i=None, rows_h=None, what=""):
    """One forced (tile_m, split_k) call and one automatic call of the dense backward; every stage checked.
    ``rows_i`` / ``rows_h``: check dg, du on these ranges of I and dx on these ranges of H (float64 time)."""
    H, I, g, act13, act2, bias = cfg
    mlp, (d1, d3, d2) = _mlp(H, I, g, dtype, act13, act2, bias, 7)
    dt = P.dt_name(dtype)
    x, dy = _act(x_kind, M, H, dtype, M), _act(dy_kind, M, H, dtype, M + 1)
    xg = x.clone().requires_grad_(True)
    mlp(xg).backward(dy)
    with torch.no_grad():
        _, _, gt, ut = mlp._forward_saving(x)
    lib = _lib.load()
    L = B.mlp_bwd_layout(M, H, I)
    assert lib.agb200_w4a16_mlp_backward_workspace_bytes(M, H, I) == L["total"]
    args = mlp._args(dtype)

    def run(tile_m, split_k):
        ws, dx = _workspace(L["total"]), torch.empty((M, H), dtype=dtype, device="cuda")
        rc = lib.agb200_w4a16_mlp_backward_ex(
            dy.data_ptr(), args.pair.p_gate, args.pair.p_up, args.p_down, gt.data_ptr(), ut.data_ptr(), dx.data_ptr(),
            M, H, I, mlp.gate_proj.group_size, mlp.down_proj.group_size, CODE[dtype], ws.data_ptr(), ws.numel(),
            torch.cuda.current_stream().cuda_stream, tile_m, split_k)
        _lib.check(rc, "agb200_w4a16_mlp_backward_ex")
        torch.cuda.synchronize()
        return dx, ws

    dx_auto, _ = run(0, 0)
    assert _bits_equal(dx_auto, xg.grad), f"{what}: the ABI's dx differs from the module's autograd dx"
    dx, ws = run(*tile)
    dgu = _part(ws, L["dgu"], (M, 2 * I), dtype)
    assert _unwritten(dgu) == 0, f"{what}: [dg | du] elements left unwritten"
    perm13 = B.sorted_perm(d1)
    if perm13 is not None:      # dx staged in w1's sorted order, then unpermuted
        assert _bits_equal(_part(ws, L["dxs"], (M, H), dtype), dx[:, torch.from_numpy(perm13).cuda()])
    dgu, g, u, dyv = _np(dgu), _np(gt), _np(ut), _np(dy)
    ci = np.concatenate([np.arange(a, b) for a, b in rows_i]) if rows_i else slice(None)
    ch = np.concatenate([np.arange(a, b) for a, b in rows_h]) if rows_h else slice(None)
    tag = f"{what} {dt} M={M} mt={tile[0]} split={tile[1]} dy={dy_kind} x={x_kind}"
    ref = B.dh_reference(dyv, B.weights(d2, dt, rows=rows_i))
    res = B.check_dgu(dgu[:, :I][:, ci], dgu[:, I:][:, ci], ref, g[:, ci], u[:, ci], dtype, what=tag)
    W1, W3 = B.weights(d1, dt, rows=rows_h), B.weights(d3, dt, rows=rows_h)
    res["dx"] = P.check(_np(dx)[:, ch], B.dx_reference(dgu[:, :I], dgu[:, I:], W1, W3), P.PATHS["dgrad"], dtype,
                        what=f"{tag} dx")
    for stage, r in res.items():
        _record(f"dense {stage}", dtype, r)
    print(f"[bwd-stages] {tag}: " + "  ".join(f"{k} {r.worst:.3f}/{100 * r.rate:.2f}%/{r.g_used:.2f}" for k, r in res.items()))


DENSE = [(1024, 2816, 128, True, True, True), (1024, 1536, 32, True, False, False), (1152, 2304, 96, False, True, True),
         (1024, 1536, -1, False, False, True), (1088, 1472, 32, True, False, True)]
DENSE_M = [1, 5, 8, 9, 64, 200, 2049]


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("cfg", range(len(DENSE)),
                         ids=["2816_g128_act_both_bias", "1536_g32_act13", "1152x2304_g96_act2_bias", "1536_g-1_bias",
                              "1088x1472_g32_act13_bias"])
@pytest.mark.parametrize("M", DENSE_M)
def test_dense_stages(dtype, cfg, M):
    """(H, I) = (1088, 1472) leaves a partial last 128-k tile in both stages (I, H not multiples of 128)."""
    i = DENSE_M.index(M) * len(DENSE) + cfg
    kinds = _kinds(dtype)
    _dense_case(dtype, M, DENSE[cfg], TILES[i % len(TILES)], kinds[i % len(kinds)], kinds[(i + 3) % len(kinds)],
                what=f"dense cfg{cfg}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [8, 300])
def test_dense_stages_llama2_7b_size(dtype, M):
    _dense_case(dtype, M, (4096, 11008, 128, True, True, False), TILES[M % len(TILES)], "offset" if M == 8 else "gauss",
                "massive", rows_i=[(11008 - 256, 11008)], rows_h=[(0, 256), (4096 - 256, 4096)], what="llama-2-7b")


# --------------------------------------------------------------------------- grouped experts
@functools.lru_cache(maxsize=None)
def _qe(E, H, I, g, dtype, act13, act2, bias, seed):
    from autogptq_b200 import QuantExperts

    ex = S.realistic_experts(E, H, I, g, P.dt_name(dtype), seed=seed, act13=act13, act2=act2, bias=bias)
    mods = {n: [make_layer(e[n], dtype=dtype) for e in ex] for n in ("w1", "w3", "w2")}
    return QuantExperts(mods["w1"], mods["w3"], mods["w2"], input_grad=True), ex


def _moe_case(dtype, E, H, I, T, k, idx, w, dy_kind, x_kind, w16=False, act=True, bias=True, idx_dtype=torch.int64,
              rows_i=None, rows_h=None, stage_tag="experts", what=""):
    qe, ex = _qe(E, H, I, 128, dtype, act, act, bias, 0)
    dt = P.dt_name(dtype)
    x, dy = _act(x_kind, T, H, dtype, T + k), _act(dy_kind, T, H, dtype, T + k + 1)
    it = torch.from_numpy(np.asarray(idx)).to(idx_dtype).cuda()
    wt = torch.from_numpy(np.asarray(w, dtype=np.float32)).to(dtype if w16 else torch.float32).cuda()
    xg, wg = x.clone().requires_grad_(True), wt.clone().requires_grad_(True)
    qe(xg, it, wg).backward(dy)
    with torch.no_grad():
        _, saved = qe._forward(x, it, wt, save=True)
    plan = qe._plan(dtype, x.device)
    lib = _lib.load()
    L = B.bwd_layout(T, k, E, H, I)
    assert lib.agb200_moe_backward_workspace_bytes(T, k, E, H, I) == L["total"]
    ws = _workspace(L["total"])
    dx = torch.empty((T, H), dtype=dtype, device="cuda")
    dw = torch.empty((T, k), dtype=wt.dtype, device="cuda")
    rc = lib.agb200_moe_backward(plan.handle, dy.data_ptr(), it.data_ptr(),
                                 _lib.MOE_INDEX_I64 if idx_dtype == torch.int64 else _lib.MOE_INDEX_I32, wt.data_ptr(),
                                 CODE[dtype] if w16 else _lib.MOE_WEIGHTS_F32, T, k, saved.data_ptr(), saved.numel(),
                                 dx.data_ptr(), dw.data_ptr(), ws.data_ptr(), ws.numel(),
                                 torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "agb200_moe_backward")
    torch.cuda.synchronize()
    tag = f"{what} {dt} T={T} k={k} mt={L['mt']} dy={dy_kind} x={x_kind} w16={w16}"
    assert _bits_equal(dx, xg.grad), f"{tag}: the ABI's dx differs from the module's autograd dx"

    Pn, rows = T * k, L["rows"]
    flat = np.asarray(idx).astype(np.int64).reshape(-1)
    valid = (flat >= 0) & (flat < E)
    prow = _part(ws, L["prow"], (Pn,), torch.int32).cpu().numpy()
    assert (prow[~valid] == -1).all(), f"{tag}: prow of an invalid id is not -1"
    pv = prow[valid]
    assert ((pv >= 0) & (pv < rows)).all() and len(np.unique(pv)) == pv.size, f"{tag}: prow not distinct rows"
    sel = torch.from_numpy(pv.astype(np.int64)).cuda()
    dyp_t = _part(ws, L["dyp"], (rows, H), dtype)[sel]
    dgu_t = _part(ws, L["dgu"], (rows, 2 * I), dtype)[sel]
    dxp_t = _part(ws, L["dxp"], (rows, H), torch.float32)[sel]
    for name, t in (("dy_pair", dyp_t), ("[dg | du]", dgu_t), ("dx_pair", dxp_t)):
        assert _unwritten(t) == 0, f"{tag}: {name} elements of valid pairs left unwritten"
    # per valid pair id (in flat order): the rows the kernels wrote
    dyp, dgu, dxp = np.zeros((Pn, H)), np.zeros((Pn, 2 * I)), np.zeros((Pn, H), dtype=np.float32)
    dyp[valid], dgu[valid], dxp[valid] = _np(dyp_t), _np(dgu_t), dxp_t.cpu().numpy()
    dyv, wv = _np(dy), wt.float().cpu().numpy()
    B.check_exact(dyp[valid], B.dy_pair(dyv, wv, dt).reshape(Pn, H)[valid], what=f"{tag} dy_pair")

    gu_off = -(-Pn * I * 2 // 256) * 256
    g_sv, u_sv = _np(saved[:Pn * I * 2].view(dtype).view(Pn, I)), _np(saved[gu_off:gu_off + Pn * I * 2].view(dtype).view(Pn, I))
    ci = np.concatenate([np.arange(a, b) for a, b in rows_i]) if rows_i else slice(None)
    ch = np.concatenate([np.arange(a, b) for a, b in rows_h]) if rows_h else slice(None)
    dh, A, gs, us, dgs, dus, refs, dxo = [], [], [], [], [], [], [], []
    dxp_nat = np.zeros_like(dxp)
    for e in range(E):
        pid = np.nonzero(flat == e)[0]
        if not pid.size:
            continue
        inv2 = S.h_order_inverse(ex[e]["w2"])
        g, u = (g_sv[pid], u_sv[pid]) if inv2 is None else (g_sv[pid][:, inv2], u_sv[pid][:, inv2])
        r = B.dh_reference(dyp[pid], B.weights(ex[e]["w2"], dt, rows=rows_i))
        dh.append(r.dh), A.append(r.A), gs.append(g[:, ci]), us.append(u[:, ci])
        dgs.append(dgu[pid, :I][:, ci]), dus.append(dgu[pid, I:][:, ci])
        p13 = B.sorted_perm(ex[e]["w1"])
        dxp_nat[pid] = dxp[pid] if p13 is None else dxp[pid][:, B.inverse(p13)]
        W1, W3 = B.weights(ex[e]["w1"], dt, rows=rows_h), B.weights(ex[e]["w3"], dt, rows=rows_h)
        refs.append(B.dx_reference(dgu[pid, :I], dgu[pid, I:], W1, W3))
        dxo.append(dxp_nat[pid][:, ch])
    cat = np.concatenate
    res = B.check_dgu(cat(dgs), cat(dus), B.DhRef(cat(dh), cat(A), H), cat(gs), cat(us), dtype, what=tag)
    res["dx_pair"] = B.check_dx_pair(cat(dxo), S.cat_refs(refs), what=tag)
    B.check_exact(_np(dx), B.dx_combine(dxp_nat.reshape(T, k, H), np.asarray(idx), E, dt), what=f"{tag} dx combine")
    for stage, r in res.items():
        _record(f"{stage_tag} {stage}", dtype, r)
    print(f"[bwd-stages] {tag}: " + "  ".join(f"{k} {r.worst:.3f}/{100 * r.rate:.2f}%/{r.g_used:.2f}" for k, r in res.items()))
    REPORT.setdefault(("experts dy_pair, dx combine bit-exact", dt), [0, 0.0, 0.0, 0.0])[0] += 1


def _routing(T, k, E, seed, invalid=None):
    """Distinct experts per token, fp32 weights summing to 1; ``invalid``: that id on ~15 % of the slots."""
    rng = np.random.default_rng(seed)
    idx = np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)
    if invalid is not None:
        idx[rng.random(idx.shape) < 0.15] = invalid
    w = rng.random((T, k)).astype(np.float32) + 0.05
    return idx, w / w.sum(axis=1, keepdims=True)


# k, T and the row tile bwd_tile picks from T·k / 8 pairs per expert
MOE_TK = [(1, 40, 32), (1, 400, 64), (1, 800, 128), (2, 5, 32), (2, 64, 32), (2, 200, 64), (2, 600, 128), (4, 32, 32),
          (4, 100, 64), (4, 300, 128)]


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("k,T,mt", MOE_TK)
def test_experts_stages(dtype, k, T, mt):
    assert B.bwd_tile(T * k, 8) == mt
    i = MOE_TK.index((k, T, mt))
    kinds = _kinds(dtype)
    i32 = i % 2 == 1
    idx, w = _routing(T, k, 8, seed=i, invalid=(-1 if i32 else 8) if i % 3 else None)
    _moe_case(dtype, 8, 1024, 1536, T, k, idx, w, kinds[i % len(kinds)], kinds[(i + 2) % len(kinds)], w16=i % 2 == 0,
              act=i % 4 < 2, bias=i % 3 != 1, idx_dtype=torch.int32 if i32 else torch.int64, what="experts")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("w16", [False, True], ids=["w32", "w16"])
def test_experts_stages_skewed_routing(dtype, w16):
    """One expert takes all 300 tokens (more than one 128-row tile), two share the second slot, the rest are empty;
    a sprinkling of invalid ids."""
    rng = np.random.default_rng(5)
    T = 300
    idx = np.stack([np.full(T, 5), rng.integers(0, 2, T)], axis=1).astype(np.int64)
    idx[rng.random(idx.shape) < 0.1] = 8
    w = rng.random((T, 2)).astype(np.float32)
    _moe_case(dtype, 8, 1024, 1536, T, 2, idx, w, "student_t", "offset", w16=w16, what="experts skewed")


@pytest.mark.parametrize("T", [8, 64])
def test_experts_stages_mixtral_size(T):
    """Mixtral-8x7B's expert shapes: the gate/up stage's reduction runs over n = 2I = 28672 terms."""
    idx, w = _routing(T, 2, 8, seed=T, invalid=8)
    _moe_case(F16, 8, 4096, 14336, T, 2, idx, w, "gauss", "offset", act=False, bias=False,
              rows_i=[(14336 - 256, 14336)], rows_h=[(0, 256), (4096 - 256, 4096)], stage_tag="experts n=28672",
              what="mixtral")


def test_report():
    """Largest err/bound, mismatch rate and γ share per stage and dtype (the DESIGN §3.12 rows)."""
    if not REPORT:
        pytest.skip("no stage check ran")
    print("\n[bwd-stages] stage                                    dtype      cases  max err/bound  max mismatch  max γ share")
    for (stage, dt), (n, w, rt, gu) in sorted(REPORT.items()):
        print(f"[bwd-stages] {stage:<40} {dt:<9} {n:>6}  {w:13.3f}  {rt:12.4f}  {gu:11.3f}")
