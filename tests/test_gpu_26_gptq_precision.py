"""The GPTQ quantiser's kernels against float64 on an H100, at real layer shapes (tests/_gptq_replay.py).

``gptq_hessian_kernel``: every element of H within its bound of the float64 running mean over the same batches, the
mismatch rate against round_f32(H*) under its limit, H bit-symmetric and two runs bit-identical.  ``gptq_quantize_kernel``:
the teacher-forced float64 replay of every row (g_idx, parameters, codes, Q, losses, packing), on Hinv from the project's
own ``add_batch`` and ``inverse_hessian_factor``.  Calibration inputs look like real ones: correlated Gaussian rows, three
massive channels (×1000) and a few near-dead ones (variance 1e-6), so the error feedback is large.
"""
import math
import time

import numpy as np
import pytest
import torch
import torch.nn as nn

from tests import _gptq_replay as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
F16, BF16 = torch.float16, torch.bfloat16
_SUMMARY: dict = {}

# Sharpness limits, set from the first H100 runs (H100 80GB HBM3, 700 W power limit) with a margin.  Measured: Hessian
# mismatch rate 33 % (fp16) / 9.1 % (bf16) of the well-conditioned elements (cases with at least 1000 of them); unclear
# codes 0.020 % (fp16) / 0.008 % (bf16).  The correctness assertions (every element within its bound, no clear code
# mismatch) are derived; only the Hessian's tensor-core factor is calibrated (tests/_gptq_replay.py, HESS_MMA).
HESS_RATE = 0.5             # share of well-conditioned elements with H != round_f32(H*)
UNCLEAR_LIMIT = 0.001       # share of codes the bound leaves undecided (the replay's own sharpness)


@pytest.fixture(scope="module", autouse=True)
def _print_summary():
    torch.zeros(1, device=DEV)                     # initialises the device before its memory statistics are read
    torch.cuda.reset_peak_memory_stats(DEV)
    t0 = time.perf_counter()
    yield
    print(f"\n[gptq precision] {time.perf_counter() - t0:.0f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated(DEV) / 2**30:.1f} GiB")
    print("\n[gptq precision] kernel    dtype     cases  max err/bound  max unclear share  max mismatch rate")
    for (k, dt), (n, worst, unclear, rate) in sorted(_SUMMARY.items()):
        print(f"[gptq precision] {k:<9} {dt:<9} {n:>5}  {worst:13.3f}  {unclear:17.5f}  {rate:17.4f}")


def _record(kernel, dtype, worst, unclear, rate):
    key = (kernel, str(dtype).replace("torch.", ""))
    n, w, u, r = _SUMMARY.get(key, (0, 0.0, 0.0, 0.0))
    _SUMMARY[key] = (n + 1, max(w, worst), max(u, unclear), max(r, rate))


def calib(T, K, dtype, seed=0, dead=()):
    """[T, K] calibration rows: Gaussian mixed through a rank-32 correlation, three channels ×1000, four near-dead
    channels (×1e-3: variance 1e-6), and the ``dead`` channels exactly zero."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    z = torch.randn(T, K, generator=g, device=DEV)
    a = torch.randn(K, 32, generator=g, device=DEV) / math.sqrt(K)
    x = z + (z @ a) @ torch.randn(32, K, generator=g, device=DEV)
    ch = torch.randperm(K, generator=g, device=DEV)
    x[:, ch[:3]] *= 1000.0
    x[:, ch[3:7]] *= 1e-3
    if len(dead):
        x[:, list(dead)] = 0
    return x.to(dtype)


# --------------------------------------------------------------------------- Hessian
def _hessian(batches, K):
    from autogptq_b200.gptq import GPTQ

    g = GPTQ(nn.Linear(K, 8, bias=False).to(DEV, F16))
    for x in batches:
        g.add_batch(x, None)
    torch.cuda.synchronize()
    return g


# (dtype, K, per-call shapes: (T,) is a 2-D input, (b, s) a 3-D one of b samples)
HESS_CASES = [
    (F16, 8, [(0,), (1,), (31,)]),
    (BF16, 8, [(2, 33), (1, 0)]),
    (F16, 120, [(33,), (4, 1)]),
    (BF16, 136, [(4097,)]),
    (F16, 520, [(2048,), (0,), (3, 31)]),
    (BF16, 520, [(31,), (1,)]),
    (F16, 4104, [(4097,), (33,)]),
    (BF16, 11008, [(2, 1024), (1,)]),
    (F16, 14336, [(2048,)]),
]


def _shape_batches(K, dtype, shapes, seed):
    out = []
    for i, sh in enumerate(shapes):
        T = int(np.prod(sh))
        out.append(calib(T, K, dtype, seed=seed + i).reshape(*sh, K))
    return out


@pytest.mark.parametrize("dtype,K,shapes", HESS_CASES, ids=[f"{'f16' if d == F16 else 'bf16'}-K{k}-{s}" for d, k, s in HESS_CASES])
def test_hessian_elements_within_bound(dtype, K, shapes):
    batches = _shape_batches(K, dtype, shapes, seed=K)
    g = _hessian(batches, K)
    ref = R.HessianReference(K, DEV)
    for b in batches:
        ref.add(b)
    assert g.nsamples == ref.n
    assert torch.equal(g.H, g.H.T), "H is not bit-symmetric"
    m = ref.check(g.H, HESS_RATE, what=f"K={K} {shapes}")
    _record("hessian", dtype, m.worst, 0.0, m.rate)
    del ref
    g2 = _hessian(batches, K)
    assert torch.equal(g.H, g2.H), "two runs differ"


def test_hessian_128_calls_of_2048_tokens():
    """The running mean of a real quantisation run: 128 calibration samples of 2048 tokens at K = 4096, plus a
    misaligned input view (the clone path)."""
    from autogptq_b200.gptq import GPTQ

    K = 4096
    g = GPTQ(nn.Linear(K, 8, bias=False).to(DEV, F16))
    ref = R.HessianReference(K, DEV)
    for i in range(128):
        x = calib(2048, K, F16, seed=1000 + i).reshape(1, 2048, K)
        g.add_batch(x, None)
        ref.add(x)
    buf = calib(34, K, F16, seed=7).reshape(-1)
    x = buf[1:1 + 33 * K].reshape(33, K)           # 2-byte offset: not 16-byte aligned
    assert x.data_ptr() % 16
    g.add_batch(x, None)
    ref.add(x)
    torch.cuda.synchronize()
    assert g.nsamples == ref.n == 129
    assert torch.equal(g.H, g.H.T)
    m = ref.check(g.H, HESS_RATE, what="128 calls")
    _record("hessian", F16, m.worst, 0.0, m.rate)


# --------------------------------------------------------------------------- quantiser
def _weights(N, K, dtype, gs, seed):
    """Gaussian rows with a spread of magnitudes, and: row 0 all zero, row 1 one ×100 outlier, row 2's first group of
    tiny weights (fp16 scale subnormal).  Returned as the fp32 values of a ``dtype`` layer."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    W = torch.randn(N, K, generator=g, device=DEV) * 0.02 * (10 ** torch.rand(N, 1, generator=g, device=DEV))
    if N > 2:
        W[0] = 0
        W[1, K // 3] *= 100
        W[2, :min(K, gs if gs > 0 else K)] *= 1e-3
    return W.to(dtype).float()


def _hinv(K, dtype, seed, dead=(), act=False, T=None):
    from autogptq_b200.gptq import GPTQ, inverse_hessian_factor

    g = GPTQ(nn.Linear(K, 8, bias=False).to(DEV, dtype))
    T = T or max(256, 2 * K)
    for i in range(0, T, 2048):
        g.add_batch(calib(min(2048, T - i), K, dtype, seed=seed + i, dead=dead), None)
    return inverse_hessian_factor(g.H, 0.01, act)


# (N, K, group_size, act-order, static, sym, dtype, dead columns (original order), Hinv kind)
Q_CASES = [
    (8, 136, 8, False, False, False, F16, (0,), "real"),              # one CTA of 8 rows; last block of 8 columns
    (24, 136, -1, True, False, True, BF16, (135,), "real"),           # second CTA has 8 rows; dead last column
    (24, 520, 40, True, False, True, BF16, (128,), "real"),           # groups straddle blocks; dead at a block boundary
    (24, 520, 96, True, True, False, F16, tuple(range(96, 192)), "real"),   # a whole dead static group
    (24, 520, 192, False, False, False, BF16, (), "real"),            # groups wider than a block
    (8, 264, 32, False, False, False, F16, (), "diag"),               # exact RTN with .5 ties
    (8, 264, 32, False, False, True, BF16, (), "diag"),
    (11008, 520, 32, False, True, True, BF16, (), "real"),
    (4104, 4096, 128, True, False, False, BF16, (), "real"),          # N % 16 == 8
    (4096, 4104, 1024, False, False, True, F16, (5,), "real"),
    (1024, 14336, 128, True, False, False, F16, (), "real"),          # Mixtral w2: 112 blocks of trailing updates
]


def _diag_weights(N, K):
    """Rows of range 15 (s = 1) made of integers and .5 ties, and a diagonal Hinv: no error feedback."""
    g = torch.Generator(device=DEV).manual_seed(3)
    W = torch.randint(-15, 16, (N, K), generator=g, device=DEV).float() / 2
    W[:, 0::32], W[:, 1::32] = -7.5, 7.5
    W[1, 32:64] = 0                                       # all-zero group: zero = rint(fl(1 / fl(2/15))) = 7
    return W


def _ids(c):
    N, K, gs, act, st, sym, dt, dead, kind = c
    return f"N{N}-K{K}-g{gs}{'-act' if act else ''}{'-static' if st else ''}{'-sym' if sym else ''}-" \
           f"{'f16' if dt == F16 else 'bf16'}{'-dead' if dead else ''}-{kind}"


@pytest.mark.parametrize("case", Q_CASES, ids=[_ids(c) for c in Q_CASES])
def test_quantize_replay(case):
    from autogptq_b200.gptq import quantize_weight

    N, K, gs, act, static, sym, dtype, dead, kind = case
    if kind == "diag":
        W0 = _diag_weights(N, K)
        Hinv = torch.diag(torch.linspace(0.5, 2.0, K, device=DEV))
        perm, dmask = None, None
    else:
        W0 = _weights(N, K, dtype, gs, seed=N + K)
        Hinv, perm, dmask = _hinv(K, dtype, seed=K, dead=dead, act=act)
        assert int(dmask.sum()) == len(dead)
        dmask = dmask if len(dead) else None
    out = quantize_weight(W0.clone(), Hinv, perm=perm, dead=dmask, group_size=gs, sym=sym, static_groups=static,
                          dtype=dtype, losses=True)
    torch.cuda.synchronize()
    m = R.check_quantize(W0, Hinv, out, perm=perm, dead=dmask, group_size=gs, sym=sym, static_groups=static,
                         dtype=dtype, what=_ids(case))
    _record("quantize", dtype, m.worst, m.unclear, m.flipped)
    if kind == "diag":
        assert m.unclear == 0.0 and m.params_unclear == 0
        if not sym:
            assert out["zero"][1, 1].item() == 7.0 and out["zero"][0, 0].item() == 8.0
    assert m.unclear <= UNCLEAR_LIMIT, m


# --------------------------------------------------------------------------- GPTQ.fasterquant end to end
def _fasterquant(layer, batches, monkeypatch, **kw):
    """Run GPTQ on ``layer``; return the GPTQ object and the (Hinv, perm, dead) that fasterquant used."""
    import autogptq_b200.gptq as gq

    seen = {}
    real = gq.inverse_hessian_factor

    def spy(H, percdamp, actorder):
        seen["f"] = real(H, percdamp, actorder)
        return seen["f"]

    monkeypatch.setattr(gq, "inverse_hessian_factor", spy)
    g = gq.GPTQ(layer)
    g.quantizer.configure(4, perchannel=True, sym=kw.pop("sym"), mse=False)
    for x in batches:
        g.add_batch(x, None)
    g.fasterquant(blocksize=128, percdamp=0.01, **kw)
    torch.cuda.synchronize()
    return g, seen["f"]


def _check_fasterquant(g, W0, Wq, f, gs, sym, static, dtype, what):
    """fasterquant's outputs bit-equal to quantize_weight on the Hinv it used, and that result through the replay.
    ``Wq``: the layer's weights afterwards ([N, K], the layer dtype)."""
    from autogptq_b200.gptq import quantize_weight

    Hinv, perm, dead = f
    dead = dead if bool(dead.any()) else None
    ref = quantize_weight(W0.clone(), Hinv, perm=perm, dead=dead, group_size=gs, sym=sym, static_groups=static,
                          dtype=dtype, losses=True)
    assert torch.equal(Wq, ref["Q"].to(dtype)), f"{what}: the layer's weights differ from quantize_weight on the same Hinv"
    assert torch.equal(g.Losses, ref["losses"])
    ql = g.quant_linear
    for name in ("qweight", "qzeros", "scales", "g_idx"):
        assert torch.equal(getattr(ql, name), ref[name]), f"{what}: {name}"
    m = R.check_quantize(W0, Hinv, ref, perm=perm, dead=dead, group_size=gs, sym=sym, static_groups=static,
                         dtype=dtype, what=what)
    _record("quantize", dtype, m.worst, m.unclear, m.flipped)
    assert m.unclear <= UNCLEAR_LIMIT, m


@pytest.mark.parametrize("N,K,gs,act,static,sym,dtype", [
    (4096, 11008, 128, True, False, False, F16),         # Llama-2-7B down_proj, act-order
    (512, 1024, 128, False, True, True, BF16),
])
def test_fasterquant_matches_quantize_weight_and_replay(N, K, gs, act, static, sym, dtype, monkeypatch):
    lin = nn.Linear(K, N, bias=True).to(DEV, dtype)
    lin.weight.data = _weights(N, K, dtype, gs, seed=5).to(dtype)
    W0 = lin.weight.data.float().clone()
    batches = [calib(1024, K, dtype, seed=11 + i).reshape(2, 512, K) for i in range(2)]
    g, f = _fasterquant(lin, batches, monkeypatch, group_size=gs, actorder=act, static_groups=static, sym=sym)
    _check_fasterquant(g, W0, lin.weight.data, f, gs, sym, static, dtype, f"fasterquant N={N} K={K}")


def test_fasterquant_conv1d(monkeypatch):
    from transformers.pytorch_utils import Conv1D

    N, K, gs = 384, 768, 128
    layer = Conv1D(N, K).to(DEV, F16)                   # weight [K, N]
    layer.weight.data = _weights(N, K, F16, gs, seed=9).t().contiguous().half()
    W0 = layer.weight.data.t().float().contiguous()
    g, f = _fasterquant(layer, [calib(512, K, F16, seed=13)], monkeypatch, group_size=gs, actorder=True,
                        static_groups=False, sym=False)
    assert layer.weight.shape == (K, N)
    _check_fasterquant(g, W0, layer.weight.data.t(), f, gs, False, False, F16, "conv1d")
