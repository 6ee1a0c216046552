"""Next-token sampling on the GPU (``agb200_sample``, DESIGN §3.21) against the float64 replay of ``tests/_sampling.py``.

Kernel grid: B ∈ {1, 3, 8} × V ∈ {1, 7, 4099, 32000, 128256, 152064, 262144} × fp16 / bf16 / fp32 logits with a row
stride above V; the rows carry parameter sets across greedy, temperature {0.3, 1, 2}, top_k {0, 1, 5, 50, V, V+10},
top_p {1, 0.9, 0.5, 1e-6} and min_p {0, 0.05}.  Every token lies in the reference K (ambiguous members allowed) and
equals the replay's draw unless the replay marks it ambiguous; greedy rows are bit-equal to torch.argmax, with planted
ties.  Two calls are bit-identical, a row's token does not depend on its index or the other rows, and a CUDA graph
replay at advancing counters equals the eager calls.  -inf is never drawn, one finite logit is always drawn, NaN and
all -inf rows give in-range tokens, idle rows write 0.  2·10^5 draws of a 64-token row pass a chi-square test against
the float64 probabilities.  BatchDecoder and ChainDecoder (dense and Mixtral): temperature 0 equals greedy generate,
sampled generate is reproducible and slot-independent, and every sampled token replays from the step's logits."""
import numpy as np
import pytest
import torch

from autogptq_b200 import BatchDecoder, SamplingParams, _lib, sample
from tests import _sampling as S

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
DTS = [F16, BF16, F32]


def _rows(params, B, dev="cuda"):
    """Device parameter tensors of B rows from a list of (temperature, top_k, top_p, min_p, seed, counter)."""
    t, k, p, m, s, c = zip(*params)
    f = lambda x, dt: torch.tensor(x, dtype=dt, device=dev)  # noqa: E731
    return (f(t, F32), f(k, torch.int32), f(p, F32), f(m, F32),
            f([v - 2 ** 64 if v >= 2 ** 63 else v for v in s], torch.int64), f(c, torch.int64))


def _logits(B, V, dtype, seed, pad=13):
    """[B, V] logits as a view of a [B, V + pad] buffer (row stride > V), LLM-like scale."""
    g = torch.Generator().manual_seed(seed)
    buf = (torch.randn(B, V + pad, generator=g) * 3).to(dtype)
    return buf.cuda()[:, :V]


def _sets(V):
    ks = [0, 1, 5, 50, V, V + 10]
    out = [(0.0, 0, 1.0, 0.0)]
    for i, t in enumerate((0.3, 1.0, 2.0)):
        for j, k in enumerate(ks):
            p = (1.0, 0.9, 0.5, 1e-6)[(i + j) % 4]
            m = (0.0, 0.05)[(i * 7 + j) % 2]
            out.append((t, k, p, m))
    return out


def _check_row(l, params, tok, counter):
    """(ambiguous) after checking one row's token against the contract."""
    t, k, p, m, seed = params
    V = l.size
    if t == 0:
        assert tok == int(np.argmax(l.astype(np.float32)))
        return False
    s = S.scaled(l, t)
    sure, amb = S.kept(s, k, p, m)
    assert sure[tok] or amb[tok], f"token {tok} outside K (V={V}, params={params})"
    want, ambiguous = S.replay(s, sure, amb, seed, counter)
    if not ambiguous:
        assert tok == want, f"token {tok}, replay {want} (V={V}, params={params}, counter={counter})"
    return ambiguous


@pytest.mark.parametrize("V", [1, 7, 4099, 32000, 128256, 152064, 262144])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16", "f32"])
def test_kernel_grid(V, dtype):
    sets = _sets(V)
    n_draws = n_amb = 0
    for B in (1, 3, 8):
        for start in range(0, len(sets), B):
            rows = [sets[(start + b) % len(sets)] for b in range(B)]
            params = [(t, k, p, m, 1000 * V + 17 * b + start, 5 + b + start) for b, (t, k, p, m) in enumerate(rows)]
            logits = _logits(B, V, dtype, seed=V + B + start)
            toks = sample(logits, *_rows(params, B)).cpu().tolist()
            l = logits.float().cpu().numpy()
            for b in range(B):
                assert 0 <= toks[b] < V
                n_amb += _check_row(l[b], params[b][:5], toks[b], params[b][5])
                n_draws += 1
            if V >= 128256 and start >= 2 * B:              # the largest rows: a sample of the sets per B
                break
    print(f"V={V} {dtype}: {n_draws} draws, {n_amb} ambiguous")
    assert n_amb <= max(1, n_draws // 20)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16", "f32"])
def test_greedy_is_torch_argmax_with_ties(dtype):
    B, V = 8, 32000
    logits = _logits(B, V, dtype, seed=3)
    for b in range(B):
        top = logits[b].max()
        idx = torch.tensor([b * 997 % V, (b * 131 + 5) % V, V - 1 - b], device="cuda")
        logits[b, idx] = top                                  # planted ties at the maximum
    logits[7].fill_(0.5)                                      # a whole row tied
    params = [(0.0, 0, 1.0, 0.0, b, b) for b in range(B)]
    toks = sample(logits, *_rows(params, B))
    assert torch.equal(toks, torch.argmax(logits, dim=-1))


def test_bit_identity_row_independence_and_graph():
    V, dtype = 152064, F16
    params = [(0.7, 50, 0.9, 0.0, 42, 9), (1.0, 0, 1.0, 0.05, 7, 10), (0.0, 0, 1.0, 0.0, 1, 11),
              (2.0, 0, 0.5, 0.0, 2 ** 64 - 1, 12), (1.0, 0, 1.0, 0.0, 3, 2 ** 33 + 1)]
    B = len(params)
    logits = _logits(B, V, dtype, seed=5)
    args = _rows(params, B)
    a = sample(logits, *args).clone()
    assert torch.equal(a, sample(logits, *args))
    # row 0's inputs at row 3 of another batch whose other rows hold different logits and parameters
    other = _logits(B, V, dtype, seed=6)
    other[3] = logits[0]
    moved = [(1.0, 5, 1.0, 0.0, 99, 1)] * B
    moved[3] = params[0]
    assert sample(other, *_rows(moved, B))[3] == a[0]
    # a graph replay at advancing counters equals the eager calls
    t, k, p, m, s, c = args
    out = torch.zeros(B, dtype=torch.int64, device="cuda")
    sample(logits, t, k, p, m, s, c, out=out)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        sample(logits, t, k, p, m, s, c, out=out)
    for step in range(4):
        c.add_(1)
        g.replay()
        eager = sample(logits, t, k, p, m, s, c.clone())
        assert torch.equal(out, eager), step


def test_special_values():
    V = 4099
    base = _logits(6, V, F32, seed=8).contiguous()
    l = base.clone()
    l[0, ::2] = float("-inf")                                 # -inf never drawn
    l[1].fill_(float("-inf"))
    l[1, 1234] = -3.0                                         # one finite logit
    l[2, 77] = float("nan")                                   # NaN: in range
    l[3].fill_(float("-inf"))                                 # all -inf: in range
    params = [(1.0, 0, 1.0, 0.0, 1, 1), (2.0, 10, 0.9, 0.1, 2, 2), (1.0, 0, 0.9, 0.0, 3, 3),
              (1.0, 5, 0.5, 0.05, 4, 4), (1.0, 0, 1.0, 0.0, 5, -1), (0.0, 0, 1.0, 0.0, 6, -5)]
    toks = sample(l, *_rows(params, 6)).cpu().tolist()
    assert toks[0] % 2 == 1
    assert toks[1] == 1234
    assert 0 <= toks[2] < V and 0 <= toks[3] < V
    assert toks[4] == 0 and toks[5] == 0                      # idle rows
    for c in range(64):                                       # -inf stays out over many draws
        p0 = [(1.0, 0, 1.0, 0.0, 1, c)]
        assert int(sample(l[:1], *_rows(p0, 1))[0]) % 2 == 1


@pytest.mark.parametrize("params", [(1.0, 0, 1.0, 0.0), (0.7, 10, 1.0, 0.0), (1.0, 0, 0.8, 0.0), (1.5, 0, 1.0, 0.05),
                                    (1.0, 20, 0.9, 0.02)])
def test_distribution(params):
    from scipy.stats import chisquare

    V, n, chunk = 64, 200000, 50000
    rng = np.random.default_rng(4)
    row = (rng.standard_normal(V) * 1.5).astype(np.float32)
    logits = torch.from_numpy(row).cuda().expand(chunk, V).contiguous()
    t, k, p, m = params
    s = S.scaled(row, t)
    sure, amb = S.kept(s, k, p, m)
    assert not amb.any()
    prob = S.probabilities(s, sure)
    counts = np.zeros(V)
    for c0 in range(0, n, chunk):
        rows = [(t, k, p, m, 2024, c0 + i) for i in range(chunk)]
        toks = sample(logits, *_rows(rows, chunk)).cpu().numpy()
        counts += np.bincount(toks, minlength=V)
    assert np.all(counts[~sure] == 0)
    pv = chisquare(counts[sure], prob[sure] * n).pvalue
    print(f"{params}: chi-square p = {pv:.3g}")
    assert pv > 1e-4


# --------------------------------------------------------------------------- decoders
def _replay_token(logits_row, sp, counter):
    l = logits_row.float().cpu().numpy()
    s = S.scaled(l, sp.temperature)
    sure, amb = S.kept(s, sp.top_k, sp.top_p, sp.min_p)
    return S.replay(s, sure, amb, sp.seed, counter)


def _prompts(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 512, (int(L),), generator=g) for L in torch.randint(3, 12, (n,), generator=g)]


@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_batch_decoder_sampling(arch):
    from tests.test_gpu_21_chain_norm import _model

    model = _model(arch, F16)
    dec = BatchDecoder(model, max_batch=4, max_length=64)
    prompts = _prompts(6)
    greedy = dec.generate(prompts, 8)
    zero = dec.generate(prompts, 8, sampling=SamplingParams(temperature=0))
    assert all(torch.equal(a, b) for a, b in zip(greedy, zero))
    sps = [SamplingParams(temperature=0.9, top_k=50, top_p=0.9, seed=100 + j) for j in range(6)]
    a = dec.generate(prompts, 8, sampling=sps)
    assert all(torch.equal(x, y) for x, y in zip(a, dec.generate(prompts, 8, sampling=sps)))
    # the same prompt and parameters in another order (so other slots and neighbours) give the same continuation
    order = [3, 0, 5, 1, 4, 2]
    b = dec.generate([prompts[j] for j in order], 8, sampling=[sps[j] for j in order])
    assert all(torch.equal(b[i], a[j]) for i, j in enumerate(order))
    torch.manual_seed(5)
    c = dec.generate(prompts, 8, sampling=SamplingParams(temperature=1.0))
    torch.manual_seed(5)
    assert all(torch.equal(x, y) for x, y in zip(c, dec.generate(prompts, 8, sampling=SamplingParams(temperature=1.0))))

    # every sampled token replays from the logits it was drawn from, counter = its position
    for s in range(4):
        dec.release(s)
    sps = [SamplingParams(temperature=t, top_k=k, top_p=p, min_p=m, seed=7 + s)
           for s, (t, k, p, m) in enumerate([(0.8, 0, 0.9, 0.0), (1.0, 20, 1.0, 0.05), (0.0, 0, 1.0, 0.0),
                                             (1.3, 0, 1.0, 0.0)])]
    ids = torch.zeros(4, dtype=torch.int64)
    n_amb = 0
    for s in (0, 1, 3):                                       # slot 2 stays idle
        dec.set_sampling(s, sps[s])
        logits = dec.prefill(s, prompts[s])
        tok = dec.sample(s, logits)
        want, amb = _replay_token(logits, sps[s], dec.positions[s])
        assert amb or tok == want
        n_amb += amb
        ids[s] = tok
    for _ in range(6):
        pos = dec.positions
        toks, logits = dec.step_sample(ids.cuda())
        toks = toks.cpu()
        assert toks[2] == 0
        for s in (0, 1, 3):
            want, amb = _replay_token(logits[s], sps[s], pos[s] + 1)
            assert amb or int(toks[s]) == want
            n_amb += amb
        ids = toks.clone()
    assert n_amb <= 2


def _chain_replay(dec, ids, out, sps):
    """Teacher-force the sampled tokens through greedy steps and replay each draw from its logits."""
    T = ids.shape[1]
    logits = dec.prefill(ids)
    n_amb = 0
    for t in range(out.shape[1] - T):
        for b, sp in enumerate(sps):
            want, amb = _replay_token(logits[b], sp, T + t)
            assert amb or int(out[b, T + t]) == want, (b, t)
            n_amb += amb
        if T + t + 1 < out.shape[1]:
            logits = dec.step(out[:, T + t].clone())
    return n_amb


@pytest.mark.parametrize("batch", [1, 2])
def test_chain_decoder_sampling(batch):
    from autogptq_b200.decoder import ChainDecoder
    from tests.test_gpu_21_chain_norm import _model

    dec = ChainDecoder(_model("llama", F16), batch=batch, max_length=64)
    ids = torch.randint(0, 512, (batch, 7), generator=torch.Generator().manual_seed(2)).cuda()
    assert torch.equal(dec.generate(ids, 10), dec.generate(ids, 10, sampling=SamplingParams(temperature=0)))
    sps = [SamplingParams(temperature=0.8, top_k=40, top_p=0.95, seed=31 + b) for b in range(batch)]
    out = dec.generate(ids, 10, sampling=sps)
    assert torch.equal(out, dec.generate(ids, 10, sampling=sps))
    assert _chain_replay(dec, ids, out, sps) <= 1


def test_chain_decoder_sampling_mixtral():
    from autogptq_b200.decoder import ChainDecoder
    from tests.test_gpu_23_moe_decoder import _model

    dec = ChainDecoder(_model(F16), batch=1, max_length=64, fused_attention=True)
    ids = torch.randint(0, 512, (1, 5), generator=torch.Generator().manual_seed(3)).cuda()
    assert torch.equal(dec.generate(ids, 8), dec.generate(ids, 8, sampling=SamplingParams(temperature=0)))
    sps = [SamplingParams(temperature=1.0, min_p=0.05, seed=5)]
    out = dec.generate(ids, 8, sampling=sps)
    assert _chain_replay(dec, ids, out, sps) <= 1


def test_refusals():
    z = torch.zeros(2, 100, device="cuda")
    params = _rows([(1.0, 0, 1.0, 0.0, 1, 1)] * 2, 2)
    with pytest.raises(NotImplementedError, match="vocabulary"):
        sample(torch.zeros(1, _lib.SAMPLE_MAX_V + 1, device="cuda"), *_rows([(1.0, 0, 1.0, 0.0, 1, 1)], 1))
    with pytest.raises(ValueError, match="contiguous last dimension"):
        sample(torch.zeros(100, 2, device="cuda").t(), *params)
    with pytest.raises(ValueError, match="top_k"):
        sample(z, params[0], params[1].long(), *params[2:])
    lib = _lib.load()
    assert lib.agb200_sample(z.data_ptr(), 99, _lib.F32, 2, 100, *(t.data_ptr() for t in params),
                             params[5].data_ptr(), None) == -1          # row_stride < V
