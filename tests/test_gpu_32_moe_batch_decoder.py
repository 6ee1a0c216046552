"""BatchDecoder over Mixtral blocks on the GPU, and the router's idle rows it relies on.

Router rows (``moe_router(..., pos=)``, ``agb200_moe_router_rows``): for random positions with some rows idle (-1),
every row's h and n and the active rows' indices, weights and logits are bit-equal to ``moe_router`` without ``pos``;
idle rows get index -1 and weight 0 and leave their logits row untouched.  ``QuantExperts._forward`` then writes an
exactly zero row for each idle row, and the plan's active-expert list is that of the active rows alone.

BatchDecoder on the random 4-layer Mixtral of ``tests/test_gpu_23_moe_decoder.py`` (attention QuantLinear, experts
QuantExperts), fp16 / bf16, max_batch 3 and 8 (one slot idle at 8): prefill logits equal HF's; 32 forced steps match
each sequence run alone through HF at batch 1 within that test's Mixtral tolerance (times the factor
``tests/test_gpu_24_batch_decoder.py`` gives fp16 at more than 4 rows), with its rule for a step whose routing parts
from HF's where a router margin is unclear (not compared; the slot's cache re-seeded from HF's); greedy tokens agree
where the margin is clear; an eager step equals its graph replay.  Admitting and releasing slots leaves the other slots'
logits bit-identical; ``generate`` equals manual steps; a paged FP8 cache is bit-equal to the static FP8 one; and
``generate(n=2)`` gives each copy the tokens of an ``n=1`` run with its seed."""
import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from autogptq_b200.sampling import SamplingParams
from tests import _precision as P
from tests._util import assert_parity
from tests.test_gpu_23_moe_decoder import L_LAYERS, TOP_K, _logit_tol, _model, _router_inputs, _RouterHook

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTS = [F16, BF16]
FP8 = torch.float8_e4m3fn


def _bits(t):
    return t.view(torch.int16) if t.dtype in DTS else t


def _np(t):
    return t.double().cpu().numpy()


# --------------------------------------------------------------------------- router rows
def _route_meta(ws, E):
    """(per-expert pair counts [E], number of active experts) of the routing tables at the start of a forward's
    workspace (``csrc/moe.cu::route_views``: counts [E], offsets [E + 1], pad_off [E + 1], active [E], meta [2])."""
    ints = ws.view(torch.int32)
    return ints[:E].cpu().tolist(), int(ints[4 * E + 2])


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_router_rows_mask_idle_rows(dtype):
    from autogptq_b200.moe import moe_router

    experts = _model(dtype).model.layers[0].mlp.experts
    H, E, k = experts.hidden_size, experts.num_experts, TOP_K
    rng = np.random.default_rng(3)
    cases = [[5, -1, 0, 17, -1, 3, 100, -1], [-1, 2], [0], [-1, -1, -1, 4], [-1] * 8, [1, 2, 3, 4, 5, 6, 7, 8]]
    cases += [[int(p) if rng.random() < 0.6 else -1 for p in rng.integers(0, 200, T)] for T in (3, 5, 8, 8)]
    for c, ps in enumerate(cases):
        T = len(ps)
        x, x2, w, _ = _router_inputs(T, H, E, dtype, seed=40 + c)
        G = _model(dtype).model.layers[0].mlp.gate.weight.detach()
        pos = torch.tensor(ps, dtype=torch.int64, device="cuda")
        act = [r for r, p in enumerate(ps) if p >= 0]
        idle = [r for r, p in enumerate(ps) if p < 0]
        sentinel = torch.full((T, E), float("nan"), dtype=dtype, device="cuda")
        lg_rows, lg_all = sentinel.clone(), torch.empty_like(sentinel)
        h, n, idx, wts, _ = moe_router(x, x2, w, 1e-5, G, k, logits=lg_rows, pos=pos)
        h0, n0, idx0, wts0, _ = moe_router(x, x2, w, 1e-5, G, k, logits=lg_all)
        torch.cuda.synchronize()
        what = f"{dtype} pos={ps}"
        assert torch.equal(_bits(h), _bits(h0)) and torch.equal(_bits(n), _bits(n0)), f"{what}: h / n differ"
        assert torch.equal(idx[act], idx0[act]) and torch.equal(wts[act], wts0[act]), f"{what}: active routing differs"
        assert torch.equal(_bits(lg_rows[act]), _bits(lg_all[act])), f"{what}: active logits differ"
        assert (idx[idle] == -1).all() and (wts[idle] == 0).all(), f"{what}: an idle row routes to an expert"
        assert lg_rows[idle].isnan().all(), f"{what}: an idle row wrote logits"

        # the experts: idle rows give exact zeros and add no expert to the plan
        plan, ws = experts._static_buffers(T, k, dtype, "cuda")
        out = torch.full((T, H), float("nan"), dtype=dtype, device="cuda")
        experts._forward(n, idx, wts, out=out, plan=plan, ws=ws)
        torch.cuda.synchronize()
        counts, n_active = _route_meta(ws, E)
        assert (_bits(out[idle]) == 0).all(), f"{what}: an idle row's expert output is not +0"
        assert not out[act].isnan().any()
        want = [0] * E
        for e in idx0[act].flatten().tolist():
            want[e] += 1
        assert counts == want and n_active == sum(c > 0 for c in want), f"{what}: {counts} / {n_active} vs {want}"
        if act:                                          # the same as the active rows routed alone
            plan_a, ws_a = experts._static_buffers(len(act), k, dtype, "cuda")
            experts._forward(n[act].contiguous(), idx0[act].contiguous(), wts0[act].contiguous(),
                             out=torch.empty((len(act), H), dtype=dtype, device="cuda"), plan=plan_a, ws=ws_a)
            torch.cuda.synchronize()
            assert _route_meta(ws_a, E) == (counts, n_active)


def test_router_rows_graph_replay_follows_pos():
    from autogptq_b200.moe import moe_router

    dtype, T, k = BF16, 8, TOP_K
    G = _model(dtype).model.layers[0].mlp.gate.weight.detach()
    H, E = G.shape[1], G.shape[0]
    x, x2, w, _ = _router_inputs(T, H, E, dtype, seed=90)
    pos = torch.full((T,), -1, dtype=torch.int64, device="cuda")
    h, n = torch.empty_like(x), torch.empty_like(x)
    idx = torch.empty((T, k), dtype=torch.int32, device="cuda")
    wts = torch.empty((T, k), dtype=torch.float32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        moe_router(x, x2, w, 1e-5, G, k, h=h, n=n, idx=idx, w=wts, pos=pos)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        moe_router(x, x2, w, 1e-5, G, k, h=h, n=n, idx=idx, w=wts, pos=pos)
    for ps in ([0, -1, 3, -1, 5, 6, -1, 9], [-1] * 7 + [2], list(range(8))):
        pos.copy_(torch.tensor(ps))
        g.replay()
        _, _, i_e, w_e, _ = moe_router(x, x2, w, 1e-5, G, k, pos=pos)
        torch.cuda.synchronize()
        assert torch.equal(idx, i_e) and torch.equal(wts, w_e), f"graph replay at pos={ps} differs from an eager call"


# --------------------------------------------------------------------------- BatchDecoder against HF
def _prompts(n, seed, lo=5, step=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 512, (lo + step * i,), generator=g).cuda() for i in range(n)]


def _routing_agrees_row(dec, s, calls, dtype):
    """(agree, unclear) of slot s's routing in every layer of the step just taken against HF's calls for that sequence
    alone, by the rule of ``tests/test_gpu_23_moe_decoder.py::_routing_agrees``: where each gap at the top-k boundary
    and above exceeds twice the largest difference between the two states' exact logits plus two ulps of the largest
    logit, the decoder's indices must equal HF's."""
    agree, unclear = True, False
    dn = P.dt_name(dtype)
    for i, (n_hf, idx_hf) in enumerate(calls):
        m = dec._moe_layers[i]
        G = _np(m["gate"])
        z_hf, z_dec = (_np(n_hf) @ G.T)[0], (_np(m["n2"][s:s + 1]) @ G.T)[0]
        l_hf = P.round_dt(z_hf, dn)
        srt = np.sort(l_hf)[::-1]
        slack = 2 * np.abs(z_hf - z_dec).max() + 2 * P.ulp(np.abs(l_hf).max(), dn)
        clear = (srt[:TOP_K] - srt[1:TOP_K + 1] > slack).all()
        same = m["idx"][s].long().tolist() == idx_hf[0].long().tolist()
        if clear:
            assert same, f"layer {i} slot {s}: decoder routes {m['idx'][s].tolist()}, HF {idx_hf[0].tolist()}"
        unclear |= not clear
        agree &= same
    return agree, unclear


# Least share of the (slot, step) pairs compared: as tests/test_gpu_23_moe_decoder.py's MIN_COMPARED (20 of 32).
MIN_COMPARED_SHARE = 20 / 32


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("max_batch", [3, 8])
def test_mixtral_batch_decoder_matches_hf(max_batch, dtype):
    from transformers import DynamicCache

    from autogptq_b200 import BatchDecoder

    model = _model(dtype)
    steps = 32
    slots = [s for s in range(max_batch) if not (max_batch == 8 and s == 5)]     # max_batch 8: slot 5 stays idle
    prompts = _prompts(len(slots), seed=max_batch)
    g = torch.Generator().manual_seed(3)
    forced = [torch.randint(0, 512, (steps,), generator=g).cuda() for _ in slots]
    dec = BatchDecoder(model, max_batch=max_batch, max_length=128)
    assert dec.moe
    # the Mixtral tolerance of ChainDecoder's test, with test_gpu_24's factor for fp16 at more than 4 rows (the skinny
    # kernel's attention projections round an ulp away more often than HF's batch-1 GEMV)
    factor = 1.5 if max_batch > _lib.GEMV_MAX_M and dtype == F16 else 1.0
    tol = factor * _logit_tol(dtype, L_LAYERS)
    hook = None
    worst, compared, parted, unclear_n, agree, total = 0.0, 0, 0, 0, 0, 0
    try:
        with torch.no_grad():
            caches = []
            for k, s in enumerate(slots):
                caches.append(DynamicCache(config=model.config))
                ref = model(input_ids=prompts[k][None], past_key_values=caches[k], use_cache=True).logits[0, -1]
                assert torch.equal(dec.prefill(s, prompts[k]), ref), "prefill logits differ from HF's"
            hook = _RouterHook(model)
            for t in range(steps):
                ids = torch.zeros(max_batch, dtype=torch.int64, device="cuda")
                for k, s in enumerate(slots):
                    ids[s] = forced[k][t]
                if t == 3:                                   # an eager step and its graph replay are bit-identical
                    p = dec.positions
                    eager = dec.step(ids, use_graph=False).clone()
                    dec.positions = p
                    got = dec.step(ids)
                    assert torch.equal(eager, got), "graph replay differs from the eager step"
                else:
                    got = dec.step(ids)
                if max_batch == 8:                           # the idle slot routes to no expert in any layer
                    assert all((m["idx"][5] == -1).all() for m in dec._moe_layers)
                for k, s in enumerate(slots):
                    hook.calls.clear()
                    r = model(input_ids=forced[k][t].view(1, 1), past_key_values=caches[k],
                              use_cache=True).logits[0, -1].float().cpu().numpy()
                    assert len(hook.calls) == L_LAYERS
                    same_routing, unclear = _routing_agrees_row(dec, s, hook.calls, dtype)
                    unclear_n += int(unclear)
                    if not same_routing:                     # only where a margin is unclear: re-seed the slot
                        parted += 1
                        for i, lay in enumerate(caches[k].layers):
                            n_pos = lay.keys.shape[2]
                            dec.k_cache[i][s, :, :n_pos].copy_(lay.keys[0])
                            dec.v_cache[i][s, :, :n_pos].copy_(lay.values[0])
                        continue
                    o = got[s].float().cpu().numpy()
                    rms = float(np.sqrt(np.mean(r.astype(np.float64) ** 2)))
                    worst = max(worst, float((np.abs(o - r) / (tol * np.abs(r) + tol * rms)).max()))
                    assert_parity(o[None], r[None], rtol=tol, atol_rms=tol,
                                  what=f"mixtral {dtype} max_batch={max_batch} slot {s} step {t}")
                    top2 = np.sort(r)[-2:]
                    if top2[1] - top2[0] > 2 * (tol * abs(top2[1]) + tol * rms):
                        assert r.argmax() == o.argmax(), f"step {t} slot {s}: greedy token differs, margin clear"
                    agree += int(r.argmax() == o.argmax())
                    total += 1
                    compared += 1
            assert dec.positions == [len(prompts[slots.index(s)]) + steps if s in slots else -1
                                     for s in range(max_batch)]
    finally:
        if hook is not None:
            hook.remove()
    print(f"[moe-batch-decoder] {dtype} max_batch={max_batch}: {compared}/{steps * len(slots)} compared, {parted} "
          f"parted ({unclear_n} with an unclear router margin), greedy agreement {agree}/{total}, tol {tol:.3g}, "
          f"largest logit err / tol {worst:.3f}")
    assert compared >= MIN_COMPARED_SHARE * steps * len(slots), f"only {compared} (slot, step) pairs compared"


# --------------------------------------------------------------------------- bit-identities
def _run_slots(model, events, steps=24, B=4):
    """Logits per step [steps][B, vocab] with slots 0..2 prefilled at the start; ``events``: {step: ("admit", slot,
    prompt) or ("release", slot)} applied before that step."""
    from autogptq_b200 import BatchDecoder

    dec = BatchDecoder(model, max_batch=B, max_length=128)
    for s, p in enumerate(_prompts(3, seed=21, lo=4, step=2)):
        dec.prefill(s, p)
    forced = torch.randint(0, 512, (steps, B), generator=torch.Generator().manual_seed(4)).cuda()
    out = []
    with torch.no_grad():
        for t in range(steps):
            ev = events.get(t)
            if ev and ev[0] == "admit":
                dec.prefill(ev[1], ev[2])
            elif ev:
                dec.release(ev[1])
            out.append(dec.step(forced[t]).clone())
    return out


def test_admit_and_release_leave_other_slots_bit_identical():
    model = _model(F16)
    base = _run_slots(model, {})
    ev = _run_slots(model, {8: ("admit", 3, _prompts(1, seed=5, lo=7)[0]), 16: ("release", 1)})
    for t in range(len(base)):
        keep = [0, 2] + ([1] if t < 16 else [])
        assert torch.equal(base[t][keep], ev[t][keep]), f"step {t}: an admit / release changed another slot's logits"


def test_generate_equals_manual_steps():
    from autogptq_b200 import BatchDecoder

    model = _model(BF16)
    prompts = _prompts(5, seed=12, lo=4, step=2)
    dec = BatchDecoder(model, max_batch=3, max_length=128)
    outs = dec.generate(prompts, 10)
    solo = BatchDecoder(model, max_batch=3, max_length=128)
    with torch.no_grad():
        for p, o in zip(prompts, outs):
            toks = [int(solo.prefill(0, p).argmax())]
            while len(toks) < 10:
                ids = torch.zeros(3, dtype=torch.int64, device="cuda")
                ids[0] = toks[-1]
                toks.append(int(solo.step(ids)[0].argmax()))
            solo.release(0)
            assert torch.equal(o[:len(p)], p) and o[len(p):].tolist() == toks


def test_paged_fp8_equals_static_fp8():
    from autogptq_b200 import BatchDecoder

    model = _model(F16)
    st = BatchDecoder(model, 4, 128, kv_cache_dtype=FP8)
    pg = BatchDecoder(model, 4, 128, kv_cache_dtype=FP8, kv_block_size=16)
    prompt = lambda n, seed: torch.randint(0, 512, (n,), generator=torch.Generator().manual_seed(seed))  # noqa: E731
    outs = []
    for d in (st, pg):
        d.set_sampling(2, SamplingParams(temperature=0.9, top_k=40, seed=11))
        log = [d.prefill(0, prompt(21, 1)), d.extend(1, prompt(6, 2)), d.extend(1, prompt(13, 3)),
               d.extend(2, prompt(8, 4))]
        for i in range(16):
            ids = torch.randint(0, 512, (4,), generator=torch.Generator().manual_seed(100 + i)).cuda()
            if i % 2:
                tok, lg = d.step_sample(ids)
                log += [tok.clone(), lg.clone()]
            else:
                log.append(d.step(ids).clone())
            if i == 6:
                d.release(0)
                log.append(d.extend(0, prompt(5, 5)))
        outs.append(log)
    for j, (a, b) in enumerate(zip(*outs)):
        assert torch.equal(a, b), f"output {j}: the paged FP8 cache differs from the static one"


def test_generate_n_samples_equal_seeded_single_runs():
    from autogptq_b200 import BatchDecoder

    pg = BatchDecoder(_model(F16), max_batch=4, max_length=128, kv_block_size=16)
    p = torch.randint(0, 512, (19,), generator=torch.Generator().manual_seed(8))
    sp = SamplingParams(temperature=0.8, top_k=50, seed=77)
    many = pg.generate([p], 16, sampling=sp, n=2)
    assert len(many) == 2
    for i in range(2):
        one = pg.generate([p], 16, sampling=SamplingParams(temperature=0.8, top_k=50, seed=77 + i))
        assert torch.equal(many[i], one[0]), f"copy {i} differs from the n=1 run with its seed"
    assert pg.kv_blocks_free == pg.kv_blocks
