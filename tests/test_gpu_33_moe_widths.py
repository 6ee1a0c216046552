"""The Mixtral decode path at the widths of real MoE checkpoints, against float64.

Grouped experts (``QuantExperts._forward(save=True)``), stage by stage with ``tests/_silu_mul.py``'s bounds (g and u,
h exactly, y_pair, the combine) on the first 256 columns of I and H, a middle tile or the last 256 (the cases take
turns), at the experts of
Mixtral-8x7B, Mixtral-8x22B, Qwen1.5-MoE-A2.7B and Qwen3-30B-A3B; fp16 / bf16, act-order on w1/w3 and w2 or none,
group size 128; every T of the decode kernel (1..8) and T = 9, 64, 300 on the tensor-core GEMM; random routings, one
expert taking every token (T = 1, 4, 7, 64), and rows routed as the masked router routes an idle row (index -1, weight 0), which must come
out exactly zero.  The plan the library builds has ``tests/_moe_layout.py``'s size.

Router (``moe_router(..., pos=)``, the masked entry BatchDecoder uses) at H 4096, 6144 and 16384 (the kernel's limit),
E 8 .. 256, k 2 .. 8, T 1..8, with and without x2: h bit-equal to rnd(x + x2), n one of its chain-norm candidates on
every row; on the active rows the logits, the top-k order (exact ties to the lower index) and the weights within
``tests/_moe_router.py``'s bounds; idle rows index -1, weight 0, logits untouched.

Decoders: a 2-layer Mixtral at 8x7B width (H 4096, I 14336, 32 / 8 heads of 128, E 8, top-2), ChainDecoder at batch 1
and 2 and BatchDecoder at max_batch 8 with three idle slots.  After one eager step every MoE block's buffers are checked
on what the block read: h1 = rnd(o + resid), n2, the router's logits / indices / weights on n2, the experts' stages on
n2 and the routing; then 16 teacher-forced steps against HF.  A Mixtral-shaped model whose experts' decode kernel does
not fit shared memory (H = 16384) is refused by both decoders before any cache is allocated.

The module prints, per stage and dtype, the largest err/bound and mismatch rate over every checked output."""
import functools
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from tests import _chain_norm as N
from tests import _moe_layout as L
from tests import _moe_router as R
from tests import _precision as P
from tests import _silu_mul as S
from tests._util import assert_parity, make_layer

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTS = [F16, BF16]
EPS = 1e-5
_SUMMARY: dict = {}           # (stage, dtype) -> [checked outputs, max err/bound, max mismatch rate]


@pytest.fixture(scope="module", autouse=True)
def _print_summary():
    yield
    print("\n[moe-widths] stage                          dtype     outputs  max err/bound  max mismatch")
    for (stage, dt), (n, worst, rate) in sorted(_SUMMARY.items()):
        print(f"[moe-widths] {stage:<30} {dt:<9} {n:>7}  {worst:13.3f}  {rate:12.4f}")


def _record(stage, dtype, worst=0.0, rate=0.0):
    e = _SUMMARY.setdefault((stage, P.dt_name(dtype)), [0, 0.0, 0.0])
    e[0] += 1
    e[1] = max(e[1], worst)
    e[2] = max(e[2], rate)


def _record_moe(prefix, dtype, res):
    for stage, r in res.items():
        _record(f"{prefix} {stage}", dtype, r.worst, r.rate)


def _np(t):
    return t.double().cpu().numpy()


def _bits(t):
    return t.view(torch.int16) if t.dtype in DTS else t


def _cols(N_):
    """First and last 256 columns and one 32-column tile in the middle."""
    mid = N_ // 2 // 32 * 32
    return [(0, 256), (mid, mid + 32), (N_ - 256, N_)]


# --------------------------------------------------------------------------- grouped experts
def _expert_dicts(E, H, I, dtype, act, seed):
    """``tests/_silu_mul.realistic_experts(E, H, I, 128, dtype, seed, act, act)``, generated one expert per thread
    (expert e of that call is the one-expert call with seed + 3e) and not kept in its cache: one dtype's experts at
    8x22B width are about 1.2 GB of packed codes.  The codes depend on the dtype (its rounded scales), so each dtype has
    its own set."""
    gen = S.realistic_experts.__wrapped__
    dt = P.dt_name(dtype)
    with ThreadPoolExecutor(8) as pool:
        return tuple(pool.map(lambda e: gen(1, H, I, 128, dt, seed=seed + 3 * e, act13=act, act2=act)[0], range(E)))


@functools.lru_cache(maxsize=1)
def _experts(E, H, I, dtype, act, seed=0):
    """(QuantExperts, host dicts); one set at a time lives on the GPU."""
    from autogptq_b200 import QuantExperts

    ex = _expert_dicts(E, H, I, dtype, act, seed)
    mods = {n: [make_layer(e[n], dtype=dtype) for e in ex] for n in ("w1", "w3", "w2")}
    return QuantExperts(mods["w1"], mods["w3"], mods["w2"]), ex


def _unpack(saved, T, k, I, H, dtype):
    """g, u [T·k, I] and y_pair [T·k, H] of ``agb200_moe_forward_saving``'s buffer."""
    Pn = T * k
    gu = -(-Pn * I * 2 // 256) * 256
    part = lambda off, n: saved[off:off + Pn * n * 2].view(dtype).view(Pn, n)   # noqa: E731
    return part(0, I), part(gu, I), part(2 * gu, H)


def _routing(T, k, E, kind, rng):
    """[T, k] int32 ids and fp32 weights summing to 1: ``random`` (k distinct experts per token), ``one_expert`` (one
    expert in every token's first slot) or ``idle`` (random, and every row r with r % 3 == 1 routed as the masked
    router routes an idle row: index -1, weight 0)."""
    idx = np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int32)
    if kind == "one_expert":
        e = int(rng.integers(E))
        for t in range(T):
            idx[t] = [e] + [int(j) for j in rng.permutation(E) if j != e][:k - 1]
    w = rng.random((T, k)).astype(np.float32) + 0.05
    w /= w.sum(axis=1, keepdims=True)
    idle = np.arange(T) % 3 == 1 if kind == "idle" else np.zeros(T, bool)
    idx[idle], w[idle] = -1, 0.0
    return idx, w, idle


def _moe_forward_check(qe, ex, x, idx, w, dtype, what, prefix, part):
    """The saving forward on x [T, H] (host), then every stage on part ``part`` (0 first, 1 middle, 2 last) of
    ``_cols`` of I and H (the float64 reference of one part of one case takes seconds at these widths, so the cases
    take turns); returns out [T, H] (host)."""
    T, k = idx.shape
    H, I = qe.hidden_size, qe.intermediate_size
    xt = torch.from_numpy(np.asarray(x, np.float32)).to(dtype).cuda()
    it, wt = torch.from_numpy(idx).cuda(), torch.from_numpy(w).cuda()
    with torch.no_grad():
        out, saved = qe._forward(xt, it, wt, save=True)
        plain = qe._forward(xt, it, wt)[0]
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(plain)), f"{what}: the plain forward differs from the saving forward"
    gs, us, ys = (_np(t) for t in _unpack(saved, T, k, I, H, dtype))
    path = "decode_mma" if T <= _lib.MOE_DECODE_MAX_T else "gemm"
    o = _np(out)
    ci, chh = _cols(I)[part % 3], _cols(H)[part % 3]
    res = S.check_moe(ex, x, idx, w, dtype, path, path, gs, us, ys, o, cols_i=ci, cols_h=chh,
                      what=f"{what} cols I {ci} H {chh}")
    _record_moe(f"{prefix} {'decode' if path == 'decode_mma' else 'gemm'}", dtype, res)
    return o


# (width, dtype, act-order): each width in both dtypes, act-order on one of them, so that every (dtype, act-order) pair
# runs at two widths (a Mixtral set is about 2.4 GB on the GPU with its tensor-core copies)
EXPERT_CASES = [("mixtral_8x7b", F16, True), ("mixtral_8x7b", BF16, False),
                ("mixtral_8x22b", F16, False), ("mixtral_8x22b", BF16, True),
                ("qwen1.5_moe_a2.7b", F16, False), ("qwen1.5_moe_a2.7b", BF16, True),
                ("qwen3_30b_a3b", F16, True), ("qwen3_30b_a3b", BF16, False)]
DECODE_KINDS = ["random", "one_expert", "idle"]


@pytest.mark.parametrize("case", range(len(EXPERT_CASES)),
                         ids=[f"{n}-{P.dt_name(d)}-{'act' if a else 'plain'}" for n, d, a in EXPERT_CASES])
def test_experts_at_real_widths(case):
    name, dtype, act = EXPERT_CASES[case]
    E, k, H, I = L.WIDTHS[name]
    qe, ex = _experts(E, H, I, dtype, act)
    dt = P.dt_name(dtype)
    acts = P.acts_for(dtype)
    rng = np.random.default_rng(case)
    cases = [(T, DECODE_KINDS[T % 3]) for T in range(1, 9)] + [(9, "random"), (64, "one_expert"), (300, "random")]
    for c, (T, kind) in enumerate(cases):
        idx, w, idle = _routing(T, k, E, kind, rng)
        akind = acts[c % len(acts)]
        x = P.activations(akind, T, H, dtype, seed=1000 + c)
        what = f"{name} {dt} act={act} T={T} {kind} {akind}"
        out = _moe_forward_check(qe, ex, x, idx, w, dtype, what, "experts", part=c)
        assert (out[idle] == 0).all(), f"{what}: an idle row's output is not exactly zero"
    # the plan the library built: the decode layout is accepted and its buffer has the restated size
    assert L.decode_layout(H, I) is not None
    assert {p.plan.numel() for p in qe._plans.values()} == {L.plan_bytes(E, I)}


# --------------------------------------------------------------------------- router
def _router_case(T, H, E, dtype, seed, kind):
    """x, x2 [T, H], norm weight [H] and router weight [E, H] (float64 host arrays of dtype values).  Router rows 1 and
    E - 1 repeat rows 0 and 2, and row 0 is scaled up, so that the exact tie of experts 0 and 1 usually falls inside
    the top-k (``tests/test_gpu_23_moe_decoder.py``'s inputs)."""
    dn = P.dt_name(dtype)
    rng = np.random.default_rng(seed)
    x = P.activations(kind, T, H, dtype, seed=seed).astype(np.float64)
    x2 = P.activations("gauss", T, H, dtype, seed=seed + 1).astype(np.float64)
    w = P.round_dt(rng.uniform(0.5, 1.5, H), dn)
    G = rng.standard_normal((E, H)) * (2.0 / np.sqrt(H))
    G[0] *= 2.0
    G[1] = G[0]
    G[E - 1] = G[2]
    return x, x2, w, P.round_dt(G, dn)


def _check_router_rows(h, n, idx, wts, logits, x, x2, w, G, k, pos, dtype, what, prefix="router", eps=EPS):
    """Every row's h and n; the active rows' logits, top-k and weights on the kernel's own n; idle rows -1 / 0 with
    their logits row left NaN (``logits`` may be None: then h, n, idx, w only)."""
    dn = P.dt_name(dtype)
    if x2 is not None:
        assert np.array_equal(h, N.add_rounded(x, x2, dn)), f"{what}: h != rnd(x + x2)"
        hh = h
    else:
        hh = x
    _record(f"{prefix} n neighbour", dtype, rate=N.check_n(n, hh, w, eps, dn, what))
    act, idle = pos >= 0, pos < 0
    assert (idx[idle] == -1).all() and (wts[idle] == 0).all(), f"{what}: an idle row routes to an expert"
    if logits is None:
        return
    assert np.isnan(logits[idle]).all(), f"{what}: an idle row wrote logits"
    if act.any():
        la = logits[act]
        _record(f"{prefix} logits", dtype, rate=R.check_logits(la, n[act], G, dn, what))
        R.check_topk(idx[act], la, k, what)
        _record(f"{prefix} weights", dtype, R.check_weights(wts[act], idx[act], la, what))


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("H", [4096, 6144, 16384])
@pytest.mark.parametrize("k", [2, 4, 8])
@pytest.mark.parametrize("E", [8, 60, 128, 256])
def test_router_rows_at_real_widths(E, k, H, dtype):
    from autogptq_b200.moe import moe_router

    dn = P.dt_name(dtype)
    rng = np.random.default_rng(E * 100 + k * 10 + H)
    for T in range(1, 9):
        for with_x2 in (False, True):
            x, x2, w, G = _router_case(T, H, E, dtype, seed=E + 7 * k + 31 * T + with_x2,
                                       kind="offset" if T % 2 else "gauss")
            if T == 1:
                pos = np.array([5 if with_x2 else -1])
            else:
                pos = rng.integers(0, 4000, T)
                pos[rng.random(T) < 0.4] = -1
                pos[0], pos[-1] = 3, -1                     # at least one active and one idle row
            cu = lambda a: torch.from_numpy(np.asarray(a)).to(dtype).cuda()   # noqa: E731
            logits = torch.full((T, E), float("nan"), dtype=dtype, device="cuda")
            h, n, idx, wts, _ = moe_router(cu(x), cu(x2) if with_x2 else None, cu(w), EPS, cu(G), k, logits=logits,
                                           pos=torch.from_numpy(pos).cuda())
            torch.cuda.synchronize()
            what = f"router E={E} k={k} H={H} T={T} x2={with_x2} {dn} pos={pos.tolist()}"
            assert (h is None) == (not with_x2)
            _check_router_rows(None if h is None else _np(h), _np(n), idx.cpu().numpy(), wts.cpu().numpy(),
                               _np(logits), x, x2 if with_x2 else None, w, G, k, pos, dtype, what)


def test_router_refuses_more_than_256_experts_and_top_9():
    from autogptq_b200.moe import moe_router

    x = torch.zeros((2, 4096), dtype=F16, device="cuda")
    w = torch.ones(4096, dtype=F16, device="cuda")
    with pytest.raises(NotImplementedError, match="257 experts"):
        moe_router(x, None, w, EPS, torch.zeros((257, 4096), dtype=F16, device="cuda"), 2)
    with pytest.raises(NotImplementedError, match="top_k 9"):
        moe_router(x, None, w, EPS, torch.zeros((16, 4096), dtype=F16, device="cuda"), 9)


# --------------------------------------------------------------------------- decoders
MX = dict(H=4096, I=14336, heads=32, kv=8, hd=128, E=8, k=2, vocab=512)


def _mixtral(dtype, H, I, heads, kv, E, k, layers, vocab=512, seed=1):
    """A random MixtralForCausalLM built on the GPU in ``dtype`` (the dense experts never exist in fp32 or on the
    host), with random RMSNorm weights and routers as in ``tests/test_gpu_23_moe_decoder.py``."""
    from transformers import MixtralConfig, MixtralForCausalLM

    cfg = MixtralConfig(hidden_size=H, intermediate_size=I, num_attention_heads=heads, num_key_value_heads=kv,
                        head_dim=128, num_hidden_layers=layers, num_local_experts=E, num_experts_per_tok=k,
                        vocab_size=vocab, max_position_embeddings=512, rms_norm_eps=EPS)
    torch.manual_seed(seed)
    with torch.device("cuda"):
        m = MixtralForCausalLM._from_config(cfg, dtype=dtype)
    with torch.no_grad():
        for mod in m.modules():
            if type(mod).__name__.endswith("RMSNorm"):
                mod.weight.uniform_(0.5, 1.5)
            if type(mod).__name__ == "MixtralTopKRouter":
                mod.weight.normal_(0.0, 2.0 / np.sqrt(H))
    m = m.eval()
    m.config._attn_implementation = "sdpa"
    return m


def _quant_attention(model, dtype):
    dt = P.dt_name(dtype)
    for i, layer in enumerate(model.model.layers):
        for j, name in enumerate(("q_proj", "k_proj", "v_proj", "o_proj")):
            lin = getattr(layer.self_attn, name)
            d = P.realistic_layer(lin.in_features, lin.out_features, 128, dt, seed=100 * i + j, wrap_groups=False)
            setattr(layer.self_attn, name, make_layer(d, dtype=dtype))


@functools.lru_cache(maxsize=1)
def _mixtral_8x7b(dtype):
    """The 2-layer model at 8x7B width and its experts' host dicts per layer (layer i: seed 1000·i)."""
    c = MX
    m = _mixtral(dtype, c["H"], c["I"], c["heads"], c["kv"], c["E"], c["k"], layers=2)
    _quant_attention(m, dtype)
    dicts = []
    for i, layer in enumerate(m.model.layers):
        ex = _expert_dicts(c["E"], c["H"], c["I"], dtype, False, seed=1000 * i)
        mods = {n: [make_layer(e[n], dtype=dtype) for e in ex] for n in ("w1", "w3", "w2")}
        from autogptq_b200 import QuantExperts

        layer.mlp.experts = QuantExperts(mods["w1"], mods["w3"], mods["w2"])
        dicts.append(ex)
    torch.cuda.empty_cache()
    return m, dicts


class _OHook:
    """Records each layer's o_proj output (BatchDecoder's o is a temporary of the step)."""

    def __init__(self, model):
        self.o = {}
        self.handles = [layer.self_attn.o_proj.register_forward_hook(self._hook(i))
                        for i, layer in enumerate(model.model.layers)]

    def _hook(self, i):
        def f(mod, inp, out):
            self.o[i] = out.detach().clone()
        return f

    def remove(self):
        for h in self.handles:
            h.remove()


def _check_moe_block(model, dicts, i, m, o, resid, pos, dtype, what):
    """Block i's MoE buffers after an eager step: h1, n2, the router's outputs (re-run with a logits buffer on the same
    inputs, bit-equal to the step's) and the experts' stages (a saving forward on n2, idx, w, bit-equal to the step's
    output).  ``pos``: the positions the step read (None: every row active).  Returns the host h1 and out."""
    from autogptq_b200.moe import moe_router

    layer = model.model.layers[i]
    ln2 = layer.post_attention_layernorm
    G = m["gate"]
    B, E, k = o.shape[0], G.shape[0], m["k"]
    logits = torch.full((B, E), float("nan"), dtype=dtype, device="cuda")
    pos_t = None if pos is None else torch.tensor(pos, dtype=torch.int64, device="cuda")
    h, n, idx, wts, _ = moe_router(o, resid, m["w2"], m["eps2"], G, k, logits=logits, pos=pos_t)
    torch.cuda.synchronize()
    for name, a, b in (("h1", h, m["h1"]), ("n2", n, m["n2"]), ("idx", idx, m["idx"]), ("w", wts, m["w"])):
        assert torch.equal(_bits(a), _bits(b)), f"{what}: the step's {name} differs from the router's on its inputs"
    pos_np = np.zeros(B, np.int64) if pos is None else np.asarray(pos)
    h1, n2 = _np(m["h1"]), _np(m["n2"])
    _check_router_rows(h1, n2, m["idx"].cpu().numpy(), m["w"].cpu().numpy(), _np(logits), _np(o), _np(resid),
                       _np(ln2.weight), _np(G), k, pos_np, dtype, what, prefix="decoder router", eps=m["eps2"])
    qe = m["experts"]
    ex = dicts[i]
    out = _moe_forward_check(qe, ex, n2, m["idx"].cpu().numpy(), m["w"].cpu().numpy(), dtype, what, "decoder experts",
                             part=i)
    assert np.array_equal(out, _np(m["out"])), f"{what}: the step's expert output differs from the saving forward's"
    assert (out[pos_np < 0] == 0).all(), f"{what}: an idle row's expert output is not exactly zero"
    return h1, out


def _hf_steps(model, dtype, prompts, forced):
    """HF's logits of each sequence alone: [sequence][0: prefill, t + 1: forced step t] and its router calls."""
    from transformers import DynamicCache

    from tests.test_gpu_23_moe_decoder import _RouterHook

    out, calls = [], []
    hook = _RouterHook(model)
    try:
        for p, f in zip(prompts, forced):
            cache = DynamicCache(config=model.config)
            hook.calls.clear()
            seq = [model(input_ids=p[None], past_key_values=cache, use_cache=True).logits[0, -1]]
            cl = [[]]
            for t in range(f.shape[0]):
                hook.calls.clear()
                seq.append(model(input_ids=f[t].view(1, 1), past_key_values=cache, use_cache=True).logits[0, -1])
                cl.append(list(hook.calls))
            out.append(seq)
            calls.append(cl)
    finally:
        hook.remove()
    return out, calls


def _compare_step(dec, rows, got, refs, calls, t, tol, dtype, what, agrees):
    """Step t of each row against HF's sequence alone; a row whose routing parts from HF's where a router margin is
    unclear is not compared from there on (``tests/test_gpu_23_moe_decoder.py``'s rule).  Returns rows compared."""
    n = 0
    for r, s in enumerate(rows):
        if s in agrees["parted"]:
            continue
        same, _ = agrees["fn"](dec, s, calls[r][t + 1], dtype)
        if not same:
            agrees["parted"].add(s)
            continue
        ref = refs[r][t + 1].float().cpu().numpy()
        assert_parity(got[s].float().cpu().numpy()[None], ref[None], rtol=tol, atol_rms=tol,
                      what=f"{what} row {s} step {t}")
        n += 1
    return n


DECODER_CASES = [(dt, d) for dt in DTS for d in ("chain_b1", "chain_b2", "batch_8")]


@pytest.mark.parametrize("dtype,decoder", DECODER_CASES, ids=[f"{P.dt_name(dt)}-{d}" for dt, d in DECODER_CASES])
def test_decoders_at_mixtral_8x7b_width(dtype, decoder):
    from autogptq_b200 import BatchDecoder
    from autogptq_b200.decoder import ChainDecoder
    from tests.test_gpu_23_moe_decoder import _logit_tol
    from tests.test_gpu_32_moe_batch_decoder import _routing_agrees_row

    model, dicts = _mixtral_8x7b(dtype)
    dt = P.dt_name(dtype)
    steps = 16
    g = torch.Generator().manual_seed(17)
    tol = _logit_tol(dtype, 2, MX["k"])
    if decoder == "batch_8":
        B, rows = 8, [0, 2, 3, 5, 6]                          # slots 1, 4 and 7 stay idle
        dec = BatchDecoder(model, max_batch=B, max_length=64)
        tol *= 1.5 if dtype == F16 else 1.0                   # test_gpu_24's fp16 allowance at more than 4 rows
    else:
        B = int(decoder[-1])
        rows = list(range(B))
        dec = ChainDecoder(model, batch=B, max_length=64, fused_attention=True)
    assert dec.moe
    # BatchDecoder: a prompt length per slot; ChainDecoder: the rows in lockstep
    prompts = [torch.randint(0, 512, (5 + 3 * r if decoder == "batch_8" else 8,), generator=g).cuda()
               for r in range(len(rows))]
    forced = [torch.randint(0, 512, (steps,), generator=g).cuda() for _ in rows]
    what = f"{decoder} {dt}"
    with torch.no_grad():
        refs, calls = _hf_steps(model, dtype, prompts, forced)
        if decoder == "batch_8":
            for r, s in enumerate(rows):
                assert torch.equal(dec.prefill(s, prompts[r]), refs[r][0]), f"{what}: prefill differs from HF's"
        else:
            got = dec.prefill(torch.stack(prompts))
            for r in rows:
                assert_parity(got[r].float().cpu().numpy()[None], refs[r][0].float().cpu().numpy()[None], rtol=tol,
                              atol_rms=tol, what=f"{what} prefill row {r}")

        def ids_at(t):
            ids = torch.zeros(B, dtype=torch.int64, device="cuda")
            for r, s in enumerate(rows):
                ids[s] = forced[r][t]
            return ids

        # one eager step, then every MoE block's buffers
        if decoder == "batch_8":
            pos = dec.positions
            hook = _OHook(model)
            try:
                got = dec.step(ids_at(0), use_graph=False)
            finally:
                hook.remove()
            resid = dec._x
            for i in range(len(model.model.layers)):
                h1, out = _check_moe_block(model, dicts, i, dec._moe_layers[i], hook.o[i], resid, pos, dtype,
                                           f"{what} block {i}")
                resid = torch.from_numpy(N.add_rounded(out, h1, dt)).to(dtype).cuda()
        else:
            got = dec.step(ids_at(0), use_graph=False)
            for i, m in enumerate(dec._moe_layers):
                _check_moe_block(model, dicts, i, m, m["o"], m["resid"], None, dtype, f"{what} block {i}")
        agrees = dict(fn=_routing_agrees_row, parted=set())       # both decoders keep n2 and idx per MoE layer
        compared = _compare_step(dec, rows, got, refs, calls, 0, tol, dtype, what, agrees)
        for t in range(1, steps):
            got = dec.step(ids_at(t))
            compared += _compare_step(dec, rows, got, refs, calls, t, tol, dtype, what, agrees)
    print(f"[moe-widths] {what}: {compared}/{steps * len(rows)} (row, step) pairs compared, rows parted at an unclear "
          f"router margin: {sorted(agrees['parted'])}, tol {tol:.3g}")
    assert compared >= steps * len(rows) // 2, f"{what}: only {compared} (row, step) pairs compared"


# --------------------------------------------------------------------------- refusal before allocation
def _refusing_mixtral(dtype):
    """One layer, H = 16384 (the router's limit), E 2, I 128, 2 / 1 heads of 128: the router takes it, the experts'
    decode kernel cannot hold 8 rows of x (``tests/_moe_layout.py``)."""
    from autogptq_b200 import QuantExperts

    H = L.REFUSED_H
    m = _mixtral(dtype, H, 128, 2, 1, 2, 2, layers=1)
    _quant_attention(m, dtype)
    dt = P.dt_name(dtype)
    ex = [S.realistic_experts.__wrapped__(1, H, 128, 128, dt, seed=3 * e)[0] for e in range(2)]
    m.model.layers[0].mlp.experts = QuantExperts(*([make_layer(e[n], dtype=dtype) for e in ex]
                                                   for n in ("w1", "w3", "w2")))
    return m


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("who", ["ChainDecoder", "BatchDecoder"])
def test_decoders_refuse_experts_before_allocating(who, dtype, monkeypatch):
    from autogptq_b200 import BatchDecoder
    from autogptq_b200.decoder import ChainDecoder

    assert L.decode_layout(L.REFUSED_H, 128) is None
    model = _refusing_mixtral(dtype)
    cls = ChainDecoder if who == "ChainDecoder" else BatchDecoder

    def no_allocate(self, rows):
        raise AssertionError(f"{who} allocated its caches before refusing experts that cannot run")

    monkeypatch.setattr(cls, "_allocate", no_allocate)
    with pytest.raises(NotImplementedError, match=rf"^{who}: model\.layers\.0\.mlp\.experts .*needs \d+ B of shared "
                                                  r"memory"):
        cls(model, **(dict(batch=1) if who == "ChainDecoder" else dict(max_batch=8)), max_length=64)
