"""The decode chain and the decoders at the widths of real GPTQ checkpoints, against float64.

Stage level: one decoder block chained as ChainDecoder chains it, starting from the block's input norm,

    x ─[rmsnorm]→ q|k|v;  q → o;  o, x ─[add_rmsnorm]→ gate|up (+h1);  gate, up ─[silu_mul]→ down;
    down, h1 ─[add_rmsnorm]→ next q|k|v (+resid)

at Qwen2-1.5B (H = 1.5 chunks of 1024 k, I = 8.75), Qwen2-7B (ragged norm prepass and publish, I = 18.5 chunks),
Mistral-7B, Llama-2-13B (I = 13.5) and the 70B widths (I = 28 and 28.875 chunks, a 4-slot ring); fp16 / bf16, M = 1, 2,
every projection act-order or none.  Each combination builds and passes, or is refused with ENOSUP; one that builds has
the ring depth and shared memory of ``tests/_chain_layout.py``.  Every y is held to the chain's DESIGN §3.12 bound on
the input the stage read (``tests/_precision.py``; normalised inputs from the ``tests/_chain_norm.py`` candidates, the
down projection's from the ``tests/_silu_mul.py`` ones) on its first and last 256 columns and a middle tile, h1 and
resid are bit-equal to rnd(a + b).  Also: one stage at K = 32768 (32 chunks, the most a stage takes), a down stage with
one group over K = 28672, group size 1024.

Model level: 2-layer random models at Mistral-7B, Qwen2-7B and Llama-2-13B widths.  ChainDecoder refuses the blocks that
do not fit before it allocates its caches; where it fits, every block's buffers after an eager step pass the same stage
checks with references built from the HF model's norms and the quantised layer dicts, then 16 teacher-forced steps
against HF.  BatchDecoder decodes 8 rows of the Qwen2-7B-width model (G = 7) against HF.

The module prints, per width and dtype, the largest err/bound and mismatch rate over every checked output."""
import functools

import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from tests import _chain_layout as CL
from tests import _chain_norm as N
from tests import _precision as P
from tests import _silu_mul as S
from tests._util import assert_parity, make_layer

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTS = [F16, BF16]
EPS = 1e-5
HD = 128
# name -> (H, I, heads, kv heads, q/k/v bias)
SHAPES = {
    "qwen2_1.5b": (1536, 8960, 12, 2, True),
    "qwen2_7b": (3584, 18944, 28, 4, True),
    "mistral_7b": (4096, 14336, 32, 8, False),
    "llama2_13b": (5120, 13824, 40, 40, False),
    "llama_70b": (8192, 28672, 64, 8, False),
    "qwen2_72b": (8192, 29568, 64, 8, True),
}
_SUMMARY: dict = {}           # (width, dtype) -> [checked outputs, max err/bound, max mismatch rate]


@pytest.fixture(scope="module", autouse=True)
def _print_summary():
    yield
    print("\n[chain-widths] width            dtype     outputs  max err/bound  max mismatch")
    for (name, dt), (n, worst, rate) in sorted(_SUMMARY.items()):
        print(f"[chain-widths] {name:<16} {dt:<9} {n:>7}  {worst:13.3f}  {rate:12.4f}")


def _record(name, dtype, r: P.Result):
    e = _SUMMARY.setdefault((name, P.dt_name(dtype)), [0, 0.0, 0.0])
    e[0] += 1
    e[1] = max(e[1], r.worst)
    e[2] = max(e[2], r.rate)


def _np(t):
    return t.double().cpu().numpy()


def _cols(N_):
    """First and last 256 columns and one 32-column tile in the middle (the whole layer when that covers it)."""
    if N_ <= 512:
        return [(0, N_)]
    mid = N_ // 2 // 32 * 32
    return [(0, 256), (mid, mid + 32), (N_ - 256, N_)]


# --------------------------------------------------------------------------- layers
_BLOCKS: dict = {}


def _block(name, dt, act, seed=0):
    """The seven layer dicts of one block (q, k, v share g_idx, as gate and up do).  Generated once per module; a
    70B-width block is about 0.45 GB packed, so only one of those is kept."""
    key = (name, dt, act, seed)
    if key not in _BLOCKS:
        H, I, nh, nkv, bias = SHAPES[name]
        if H == 8192:
            for k in [k for k in _BLOCKS if SHAPES[k[0]][0] == 8192]:
                del _BLOCKS[k]
        s = 1000 * seed
        q = P.wide_layer(H, nh * HD, 128, dt, seed=s + 1, act_order=act, bias=bias)
        gate = P.wide_layer(H, I, 128, dt, seed=s + 401, act_order=act)
        _BLOCKS[key] = dict(
            q=q, k=P.wide_layer(H, nkv * HD, 128, dt, seed=s + 101, bias=bias, g_idx=q["g_idx"]),
            v=P.wide_layer(H, nkv * HD, 128, dt, seed=s + 201, bias=bias, g_idx=q["g_idx"]),
            o=P.wide_layer(nh * HD, H, 128, dt, seed=s + 301, act_order=act),
            gate=gate, up=P.wide_layer(H, I, 128, dt, seed=s + 501, g_idx=gate["g_idx"]),
            down=P.wide_layer(I, H, 128, dt, seed=s + 601, act_order=act))
    return _BLOCKS[key]


def _blank_layer(K, N_, act, group_size=128):
    """A layer whose weights do not matter (a chain that is refused before it runs): zero codes, unit scales."""
    G = K // group_size
    g_idx = np.arange(K, dtype=np.int32) // group_size
    if act:
        g_idx = g_idx[np.random.default_rng(K).permutation(K)]
    return dict(qweight=np.zeros((K // 8, N_), np.int32), qzeros=np.zeros((G, N_ // 8), np.int32),
                scales=np.ones((G, N_), np.float32), g_idx=g_idx, bias=None, K=K, N=N_, group_size=group_size)


def _blank_block(name, act):
    H, I, nh, nkv, _ = SHAPES[name]
    q = _blank_layer(H, nh * HD, act)
    kv = dict(q, N=nkv * HD, qweight=q["qweight"][:, :nkv * HD], qzeros=q["qzeros"][:, :nkv * HD // 8],
              scales=q["scales"][:, :nkv * HD])
    g = _blank_layer(H, I, act)
    return dict(q=q, k=kv, v=kv, o=_blank_layer(nh * HD, H, act), gate=g, up=g, down=_blank_layer(I, H, act))


def _norm_weight(K, dtype, seed):
    rng = np.random.default_rng(seed)
    return P.round_dt(rng.uniform(0.05, 1.0, size=K) * np.where(rng.random(K) < 0.3, -1, 1), P.dt_name(dtype))


# --------------------------------------------------------------------------- the stage checks
def _check_cols(name, tag, y, d, ref_of, dtype):
    """y on ``_cols`` against the references ``ref_of(cols)``, as one set of columns: the mismatch rate is a rate over
    the layer's checked outputs, not over one 32-column tile."""
    cols = _cols(d["N"])
    refs = [ref_of(c) for c in cols]
    cat = lambda f: np.concatenate([getattr(r, f) for r in refs], axis=1)   # noqa: E731
    ref = P.Ref(cat("ystar"), cat("A"), cat("F"), refs[0].n_terms, refs[0].bad_rows, cat("A0"))
    ys = np.concatenate([y[:, c0:c1] for c0, c1 in cols], axis=1)
    _record(name, dtype, P.check(ys, ref, P.PATHS["chain"], dtype, what=f"{tag} cols {cols}"))


def _check_normed(name, tag, y, d, h, w, eps, dtype):
    _check_cols(name, tag, y, d, lambda c: N.reference_y(d, h, w, eps, dtype, c), dtype)


def _check_plain(name, tag, y, d, x, dtype):
    _check_cols(name, tag, y, d, lambda c: P.reference(d, x, P.PATHS["chain"], dtype, cols=c), dtype)


def _check_down(name, tag, y, d, g, u, dtype):
    _check_cols(name, tag, y, d, lambda c: S.reference_down(d, g, u, P.PATHS["chain"], dtype, cols=c), dtype)


def _check_sum(h, a, b, dtype, what):
    assert np.array_equal(h, N.add_rounded(a, b, dtype)), f"{what} != rnd(a + b) of what the stage read"


def _check_block(name, ds, bufs, w_in, w_post, eps_in, eps_post, dtype, tag, w_next=None, eps_next=None):
    """One block's outputs (host float64 arrays in ``bufs``: the residual h_in, whose norm q|k|v read, q, k, v, o's
    input a, o, h1, gate, up, down, and with ``w_next`` the next block's q2, k2, v2 (layer dicts ``bufs["next"]``) and
    resid) on the inputs the stages read."""
    b = bufs
    for n in ("q", "k", "v"):
        _check_normed(name, f"{tag} {n}", b[n], ds[n], b["h_in"], w_in, eps_in, dtype)
    _check_plain(name, f"{tag} o", b["o"], ds["o"], b["a"], dtype)
    _check_sum(b["h1"], b["o"], b["h_in"], dtype, f"{tag} h1")
    for n in ("gate", "up"):
        _check_normed(name, f"{tag} {n}", b[n], ds[n], b["h1"], w_post, eps_post, dtype)
    _check_down(name, f"{tag} down", b["down"], ds["down"], b["gate"], b["up"], dtype)
    if w_next is not None:
        _check_sum(b["resid"], b["down"], b["h1"], dtype, f"{tag} resid")
        dn = b["next"]
        for n in ("q", "k", "v"):
            _check_normed(name, f"{tag} next {n}", b[f"{n}2"], dn[n], b["resid"], w_next, eps_next, dtype)


def _assert_layout(ch, M, stages):
    want = CL.layout(M, stages)
    info = ch.info()
    assert (info["ring_slots"], info["smem_bytes"]) == want, (info, want)
    return info


def _assert_refused(ch):
    with pytest.raises(_lib.B200KernelError) as e:
        ch.build()
    assert e.value.code == _lib.ENOSUP, str(e.value)


# --------------------------------------------------------------------------- stage level
@pytest.mark.parametrize("M", [1, 2])
@pytest.mark.parametrize("act", [False, True], ids=["plain", "act_order"])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("name", list(SHAPES))
def test_block_chain(name, dtype, act, M):
    from autogptq_b200.chain import DecodeChain

    H, I, nh, nkv, _ = SHAPES[name]
    dt = P.dt_name(dtype)
    stages = [(H, True), (nh * HD, act), (H, True), (I, act), (H, True)]
    want = CL.layout(M, stages)
    assert want == CL.layout(M, CL.block_stages(H, I, act)), "the stage-level chain has ChainDecoder's layout"
    ds = _block(name, dt, act) if want is not None else _blank_block(name, act)
    Lq, Lk, Lv, Lo, Lg, Lu, Ld = (make_layer(ds[n], dtype=dtype) for n in ("q", "k", "v", "o", "gate", "up", "down"))
    wn = [_norm_weight(H, dtype, s) for s in (1, 2, 3)]
    wt = [torch.from_numpy(w).to(dtype).cuda() for w in wn]
    ch = DecodeChain(M=M, dtype=dtype)
    x = ch.input(H)
    q, k, v = ch.stage([Lq, Lk, Lv], x, x_mode="rmsnorm", norm_weight=wt[0], norm_eps=EPS)
    (o,) = ch.stage([Lo], q)
    gate, up, h1 = ch.stage([Lg, Lu], o, x2=x, x_mode="add_rmsnorm", norm_weight=wt[1], norm_eps=EPS)
    (down,) = ch.stage([Ld], gate, x2=up, x_mode="silu_mul")
    q2, k2, v2, resid = ch.stage([Lq, Lk, Lv], down, x2=h1, x_mode="add_rmsnorm", norm_weight=wt[2], norm_eps=EPS)
    if want is None:
        _assert_refused(ch)
        print(f"[chain-widths] {name} {dt} M={M} act={act}: refused (ENOSUP)")
        return
    ch.build()
    info = _assert_layout(ch, M, stages)
    print(f"[chain-widths] {name} {dt} M={M} act={act}: {info['ring_slots']} slots, {info['smem_bytes']} B")
    for launch, kind in enumerate(("offset", "massive", "row_scale")):
        x.copy_(torch.from_numpy(P.activations(kind, M, H, dtype, seed=50 + launch)).to(dtype).cuda())
        ch.run()
        torch.cuda.synchronize()
        b = {n: _np(t) for n, t in dict(h_in=x, q=q, k=k, v=v, o=o, h1=h1, gate=gate, up=up, down=down, q2=q2, k2=k2,
                                          v2=v2, resid=resid).items()}
        b["a"], b["next"] = b["q"], ds
        _check_block(name, ds, b, wn[0], wn[1], EPS, EPS, dtype, f"{name} {dt} M={M} act={act} {kind}",
                     w_next=wn[2], eps_next=EPS)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_widest_stages(dtype):
    """One stage at K = 32768 (32 chunks: every bit of the per-warp chunk mask), a down-shaped stage whose one group
    covers K = 28672 (bpg_log2 = 31) and an act-order layer with group size 1024, at M = 1 and 2 (K = 32768 is refused
    at M = 2: its digits leave no room for 3 slots)."""
    from autogptq_b200.chain import DecodeChain

    dt = P.dt_name(dtype)
    cases = [("K=32768", P.wide_layer(32768, 512, 128, dt, seed=71, bias=True), False),
             ("K=28672 one group", P.wide_layer(28672, 1024, -1, dt, seed=72), False),
             ("g=1024 act-order", P.wide_layer(14336, 1024, 1024, dt, seed=73, act_order=True), True)]
    for what, d, staged in cases:
        lay = make_layer(d, dtype=dtype)
        for M in (1, 2):
            ch = DecodeChain(M=M, dtype=dtype)
            x = ch.input(d["K"])
            (y,) = ch.stage([lay], x)
            if CL.layout(M, [(d["K"], staged)]) is None:
                _assert_refused(ch)
                continue
            ch.build()
            _assert_layout(ch, M, [(d["K"], staged)])
            for launch, kind in enumerate(("offset", "massive", "row_scale")):
                x.copy_(torch.from_numpy(P.activations(kind, M, d["K"], dtype, seed=60 + launch)).to(dtype).cuda())
                ch.run()
                torch.cuda.synchronize()
                _check_plain(f"stage {what}", f"{what} {dt} M={M} {kind}", _np(y), d, _np(x), dtype)
    assert CL.layout(2, [(32768, False)]) is None


# --------------------------------------------------------------------------- model level
MODELS = ["mistral_7b", "qwen2_7b", "llama2_13b"]


@functools.lru_cache(maxsize=1)
def _model(name, dtype, act=False):
    """A 2-layer random model at the width's shapes (vocab 512) whose projections are QuantLinears of the ``_block``
    dicts (layer i: seed i); returns (model, per-layer dicts)."""
    from transformers import LlamaConfig, LlamaForCausalLM, Qwen2Config, Qwen2ForCausalLM

    H, I, nh, nkv, bias = SHAPES[name]
    common = dict(hidden_size=H, intermediate_size=I, num_attention_heads=nh, num_key_value_heads=nkv, head_dim=HD,
                  num_hidden_layers=2, vocab_size=512, max_position_embeddings=512, rms_norm_eps=EPS)
    torch.manual_seed(1)
    with torch.device("cuda"):                       # the nn.Linear weights are replaced at once: initialise on the GPU
        if bias:
            m = Qwen2ForCausalLM(Qwen2Config(**common, use_sliding_window=False))
        else:
            m = LlamaForCausalLM(LlamaConfig(**common))
    m = m.to(dtype).eval()
    m.config._attn_implementation = "sdpa"
    with torch.no_grad():                           # random norm weights, as trained models have
        for mod in m.modules():
            if type(mod).__name__.endswith("RMSNorm"):
                mod.weight.uniform_(0.5, 1.5)
    dt = P.dt_name(dtype)
    dicts = []
    for i, layer in enumerate(m.model.layers):
        ds = _block(name, dt, act, seed=i)
        for mod, names in ((layer.self_attn, ("q", "k", "v", "o")), (layer.mlp, ("gate", "up", "down"))):
            for n in names:
                setattr(mod, f"{n}_proj", make_layer(ds[n], dtype=dtype))
        dicts.append(ds)
    return m, dicts


def _logit_tol(dtype, n_layers):
    """``tests/test_gpu_21_chain_norm.py``'s: 12 roundings per block, each up to 2^-p of the rms."""
    p = 11 if dtype == F16 else 8
    return 12 * n_layers * 2.0 ** -p


def _refusing_model(name, dtype):
    """The model at the width's shapes with act-order on every projection, without running anything (blank weights)."""
    from transformers import LlamaConfig, LlamaForCausalLM, Qwen2Config, Qwen2ForCausalLM

    H, I, nh, nkv, bias = SHAPES[name]
    common = dict(hidden_size=H, intermediate_size=I, num_attention_heads=nh, num_key_value_heads=nkv, head_dim=HD,
                  num_hidden_layers=2, vocab_size=512, max_position_embeddings=512, rms_norm_eps=EPS)
    with torch.device("cuda"):
        m = (Qwen2ForCausalLM(Qwen2Config(**common, use_sliding_window=False)) if bias
             else LlamaForCausalLM(LlamaConfig(**common)))
    m = m.to(dtype).eval()
    ds = _blank_block(name, True)
    for layer in m.model.layers:
        for mod, names in ((layer.self_attn, ("q", "k", "v", "o")), (layer.mlp, ("gate", "up", "down"))):
            for n in names:
                d = dict(ds[n], bias=np.zeros(ds[n]["N"], np.float32)) if bias and n in ("q", "k", "v") else ds[n]
                setattr(mod, f"{n}_proj", make_layer(d, dtype=dtype))
    return m


REFUSED = [(n, M, act) for n in MODELS for (M, act), slots in CL.H100_SLOTS[n].items() if slots is None]


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("name,batch,act", REFUSED, ids=[f"{n}-b{M}-{'act' if a else 'plain'}" for n, M, a in REFUSED])
def test_chain_decoder_refuses_before_allocating(name, batch, act, dtype, monkeypatch):
    from autogptq_b200.decoder import ChainDecoder

    model = _model(name, dtype)[0] if not act else _refusing_model(name, dtype)

    def no_allocate(self, rows):
        raise AssertionError("ChainDecoder allocated its caches before refusing a block whose chain does not fit")

    monkeypatch.setattr(ChainDecoder, "_allocate", no_allocate)
    with pytest.raises(NotImplementedError, match=rf"model\.layers\.0 at batch {batch} .*needs \d+ B of shared "
                                                  r"memory .*more than the \d+ B a block may opt in to"):
        ChainDecoder(model, batch=batch, max_length=64)


def _decoder_block_buffers(dec, i):
    """Host copies of block i's buffers: its q|k|v (``_qkv``), the attention output (``_attn_in``) and, from the stage
    records of the chain that starts at o_i, o, gate, up, h1, down and the next q|k|v and residual."""
    ch = dec.chains[i + 1]
    st = ch._stages                         # (layers, x, x2, mode, parts, stride, ys, peer_tables, perm, norm)
    q, k, v = dec._qkv[i]
    b = dict(q=_np(q), k=_np(k), v=_np(v), a=_np(dec._attn_in[i]), o=_np(st[0][6][0]), gate=_np(st[1][6][0]),
             up=_np(st[1][6][1]), h1=_np(st[1][9][2]), down=_np(st[2][6][0]))
    if len(st) > 3:
        q2, k2, v2 = st[3][6]
        b.update(q2=_np(q2), k2=_np(k2), v2=_np(v2), resid=_np(st[3][9][2]))
    return b


@pytest.mark.parametrize("fused", [False, True], ids=["torch_attn", "fused_attn"])
@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("name", MODELS)
def test_chain_decoder_blocks_and_logits(name, dtype, batch, fused):
    from transformers import DynamicCache

    from autogptq_b200.decoder import ChainDecoder

    if CL.H100_SLOTS[name][(batch, False)] is None:
        pytest.skip("refused: test_chain_decoder_refuses_before_allocating")
    model, dicts = _model(name, dtype)
    layers = model.model.layers
    T0, steps = 8, 16
    g = torch.Generator().manual_seed(7 + batch)
    prompt = torch.randint(0, 512, (batch, T0), generator=g).cuda()
    forced = torch.randint(0, 512, (batch, steps), generator=g).cuda()
    dec = ChainDecoder(model, batch=batch, max_length=64, fused_attention=fused)
    H, I = SHAPES[name][:2]
    for ch in dec.chains[1:]:
        assert (ch.info()["ring_slots"], ch.info()["smem_bytes"]) == CL.layout(
            batch, CL.block_stages(H, I, False)[:len(ch._stages)]), ch.info()
    tol = _logit_tol(dtype, 2)
    dt = P.dt_name(dtype)
    with torch.no_grad():
        cache = DynamicCache(config=model.config)
        ref = model(input_ids=prompt, past_key_values=cache, use_cache=True).logits[:, -1]
        assert torch.equal(dec.prefill(prompt), ref)
        for t in range(steps):
            ids = forced[:, t]
            ref = model(input_ids=ids[:, None], past_key_values=cache, use_cache=True).logits[:, -1].float()
            if t == 0:                               # every block's buffers after one eager step
                got = dec.step(ids, use_graph=False).float()
                h_in = _np(dec._x0)
                for i, layer in enumerate(layers):        # block i + 1's q|k|v are checked as block i + 1's
                    ln1, ln2 = layer.input_layernorm, layer.post_attention_layernorm
                    b = _decoder_block_buffers(dec, i)
                    b["h_in"] = h_in
                    tag = f"ChainDecoder {name} {dt} batch={batch} fused={fused} block {i}"
                    _check_block(name, dicts[i], b, _np(ln1.weight), _np(ln2.weight), float(ln1.variance_epsilon),
                                 float(ln2.variance_epsilon), dtype, tag)
                    if i + 1 < len(layers):
                        _check_sum(b["resid"], b["down"], b["h1"], dtype, f"{tag} resid")
                        h_in = b["resid"]
            else:
                got = dec.step(ids).float()
            assert_parity(got.cpu().numpy(), ref.cpu().numpy(), rtol=tol, atol_rms=tol,
                          what=f"{name} {dt} batch={batch} fused={fused} step {t}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_batch_decoder_qwen2_7b_width(dtype):
    """8 rows, G = 7 (28 heads over 4 kv heads): the rows attention kernel at Qwen2-7B's grouping, teacher-forced."""
    from transformers import DynamicCache

    from autogptq_b200 import BatchDecoder

    model, _ = _model("qwen2_7b", dtype)
    steps, B = 8, 8
    g = torch.Generator().manual_seed(11)
    prompts = [torch.randint(0, 512, (4 + 3 * i,), generator=g).cuda() for i in range(B)]
    forced = torch.randint(0, 512, (B, steps), generator=g).cuda()
    # 8 rows run the projections on the mma.sync skinny kernel: test_gpu_24_batch_decoder.py's fp16 allowance
    tol = _logit_tol(dtype, 2) * (1.5 if dtype == F16 else 1.0)
    dec = BatchDecoder(model, max_batch=B, max_length=64)
    with torch.no_grad():
        refs = []
        for p, f in zip(prompts, forced):
            cache = DynamicCache(config=model.config)
            seq = [model(input_ids=p[None], past_key_values=cache, use_cache=True).logits[0, -1]]
            for t in range(steps):
                seq.append(model(input_ids=f[t].view(1, 1), past_key_values=cache, use_cache=True).logits[0, -1])
            refs.append(seq)
        for s in range(B):
            assert torch.equal(dec.prefill(s, prompts[s]), refs[s][0]), "prefill logits differ from HF's"
        for t in range(steps):
            got = dec.step(forced[:, t]).float().cpu().numpy()
            r = torch.stack([refs[s][t + 1] for s in range(B)]).float().cpu().numpy()
            assert_parity(got, r, rtol=tol, atol_rms=tol, what=f"BatchDecoder qwen2_7b {P.dt_name(dtype)} step {t}")
