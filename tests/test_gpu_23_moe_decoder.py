"""The MoE router kernel on the GPU, and ChainDecoder on a Mixtral model against the transformers model it runs.

Kernel level (``autogptq_b200.moe.moe_router``), every output checked on the inputs the kernel actually saw
(``tests/_moe_router.py``, ``tests/_chain_norm.py``):
* h bit-equal to torch's x + x2;
* n one of its two chain-norm candidates;
* the logits one of their two candidates around the float64 dot product of the kernel's own n;
* the indices equal to the reference wherever the gap to the next expert is clear, and every exact tie (duplicated
  router rows) resolved to the lower index;
* the weights within their bound, summing to 1 within fp32 rounding;
* repeat bit-identity, CUDA-graph replay on new inputs, massive-channel activations.

Model level: a small random Mixtral (H 1024, I 2048, 8 experts, top-2, 4 layers, 8/2 heads) whose attention
projections are QuantLinear and whose experts are QuantExperts, 32 teacher-forced ChainDecoder steps against the HF
model with a DynamicCache, at batch 1 / 2, fp16 / bf16, torch / fused attention."""
import functools

import numpy as np
import pytest
import torch

from tests import _chain_norm as N
from tests import _moe_router as R
from tests import _precision as P
from tests._util import assert_parity, make_layer

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTS = [F16, BF16]


def _np(t):
    return t.double().cpu().numpy()


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16)) if a.dtype in DTS else torch.equal(a, b)


def _router_inputs(T, H, E, dtype, seed, kind="gauss"):
    """x, x2 [T, H], norm weight [H], router weight [E, H] on the GPU.  Rows 1 and E - 1 of the router repeat rows 0 and
    2, and row 0 is scaled up so that the tie of experts 0 and 1 usually falls inside the top-k."""
    dn = P.dt_name(dtype)
    rng = np.random.default_rng(seed)
    x = torch.from_numpy(P.activations(kind, T, H, dtype, seed=seed)).to(dtype).cuda()
    x2 = torch.from_numpy(P.activations("gauss", T, H, dtype, seed=seed + 1)).to(dtype).cuda()
    w = torch.from_numpy(P.round_dt(rng.uniform(0.5, 1.5, H), dn)).to(dtype).cuda()
    G = rng.standard_normal((E, H)) * (2.0 / np.sqrt(H))
    G[0] *= 2.0
    G[1] = G[0]
    G[E - 1] = G[2]
    return x, x2, w, torch.from_numpy(P.round_dt(G, dn)).to(dtype).cuda()


def _run(x, x2, w, G, k, eps=1e-5):
    from autogptq_b200.moe import moe_router

    logits = torch.empty((x.shape[0], G.shape[0]), dtype=x.dtype, device=x.device)
    return moe_router(x, x2, w, eps, G, k, logits=logits)


def _check(x, x2, w, G, k, outs, dtype, what, eps=1e-5):
    h, n, idx, wts, logits = outs
    dn = P.dt_name(dtype)
    if x2 is not None:
        assert _bits_equal(h, x + x2), f"{what}: h differs from x + x2"
        hh = _np(h)
    else:
        assert h is None
        hh = _np(x)
    N.check_n(_np(n), hh, _np(w), eps, dn, what)
    R.check_logits(_np(logits), _np(n), _np(G), dn, what)
    l = _np(logits)
    R.check_topk(idx.cpu().numpy(), l, k, what)
    return R.check_weights(wts.cpu().numpy(), idx.cpu().numpy(), l, what)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("H", [1024, 4096, 6144])
@pytest.mark.parametrize("k", [1, 2, 4])
@pytest.mark.parametrize("E", [4, 8, 16, 64])
def test_router_kernel(E, k, H, dtype):
    worst = 0.0
    for T in (1, 2, 8):
        for with_x2 in (False, True):
            x, x2, w, G = _router_inputs(T, H, E, dtype, seed=E * 1000 + k * 100 + T)
            x2 = x2 if with_x2 else None
            outs = _run(x, x2, w, G, k)
            torch.cuda.synchronize()
            worst = max(worst, _check(x, x2, w, G, k, outs, dtype, f"E={E} k={k} H={H} T={T} x2={with_x2} {dtype}"))
            ties = outs[2].cpu().numpy()
            assert ((ties == 1).any(axis=1) <= (ties == 0).any(axis=1)).all()    # expert 1 only after its twin 0
    print(f"[moe-router] E={E} k={k} H={H} {dtype}: largest weight err/bound {worst:.3f}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_router_massive_channels_and_repeat_identity(dtype):
    """Rows with three channels ×1000 (the §3.12 outlier rows), and two calls bit-identical."""
    x, x2, w, G = _router_inputs(8, 4096, 8, dtype, seed=7, kind="massive")
    a = _run(x, x2, w, G, 2)
    b = _run(x, x2, w, G, 2)
    torch.cuda.synchronize()
    _check(x, x2, w, G, 2, a, dtype, f"massive {dtype}")
    for u, v in zip(a, b):
        assert _bits_equal(u, v), "two calls differ"


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_router_graph_replay_with_new_inputs(dtype):
    from autogptq_b200.moe import moe_router

    T, H, E, k = 2, 4096, 8, 2
    x, x2, w, G = _router_inputs(T, H, E, dtype, seed=21)
    h, n = torch.empty_like(x), torch.empty_like(x)
    idx = torch.empty((T, k), dtype=torch.int32, device="cuda")
    wts = torch.empty((T, k), dtype=torch.float32, device="cuda")
    logits = torch.empty((T, E), dtype=dtype, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        moe_router(x, x2, w, 1e-5, G, k, h=h, n=n, idx=idx, w=wts, logits=logits)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        moe_router(x, x2, w, 1e-5, G, k, h=h, n=n, idx=idx, w=wts, logits=logits)
    for seed in (22, 23):
        nx, nx2, _, _ = _router_inputs(T, H, E, dtype, seed=seed)
        x.copy_(nx)
        x2.copy_(nx2)
        g.replay()
        eager = _run(x, x2, w, G, k)
        torch.cuda.synchronize()
        for u, v in zip((h, n, idx, wts, logits), eager):
            assert _bits_equal(u, v), "graph replay differs from an eager call"
        _check(x, x2, w, G, k, (h, n, idx, wts, logits), dtype, f"graph replay {dtype}")


# --------------------------------------------------------------------------- model level
L_LAYERS, E_EXPERTS, TOP_K = 4, 8, 2


def _quantize_mixtral(model, dtype):
    """Attention projections -> QuantLinear of realistic random 4-bit layers; each block's experts -> QuantExperts of
    such layers."""
    from autogptq_b200 import QuantExperts

    dt = P.dt_name(dtype)
    k = 0

    def quant(K, Nf):
        nonlocal k
        d = P.realistic_layer(K, Nf, 128, dt, seed=k, wrap_groups=False)
        k += 1
        return make_layer(d, dtype=dtype)

    cfg = model.config
    H, I = cfg.hidden_size, cfg.intermediate_size
    for layer in model.model.layers:
        for name in ("q_proj", "k_proj", "v_proj", "o_proj"):
            lin = getattr(layer.self_attn, name)
            setattr(layer.self_attn, name, quant(lin.in_features, lin.out_features))
        E = cfg.num_local_experts
        w1, w3, w2 = [quant(H, I) for _ in range(E)], [quant(H, I) for _ in range(E)], [quant(I, H) for _ in range(E)]
        layer.mlp.experts = QuantExperts(w1, w3, w2)
    return model


@functools.lru_cache(maxsize=None)
def _model(dtype):
    from transformers import MixtralConfig, MixtralForCausalLM

    cfg = MixtralConfig(hidden_size=1024, intermediate_size=2048, num_attention_heads=8, num_key_value_heads=2,
                        num_hidden_layers=L_LAYERS, num_local_experts=E_EXPERTS, num_experts_per_tok=TOP_K,
                        vocab_size=512, max_position_embeddings=512, rms_norm_eps=1e-5)
    torch.manual_seed(1)
    m = MixtralForCausalLM(cfg)
    with torch.no_grad():
        for mod in m.modules():
            if type(mod).__name__.endswith("RMSNorm"):
                mod.weight.uniform_(0.5, 1.5)
            if type(mod).__name__ == "MixtralTopKRouter":
                mod.weight.normal_(0.0, 2.0 / np.sqrt(cfg.hidden_size))
    m = m.to(dtype).cuda().eval()
    m.config._attn_implementation = "sdpa"
    return _quantize_mixtral(m, dtype)


def _logit_tol(dtype, n_layers, k=TOP_K):
    """As tests/test_gpu_21_chain_norm.py (12 roundings per dense block, each about one ulp, summed over the blocks),
    with two more per routed expert: an MoE block rounds g, u, silu·mul and the down output of each of its k experts
    and then their weighted sum, where a dense block rounds one of each.  Doubled: the routing weights pass on a logit
    difference with gain w(1 − w) times the gap between the two experts' outputs, which is O(rms), and the caches carry
    these differences from step to step (measured on the H100: up to 1.44 of the undoubled value, fp16, batch 2)."""
    p = 11 if dtype == F16 else 8
    return 2 * (12 + 2 * k) * n_layers * 2.0 ** -p


# Least number of the 32 steps compared.  A step whose routing parts from HF's (possible only where a router margin is
# unclear, which _routing_agrees checks) is not compared, and the decoder's cache is re-seeded from HF's after it.  On
# this random model that happened on up to about one step in five (fused attention, batch 2, H100).
MIN_COMPARED = 20


class _RouterHook:
    """Records the input and top-k indices of every MixtralTopKRouter call of the HF model."""

    def __init__(self, model):
        self.calls = []
        self.handles = [layer.mlp.gate.register_forward_hook(self) for layer in model.model.layers]

    def __call__(self, mod, inp, out):
        self.calls.append((inp[0].detach().reshape(-1, mod.hidden_dim).clone(), out[2].detach().clone()))

    def remove(self):
        for h in self.handles:
            h.remove()


def _routing_agrees(dec, calls, model, dtype):
    """(agree, unclear) over the layers of one step: HF's decisions against the decoder's.  A layer's reference margin
    is clear when each gap between HF's sorted logits at the top-k boundary and above exceeds twice the largest
    difference between the two states' exact logits plus two ulps of the largest logit (the rounding of either
    side); there the decoder's indices must equal HF's."""
    agree, unclear = True, False
    dn = P.dt_name(dtype)
    for i, (n_hf, idx_hf) in enumerate(calls):
        m = dec._moe_layers[i]
        G = _np(m["gate"])
        z_hf, z_dec = _np(n_hf) @ G.T, _np(m["n2"]) @ G.T
        l_hf = P.round_dt(z_hf, dn)
        idx_dec = m["idx"].long().cpu().numpy()
        idx_ref = idx_hf.long().cpu().numpy()
        for t in range(l_hf.shape[0]):
            s = np.sort(l_hf[t])[::-1]
            slack = 2 * np.abs(z_hf[t] - z_dec[t]).max() + 2 * P.ulp(np.abs(l_hf[t]).max(), dn)
            clear = (s[:TOP_K] - s[1:TOP_K + 1] > slack).all()
            same = idx_dec[t].tolist() == idx_ref[t].tolist()
            if clear:
                assert same, f"layer {i} row {t}: decoder routes {idx_dec[t].tolist()}, HF {idx_ref[t].tolist()}"
            unclear |= not clear
            agree &= same
    return agree, unclear


@pytest.mark.parametrize("fused", [False, True], ids=["torch_attn", "fused_attn"])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("batch", [1, 2])
def test_mixtral_decoder_matches_hf(batch, dtype, fused):
    from transformers import DynamicCache

    from autogptq_b200.decoder import ChainDecoder

    model = _model(dtype)
    T0, steps = 8, 32
    g = torch.Generator().manual_seed(5 + batch)
    prompt = torch.randint(0, 512, (batch, T0), generator=g).cuda()
    forced = torch.randint(0, 512, (batch, steps), generator=g).cuda()
    dec = ChainDecoder(model, batch=batch, max_length=128, fused_attention=fused)
    assert dec.moe
    tol = _logit_tol(dtype, L_LAYERS)
    hook = None
    try:
        with torch.no_grad():
            cache = DynamicCache(config=model.config)
            ref = model(input_ids=prompt, past_key_values=cache, use_cache=True).logits[:, -1]
            got = dec.prefill(prompt)
            assert torch.equal(got, ref)
            hook = _RouterHook(model)
            compared = unclear_steps = parted = agree = total = 0
            for t in range(steps):
                ids = forced[:, t]
                hook.calls.clear()
                ref = model(input_ids=ids[:, None], past_key_values=cache, use_cache=True).logits[:, -1].float()
                if t == 3:                                   # an eager step and its graph replay are bit-identical
                    p = dec.position
                    eager = dec.step(ids, use_graph=False).clone()
                    dec.position = p
                    got = dec.step(ids).float()
                    assert torch.equal(eager.float(), got), "graph replay differs from the eager step"
                else:
                    got = dec.step(ids).float()
                assert len(hook.calls) == L_LAYERS
                same_routing, unclear = _routing_agrees(dec, hook.calls, model, dtype)
                unclear_steps += int(unclear)
                if not same_routing:              # only possible where a margin is unclear: the caches part here
                    parted += 1
                    for i, lay in enumerate(cache.layers):
                        n_pos = lay.keys.shape[2]
                        dec.k_cache[i][:, :, :n_pos].copy_(lay.keys)
                        dec.v_cache[i][:, :, :n_pos].copy_(lay.values)
                    continue
                r, o = ref.cpu().numpy(), got.cpu().numpy()
                assert_parity(o, r, rtol=tol, atol_rms=tol, what=f"mixtral {dtype} batch={batch} step {t}")
                top2 = np.sort(r, axis=-1)[:, -2:]
                margin = top2[:, 1] - top2[:, 0]
                rms = float(np.sqrt(np.mean(r.astype(np.float64) ** 2)))
                clear = margin > 2 * (tol * np.abs(top2[:, 1]) + tol * rms)
                same = r.argmax(-1) == o.argmax(-1)
                assert same[clear].all(), f"step {t}: greedy token differs where the reference margin is clear"
                agree += int(same.sum())
                total += same.size
                compared += 1
    finally:
        if hook is not None:
            hook.remove()
    print(f"[moe-decoder] batch={batch} {dtype} fused={fused}: {compared}/{steps} steps compared, {parted} parted "
          f"({unclear_steps} with an unclear router margin), greedy agreement {agree}/{total}, tol {tol:.3g}")
    assert compared >= MIN_COMPARED, f"only {compared} of {steps} steps were compared ({parted} parted)"


def test_mixtral_generate_matches_steps():
    from autogptq_b200.decoder import ChainDecoder

    model = _model(F16)
    dec = ChainDecoder(model, batch=1, max_length=64, fused_attention=True)
    prompt = torch.randint(0, 512, (1, 8), generator=torch.Generator().manual_seed(9)).cuda()
    out = dec.generate(prompt, 12)
    assert out.shape == (1, 20) and torch.equal(out[:, :8], prompt)
    dec2 = ChainDecoder(model, batch=1, max_length=64, fused_attention=True)
    logits = dec2.prefill(prompt)
    toks = []
    for _ in range(12):
        tok = logits.argmax(-1)
        toks.append(int(tok))
        logits = dec2.step(tok, use_graph=False)
    assert out[0, 8:].tolist() == toks
