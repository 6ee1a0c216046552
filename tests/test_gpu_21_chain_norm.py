"""The decode chain's norm stage inputs on the GPU, and ChainDecoder against the transformers model it runs.

Stage level (Llama-2-7B shapes, one H = 8192 stage; fp16 / bf16; M = 1, 2; plain and act-order layers):

    x_ext ─[rmsnorm]→ A (H→H)          RMSNorm of an external input
    y_a, r_ext ─[add_rmsnorm]→ B (H→H), h1 = rnd(y_a + r_ext)    one operand a chain output, the other external
    y_b, h1 ─[add_rmsnorm]→ C (H→I), h2 = rnd(y_b + h1)          both chain outputs, h1 found by pointer

* h1 and h2 are bit-equal to rnd(a + b) of what the stage read;
* each y is within the chain's DESIGN §3.12 bound (``tests/_precision.py``) against float64 on the host-side n,
  widened by Σ|n_alt − n|·|W| where n has two candidates (``tests/_chain_norm.py``, ``check_y``);
* three consecutive launches (tags are never reset) each pass, and two launches on one input are bit-identical.

Model level: a small random Llama and a Qwen2 with q/k/v biases, 32 teacher-forced ChainDecoder steps against the HF
model with the same QuantLinears and a DynamicCache (tolerance derived at ``_logit_tol``)."""
import functools

import numpy as np
import pytest
import torch

from tests import _chain_norm as N
from tests import _precision as P
from tests._util import assert_parity, make_layer

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTS = [F16, BF16]


def _np(t):
    return t.double().cpu().numpy()


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


@functools.lru_cache(maxsize=None)
def _layers(H, I, dt, act):
    return (P.wide_layer(H, H, 128, dt, seed=60, act_order=act, bias=True),
            P.wide_layer(H, H, 128, dt, seed=61, act_order=act),
            P.wide_layer(H, I, 128, dt, seed=62, act_order=act, bias=True))


def _weight(K, dtype, seed):
    rng = np.random.default_rng(seed)
    return P.round_dt(rng.uniform(0.05, 3.0, size=K) * np.where(rng.random(K) < 0.3, -1, 1), P.dt_name(dtype))


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 2])
@pytest.mark.parametrize("H,I,act", [(4096, 11008, False), (4096, 11008, True), (8192, 1024, False)],
                         ids=["llama7b", "llama7b_act_order", "h8192"])
def test_norm_stages(dtype, M, H, I, act):
    from autogptq_b200.chain import DecodeChain

    dt = P.dt_name(dtype)
    da, db, dc = _layers(H, I, dt, act)
    A, B, C = (make_layer(d, dtype=dtype) for d in (da, db, dc))
    wa, wb, wc = (_weight(H, dtype, s) for s in (1, 2, 3))
    eps = 1e-5
    wt = [torch.from_numpy(w).to(dtype).cuda() for w in (wa, wb, wc)]
    ch = DecodeChain(M=M, dtype=dtype)
    x_ext, r_ext = ch.input(H), ch.input(H)
    (ya,) = ch.stage([A], x_ext, x_mode="rmsnorm", norm_weight=wt[0], norm_eps=eps)
    yb, h1 = ch.stage([B], ya, x2=r_ext, x_mode="add_rmsnorm", norm_weight=wt[1], norm_eps=eps)
    yc, h2 = ch.stage([C], yb, x2=h1, x_mode="add_rmsnorm", norm_weight=wt[2], norm_eps=eps)
    ch.build()
    cols_h = (H - 256, H)
    cols_i = (I - 256, I) if I > 1024 else None
    for launch, kind in enumerate(("massive", "offset", "gauss")):
        x = P.activations(kind, M, H, dtype, seed=30 + launch)
        r = P.round_dt(P.activations("gauss", M, H, dtype, seed=40 + launch) * 4.0, dt)
        x_ext.copy_(torch.from_numpy(x).to(dtype).cuda())
        r_ext.copy_(torch.from_numpy(r).to(dtype).cuda())
        ch.run()
        torch.cuda.synchronize()
        outs = [t.clone() for t in (ya, yb, yc, h1, h2)]
        ch.run()
        torch.cuda.synchronize()
        for a, b in zip(outs, (ya, yb, yc, h1, h2)):
            assert _bits_equal(a, b), "two launches on one input differ"
        xs, yan, ybn, rn = _np(x_ext), _np(ya), _np(yb), _np(r_ext)
        h1n, h2n = _np(h1), _np(h2)
        assert np.array_equal(h1n, N.add_rounded(yan, rn, dtype)), f"h1 != rnd(y_a + r) ({kind})"
        assert np.array_equal(h2n, N.add_rounded(ybn, h1n, dtype)), f"h2 != rnd(y_b + h1) ({kind})"
        tag = f"{dt} M={M} H={H} act={act} {kind} launch {launch}"
        N.check_y(yan, da, xs, wa, eps, dtype, cols_h, f"rmsnorm stage {tag}")
        N.check_y(ybn, db, h1n, wb, eps, dtype, cols_h, f"add_rmsnorm stage (external residual) {tag}")
        N.check_y(_np(yc), dc, h2n, wc, eps, dtype, cols_i, f"add_rmsnorm stage (chain residual) {tag}")


def test_chain_without_norm_stages_keeps_its_shape():
    """A bench.py-shaped chain (q|k|v, o, gate|up, silu_mul down of a Llama-2-7B block, twice) has the same ring depth
    and shared memory as before norm stages existed: the norm staging only costs a chain that has a norm stage."""
    from autogptq_b200.chain import DecodeChain

    dt = "float16"
    mk = lambda K, N, s: make_layer(P.realistic_layer(K, N, 128, dt, seed=s, wrap_groups=False))
    qkv = [mk(4096, 4096, s) for s in (1, 2, 3)]
    o, g, u, d = mk(4096, 4096, 4), mk(4096, 11008, 5), mk(4096, 11008, 6), mk(11008, 4096, 7)
    info = {}
    for M in (1, 2):
        ch = DecodeChain(M=M)
        x = ch.input(4096)
        for _ in range(2):
            q, _, _ = ch.stage(qkv, x)
            (x,) = ch.stage([o], q)
            ga, up = ch.stage([g, u], x)
            (x,) = ch.stage([d], ga, x2=up, x_mode="silu_mul")
        ch.build()
        info[M] = ch.info()
        # the same chain with the block's norms: ring slots shrink by the staged x (M * 4096 * 2 bytes)
        ch2 = DecodeChain(M=M)
        x = ch2.input(4096)
        w = torch.ones(4096, dtype=F16, device="cuda")
        q, _, _ = ch2.stage(qkv, x, x_mode="rmsnorm", norm_weight=w)
        (y,) = ch2.stage([o], q)
        ga, up, h = ch2.stage([g, u], y, x2=x, x_mode="add_rmsnorm", norm_weight=w)
        (y,) = ch2.stage([d], ga, x2=up, x_mode="silu_mul")
        ch2.build()
        i2 = ch2.info()
        assert i2["smem_bytes"] - i2["ring_slots"] * 17 * 1024 == (
            info[M]["smem_bytes"] - info[M]["ring_slots"] * 17 * 1024 + M * 4096 * 2), (info[M], i2)
        print(f"[chain-norm] M={M}: without norm stages {info[M]}, with {i2}")
    assert (info[1]["ring_slots"], info[1]["smem_bytes"]) == BASE_INFO[1], info[1]
    assert (info[2]["ring_slots"], info[2]["smem_bytes"]) == BASE_INFO[2], info[2]


# (ring slots, dynamic shared memory bytes) of that chain before norm stages existed, on an H100 80GB HBM3
BASE_INFO = {1: (10, 232088), 2: (7, 231064)}


# --------------------------------------------------------------------------- model level
def _quantize_model(model, dtype, seed=0):
    """Replace every nn.Linear projection of the decoder layers by a QuantLinear of a realistic random 4-bit layer
    (bias kept when the Linear has one)."""
    dt = P.dt_name(dtype)
    k = seed
    for layer in model.model.layers:
        for mod, names in ((layer.self_attn, ("q_proj", "k_proj", "v_proj", "o_proj")),
                           (layer.mlp, ("gate_proj", "up_proj", "down_proj"))):
            for name in names:
                lin = getattr(mod, name)
                d = P.realistic_layer(lin.in_features, lin.out_features, 128, dt, seed=k, bias=lin.bias is not None,
                                      wrap_groups=False)
                k += 1
                setattr(mod, name, make_layer(d, dtype=dtype))
    return model


@functools.lru_cache(maxsize=None)
def _model(arch, dtype):
    from transformers import LlamaConfig, LlamaForCausalLM, Qwen2Config, Qwen2ForCausalLM

    common = dict(hidden_size=1024, intermediate_size=2816, num_attention_heads=8, num_key_value_heads=2,
                  num_hidden_layers=4, vocab_size=512, max_position_embeddings=512, rms_norm_eps=1e-5)
    torch.manual_seed(1)
    if arch == "llama":
        m = LlamaForCausalLM(LlamaConfig(**common))
    else:
        m = Qwen2ForCausalLM(Qwen2Config(**common, use_sliding_window=False))
    with torch.no_grad():                               # random norm weights, as trained models have
        for mod in m.modules():
            if type(mod).__name__.endswith("RMSNorm"):
                mod.weight.uniform_(0.5, 1.5)
    m = m.to(dtype).cuda().eval()
    m.config._attn_implementation = "sdpa"
    return _quantize_model(m, dtype)


def _logit_tol(dtype, n_layers):
    """Logit tolerance between two correct implementations.  Each rounded activation of a block (h1, n2, g, u, the
    silu·mul h, down, h2, the next norm, q/k/v, the attention output, o) may differ by about one ulp of the dtype
    between the chain and the HF path (§3.12 bound, norm candidates, a different attention kernel): 12 roundings per
    block, each moving an O(rms) value by at most 2^-p relative, passed on with gain ~1 by the norms.  Summed linearly
    over the blocks: tol = 12·L·2^-p relative to rms, and the same relative to each logit (p = 11 fp16, 8 bf16)."""
    p = 11 if dtype == F16 else 8
    return 12 * n_layers * 2.0 ** -p


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_decoder_matches_hf(arch, dtype, batch):
    from transformers import DynamicCache

    from autogptq_b200.decoder import ChainDecoder

    model = _model(arch, dtype)
    T0, steps = 16, 32
    g = torch.Generator().manual_seed(5 + batch)
    prompt = torch.randint(0, 512, (batch, T0), generator=g).cuda()
    forced = torch.randint(0, 512, (batch, steps), generator=g).cuda()
    dec = ChainDecoder(model, batch=batch, max_length=128)
    tol = _logit_tol(dtype, 4)
    with torch.no_grad():
        cache = DynamicCache(config=model.config)
        ref = model(input_ids=prompt, past_key_values=cache, use_cache=True).logits[:, -1]
        got = dec.prefill(prompt)
        assert torch.equal(got, ref)
        agree = total = 0
        for t in range(steps):
            ids = forced[:, t]
            ref = model(input_ids=ids[:, None], past_key_values=cache, use_cache=True).logits[:, -1].float()
            if t == 3:                                   # an eager step and its graph replay are bit-identical
                p = dec.position
                eager = dec.step(ids, use_graph=False).clone()
                dec.position = p
                got = dec.step(ids).float()
                assert torch.equal(eager.float(), got), "graph replay differs from the eager step"
            else:
                got = dec.step(ids).float()
            r, o = ref.cpu().numpy(), got.cpu().numpy()
            assert_parity(o, r, rtol=tol, atol_rms=tol, what=f"{arch} {dtype} batch={batch} step {t}")
            top2 = np.sort(r, axis=-1)[:, -2:]
            margin = top2[:, 1] - top2[:, 0]
            rms = float(np.sqrt(np.mean(r.astype(np.float64) ** 2)))
            clear = margin > 2 * (tol * np.abs(top2[:, 1]) + tol * rms)
            same = r.argmax(-1) == o.argmax(-1)
            assert same[clear].all(), f"step {t}: greedy token differs where the reference margin is clear"
            agree += int(same.sum())
            total += same.size
        print(f"[chain-norm] decoder {arch} {dtype} batch={batch}: greedy agreement {agree}/{total}, tol {tol:.3g}")


def test_decoder_generate_runs_and_matches_steps():
    from autogptq_b200.decoder import ChainDecoder

    model = _model("llama", F16)
    dec = ChainDecoder(model, batch=1, max_length=64)
    prompt = torch.randint(0, 512, (1, 8), generator=torch.Generator().manual_seed(9)).cuda()
    out = dec.generate(prompt, 12)
    assert out.shape == (1, 20) and torch.equal(out[:, :8], prompt)
    dec2 = ChainDecoder(model, batch=1, max_length=64)
    logits = dec2.prefill(prompt)
    toks = []
    for _ in range(12):
        tok = logits.argmax(-1)
        toks.append(int(tok))
        logits = dec2.step(tok, use_graph=False)
    assert out[0, 8:].tolist() == toks
