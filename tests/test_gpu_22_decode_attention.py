"""The decode attention kernel (``agb200_decode_attention``) on the GPU, and ChainDecoder(fused_attention=True) against
the transformers model it runs.

Kernel level, against transformers' rotary embedding on the same q / k (``tests/_attention.py``):
* the new cache entries at pos are bit-equal to apply_rotary_pos_emb's k̂ (v trivially);
* o is within the derived bound of the float64 reference on torch's q̂ and the cache, and mismatches round(o*) at
  most at DESIGN §3.12's rates (5 % fp16, 1 % bf16) where the budget is at most one ulp;
* positions above pos (NaN-filled) are untouched and unread: the output equals the run with zeros there; positions
  below pos are unchanged; two calls are bit-identical; a CUDA graph captured at one position replays at later ones.

Model level: the small random Llama and Qwen2 of ``tests/test_gpu_21_chain_norm.py`` and a Llama with llama3 rope
scaling, 32 teacher-forced steps against HF at that module's logit tolerance."""
import functools

import numpy as np
import pytest
import torch

from tests import _attention as A
from tests import _precision as P
from tests._util import assert_parity
from tests.test_gpu_21_chain_norm import _logit_tol, _model, _quantize_model

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTS = [F16, BF16]
SHAPES = [(32, 32, 128), (32, 8, 128), (28, 4, 128), (64, 8, 128), (14, 2, 64)]
POSITIONS = [0, 1, 15, 16, 17, 255, 1000, 4095]
MAXLEN = 4096
WORST = {}


def _bits(t):
    return t.view(torch.int16)


@functools.lru_cache(maxsize=None)
def _rotary(hd, kind="default"):
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding

    params = {"rope_type": "default", "rope_theta": 10000.0}
    if kind == "llama3":
        params = {"rope_type": "llama3", "rope_theta": 500000.0, "factor": 8.0, "low_freq_factor": 1.0,
                  "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}
    cfg = LlamaConfig(hidden_size=hd * 2, num_attention_heads=2, num_key_value_heads=2, head_dim=hd,
                      max_position_embeddings=32768, rope_parameters=params)
    return LlamaRotaryEmbedding(cfg, device="cuda")


class Case:
    """Random q / k / v and caches of one shape; rows above pos hold NaN."""

    def __init__(self, nh, nkv, hd, B, dtype, L, pos, seed=0, outliers=False, kind="default"):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.nh, self.nkv, self.hd, self.B, self.dtype, self.L = nh, nkv, hd, B, dtype, L
        self.q = torch.randn(B, nh * hd, generator=g, device="cuda").to(dtype)
        self.k = torch.randn(B, nkv * hd, generator=g, device="cuda").to(dtype)
        self.v = torch.randn(B, nkv * hd, generator=g, device="cuda").to(dtype)
        self.kc = torch.randn(B, nkv, L, hd, generator=g, device="cuda").to(dtype)
        self.vc = torch.randn(B, nkv, L, hd, generator=g, device="cuda").to(dtype)
        if outliers:                     # a few 100x channels in q and k: the softmax is dominated by few positions
            for t in (self.q, self.k):
                t.view(B, -1, hd)[:, :, 3] *= 100
                t.view(B, -1, hd)[:, :, hd // 2 + 7] *= 100
            self.kc[:, :, :, 3] *= 100
            self.kc[:, :, :, hd // 2 + 7] *= 100
        self.rot = _rotary(hd, kind)
        self.pos = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.out = torch.empty(B, nh * hd, dtype=dtype, device="cuda")
        self.k0, self.v0 = self.kc.clone(), self.vc.clone()
        self.p = -1
        self.set_pos(pos)

    def set_pos(self, pos):
        """Advance to pos: rows the kernel has not written below pos get random values, rows above pos NaN."""
        self.kc[:, :, self.p + 1:pos] = self.k0[:, :, self.p + 1:pos]
        self.vc[:, :, self.p + 1:pos] = self.v0[:, :, self.p + 1:pos]
        self.p = pos
        self.pos.fill_(pos)
        self.kc[:, :, pos + 1:] = float("nan")
        self.vc[:, :, pos + 1:] = float("nan")

    def run(self, out=None, ws=None):
        from autogptq_b200.attention import decode_attention

        return decode_attention(self.q, self.k, self.v, self.kc, self.vc, self.pos, self.rot.inv_freq,
                                self.rot.attention_scaling, self.hd ** -0.5, self.out if out is None else out, ws)

    def torch_rope(self):
        from transformers.models.llama.modeling_llama import apply_rotary_pos_emb

        B, hd = self.B, self.hd
        cos, sin = self.rot(self.q.view(B, 1, -1), self.pos.view(1, 1).expand(B, 1))
        qh, kh = apply_rotary_pos_emb(self.q.view(B, 1, self.nh, hd).transpose(1, 2),
                                      self.k.view(B, 1, self.nkv, hd).transpose(1, 2), cos, sin)
        return qh[:, :, 0], kh[:, :, 0]

    def check_output(self, what):
        qh, _ = self.torch_rope()
        n = self.p + 1
        d = P.dt_name(self.dtype)
        o, p, s, qk, Vr = A.reference(qh.double().cpu().numpy(), self.kc[:, :, :n].double().cpu().numpy(),
                                      self.vc[:, :, :n].double().cpu().numpy(), self.hd ** -0.5)
        b, budget = A.bound(o, p, s, qk, Vr, self.hd ** -0.5, self.hd, d)
        got = self.out.view(self.B, self.nh, self.hd).double().cpu().numpy()
        worst, rate, n_cond = A.check(got, o, b, budget, d, what)
        w = WORST.setdefault(d, [0.0, 0, 0])
        w[0] = max(w[0], worst)
        w[1] += int(rate * n_cond + 0.5)
        w[2] += n_cond
        return worst, rate


@pytest.mark.parametrize("pos", POSITIONS)
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_kernel(shape, B, dtype, pos):
    nh, nkv, hd = shape
    c = Case(nh, nkv, hd, B, dtype, MAXLEN, pos, seed=pos + 31 * B)
    before = c.kc.clone(), c.vc.clone()
    c.run()
    torch.cuda.synchronize()
    _, kh = c.torch_rope()
    assert torch.equal(_bits(c.kc[:, :, pos]), _bits(kh)), "cache k̂ differs from apply_rotary_pos_emb"
    assert torch.equal(_bits(c.vc[:, :, pos]), _bits(c.v.view(B, nkv, hd)))
    for cache, old in zip((c.kc, c.vc), before):
        assert torch.equal(_bits(cache[:, :, :pos]), _bits(old[:, :, :pos])), "a position below pos changed"
        assert torch.equal(_bits(cache[:, :, pos + 1:]), _bits(old[:, :, pos + 1:])), "a position above pos changed"
    c.check_output(f"{shape} B={B} {dtype} pos={pos}")
    first = c.out.clone()
    c.run()
    assert torch.equal(_bits(c.out), _bits(first)), "two calls differ"
    c.kc[:, :, pos + 1:] = 0
    c.vc[:, :, pos + 1:] = 0
    c.run()
    assert torch.equal(_bits(c.out), _bits(first)), "the output depends on positions above pos"


@pytest.mark.parametrize("pos", [8191, 16383])
def test_kernel_long_context(pos):
    c = Case(32, 32, 128, 1, F16, 16384, pos, seed=5)
    c.run()
    _, kh = c.torch_rope()
    assert torch.equal(_bits(c.kc[:, :, pos]), _bits(kh))
    c.check_output(f"7B 16384 pos={pos}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("shape", [(32, 8, 128), (14, 2, 64)], ids=["32x8x128", "14x2x64"])
def test_kernel_outliers(shape, dtype):
    nh, nkv, hd = shape
    for pos in (17, 1000):
        c = Case(nh, nkv, hd, 2, dtype, 2048, pos, seed=9, outliers=True)
        c.run()
        _, kh = c.torch_rope()
        assert torch.equal(_bits(c.kc[:, :, pos]), _bits(kh))
        c.check_output(f"outliers {shape} {dtype} pos={pos}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_kernel_llama3_rope(dtype):
    c = Case(32, 8, 128, 1, dtype, 16384, 12000, seed=11, kind="llama3")
    c.run()
    _, kh = c.torch_rope()
    assert torch.equal(_bits(c.kc[:, :, 12000]), _bits(kh))
    c.check_output(f"llama3 {dtype}")


def test_graph_replay_follows_pos():
    from autogptq_b200.attention import decode_attention_workspace

    c = Case(32, 8, 128, 2, BF16, 4096, 100, seed=13)
    ws = decode_attention_workspace(2, 32, 8, 128, 4096, "cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        c.run(ws=ws)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c.run(ws=ws)
    for pos in (101, 517, 4095):
        c.set_pos(pos)
        g.replay()
        torch.cuda.synchronize()
        got = c.out.clone()
        c.run(ws=ws)
        assert torch.equal(_bits(got), _bits(c.out)), f"graph replay at pos {pos} differs from the eager call"
        c.check_output(f"graph pos={pos}")


def test_refusals_and_errors():
    from autogptq_b200.attention import decode_attention

    c = Case(32, 2, 128, 1, F16, 64, 3)
    with pytest.raises(NotImplementedError, match="16 query heads"):
        c.run()
    c = Case(32, 8, 128, 1, F16, 64, 3)
    with pytest.raises(ValueError, match="contiguous"):
        strided = torch.empty(1, 2 * 32 * 128, dtype=F16, device="cuda")[:, ::2]
        decode_attention(c.q, c.k, c.v, c.kc, c.vc, c.pos, c.rot.inv_freq, 1.0, 0.1, strided)
    with pytest.raises(ValueError, match="workspace"):
        c.run(ws=torch.zeros(16, dtype=torch.uint8, device="cuda"))


def test_print_worst():
    """Summary line for DESIGN §3.12 (runs after the matrix in file order)."""
    for d, (w, mism, n) in WORST.items():
        print(f"[decode-attention] {d}: largest err/bound {w:.3f}, mismatch {mism}/{n} = {mism / max(n, 1):.4%}")


# --------------------------------------------------------------------------- model level
@functools.lru_cache(maxsize=None)
def _llama3_model(dtype):
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2816, num_attention_heads=8, num_key_value_heads=2,
                      num_hidden_layers=4, vocab_size=512, max_position_embeddings=512, rms_norm_eps=1e-5,
                      rope_parameters={"rope_type": "llama3", "rope_theta": 500000.0, "factor": 8.0,
                                       "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                       "original_max_position_embeddings": 64})
    torch.manual_seed(1)
    m = LlamaForCausalLM(cfg)
    with torch.no_grad():
        for mod in m.modules():
            if type(mod).__name__.endswith("RMSNorm"):
                mod.weight.uniform_(0.5, 1.5)
    m = m.to(dtype).cuda().eval()
    m.config._attn_implementation = "sdpa"
    return _quantize_model(m, dtype)


def _get_model(arch, dtype):
    return _llama3_model(dtype) if arch == "llama3" else _model(arch, dtype)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("arch", ["llama", "qwen2", "llama3"])
def test_decoder_fused_attention_matches_hf(arch, dtype, batch):
    from transformers import DynamicCache

    from autogptq_b200.decoder import ChainDecoder

    model = _get_model(arch, dtype)
    T0, steps = 16, 32
    g = torch.Generator().manual_seed(5 + batch)
    prompt = torch.randint(0, 512, (batch, T0), generator=g).cuda()
    forced = torch.randint(0, 512, (batch, steps), generator=g).cuda()
    dec = ChainDecoder(model, batch=batch, max_length=128, fused_attention=True)
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
        print(f"[decode-attention] decoder {arch} {dtype} batch={batch}: greedy agreement {agree}/{total}")


def test_decoder_fused_generate_matches_steps():
    from autogptq_b200.decoder import ChainDecoder

    model = _model("llama", F16)
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
