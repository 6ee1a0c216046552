"""Prefill attention on the GPU (``agb200_prefill_attention`` / ``_fp8``) and the decoders' ``extend``.

Kernel grid: fp16 / bf16 × hd 64 / 128 × G 1 / 4 / 8 × 16-bit / FP8 cache × (start, T) ∈ {(0,1), (0,17), (0,64), (0,333),
(100,1), (100,63), (4000,96)}, at B = 1 and at B = 3 with a different start per row:
* the new cache rows are bit-equal to apply_rotary_pos_emb(k) and v (16-bit) or to ``quantize_kv`` of them (FP8); every
  other cache byte is unchanged (every position at or past each row's start holds NaN, code 0x7F, NaN scales before the
  call, so a read past the new rows would show);
* every output element is within the ``tests/_prefill_attention.py`` bound of the float64 reference over the cache as
  stored, at the mismatch rates of ``tests/_attention.py``;
* two calls are bit-identical; changing row j's inputs and history leaves the other rows bit-identical.
FP8 histories scale their v rows by 2^-10, 1 and 2^10 in turn, so v scales differ by 2^20 inside every tile.  A row
whose tokens do not fit gets NaN and no cache write.  Chunking (333 = 100 + 200 + 33) writes the same cache bytes as
one call; a T = 1 call writes the same bytes as the decode step.

Model level (the 4-layer Llama and Qwen2 of ``tests/test_gpu_21_chain_norm``): ``BatchDecoder.extend`` on an idle slot
against HF's prefill (layer 0's cache rows bit-equal, logits within ``_logit_tol``, then 32 teacher-forced steps), a
multi-turn conversation, chunked against one call, other slots untouched, ``ChainDecoder.extend``, and FP8 against HF
attending over the decoder's own FP8 rows (HF quantising its own rows, and HF unquantised, printed)."""
import numpy as np
import pytest
import torch

from tests import _attention as A
from tests import _prefill_attention as PA
from tests import _precision as P
from tests._util import assert_parity
from tests.test_gpu_21_chain_norm import _logit_tol, _model
from tests.test_gpu_24_batch_decoder import _rotary
from tests.test_gpu_25_kv_fp8 import _dec_rows, _quantising_cache, _Stats

pytestmark = pytest.mark.gpu

F16, BF16, FP8 = torch.float16, torch.bfloat16, torch.float8_e4m3fn
DTS = [F16, BF16]
L = 4224
CASES = [(0, 1), (0, 17), (0, 64), (0, 333), (100, 1), (100, 63), (4000, 96)]
FIGURES = {"float16": [0.0, 0, 0], "bfloat16": [0.0, 0, 0]}     # largest err/bound, mismatches, elements counted


def _bits(t):
    return t.view(torch.uint8) if t.dtype == FP8 else t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _q(x):
    from autogptq_b200.attention import quantize_kv

    return quantize_kv(x)


class Rows:
    """B rows of T new tokens at ``starts``: random q / k / v, a random history before each start and NaN (FP8: code
    0x7F, NaN scales) from it on."""

    def __init__(self, n_kv, G, hd, B, dtype, fp8, starts, T, seed=0, length=L):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.nh, self.nkv, self.hd, self.B, self.T, self.dtype, self.fp8 = n_kv * G, n_kv, hd, B, T, dtype, fp8
        self.length = length
        self.g = g
        r = lambda *s: torch.randn(*s, generator=g, device="cuda").to(dtype)
        self.q, self.k, self.v = r(B, T, self.nh * hd), r(B, T, n_kv * hd), r(B, T, n_kv * hd)
        self.rot = _rotary(hd)
        self.kc, self.vc = r(B, n_kv, length, hd) * 3, r(B, n_kv, length, hd)
        if fp8:
            tilt = 2.0 ** (10 * (torch.arange(length, device="cuda") % 3 - 1))
            self.vc = (self.vc.float() * tilt[:, None]).to(dtype)
            (self.kc, self.ks), (self.vc, self.vs) = _q(self.kc), _q(self.vc)
        else:
            self.ks = self.vs = None
        self.starts = list(starts)
        for b, s in enumerate(starts):
            self.blank(b, s)
        self.start = torch.tensor(self.starts, dtype=torch.int64, device="cuda")
        self.out = torch.empty(B, T, self.nh * hd, dtype=dtype, device="cuda")

    def caches(self):
        return (self.kc, self.vc) + ((self.ks, self.vs) if self.fp8 else ())

    def blank(self, b, s):
        for t in self.caches():
            if t.dtype == FP8:
                t.view(torch.uint8)[b, :, max(s, 0):] = 0x7F
            else:
                t[b, :, max(s, 0):] = float("nan")

    def run(self, q=None, k=None, v=None, start=None, out=None):
        from autogptq_b200.attention import prefill_attention

        kw = dict(k_scale=self.ks, v_scale=self.vs) if self.fp8 else {}
        return prefill_attention(self.q if q is None else q, self.k if k is None else k, self.v if v is None else v,
                                 self.kc, self.vc, self.start if start is None else start, self.rot.inv_freq,
                                 self.rot.attention_scaling, self.hd ** -0.5, self.out if out is None else out, **kw)

    def expected(self, before, starts, q=None, k=None, v=None):
        """The caches after a call from ``before``: new rows of the rows that fit, everything else unchanged."""
        q, k, v = (self.q if q is None else q), (self.k if k is None else k), (self.v if v is None else v)
        from transformers.models.llama.modeling_llama import apply_rotary_pos_emb

        B, T, hd = q.shape[0], q.shape[1], self.hd
        pid = torch.tensor(starts, device="cuda").clamp(min=0)[:, None] + torch.arange(T, device="cuda")[None]
        cos, sin = self.rot(q, pid)
        _, kh = apply_rotary_pos_emb(q.view(B, T, -1, hd).transpose(1, 2), k.view(B, T, -1, hd).transpose(1, 2),
                                     cos, sin)
        vh = v.view(B, T, -1, hd).transpose(1, 2)
        new = (kh, vh) if not self.fp8 else (lambda a, b: (a[0], b[0], a[1], b[1]))(_q(kh), _q(vh))
        exp = [_bits(t).clone() for t in before]
        for b, s in enumerate(starts):
            if 0 <= s and s + T <= self.length:
                for e, n in zip(exp, new):
                    e[b, :, s:s + T] = _bits(n[b].contiguous())
        return exp

    def check_caches(self, exp, what):
        for t, e in zip(self.caches(), exp):
            assert torch.equal(_bits(t), e), f"{what}: a cache byte differs from the expected write"

    def qhat(self, starts, q=None):
        from transformers.models.llama.modeling_llama import apply_rotary_pos_emb

        q = self.q if q is None else q
        B, T, hd = q.shape[0], q.shape[1], self.hd
        pid = torch.tensor(starts, device="cuda").clamp(min=0)[:, None] + torch.arange(T, device="cuda")[None]
        cos, sin = self.rot(q, pid)
        qh, _ = apply_rotary_pos_emb(q.view(B, T, -1, hd).transpose(1, 2), q.view(B, T, -1, hd).transpose(1, 2),
                                     cos, sin)
        return qh.transpose(1, 2)                                   # [B, T, H, hd]

    def check_output(self, what, starts=None, q=None, out=None, rows=None):
        """Every row that fits within the bound over its cache as stored; the others NaN."""
        starts = self.starts if starts is None else starts
        out = self.out if out is None else out
        T = out.shape[1]
        qh = self.qhat(starts, q).double()
        if self.fp8:
            K = self.kc.double() * self.ks.double()[..., None]
            V = self.vc.double() * self.vs.double()[..., None]
        else:
            K, V = self.kc.double(), self.vc.double()
        dn, sc = P.dt_name(self.dtype), self.hd ** -0.5
        G = self.nh // self.nkv
        o_all = out.view(out.shape[0], T, self.nh, self.hd)
        for b, s in enumerate(starts):
            if rows is not None and b not in rows:
                continue
            if not (0 <= s and s + T <= self.length):
                assert torch.isnan(o_all[b].float()).all(), f"{what}: row {b} does not fit but is not NaN"
                continue
            o, p, sco, qk, Vr = PA.reference(qh[b], K[b], V[b], s, sc)
            Aw = None
            if self.fp8:
                R = self.vs[b, :, :s + T].double().amax(dim=-1)
                Aw = (self.vc[b, :, :s + T].double().abs() * R[:, None, None]).repeat_interleave(G, dim=0)
            bd, budget = PA.bound(o, p, sco, qk, Vr, sc, self.hd, dn, Aw)
            w, m, n = PA.check(o_all[b].double().cpu().numpy(), o, bd, budget, dn, f"{what} row {b} start {s}")
            fig = FIGURES[dn]
            fig[0], fig[1], fig[2] = max(fig[0], w), fig[1] + m, fig[2] + n


def _report(what):
    for dn, (w, m, n) in FIGURES.items():
        print(f"[prefill-attn] {what} {dn}: largest err/bound so far {w:.3f}, mismatches {m}/{n}")


@pytest.mark.parametrize("start,T", CASES, ids=[f"s{s}_T{t}" for s, t in CASES])
@pytest.mark.parametrize("fp8", [False, True], ids=["c16", "fp8"])
@pytest.mark.parametrize("G", [1, 4, 8])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_prefill_attention_grid(dtype, hd, G, fp8, start, T):
    for B, starts in ((1, [start]), (3, [start, start // 2 + 3, start + 1])):
        c = Rows(2, G, hd, B, dtype, fp8, starts, T, seed=start * 7 + T + G * 1000 + hd + B)
        before = [t.clone() for t in c.caches()]
        exp = c.expected(before, starts)
        c.run()
        torch.cuda.synchronize()
        what = f"{dtype} hd={hd} G={G} fp8={fp8} B={B} starts={starts} T={T}"
        c.check_caches(exp, what)
        c.check_output(what)
        first, caches1 = c.out.clone(), [t.clone() for t in c.caches()]
        for t, b in zip(c.caches(), before):
            t.copy_(b)
        c.run()
        assert torch.equal(_bits(c.out), _bits(first)), f"{what}: two calls differ"
        if B < 2:
            continue
        # row j's inputs and history change: every other row's output and cache rows stay bit-identical
        j = B - 1
        for t, b in zip(c.caches(), before):
            t.copy_(b)
        for t in (c.q, c.k, c.v):
            t[j] = torch.randn(t[j].shape, generator=c.g, device="cuda").to(dtype)
        hist = _bits(c.kc)[j, :, :starts[j]]
        hist.copy_(hist.flip(1).clone())
        c.run()
        assert torch.equal(_bits(c.out[:j]), _bits(first[:j])), f"{what}: row {j} changed other rows' outputs"
        for t, u in zip(c.caches(), caches1):
            assert torch.equal(_bits(t[:j]), _bits(u[:j])), f"{what}: row {j} changed other rows' caches"
        c.check_output(what + f" (row {j} changed)", rows=[j])
    _report(f"grid hd={hd} G={G} fp8={fp8}")


@pytest.mark.parametrize("fp8", [False, True], ids=["c16", "fp8"])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_prefill_attention_row_out_of_range(dtype, fp8):
    """start + T > max_length and start < 0: NaN out, the row's cache untouched; the row that fits is unaffected."""
    c = Rows(2, 4, 128, 3, dtype, fp8, [L - 40, 7, -1], 41, seed=5)
    before = [t.clone() for t in c.caches()]
    exp = c.expected(before, c.starts)
    c.run()
    torch.cuda.synchronize()
    c.check_caches(exp, "out of range")
    c.check_output(f"out of range {dtype} fp8={fp8}")


@pytest.mark.parametrize("fp8", [False, True], ids=["c16", "fp8"])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_prefill_attention_chunks_write_the_same_cache(dtype, fp8):
    """One call of 333 tokens against calls of 100, 200 and 33: the same cache bytes; each output within the bound."""
    for s0 in (0, 50):
        one = Rows(2, 4, 128, 2, dtype, fp8, [s0, s0 + 9], 333, seed=11 + s0)
        before = [t.clone() for t in one.caches()]
        one.run()
        one.check_output(f"chunks: one call {dtype} fp8={fp8} start {s0}")
        full = [t.clone() for t in one.caches()]
        for t, b in zip(one.caches(), before):
            t.copy_(b)
        off = 0
        for n in (100, 200, 33):
            st = [s + off for s in one.starts]
            sl = slice(off, off + n)
            q, k, v = (x[:, sl].contiguous() for x in (one.q, one.k, one.v))
            out = torch.empty(2, n, one.nh * one.hd, dtype=dtype, device="cuda")
            one.run(q, k, v, torch.tensor(st, dtype=torch.int64, device="cuda"), out)
            one.check_output(f"chunk {off}+{n} {dtype} fp8={fp8}", starts=st, q=q, out=out)
            off += n
        for t, u in zip(one.caches(), full):
            assert torch.equal(_bits(t), _bits(u)), "chunked calls wrote different cache bytes"
    _report(f"chunks fp8={fp8}")


@pytest.mark.parametrize("fp8", [False, True], ids=["c16", "fp8"])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_prefill_one_token_writes_what_the_decode_step_writes(dtype, fp8):
    from autogptq_b200.attention import decode_attention_rows

    c = Rows(8, 4, 128, 3, dtype, fp8, [0, 33, 700], 1, seed=3, length=1024)
    caches = [t.clone() for t in c.caches()]
    c.run()
    c.check_output(f"T=1 {dtype} fp8={fp8}")
    out = torch.empty(3, c.nh * c.hd, dtype=dtype, device="cuda")
    kw = dict(k_scale=caches[2], v_scale=caches[3]) if fp8 else {}
    decode_attention_rows(c.q[:, 0].contiguous(), c.k[:, 0].contiguous(), c.v[:, 0].contiguous(), caches[0],
                          caches[1], c.start.clone(), c.rot.inv_freq, c.rot.attention_scaling, c.hd ** -0.5, out, **kw)
    for t, u in zip(c.caches(), caches):
        assert torch.equal(_bits(t), _bits(u)), "the prefill and decode kernels wrote different cache bytes"
    # the decode step's output against its own bound, over the same cache
    qh = c.qhat(c.starts)[:, 0].double().cpu().numpy()
    K = (c.kc.double() * c.ks.double()[..., None]) if fp8 else c.kc.double()
    V = (c.vc.double() * c.vs.double()[..., None]) if fp8 else c.vc.double()
    for b, s in enumerate(c.starts):
        o, p, sc, qk, Vr = A.reference(qh[b:b + 1], K[b:b + 1, :, :s + 1].cpu().numpy(),
                                       V[b:b + 1, :, :s + 1].cpu().numpy(), c.hd ** -0.5)
        bd, budget = A.bound(o, p, sc, qk, Vr, c.hd ** -0.5, c.hd, P.dt_name(dtype))
        A.check(out[b:b + 1].view(1, c.nh, c.hd).double().cpu().numpy(), o, bd, budget, P.dt_name(dtype),
                f"decode row {b}")


def test_prefill_attention_argument_errors():
    from autogptq_b200.attention import prefill_attention

    c = Rows(2, 4, 128, 2, F16, True, [0, 5], 8, seed=1, length=256)
    args = (c.q, c.k, c.v, c.kc, c.vc, c.start, c.rot.inv_freq, 1.0, 0.1, c.out)
    with pytest.raises(ValueError, match=r"^prefill_attention: a torch\.float8_e4m3fn cache needs k_scale and v_scale"):
        prefill_attention(*args)
    with pytest.raises(ValueError, match=r"^start must be 2 int64 element\(s\), got torch\.int64 with 1 elements$"):
        prefill_attention(*args[:5], c.start[:1].clone(), *args[6:], k_scale=c.ks, v_scale=c.vs)
    with pytest.raises(ValueError, match=r"^k must be \[2, 8, 256\], got \[2, 7, 256\]$"):
        prefill_attention(c.q, c.k[:, :7].contiguous(), *args[2:], k_scale=c.ks, v_scale=c.vs)
    with pytest.raises(NotImplementedError, match=r"^prefill_attention: batch 9; the kernel takes 1\.\.8"):
        z = torch.zeros
        prefill_attention(z(9, 1, 128, dtype=F16, device="cuda"), z(9, 1, 128, dtype=F16, device="cuda"),
                          z(9, 1, 128, dtype=F16, device="cuda"), z(9, 1, 16, 128, dtype=F16, device="cuda"),
                          z(9, 1, 16, 128, dtype=F16, device="cuda"), z(9, dtype=torch.int64, device="cuda"),
                          c.rot.inv_freq, 1.0, 0.1, z(9, 1, 128, dtype=F16, device="cuda"))


# --------------------------------------------------------------------------- decoders
def _parity(o, r, tol, what, stats=None):
    o, r = o.float().cpu().numpy().reshape(-1, o.shape[-1]), r.float().cpu().numpy().reshape(-1, r.shape[-1])
    assert_parity(o, r, rtol=tol, atol_rms=tol, what=what)
    if stats is not None:
        rms = float(np.sqrt(np.mean(r.astype(np.float64) ** 2)))
        stats[0] = max(stats[0], float((np.abs(o - r) / (tol * np.abs(r) + tol * rms)).max()))


def _tokens(n, seed):
    return torch.randint(0, 512, (n,), generator=torch.Generator().manual_seed(seed)).cuda()


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_batch_extend_matches_hf_prefill(arch, dtype):
    from transformers import DynamicCache

    from autogptq_b200 import BatchDecoder

    model = _model(arch, dtype)
    tol, worst = _logit_tol(dtype, 4), [0.0]
    prompt, forced = _tokens(40, 1), _tokens(32, 2)
    dec = BatchDecoder(model, max_batch=3, max_length=128)
    with torch.no_grad():
        cache = DynamicCache(config=model.config)
        r0 = model(input_ids=prompt[None], past_key_values=cache, use_cache=True).logits[0, -1]
        got = dec.extend(1, prompt)
        assert dec.positions == [-1, 40, -1]
        assert torch.equal(_bits(dec.k_cache[0][1, :, :40]), _bits(cache.layers[0].keys[0])), "layer 0 keys differ"
        assert torch.equal(_bits(dec.v_cache[0][1, :, :40]), _bits(cache.layers[0].values[0])), "layer 0 values differ"
        _parity(got, r0, tol, f"{arch} {dtype} extend", worst)
        for t in range(32):
            ids = torch.zeros(3, dtype=torch.int64, device="cuda")
            ids[1] = forced[t]
            o = dec.step(ids)[1]
            r = model(input_ids=forced[t].view(1, 1), past_key_values=cache, use_cache=True).logits[0, -1]
            _parity(o, r, tol, f"{arch} {dtype} step {t} after extend", worst)
    print(f"[prefill-attn] BatchDecoder.extend {arch} {dtype}: largest logit err / tol {worst[0]:.3f}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_batch_extend_multi_turn(arch, dtype):
    """Prefill 40 tokens, 10 forced steps, extend 25 tokens, 10 more steps: against HF over the whole sequence."""
    from transformers import DynamicCache

    from autogptq_b200 import BatchDecoder

    model = _model(arch, dtype)
    tol, worst = _logit_tol(dtype, 4), [0.0]
    prompt, turn, forced = _tokens(40, 3), _tokens(25, 4), _tokens(20, 5)
    dec = BatchDecoder(model, max_batch=2, max_length=128)
    with torch.no_grad():
        cache = DynamicCache(config=model.config)
        model(input_ids=prompt[None], past_key_values=cache, use_cache=True)
        dec.prefill(0, prompt)

        def steps(ts):
            for t in ts:
                ids = torch.zeros(2, dtype=torch.int64, device="cuda")
                ids[0] = forced[t]
                o = dec.step(ids)[0]
                r = model(input_ids=forced[t].view(1, 1), past_key_values=cache, use_cache=True).logits[0, -1]
                _parity(o, r, tol, f"{arch} {dtype} multi-turn step {t}", worst)

        steps(range(10))
        r = model(input_ids=turn[None], past_key_values=cache, use_cache=True).logits[0, -1]
        _parity(dec.extend(0, turn), r, tol, f"{arch} {dtype} extend of the second turn", worst)
        assert dec.positions == [75, -1]
        steps(range(10, 20))
    print(f"[prefill-attn] multi-turn {arch} {dtype}: largest logit err / tol {worst[0]:.3f}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_batch_extend_in_chunks(dtype):
    from autogptq_b200 import BatchDecoder

    model = _model("llama", dtype)
    tol = _logit_tol(dtype, 4)
    prompt, forced = _tokens(45, 6), _tokens(8, 7)
    a = BatchDecoder(model, max_batch=2, max_length=128)
    b = BatchDecoder(model, max_batch=2, max_length=128)
    with torch.no_grad():
        la = a.extend(0, prompt)
        for off in range(0, 45, 16):
            lb = b.extend(0, prompt[off:off + 16])
        assert a.positions == b.positions == [45, -1]
        _parity(lb, la, tol, f"{dtype} chunks of 16 against one call")
        for t in range(8):
            ids = torch.zeros(2, dtype=torch.int64, device="cuda")
            ids[0] = forced[t]
            _parity(b.step(ids)[0], a.step(ids)[0].clone(), tol, f"{dtype} step {t} after chunks")


def test_batch_extend_leaves_other_slots_bit_identical():
    from autogptq_b200 import BatchDecoder

    model = _model("llama", F16)
    forced = torch.randint(0, 512, (12, 4), generator=torch.Generator().manual_seed(8)).cuda()

    def run(extend_at):
        dec = BatchDecoder(model, max_batch=4, max_length=128)
        with torch.no_grad():
            dec.prefill(0, _tokens(9, 10))
            dec.extend(2, _tokens(14, 11))
            out, snap = [], None
            for t in range(12):
                if t == extend_at:
                    keep = [[c[s].clone() for c in dec.k_cache + dec.v_cache] for s in (0, 2)]
                    pos = dec.positions
                    dec.extend(1, _tokens(21, 12))
                    assert dec.positions == [pos[0], 21, pos[2], -1]
                    snap = [[c[s] for c in dec.k_cache + dec.v_cache] for s in (0, 2)]
                    for k, s in zip(keep, snap):
                        assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(k, s)), "another slot's cache changed"
                out.append(dec.step(forced[t]).clone())
        return out

    base, ev = run(None), run(5)
    for t in range(12):
        assert torch.equal(base[t][[0, 2]], ev[t][[0, 2]]), f"step {t}: an extend changed another slot's logits"


@pytest.mark.parametrize("fused", [False, True], ids=["torch_attn", "fused_attn"])
@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_chain_extend_matches_hf(dtype, batch, fused):
    from transformers import DynamicCache

    from autogptq_b200.decoder import ChainDecoder

    model = _model("llama", dtype)
    tol, worst = _logit_tol(dtype, 4), [0.0]
    g = torch.Generator().manual_seed(20 + batch)
    prompt = torch.randint(0, 512, (batch, 30), generator=g).cuda()
    more = torch.randint(0, 512, (batch, 12), generator=g).cuda()
    forced = torch.randint(0, 512, (16, batch), generator=g).cuda()
    dec = ChainDecoder(model, batch=batch, max_length=128, fused_attention=fused)
    with torch.no_grad():
        cache = DynamicCache(config=model.config)
        r = model(input_ids=prompt, past_key_values=cache, use_cache=True).logits[:, -1]
        _parity(dec.extend(prompt), r, tol, f"chain extend {dtype} B={batch}", worst)
        for t in range(16):
            if t == 8:
                r = model(input_ids=more, past_key_values=cache, use_cache=True).logits[:, -1]
                _parity(dec.extend(more), r, tol, f"chain extend of 12 more {dtype} B={batch}", worst)
            r = model(input_ids=forced[t].view(batch, 1), past_key_values=cache, use_cache=True).logits[:, -1]
            _parity(dec.step(forced[t]), r, tol, f"chain step {t} {dtype} B={batch} fused={fused}", worst)
        assert dec.position == 30 + 12 + 16
    print(f"[prefill-attn] ChainDecoder.extend {dtype} batch={batch} fused={fused}: largest err / tol {worst[0]:.3f}")


def _qdq_attention(module, query, key, value, attention_mask, **kwargs):
    """SDPA over keys and values passed through the FP8 cache format (test-registered attention function)."""
    from transformers.integrations.sdpa_attention import sdpa_attention_forward

    from autogptq_b200.attention import dequantize_kv

    qdq = lambda x: dequantize_kv(*_q(x)).to(x.dtype)  # noqa: E731
    return sdpa_attention_forward(module, query, qdq(key), qdq(value), attention_mask, **kwargs)


def _prompt_rows(dec, i, slot, n):
    """Layer i's cache rows 0 .. n - 1 of ``slot``, dequantised to the dtype: [1, n_kv, n, hd]."""
    from autogptq_b200.attention import dequantize_kv

    return tuple(dequantize_kv(c[i][slot, :, :n], s[i][slot, :, :n]).to(dec.dtype)[None]
                 for c, s in ((dec.k_cache, dec.k_scale), (dec.v_cache, dec.v_scale)))


# The asserted reference attends over the decoder's own FP8 rows, for the prompt as for the steps (the scheme of
# tests/test_gpu_25_kv_fp8.py, see the comment above its ``_qdq``): HF's k̂ of a later layer may differ from the
# decoder's by an ulp, and next to an E4M3 midpoint that ulp moves a code by a whole step.  The registered attention
# function checks each layer's rows against HF's own (``_near_rows``) and attends over them.  HF quantising its own
# rows, and HF unquantised, are printed.
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_fp8_batch_extend_matches_hf(arch, dtype):
    from transformers import AttentionInterface, DynamicCache
    from transformers.integrations.sdpa_attention import sdpa_attention_forward

    from autogptq_b200 import BatchDecoder
    from tests.test_gpu_25_kv_fp8 import _near_rows

    model = _model(arch, dtype)
    tol = _logit_tol(dtype, 4)
    n = 40
    prompt, forced = _tokens(n, 13), _tokens(16, 14)
    dec = BatchDecoder(model, max_batch=2, max_length=128, kv_cache_dtype=FP8)
    st, own, plain = _Stats(tol, 1.0), _Stats(tol, 1.0), _Stats(tol, 1.0)
    moved = dict(tol=tol, moved=0, rows=0)

    def dec_rows_attention(module, query, key, value, attention_mask, **kwargs):
        k, v = _prompt_rows(dec, module.layer_idx, 1, n)
        _near_rows(k, key, moved)
        _near_rows(v, value, moved)
        return sdpa_attention_forward(module, query, k, v, attention_mask, **kwargs)

    AttentionInterface.register("agb_test_qdq_sdpa", _qdq_attention)
    AttentionInterface.register("agb_test_dec_rows_sdpa", dec_rows_attention)
    impl = model.config._attn_implementation
    with torch.no_grad():
        got = dec.extend(1, prompt)
        r_plain = model(input_ids=prompt[None]).logits[0, -1]
        cache = DynamicCache(config=model.config)
        try:
            model.config._attn_implementation = "agb_test_qdq_sdpa"
            r_own = model(input_ids=prompt[None]).logits[0, -1]
            model.config._attn_implementation = "agb_test_dec_rows_sdpa"
            r = model(input_ids=prompt[None], past_key_values=cache, use_cache=True).logits[0, -1]
        finally:
            model.config._attn_implementation = impl
        g = got[None].float().cpu().numpy()
        st.add(g, r[None].float().cpu().numpy(), f"{arch} {dtype} fp8 extend", True)
        own.add(g, r_own[None].float().cpu().numpy(), "", False)
        plain.add(g, r_plain[None].float().cpu().numpy(), "", False)
        for i, lay in enumerate(cache.layers):
            lay.keys, lay.values = _prompt_rows(dec, i, 1, n)
        _quantising_cache(cache, moved)
        for t in range(16):
            ids = torch.zeros(2, dtype=torch.int64, device="cuda")
            ids[1] = forced[t]
            o = dec.step(ids)[1]
            for i, lay in enumerate(cache.layers):
                lay.rows = _dec_rows(dec, i, 1, n + t)
            r = model(input_ids=forced[t].view(1, 1), past_key_values=cache, use_cache=True).logits[0, -1]
            st.add(o[None].float().cpu().numpy(), r[None].float().cpu().numpy(), f"{arch} {dtype} fp8 step {t}", True)
    print(f"[prefill-attn] FP8 BatchDecoder.extend {arch} {dtype}: vs HF over the decoder's FP8 rows: largest err/tol "
          f"{st.worst:.3f}, greedy {st.agree}/{st.total}; rows unlike HF's own quantised ones "
          f"{moved['moved']}/{moved['rows']}; extend vs HF quantising its own rows (not asserted): err/tol "
          f"{own.worst:.3f}; vs unquantised HF (not asserted): err/tol {plain.worst:.3f}")
