"""The FP8 KV cache on the GPU: ``agb200_decode_attention_rows_fp8`` / ``agb200_decode_attention_fp8``, ``quantize_kv``
on CUDA, and BatchDecoder / ChainDecoder with ``kv_cache_dtype=torch.float8_e4m3fn`` against transformers attending
over the decoder's dequantised cache (see the comment above ``_qdq`` for why the decoder's rows, not HF's own).

Attention, B ∈ {1, 2, 3, 5, 8} × fp16 / bf16 × hd {64, 128} × G {1, 4, 6, 7, 8}, rows at positions 0, 31, 32, 33, L - 1 and
idle, as ``tests/test_gpu_24_batch_decoder.py``:
* each active row's new codes and scales are bit-equal to ``quantize_kv`` of apply_rotary_pos_emb(k) and of v; every
  other code and scale byte is unchanged (positions above each row hold code 0x7F and NaN scales, so a read past the
  position would show);
* active rows are within the ``tests/_attention.py`` bound of the float64 reference over the dequantised cache (every
  scale is a power of two, so the kernel's arithmetic is the 16-bit kernel's on those values); idle rows are zero;
* two calls are bit-identical; changing row j leaves every other row bit-identical; a CUDA graph replays as the eager
  calls; with one shared position and B <= 2 the lockstep FP8 entry equals the rows entry.
Long contexts (max_length 4096 and 16384, small and large B·n_kv): every check above at positions where a CTA runs
5 to 8 tiles, so the ring of tile buffers wraps and a partial last tile follows full ones.

Model level: the reference is HF attending over the decoder's own FP8 cache, not HF quantising its own new rows (see
the comment above ``_qdq``)."""
import numpy as np
import pytest
import torch

from autogptq_b200 import _lib
from tests import _attention as A
from tests import _precision as P
from tests._util import assert_parity
from tests.test_gpu_21_chain_norm import _logit_tol, _model
from tests.test_gpu_24_batch_decoder import _hf_runs, _positions, _prompts, _rotary

pytestmark = pytest.mark.gpu

F16, BF16, FP8 = torch.float16, torch.bfloat16, torch.float8_e4m3fn
DTS = [F16, BF16]
L = 256


def _bits(t):
    return t.view(torch.uint8) if t.dtype == FP8 else t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _q(x):
    from autogptq_b200.attention import quantize_kv

    return quantize_kv(x)


def _dq(codes, scale):
    from autogptq_b200.attention import dequantize_kv

    return dequantize_kv(codes, scale)


class Rows8:
    """Random q / k / v and FP8 caches of B independent rows; positions above each row's position hold code 0x7F (NaN)
    and NaN scales."""

    def __init__(self, n_kv, G, hd, B, dtype, pos, seed=0, length=L):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.nh, self.nkv, self.hd, self.B, self.dtype = n_kv * G, n_kv, hd, B, dtype
        r = lambda *s: torch.randn(*s, generator=g, device="cuda").to(dtype)
        self.q, self.k, self.v = r(B, self.nh * hd), r(B, n_kv * hd), r(B, n_kv * hd)
        self.kc, self.ks = _q(r(B, n_kv, length, hd) * 3)
        self.vc, self.vs = _q(r(B, n_kv, length, hd))
        self.rot = _rotary(hd)
        self.pos = torch.zeros(B, dtype=torch.int64, device="cuda")
        self.out = torch.empty(B, self.nh * hd, dtype=dtype, device="cuda")
        self.orig = [t.clone() for t in (self.kc, self.ks, self.vc, self.vs)]
        self.p = [-1] * B
        self.set_pos(pos)

    def caches(self):
        return self.kc, self.ks, self.vc, self.vs

    def set_pos(self, pos):
        """Move each row to its position: positions a row skips get their original values, those above it NaN."""
        for b, p in enumerate(pos):
            lo = self.p[b] + 1
            for t, o in zip(self.caches(), self.orig):
                if p > lo:
                    t[b, :, lo:p] = o[b, :, lo:p]
                if t.dtype == FP8:
                    t.view(torch.uint8)[b, :, p + 1:] = 0x7F
                else:
                    t[b, :, p + 1:] = float("nan")
        self.p = list(pos)
        self.pos.copy_(torch.tensor(self.p))

    def run(self, out=None, ws=None):
        from autogptq_b200.attention import decode_attention_rows

        return decode_attention_rows(self.q, self.k, self.v, self.kc, self.vc, self.pos, self.rot.inv_freq,
                                     self.rot.attention_scaling, self.hd ** -0.5, self.out if out is None else out, ws,
                                     k_scale=self.ks, v_scale=self.vs)

    def torch_rope(self):
        from transformers.models.llama.modeling_llama import apply_rotary_pos_emb

        B, hd = self.B, self.hd
        pid = self.pos.clamp(min=0).view(B, 1)
        cos, sin = self.rot(self.q.view(B, 1, -1), pid)
        qh, kh = apply_rotary_pos_emb(self.q.view(B, 1, self.nh, hd).transpose(1, 2),
                                      self.k.view(B, 1, self.nkv, hd).transpose(1, 2), cos, sin)
        return qh[:, :, 0], kh[:, :, 0]

    def check_caches(self, before):
        """New codes and scales bit-equal to quantize_kv of torch's k̂ and of v; every other byte unchanged."""
        _, kh = self.torch_rope()
        kq, vq = _q(kh), _q(self.v.view(self.B, self.nkv, self.hd))
        for cache, old, new in zip(self.caches(), before, (kq[0], kq[1], vq[0], vq[1])):
            exp = _bits(old).clone()
            for b, p in enumerate(self.p):
                if p >= 0:
                    exp[b, :, p] = _bits(new[b])
            assert torch.equal(_bits(cache), exp), "a cache code or scale differs from the expected write"

    def check_output(self, what):
        qh, _ = self.torch_rope()
        K, V = _dq(self.kc, self.ks), _dq(self.vc, self.vs)
        out = self.out.view(self.B, self.nh, self.hd).double().cpu().numpy()
        qh, K, V = qh.double().cpu().numpy(), K.double().cpu().numpy(), V.double().cpu().numpy()
        dn, sc = P.dt_name(self.dtype), self.hd ** -0.5
        for b, p in enumerate(self.p):          # tests/_batch_attention.py's check_rows, keeping the figures
            if p < 0:
                assert (out[b] == 0).all(), f"{what}: idle row {b} is not zero"
                continue
            ob, pb, sb, qk, Vr = A.reference(qh[b:b + 1], K[b:b + 1, :, :p + 1], V[b:b + 1, :, :p + 1], sc)
            bd, budget = A.bound(ob, pb, sb, qk, Vr, sc, self.hd, dn)
            w, rate, n = A.check(out[b:b + 1], ob, bd, budget, dn, f"{what} row {b} pos {p}")
            fig = FIGURES[dn]
            fig[0], fig[1], fig[2] = max(fig[0], w), fig[1] + round(rate * n), fig[2] + n


FIGURES = {"float16": [0.0, 0, 0], "bfloat16": [0.0, 0, 0]}     # largest err/bound, mismatches, elements counted


def _report(what):
    for dn, (w, m, n) in FIGURES.items():
        print(f"[kv-fp8] {what} {dn}: largest err/bound so far {w:.3f}, mismatch rate {m}/{n}")


@pytest.mark.parametrize("G", [1, 4, 6, 7, 8])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("B", [1, 2, 3, 5, 8])
def test_fp8_attention_rows(B, dtype, hd, G):
    for shift in (0, 2, 3, 5):
        pos = _positions(B, shift)
        c = Rows8(2, G, hd, B, dtype, pos, seed=B * 100 + G * 10 + shift)
        before = [t.clone() for t in c.caches()]
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
        keep = [t.clone() for t in c.caches()]
        g = torch.Generator(device="cuda").manual_seed(7 + shift)
        for t in (c.q, c.k, c.v):
            t[j] = torch.randn(t.shape[1], generator=g, device="cuda").to(dtype)
        for pair in ((0, 1), (2, 3)):
            codes, sc = _q(torch.randn(c.kc[j].shape, generator=g, device="cuda").to(dtype))
            for i, t in zip(pair, (codes, sc)):
                c.caches()[i][j] = t
                c.orig[i][j] = t
        c.set_pos(c.p[:j] + [17 if c.p[j] != 17 else -1])
        before = [t.clone() for t in c.caches()]
        c.run()
        assert torch.equal(_bits(c.out[:j]), _bits(first[:j])), f"row {j} changed other rows' outputs"
        for t, k in zip(c.caches(), keep):
            assert torch.equal(_bits(t[:j]), _bits(k[:j])), f"row {j} changed other rows' caches"
        c.check_caches(before)
        c.check_output(f"B={B} {dtype} hd={hd} G={G} pos={c.p} (row {j} changed)")
    _report(f"grid B={B} hd={hd} G={G}")


def _splits(B, n_heads, n_kv, hd, length):
    """The kernel's split count S, read back from the workspace size: counter words, then S partials per (b, kv head)
    of attn_part_floats(G, hd) = G·hd + 16 floats (csrc/attention.cu)."""
    lib = _lib.load()
    ws = int(lib.agb200_decode_attention_workspace_bytes(B, n_heads, n_kv, hd, length))
    counters = -(-B * n_kv * 4 // 256) * 256
    return (ws - counters) // (B * n_kv * (n_heads // n_kv * hd + 16) * 4)


LONG = {"B2_kv2_16384": (2, 2, 16384, [16383, 10000]),
        "B8_kv4_4096": (8, 4, 4096, [4095, 2047, 1000, -1, 700, 3500, 160, 4000])}


@pytest.mark.parametrize("G", [1, 8])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("shape", list(LONG))
def test_fp8_attention_rows_long_context(shape, dtype, hd, G):
    """The ring of tile buffers in steady state: CTAs of 5 to 8 tiles, the last one partial."""
    B, n_kv, length, pos = LONG[shape]
    S = _splits(B, n_kv * G, n_kv, hd, length)
    tiles = [-(-(-(-(p + 1) // S)) // 32) for p in pos if p >= 0]
    assert max(tiles) >= 5 and min(t for t in tiles if t > 1) < max(tiles), f"S={S}: tiles per CTA {tiles}"
    c = Rows8(n_kv, G, hd, B, dtype, pos, seed=length + B + G, length=length)
    before = [t.clone() for t in c.caches()]
    c.run()
    torch.cuda.synchronize()
    c.check_caches(before)
    c.check_output(f"{shape} {dtype} hd={hd} G={G} S={S} tiles={tiles}")
    first = c.out.clone()
    c.run()
    assert torch.equal(_bits(c.out), _bits(first)), "two calls differ"
    if B <= 2:                                   # the lockstep entry at one shared position, same kernel
        from autogptq_b200.attention import decode_attention

        c.set_pos([pos[0]] * B)
        caches, out = [t.clone() for t in c.caches()], torch.empty_like(c.out)
        kc, ks, vc, vs = caches
        p1 = torch.tensor([pos[0]], dtype=torch.int64, device="cuda")
        decode_attention(c.q, c.k, c.v, kc, vc, p1, c.rot.inv_freq, c.rot.attention_scaling, c.hd ** -0.5, out,
                         k_scale=ks, v_scale=vs)
        c.run()
        assert torch.equal(_bits(c.out), _bits(out)), "the lockstep entry differs from the rows entry"
        c.check_output(f"{shape} {dtype} hd={hd} G={G} shared pos {pos[0]}")
    _report(f"long {shape} hd={hd} G={G}")


@pytest.mark.parametrize("B", [3, 8])
def test_fp8_attention_rows_graph_replay(B):
    from autogptq_b200.attention import decode_attention_workspace

    c = Rows8(8, 4, 128, B, BF16, _positions(B, 1), seed=13)
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
def test_fp8_lockstep_entry_equals_rows_entry(B, dtype):
    from autogptq_b200.attention import decode_attention

    for pos in (0, 33, L - 1):
        a = Rows8(8, 4, 128, B, dtype, [pos] * B, seed=pos)
        caches, out = [t.clone() for t in a.caches()], torch.empty_like(a.out)
        p1 = torch.tensor([pos], dtype=torch.int64, device="cuda")
        kc, ks, vc, vs = caches
        decode_attention(a.q, a.k, a.v, kc, vc, p1, a.rot.inv_freq, a.rot.attention_scaling, a.hd ** -0.5, out,
                         k_scale=ks, v_scale=vs)
        a.run()
        assert torch.equal(_bits(a.out), _bits(out)), f"pos {pos}: outputs differ from decode_attention"
        for t, u in zip(a.caches(), caches):
            assert torch.equal(_bits(t), _bits(u))


def test_fp8_attention_refusals():
    from autogptq_b200.attention import decode_attention_rows

    c = Rows8(8, 4, 128, 3, F16, [1, 2, 3])
    args = (c.q, c.k, c.v, c.kc, c.vc, c.pos, c.rot.inv_freq, 1.0, 0.1, c.out)
    with pytest.raises(ValueError, match="needs k_scale and v_scale"):
        decode_attention_rows(*args)
    with pytest.raises(ValueError, match="k_scale must be"):
        decode_attention_rows(*args, k_scale=c.ks[:, :, :8].contiguous(), v_scale=c.vs)
    with pytest.raises(ValueError, match="the activations"):
        decode_attention_rows(c.q, c.k.to(BF16), *args[2:], k_scale=c.ks, v_scale=c.vs)
    with pytest.raises(ValueError, match="go with a"):
        decode_attention_rows(c.q, c.k, c.v, c.q.new_zeros(3, 8, L, 128), c.q.new_zeros(3, 8, L, 128), *args[5:],
                              k_scale=c.ks, v_scale=c.vs)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_quantize_kv_cuda_equals_cpu(dtype):
    g = torch.Generator().manual_seed(2)
    mags = [2.0 ** k for k in range(-12, 14, 2)] if dtype == F16 else [2.0 ** k for k in range(-100, 100, 9)]
    x = torch.cat([(torch.randn(64, 128, generator=g, dtype=torch.float64) * m).to(dtype) for m in mags])
    x[::9] = 0
    x[1::9, ::3] = 2.0 ** -9 * 0.5 * x[1::9, ::3].abs().amax(-1, keepdim=True) / 448      # ties near zero
    cc, cs = _q(x)
    gc, gs = _q(x.cuda())
    assert torch.equal(_bits(gc).cpu(), _bits(cc)) and torch.equal(_bits(gs).cpu(), _bits(cs))


# --------------------------------------------------------------------------- decoders
# The reference attends over the decoder's own cache.  Quantisation is discontinuous: a new row's k̂ or v from HF and
# from the decoder may differ by an ulp (the tolerance below allows it), and next to an E4M3 rounding midpoint or a
# scale boundary that ulp moves a code by a whole E4M3 step (6-12 %) or the row to another grid.  So HF's cache takes
# the decoder's new rows (dequantised), after checking that they are HF's own quantised rows up to such moves; what
# remains between the two is the 16-bit arithmetic that ``_logit_tol`` covers.  The kernel's quantisation of its own
# inputs is pinned bit for bit above.
def _qdq(x):
    c, s = _q(x)
    return _dq(c, s).to(x.dtype)


def _near_rows(got, x, stats):
    """The decoder's dequantised rows against HF's unquantised rows x: apart by at most half an E4M3 step (of a grid up
    to twice as coarse, for a row that moved to the next scale) plus the 16-bit difference ``stats["tol"]`` allows,
    relative to the row's largest value, twice over (this catches a wrong row, position or layer).  Counts the rows
    that differ from HF's own quantised rows."""
    g, h = got.float(), x.float()
    a = h.abs().amax(-1, keepdim=True)
    bound = 2.0 ** -4 * h.abs() + 2.0 ** -9 * (a / 224.0) + 2 * stats["tol"] * a
    assert ((g - h).abs() <= bound).all(), "a new cache row is not HF's row, quantised"
    stats["moved"] += int((g != _qdq(x).float()).any(-1).sum())
    stats["rows"] += g[..., 0].numel()


def _quantising_cache(cache, stats):
    """A prefilled DynamicCache made to hold dequant(quant(x)) of its rows; each later update appends the rows set in
    ``layer.rows`` (the decoder's) after checking them against the update's own rows quantised."""
    def update(self, key_states, value_states, *args, **kwargs):
        rows = self.rows
        self.rows = None
        for got, x in zip(rows, (key_states, value_states)):
            _near_rows(got, x, stats)
        return super(type(self), self).update(*rows, *args, **kwargs)

    for lay in cache.layers:
        lay.keys, lay.values = _qdq(lay.keys), _qdq(lay.values)
        lay.__class__ = type("Quantising" + type(lay).__name__, (type(lay),), {"update": update})
        lay.rows = None
    return cache


def _dec_rows(dec, i, index, pos):
    """Layer i's cache rows at ``pos`` for ``index`` (slot or all rows), dequantised to the dtype: [b, n_kv, 1, hd]."""
    k = _dq(dec.k_cache[i][index][..., pos, :], dec.k_scale[i][index][..., pos])
    v = _dq(dec.v_cache[i][index][..., pos, :], dec.v_scale[i][index][..., pos])
    return tuple(t.to(dec.dtype).reshape(-1, t.shape[-2], 1, t.shape[-1]) for t in (k, v))


class _Stats:
    """Largest logit error over tol and greedy agreement (printed against the unquantised run, asserted otherwise)."""

    def __init__(self, tol, factor):
        self.tol, self.factor, self.worst, self.agree, self.total = tol, factor, 0.0, 0, 0

    def add(self, o, r, what, check):
        rms = float(np.sqrt(np.mean(r.astype(np.float64) ** 2)))
        tol = self.tol
        self.worst = max(self.worst, float((np.abs(o - r) / (tol * np.abs(r) + tol * rms)).max()))
        same = r.argmax(-1) == o.argmax(-1)
        if check:
            assert_parity(o, r, rtol=self.factor * tol, atol_rms=self.factor * tol, what=what)
            top2 = np.sort(r, axis=-1)[:, -2:]
            clear = top2[:, 1] - top2[:, 0] > 2 * self.factor * (tol * np.abs(top2[:, 1]) + tol * rms)
            assert same[clear].all(), f"{what}: greedy token differs where the reference margin is clear"
        self.agree += int(same.sum())
        self.total += same.size


def _batch_decoder_vs_hf(arch, dtype, max_batch, slots, prompts, steps, max_length):
    """BatchDecoder(kv_cache_dtype=FP8) with ``prompts`` in ``slots``, ``steps`` teacher-forced steps, against HF on
    each sequence alone over the decoder's cache (asserted) and over an unquantised cache (printed)."""
    from transformers import DynamicCache

    from autogptq_b200 import BatchDecoder

    model = _model(arch, dtype)
    g = torch.Generator().manual_seed(3)
    forced = [torch.randint(0, 512, (steps,), generator=g).cuda() for _ in slots]
    plain = _hf_runs(model, prompts, forced, steps)
    dec = BatchDecoder(model, max_batch=max_batch, max_length=max_length, kv_cache_dtype=FP8)
    tol = _logit_tol(dtype, 4)
    factor = 1.5 if max_batch > _lib.GEMV_MAX_M and dtype == F16 else 1.0     # as tests/test_gpu_24_batch_decoder.py
    st, sp, moved = _Stats(tol, factor), _Stats(tol, factor), dict(tol=factor * tol, moved=0, rows=0)
    caches = []
    with torch.no_grad():
        for k, s in enumerate(slots):
            cache = DynamicCache(config=model.config)
            r0 = model(input_ids=prompts[k][None], past_key_values=cache, use_cache=True).logits[0, -1]
            assert torch.equal(dec.prefill(s, prompts[k]), r0), "prefill logits differ from HF's"
            caches.append(_quantising_cache(cache, moved))
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
            ref = []
            for k, s in enumerate(slots):
                pos = len(prompts[k]) + t
                for i, lay in enumerate(caches[k].layers):
                    lay.rows = _dec_rows(dec, i, s, pos)
                ref.append(model(input_ids=forced[k][t].view(1, 1), past_key_values=caches[k],
                                 use_cache=True).logits[0, -1])
            o = got[slots].float().cpu().numpy()
            what = f"{arch} {dtype} max_batch={max_batch} max_length={max_length} step {t}"
            st.add(o, torch.stack(ref).float().cpu().numpy(), what, True)
            sp.add(o, torch.stack([plain[k][t + 1] for k in range(len(slots))]).float().cpu().numpy(), what, False)
    print(f"[kv-fp8] BatchDecoder {arch} {dtype} max_batch={max_batch} max_length={max_length}: vs HF on the "
          f"decoder's FP8 cache: greedy {st.agree}/{st.total}, largest err/tol {st.worst:.3f}; new rows unlike HF's "
          f"own quantised ones {moved['moved']}/{moved['rows']}; vs HF unquantised (not asserted): greedy "
          f"{sp.agree}/{sp.total}, largest err/tol {sp.worst:.3f}")


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("max_batch", [3, 8])
@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_fp8_batch_decoder_matches_hf(arch, max_batch, dtype):
    slots = [s for s in range(max_batch) if not (max_batch == 8 and s == 5)]     # max_batch 8: slot 5 stays idle
    _batch_decoder_vs_hf(arch, dtype, max_batch, slots, _prompts(len(slots), seed=max_batch), 32, 128)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
def test_fp8_batch_decoder_long_context(dtype):
    """Prompts of 4300 and 2000 tokens in slots 0 and 5 of 8: the attention's CTAs run 5 and 2 tiles per split."""
    S = _splits(8, 8, 2, 128, 4400)
    assert -(-(-(-4301 // S)) // 32) >= 5, f"S={S}"
    _batch_decoder_vs_hf("llama", dtype, 8, [0, 5], _prompts(2, seed=17, lo=4300, step=-2300), 8, 4400)


@pytest.mark.parametrize("dtype", DTS, ids=["f16", "bf16"])
@pytest.mark.parametrize("batch", [1, 2])
def test_fp8_chain_decoder_matches_hf(batch, dtype):
    from transformers import DynamicCache

    from autogptq_b200.decoder import ChainDecoder

    model = _model("llama", dtype)
    steps = 32
    g = torch.Generator().manual_seed(9)
    prompt = torch.randint(0, 512, (batch, 13), generator=g).cuda()
    forced = torch.randint(0, 512, (steps, batch), generator=g).cuda()
    dec = ChainDecoder(model, batch=batch, max_length=128, fused_attention=True, kv_cache_dtype=FP8)
    tol = _logit_tol(dtype, 4)
    st, moved = _Stats(tol, 1.0), dict(tol=tol, moved=0, rows=0)
    with torch.no_grad():
        cache = DynamicCache(config=model.config)
        r0 = model(input_ids=prompt, past_key_values=cache, use_cache=True).logits[:, -1]
        assert torch.equal(dec.prefill(prompt), r0), "prefill logits differ from HF's"
        _quantising_cache(cache, moved)
        for t in range(steps):
            got = dec.step(forced[t])
            for i, lay in enumerate(cache.layers):
                lay.rows = _dec_rows(dec, i, slice(None), 13 + t)
            r = model(input_ids=forced[t].view(batch, 1), past_key_values=cache, use_cache=True).logits[:, -1]
            st.add(got.float().cpu().numpy(), r.float().cpu().numpy(), f"ChainDecoder fp8 B={batch} {dtype} step {t}",
                   True)
    print(f"[kv-fp8] ChainDecoder batch={batch} {dtype}: greedy {st.agree}/{st.total}, largest err/tol {st.worst:.3f}; "
          f"new rows unlike HF's own quantised ones {moved['moved']}/{moved['rows']}")


def _run_slots(model, events, steps=30, B=4):
    from autogptq_b200 import BatchDecoder

    dec = BatchDecoder(model, max_batch=B, max_length=128, kv_cache_dtype=FP8)
    prompts = _prompts(3, seed=21, lo=7, step=5)
    for s, p in enumerate(prompts):
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


def test_fp8_admit_and_release_leave_other_slots_bit_identical():
    model = _model("llama", F16)
    base = _run_slots(model, {})
    late = _prompts(1, seed=5, lo=11)[0]
    ev = _run_slots(model, {10: ("admit", 3, late), 20: ("release", 1)})
    for t in range(len(base)):
        keep = [0, 2] + ([1] if t < 20 else [])
        assert torch.equal(base[t][keep], ev[t][keep]), f"step {t}: an admit / release changed another slot's logits"


def test_fp8_reused_slot_equals_fresh_decoder():
    from autogptq_b200 import BatchDecoder

    model = _model("llama", BF16)
    long_p, short_p = _prompts(2, seed=8, lo=40, step=-30)
    ids = torch.randint(0, 512, (6, 4), generator=torch.Generator().manual_seed(6)).cuda()
    with torch.no_grad():
        dec = BatchDecoder(model, max_batch=4, max_length=128, kv_cache_dtype=FP8)
        dec.prefill(0, long_p)
        dec.prefill(2, short_p)
        for t in range(12):
            dec.step(ids[t % 6])
        dec.release(0)
        dec.release(2)
        a = [dec.prefill(0, short_p).clone()] + [dec.step(ids[t]).clone()[0] for t in range(6)]
        fresh = BatchDecoder(model, max_batch=4, max_length=128, kv_cache_dtype=FP8)
        b = [fresh.prefill(0, short_p).clone()] + [fresh.step(ids[t]).clone()[0] for t in range(6)]
    for t, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f"step {t}: a reused slot differs from a fresh decoder"


def test_fp8_cache_memory():
    from autogptq_b200 import BatchDecoder

    model = _model("qwen2", BF16)
    nbytes = lambda ts: sum(t.numel() * t.element_size() for t in ts)
    a = BatchDecoder(model, max_batch=8, max_length=512)
    b = BatchDecoder(model, max_batch=8, max_length=512, kv_cache_dtype=FP8)
    assert a.k_scale is None and b.k_cache[0].dtype == FP8 and b.k_scale[0].shape == (8, 2, 512)
    hd = a.head_dim
    full = nbytes(a.k_cache + a.v_cache)
    small = nbytes(b.k_cache + b.v_cache + b.k_scale + b.v_scale)
    assert small * 2 * hd == full * (hd + 4), f"{small} bytes against {full}"
