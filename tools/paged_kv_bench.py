"""The paged KV cache (DESIGN §3.22) against the static one, in one run:

    python tools/paged_kv_bench.py [--reps 20] [--repeats 3] [--layers 8] [--steps 64] [--parts attn,step,bytes,gen]

1. attn: the per-row decode attention of one layer, paged (scrambled table) against static on the same contents, at
   Llama-2-7B (32 kv heads) and Llama-3-8B (8 kv heads) shapes, hd 128, B 1 and 8 with every row at the context's
   last position, contexts 512 .. 16384, block sizes 16 / 64 / 256, 16-bit and FP8: µs per call (CUDA graph of ``reps``
   calls, events) and the cache bytes read per second.
2. step: the BatchDecoder step (fp16, synthetic Llama-2-7B-shaped GPTQ model of ``--layers`` layers) at 8 rows with
   ragged positions 256..768 and 7000..8000, static against paged (block size 16), ms per step.
3. bytes: the cache bytes of one 30K-token slot and seven 1K-token slots at max_length 32768, Llama-2-7B shapes,
   static against paged (block size 16), computed from the shapes.
4. gen: ``generate(n=4)`` from one 2048-token prompt against four separate copies of it (n=1, the same four seeds), on
   the paged decoder: seconds and the most pool blocks in use.

Each comparison alternates its arms and runs ``repeats`` times; the JSON line has every repeat, the GPU name and power
limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.batch_decoder_bench import ragged  # noqa: E402
from tools.chain_decoder_bench import build_model, gpu_facts, time_graph, timed_steps  # noqa: E402

FP8 = torch.float8_e4m3fn


def attn_part(reps, repeats):
    from autogptq_b200.attention import decode_attention_rows, decode_attention_rows_paged, decode_attention_workspace
    from tests import _paged as PG

    dev, hd, nh, out = "cuda", 128, 32, []
    inv = (1.0 / 10000.0 ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd)).to(dev)
    for model, nkv in (("llama2-7b", 32), ("llama3-8b", 8)):
        for B in (1, 8):
            for ctx in (512, 1024, 2048, 4096, 8192, 16384):
                for fp8 in (False, True):
                    g = torch.Generator(device=dev).manual_seed(ctx)
                    shape = (B, nkv, ctx, hd)
                    kc = torch.randn(shape, generator=g, device=dev).half()
                    vc = torch.randn(shape, generator=g, device=dev).half()
                    kw = {}
                    if fp8:
                        from autogptq_b200.attention import quantize_kv
                        (kc, ks), (vc, vs) = quantize_kv(kc), quantize_kv(vc)
                        kw = dict(k_scale=ks, v_scale=vs)
                    q = torch.randn((B, nh * hd), generator=g, device=dev).half()
                    k = torch.randn((B, nkv * hd), generator=g, device=dev).half()
                    v = torch.randn((B, nkv * hd), generator=g, device=dev).half()
                    pos = torch.full((B,), ctx - 1, dtype=torch.int64, device=dev)
                    o = torch.empty_like(q)
                    ws = decode_attention_workspace(B, nh, nkv, hd, ctx, dev)
                    arms = {"static": lambda: decode_attention_rows(q, k, v, kc, vc, pos, inv, 1.0, hd ** -0.5, o, ws,
                                                                    **kw)}
                    pools = {}
                    for bs in (16, 64, 256):
                        mb = ctx // bs
                        table = PG.make_table(B, mb, B * mb, "scrambled", seed=bs)
                        pk, pv = (torch.empty((B * mb, nkv, bs, hd), dtype=kc.dtype, device=dev) for _ in range(2))
                        PG.scatter(pk.view(torch.uint8) if fp8 else pk, table, kc.view(torch.uint8) if fp8 else kc)
                        PG.scatter(pv.view(torch.uint8) if fp8 else pv, table, vc.view(torch.uint8) if fp8 else vc)
                        pkw = {}
                        if fp8:
                            pks, pvs = (torch.empty((B * mb, nkv, bs), device=dev) for _ in range(2))
                            PG.scatter(pks, table, ks)
                            PG.scatter(pvs, table, vs)
                            pkw = dict(k_scale=pks, v_scale=pvs)
                        t = torch.from_numpy(table).to(dev)
                        pools[bs] = (pk, pv, t, pkw)
                        arms[f"paged{bs}"] = (lambda pk=pk, pv=pv, t=t, pkw=pkw: decode_attention_rows_paged(
                            q, k, v, pk, pv, t, pos, inv, 1.0, hd ** -0.5, o, ws, **pkw))
                    times = {a: [] for a in arms}
                    for _ in range(repeats):
                        for a, fn in arms.items():
                            times[a].append(time_graph(fn, reps) * 1e3)      # µs per call
                    per_row = 2 * ctx * nkv * (hd * (1 if fp8 else 2) + (4 if fp8 else 0))
                    rec = {"model": model, "B": B, "ctx": ctx, "kv": "fp8" if fp8 else "fp16",
                           "us": {a: [round(x, 2) for x in ts] for a, ts in times.items()},
                           "GBps": {a: round(B * per_row / (min(ts) * 1e-6) / 1e9, 1) for a, ts in times.items()}}
                    print(json.dumps(rec), flush=True)
                    out.append(rec)
                    del pools, arms, kc, vc
    return out


def _fill(dec, s, T, gen):
    """Synthetic N(0, 1) keys and values at positions :T of slot s (blocks reserved first on a paged cache)."""
    dec._cache.reserve({s: T})
    for i, k in enumerate(dec.k_cache):
        shape = (1, dec.n_kv, T, dec.head_dim)
        x = [torch.randn(shape, generator=gen, device=k.device).half() for _ in range(2)]
        dec._cache.store(i, slice(s, s + 1), *x)
    dec._pos[s] = T
    dec._host_pos[s] = T


def step_part(layers, steps, repeats):
    from autogptq_b200.batch_decoder import BatchDecoder

    dev, out = "cuda", []
    model = build_model(layers, 8, dev)
    for lo, hi in ((256, 768), (7000, 8000)):
        lengths = ragged(8, (lo + hi) // 2, (hi - lo) // 2)
        L = hi + steps * (repeats + 2) + 64
        decs = {"static": BatchDecoder(model, 8, L), "paged16": BatchDecoder(model, 8, L, kv_block_size=16)}
        gen = torch.Generator(device=dev).manual_seed(2)
        for d in decs.values():
            for s, T in enumerate(lengths):
                _fill(d, s, T, gen)
        tok = torch.randint(0, 32000, (8,), device=dev, generator=gen)
        times = {a: [] for a in decs}
        for d in decs.values():
            for _ in range(3):
                d.step(tok)
        for _ in range(repeats):
            for a, d in decs.items():
                times[a].append(timed_steps(lambda t, d=d: d.step(t).argmax(-1), tok, steps))
        rec = {"positions": [lo, hi], "layers": layers, "ms_per_step": {a: [round(x, 3) for x in ts]
                                                                        for a, ts in times.items()}}
        print(json.dumps(rec), flush=True)
        out.append(rec)
        del decs
        torch.cuda.empty_cache()
    return out


def bytes_part():
    n_kv, hd, layers, elt, bs = 32, 128, 32, 2, 16
    per_token = 2 * n_kv * hd * elt * layers
    static = 8 * 32768 * per_token
    blocks = -(-30000 // bs) + 7 * -(-1000 // bs)
    paged = blocks * bs * per_token
    return {"static_GB": round(static / 1e9, 2), "paged_GB": round(paged / 1e9, 2), "blocks": blocks,
            "fp8_static_GB": round(8 * 32768 * 2 * n_kv * (hd + 4) * layers / 1e9, 2),
            "fp8_paged_GB": round(blocks * bs * 2 * n_kv * (hd + 4) * layers / 1e9, 2)}


def gen_part(layers, repeats):
    from autogptq_b200.batch_decoder import BatchDecoder
    from autogptq_b200.sampling import SamplingParams

    dev = "cuda"
    model = build_model(layers, 8, dev)
    dec = BatchDecoder(model, 8, 2048 + 128, kv_block_size=16)
    p = torch.randint(0, 32000, (2048,), generator=torch.Generator().manual_seed(3))
    sp = [SamplingParams(temperature=0.8, top_k=50, seed=10 + i) for i in range(4)]
    peak = [0]
    reserve = dec._cache.reserve

    def tracked(need):
        reserve(need)
        peak[0] = max(peak[0], dec.kv_blocks - dec.kv_blocks_free)
    dec._cache.reserve = tracked

    def fork():
        return dec.generate([p], 64, sampling=sp[0], n=4)

    def separate():
        return dec.generate([p] * 4, 64, sampling=sp)
    res = {"fork": {"s": [], "peak_blocks": 0}, "separate": {"s": [], "peak_blocks": 0}}
    fork(), separate()                                     # capture and warm up
    for _ in range(repeats):
        for name, fn in (("fork", fork), ("separate", separate)):
            peak[0] = 0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            res[name]["s"].append(round(time.perf_counter() - t0, 3))
            res[name]["peak_blocks"] = peak[0]
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--parts", default="attn,step,bytes,gen")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("paged_kv_bench needs a CUDA device")
    name, power = gpu_facts()
    parts = args.parts.split(",")
    rec = {"gpu": name, "power_limit": power}
    with torch.no_grad():
        if "bytes" in parts:
            rec["bytes"] = bytes_part()
        if "attn" in parts:
            rec["attn"] = attn_part(args.reps, args.repeats)
        if "step" in parts:
            rec["step"] = step_part(args.layers, args.steps, args.repeats)
        if "gen" in parts:
            rec["gen"] = gen_part(args.layers, args.repeats)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
