"""Aggregate decode throughput of a Llama-2-7B-shaped GPTQ model with BatchDecoder at max_batch 1, 2, 4 and 8 (every
slot active, ragged positions), next to ChainDecoder(fused_attention=True) at batch 1 and 2 from the same run.

    python tools/batch_decoder_bench.py [--layers 32] [--batches 1,2,4,8] [--steps 128] [--prompt 512] [--spread 256]
                                        [--max-length 0] [--kv-cache {dtype,fp8,both}]

Weights are synthetic, built as ``tools/chain_decoder_bench.py`` builds them (fp16).  Slot s starts at a prompt length
spread evenly over [prompt - spread, prompt + spread]; the caches are filled synthetically and the positions set, instead
of running an HF prefill.  ChainDecoder runs its sequences in lockstep at ``prompt`` tokens.  The decoders alternate:
chain batch 1, chain batch 2, then each BatchDecoder size, and the two chain runs again.

Each BatchDecoder record has ms per step, aggregate tokens/s (max_batch tokens per step) and the split of a step into the
linear layers (q|k|v, o, gate|up, down), the attentions, the norms (add_rmsnorm) and the rest (embedding, lm_head,
position update, launch gaps), each part captured in a CUDA graph of its own and replayed.  ``--kv-cache fp8`` runs both
decoders with ``kv_cache_dtype=torch.float8_e4m3fn`` (synthetic rows quantised into the cache); ``both`` runs each
configuration with the 16-bit cache and then the FP8 one.  ``--max-length`` raises every decoder's max_length to at
least that value.  Prints one JSON line with
the GPU name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.chain_decoder_bench import build_model, gpu_facts, time_graph, timed_steps  # noqa: E402


def ragged(B, prompt, spread):
    """Prompt lengths of B slots spread evenly over [prompt - spread, prompt + spread]."""
    if B == 1:
        return [prompt]
    return [prompt - spread + (2 * spread * s) // (B - 1) for s in range(B)]


def _fill(dec, rows, T, gen):
    """Synthetic keys and values N(0, 1) in positions :T of the decoder's cache rows ``rows`` (quantised for FP8)."""
    n = len(range(dec._cache.rows)[rows])
    for i, k in enumerate(dec.k_cache):
        x = [torch.randn((n, dec.n_kv, T, dec.head_dim), generator=gen, device=k.device).half() for _ in range(2)]
        dec._cache.store(i, rows, *x)


def _kv_dtype(kv):
    return torch.float8_e4m3fn if kv == "fp8" else None


@torch.no_grad()
def batch_decoder(model, B, lengths, S, dev, kv="dtype", min_length=0):
    """One BatchDecoder run with every slot active at the given lengths: ms per step, tokens/s and the split."""
    from autogptq_b200.batch_decoder import BatchDecoder
    from autogptq_b200.mlp import forward_gate_up
    from autogptq_b200.moe import add_rmsnorm
    from autogptq_b200.qlinear import forward_group

    dec = BatchDecoder(model, max_batch=B, max_length=max(min_length, max(lengths) + S + 8),
                       kv_cache_dtype=_kv_dtype(kv))
    gen = torch.Generator(device=dev).manual_seed(2)
    for s, T in enumerate(lengths):
        _fill(dec, slice(s, s + 1), T, gen)
    dec.positions = lengths
    tok = torch.randint(0, 32000, (B,), device=dev, generator=gen)
    for _ in range(3):                                   # capture + warm replays
        tok = dec.step(tok).argmax(-1)
    dec.positions = lengths
    ms = timed_steps(lambda t: dec.step(t).argmax(-1), tok, S)

    # split: each part alone as one graph, at the middle of the timed window
    dec.positions = [T + S // 2 for T in lengths]
    plans = dec._plans

    def linears():
        for attn, mlp, *_ in plans:
            forward_group([attn.q_proj, attn.k_proj, attn.v_proj], dec._n1)
            attn.o_proj(dec._attn_out)
            mlp.down_proj(forward_gate_up(mlp.gate_proj, mlp.up_proj, dec._n2))

    q = [forward_group([a.q_proj, a.k_proj, a.v_proj], dec._n1) for a, *_ in plans]

    def attentions():
        for i, (qq, kk, vv) in enumerate(q):
            dec._cache.decode(i, qq, kk, vv, dec._pos, dec._inv_freq, dec._attn_scaling, dec.scaling, dec._attn_out,
                              dec._attn_ws)

    def norms():
        w, eps = plans[0][2]
        add_rmsnorm(dec._x, None, w, eps, n=dec._n1)
        for _, _, _, (w2, eps2), _ in plans:
            add_rmsnorm(dec._x, dec._resid, w2, eps2, h=dec._h1, n=dec._n2)
            add_rmsnorm(dec._x, dec._h1, w2, eps2, h=dec._resid, n=dec._n1)

    L = dec.max_length
    lin_ms = time_graph(linears, 20)
    attn_ms = time_graph(attentions, 20)
    norm_ms = time_graph(norms, 20)
    del dec, q
    torch.cuda.empty_cache()
    return {"max_batch": B, "kv_cache": kv, "lengths": lengths, "max_length": L, "ms_per_step": ms,
            "tokens_per_s": 1000.0 * B / ms,
            "split_ms": {"linear": lin_ms, "attention": attn_ms, "norms": norm_ms,
                         "rest": ms - lin_ms - attn_ms - norm_ms}}


@torch.no_grad()
def chain_decoder(model, B, T, S, dev, kv="dtype", min_length=0):
    """ChainDecoder(fused_attention=True) with B sequences in lockstep at a synthetic cache of T positions."""
    from autogptq_b200.decoder import ChainDecoder

    dec = ChainDecoder(model, batch=B, max_length=max(min_length, T + S + 8), fused_attention=True,
                       kv_cache_dtype=_kv_dtype(kv))
    gen = torch.Generator(device=dev).manual_seed(2)
    _fill(dec, slice(None), T, gen)
    dec.position = T
    tok = torch.randint(0, 32000, (B,), device=dev, generator=gen)
    for _ in range(3):
        tok = dec.step(tok).argmax(-1)
    dec.position = T
    ms = timed_steps(lambda t: dec.step(t).argmax(-1), tok, S)
    del dec
    torch.cuda.empty_cache()
    return {"batch": B, "kv_cache": kv, "prompt": T, "ms_per_step": ms, "tokens_per_s": 1000.0 * B / ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--prompt", type=int, default=512)
    ap.add_argument("--spread", type=int, default=256)
    ap.add_argument("--max-length", type=int, default=0)
    ap.add_argument("--kv-cache", choices=("dtype", "fp8", "both"), default="dtype")
    args = ap.parse_args()
    kvs = ["dtype", "fp8"] if args.kv_cache == "both" else [args.kv_cache]
    batches = [int(b) for b in args.batches.split(",")]
    plan = {B: ragged(B, args.prompt, args.spread) for B in batches}
    if not torch.cuda.is_available():
        raise SystemExit(f"batch_decoder_bench: no CUDA device (plan: {json.dumps(plan)})")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power = gpu_facts()
    model = build_model(args.layers, 1, dev)
    rec = {"gpu": name, "power_limit": power, "layers": args.layers, "steps": args.steps, "dtype": "float16",
           "chain_decoder": [], "batch_decoder": []}
    for B in (1, 2):
        for kv in kvs:
            rec["chain_decoder"].append(chain_decoder(model, B, args.prompt, args.steps, dev, kv, args.max_length))
    for B in batches:
        for kv in kvs:
            r = batch_decoder(model, B, plan[B], args.steps, dev, kv, args.max_length)
            rec["batch_decoder"].append(r)
            print(f"# {json.dumps(r)}", file=sys.stderr, flush=True)
    for B in (1, 2):
        for kv in kvs:
            rec["chain_decoder"].append(chain_decoder(model, B, args.prompt, args.steps, dev, kv, args.max_length))
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
