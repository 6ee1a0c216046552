"""Aggregate decode throughput of a Mixtral-8x7B-shaped GPTQ model with BatchDecoder at 1, 2, 4 and 8 active rows
(ragged positions), plus 2 active rows of 8 slots, next to ChainDecoder(fused_attention=True) at batch 1 and 2.

    python tools/moe_batch_decoder_bench.py [--layers 32] [--batches 1,2,4,8] [--steps 64] [--prompt 512]
                                            [--spread 256] [--rounds 3]

The model is ``tools/moe_decoder_bench.py``'s (H 4096, I 14336, 8 experts, top-2, 32/8/128 heads, synthetic 4-bit
weights, about 23 GB of experts).  Slot s starts at a prompt length spread evenly over [prompt - spread, prompt + spread]
(``tools/batch_decoder_bench.py``); caches are filled synthetically and positions set instead of an HF prefill, so the
experts' tensor-core copies are never built.  The configurations alternate, ``--rounds`` times over: chain batch 1, chain
batch 2, each BatchDecoder size, then 2 of 8 slots.

Each BatchDecoder record has ms per step and aggregate tokens/s (active rows per step), and per step: the experts' time
(every layer's ``QuantExperts`` forward on the last step's routing, captured in one graph and replayed), the distinct
experts hit per layer (counted on the host from each layer's routing over ``--hit-steps`` further steps), the expert
bytes those hits stream and the rate that gives.  ``hits_if_idle_routed`` counts, from the same steps, the experts the
idle rows' own router logits (their n2 · gateᵀ on the host) would have added had they been routed: what masking them
saves.  Prints one JSON line with the GPU name and power limit read in the same run; ``summary`` holds, per
configuration, the median tokens/s over the rounds and its range."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.batch_decoder_bench import _fill, chain_decoder, ragged  # noqa: E402
from tools.chain_decoder_bench import gpu_facts, time_graph, timed_steps  # noqa: E402
from tools.moe_decoder_bench import build_model  # noqa: E402


def expert_bytes(experts) -> int:
    """Packed bytes of one expert of a layer: w1, w3 and w2 with their zeros and scales."""
    return sum(t.numel() * t.element_size() for lin in (experts.w1[0], experts.w3[0], experts.w2[0])
               for t in (lin.qweight, lin.qzeros, lin.scales))


def _hits(dec, active):
    """(distinct experts hit per layer, those plus the idle rows' host-side top-k) of the step just taken."""
    hit, would = [], []
    idle = [s for s in range(dec.max_batch) if s not in active]
    for m in dec._moe_layers:
        idx = m["idx"].cpu()
        got = {int(e) for e in idx.flatten().tolist() if e >= 0}
        assert all((idx[s] == -1).all() for s in idle), "an idle row was routed"
        hit.append(len(got))
        if idle:
            logits = m["n2"][idle].float() @ m["gate"].float().t()
            got |= set(logits.topk(m["k"], dim=-1).indices.flatten().tolist())
        would.append(len(got))
    return hit, would


@torch.no_grad()
def batch_decoder(model, B, lengths, S, hit_steps, dev):
    """One BatchDecoder run of max_batch B whose slots hold ``lengths`` (-1: idle): ms per step, tokens/s, expert
    time, hits and bytes."""
    from autogptq_b200.batch_decoder import BatchDecoder

    active = [s for s, T in enumerate(lengths) if T >= 0]
    dec = BatchDecoder(model, max_batch=B, max_length=max(lengths) + S + hit_steps + 8)
    gen = torch.Generator(device=dev).manual_seed(2)
    for s in active:
        _fill(dec, (s, slice(None)), lengths[s], gen)
    dec.positions = lengths
    tok = torch.randint(0, 32000, (B,), device=dev, generator=gen)
    for _ in range(3):                                   # capture + warm replays
        tok = dec.step(tok).argmax(-1)
    dec.positions = lengths
    ms = timed_steps(lambda t: dec.step(t).argmax(-1), tok, S)

    def experts():
        for m in dec._moe_layers:
            m["experts"]._forward(m["n2"], m["idx"], m["w"], out=m["out"], plan=m["plan"], ws=m["ws"])

    experts_ms = time_graph(experts, 20)
    hits, would = [], []
    for _ in range(hit_steps):
        tok = dec.step(tok).argmax(-1)
        h, w = _hits(dec, active)
        hits += h
        would += w
    per = expert_bytes(dec._moe_layers[0]["experts"])
    L = len(dec._moe_layers)
    mean_hits = sum(hits) / len(hits)
    del dec
    torch.cuda.empty_cache()
    return {"max_batch": B, "active": len(active), "lengths": lengths, "ms_per_step": ms,
            "tokens_per_s": 1000.0 * len(active) / ms, "experts_ms_per_step": experts_ms,
            "experts_hit_per_layer": mean_hits, "hits_if_idle_routed": sum(would) / len(would),
            "expert_gb_per_step": mean_hits * per * L / 1e9,
            "expert_tb_per_s": mean_hits * per * L / (experts_ms * 1e-3) / 1e12}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--hit-steps", type=int, default=8)
    ap.add_argument("--prompt", type=int, default=512)
    ap.add_argument("--spread", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    configs = [("chain", 1, None), ("chain", 2, None)]
    configs += [("batch", B, ragged(B, args.prompt, args.spread)) for B in (int(b) for b in args.batches.split(","))]
    configs.append(("batch", 8, ragged(2, args.prompt, args.spread) + [-1] * 6))
    if not torch.cuda.is_available():
        raise SystemExit(f"moe_batch_decoder_bench: no CUDA device (plan: {json.dumps(configs)})")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power = gpu_facts()
    model = build_model(args.layers, dev)
    rec = {"gpu": name, "power_limit": power, "layers": args.layers, "steps": args.steps, "dtype": "float16",
           "expert_mb_per_layer": expert_bytes(model.model.layers[0].mlp.experts) / 1e6, "runs": []}
    rates = {}
    for rnd in range(args.rounds):
        for kind, B, lengths in configs:
            if kind == "chain":
                r = chain_decoder(model, B, args.prompt, args.steps, dev)
                key = f"chain_b{B}"
            else:
                r = batch_decoder(model, B, lengths, args.steps, args.hit_steps, dev)
                key = f"batch_{r['active']}_of_{B}"
            r.update(kind=kind, round=rnd)
            rec["runs"].append(r)
            rates.setdefault(key, []).append(r["tokens_per_s"])
            print(f"# {json.dumps(r)}", file=sys.stderr, flush=True)
    rec["summary"] = {k: {"tokens_per_s_median": statistics.median(v), "min": min(v), "max": max(v)}
                      for k, v in rates.items()}
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
