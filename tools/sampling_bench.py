"""Cost of next-token sampling (DESIGN §3.21): the sampling kernel against torch, and sampled against greedy decoding.

    python tools/sampling_bench.py [--reps 200] [--layers 32] [--prompt 32] [--new 128] [--rounds 3] [--skip-decode]

1. Kernel: median µs over CUDA-graph replays of ``autogptq_b200.sample`` at B ∈ {1, 8} × V ∈ {32000, 128256, 152064},
   fp16 and fp32 logits, with every filter on (temperature 0.7, top_k 50, top_p 0.9, min_p 0.05), with temperature only,
   and greedy; next to torch doing the same work: transformers' four warpers (temperature, top-k, top-p with its full
   sort, min-p) and ``torch.multinomial`` over the softmax, captured in a graph too (or timed eagerly, with the reason,
   when the capture fails), and ``torch.argmax`` for greedy.
2. Decoding: tokens/s of ``BatchDecoder.generate`` on the 8 rows of the Llama-2-7B-shaped synthetic model of
   ``tools/batch_decoder_bench.py`` (fp16 weights, 8 prompts of ``--prompt`` tokens, ``--new`` new tokens each, no EOS),
   greedy against sampled (temperature 0.7, top_p 0.9, top_k 50), alternating the two ``--rounds`` times in one run.

Prints one JSON line with the GPU name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.chain_decoder_bench import build_model, gpu_facts  # noqa: E402


def median_us(fn, reps: int):
    """Median µs of one replay of ``fn`` captured in a CUDA graph (each replay timed by events), and how it was run."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    how = "graph"
    try:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        run = g.replay
    except Exception as e:          # noqa: BLE001 - torch ops that cannot be captured are timed eagerly
        torch.cuda.synchronize()
        how, run = f"eager ({type(e).__name__})", fn
    for _ in range(5):
        run()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        run()
        b.record()
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) * 1000 for a, b in ev), how


def torch_sampler(logits, t, k, p, m):
    """transformers' warpers in generate's order, then torch.multinomial (one generator for the batch)."""
    from transformers.generation.logits_process import (MinPLogitsWarper, TemperatureLogitsWarper, TopKLogitsWarper,
                                                        TopPLogitsWarper)

    warpers = [TemperatureLogitsWarper(t)]
    if k:
        warpers.append(TopKLogitsWarper(k))
    if p < 1:
        warpers.append(TopPLogitsWarper(p))
    if m:
        warpers.append(MinPLogitsWarper(m))

    def run():
        x = logits.float()
        for w in warpers:
            x = w(None, x)
        return torch.multinomial(torch.softmax(x, dim=-1), 1)
    return run


@torch.no_grad()
def kernel_table(reps: int):
    from autogptq_b200 import sample

    rows = []
    dev = torch.device("cuda")
    for B in (1, 8):
        for V in (32000, 128256, 152064):
            for dt in (torch.float16, torch.float32):
                logits = (torch.randn(B, V, device=dev) * 3).to(dt)
                for name, (t, k, p, m) in (("all", (0.7, 50, 0.9, 0.05)), ("temperature", (1.0, 0, 1.0, 0.0)),
                                           ("greedy", (0.0, 0, 1.0, 0.0))):
                    args = (torch.full((B,), t, device=dev), torch.full((B,), k, dtype=torch.int32, device=dev),
                            torch.full((B,), p, device=dev), torch.full((B,), m, device=dev),
                            torch.arange(B, dtype=torch.int64, device=dev), torch.arange(B, dtype=torch.int64, device=dev))
                    out = torch.empty(B, dtype=torch.int64, device=dev)
                    us, _ = median_us(lambda: sample(logits, *args, out=out), reps)
                    if name == "greedy":
                        ref, how = median_us(lambda: torch.argmax(logits, dim=-1), reps)
                    else:
                        ref, how = median_us(torch_sampler(logits, t, k, p, m), reps)
                    rows.append({"B": B, "V": V, "dtype": str(dt).replace("torch.", ""), "params": name,
                                 "kernel_us": round(us, 2), "torch_us": round(ref, 2), "torch_run": how})
                    print(json.dumps(rows[-1]), flush=True)
    return rows


@torch.no_grad()
def decode_table(layers: int, prompt: int, new: int, rounds: int):
    from autogptq_b200 import BatchDecoder, SamplingParams

    dev = torch.device("cuda")
    model = build_model(layers, 8, dev)
    dec = BatchDecoder(model, max_batch=8, max_length=prompt + new + 8)
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(0, 32000, (prompt,), generator=g) for _ in range(8)]
    sampled = SamplingParams(temperature=0.7, top_p=0.9, top_k=50, seed=1)
    runs = {"greedy": [], "sampled": []}
    for kind in ("greedy", "sampled"):                    # warm-up: graph captures, library workspaces
        dec.generate(prompts, 4, sampling=None if kind == "greedy" else sampled)
    for _ in range(rounds):
        for kind in ("greedy", "sampled"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            outs = dec.generate(prompts, new, sampling=None if kind == "greedy" else sampled)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            n = sum(int(o.numel()) - prompt for o in outs)
            runs[kind].append(n / dt)
    med = {k: statistics.median(v) for k, v in runs.items()}
    return {"layers": layers, "prompt": prompt, "new_tokens": new, "rows": 8,
            "tokens_per_s": {k: [round(x, 1) for x in v] for k, v in runs.items()},
            "median_tokens_per_s": {k: round(v, 1) for k, v in med.items()},
            "sampled_cost_pct": round(100 * (1 - med["sampled"] / med["greedy"]), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--prompt", type=int, default=32)
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-decode", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampling_bench needs a CUDA device")
    name, power = gpu_facts()
    rec = {"gpu": name, "power_limit": power, "kernel": kernel_table(args.reps)}
    if not args.skip_decode:
        rec["decode"] = decode_table(args.layers, args.prompt, args.new, args.rounds)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
