#!/usr/bin/env python
"""Weight-stream settings of the decode chain on bench.py's Llama-2-7B token (measurement aid, not a bench value).

    python tools/chain_lookahead_sweep.py [--blocks 32] [--reps 50] [--repeat 1] [--base knob=v,...]
                                          [--vary knob=v1,v2,...]... [--grid knob=v1,v2,...]...

Knobs (read by agb200_chain_create; "d" = the library default):
    slots      ring slots          AGB200_CHAIN_SLOTS
    inflight   in-flight cap       AGB200_CHAIN_INFLIGHT (0 = off)
    backoff    poll back-off       AGB200_CHAIN_POLL_BACKOFF (cycles)
    lookahead  L2 lookahead slots  AGB200_CHAIN_L2_LOOKAHEAD (clamped to the chain's maximum)

Every --vary changes one knob from --base; the --grid lists form a cartesian product on top of --base.  The whole list
of configurations runs --repeat times, interleaved.  Each measurement prints one JSON line: GPU name and power limit
(read at start), the settings the chain reports, us per token and GB/s of algorithmic bytes (CUDA-graph replays, CUDA
events), a digest of the token's output, and from one profiled launch the producer's blocked fraction and the consumer
profile (``DecodeChain.profile()``)."""
import argparse
import hashlib
import itertools
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

KNOBS = {"slots": "AGB200_CHAIN_SLOTS", "inflight": "AGB200_CHAIN_INFLIGHT", "backoff": "AGB200_CHAIN_POLL_BACKOFF",
         "lookahead": "AGB200_CHAIN_L2_LOOKAHEAD"}
CONSUMER = ["total", "wait_x", "convert", "wait_w", "mma", "flush", "tile_end", "stage_end"]


def profile_summary(pr):
    """DecodeChain.profile() [grid, 4, 8] -> consumer fractions of their total cycles and the producer's counters."""
    pr = pr.astype("float64")
    cons, prod = pr[:, :3, :], pr[:, 3, :]
    tot = cons[:, :, 0].mean()
    consumer = {"total_cycles": round(tot), **{c: round(float(cons[:, :, i].mean() / tot), 3) for i, c in enumerate(CONSUMER) if i > 0}}
    ptot = prod[:, 0]
    producer = {"total_cycles": round(float(ptot.mean())),
                "blocked_full_frac": round(float((prod[:, 1] / ptot).mean()), 4),
                "blocked_full_frac_max_cta": round(float((prod[:, 1] / ptot).max()), 4),
                "blocked_inflight_frac": round(float((prod[:, 2] / ptot).mean()), 4),
                "slots_issued": int(prod[:, 3].sum()), "slots_issued_per_cta": [int(prod[:, 3].min()), int(prod[:, 3].max())],
                "slots_prefetched_l2": int(prod[:, 4].sum())}
    return consumer, producer


def gpu_facts():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, watts, mhz = [c.strip() for c in out.split(",")]
        return {"gpu": name, "power_limit_w": float(watts), "sm_max_mhz": float(mhz)}
    except Exception as exc:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "nvidia_smi": str(exc)[:100]}


def parse_lists(items):
    out = []
    for it in items or []:
        k, v = it.split("=", 1)
        if k not in KNOBS:
            raise SystemExit(f"unknown knob {k!r} (one of {sorted(KNOBS)})")
        out.append((k, v.split(",")))
    return out


def configs(args):
    base = dict((k, v[0]) for k, v in parse_lists(args.base.split(";") if args.base else []))
    plan = [dict(base)]
    for k, vals in parse_lists(args.vary):
        plan += [{**base, k: v} for v in vals]
    grid = parse_lists(args.grid)
    if grid:
        keys = [k for k, _ in grid]
        plan += [{**base, **dict(zip(keys, combo))} for combo in itertools.product(*[v for _, v in grid])]
    seen, uniq = set(), []
    for c in plan:
        key = tuple(sorted(c.items()))
        if key not in seen:
            seen.add(key)
            uniq.append(c)
    return uniq


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--repeat", type=int, default=1)
    ap.add_argument("--base", default="", help="knob=value pairs separated by ';' (default: library defaults)")
    ap.add_argument("--vary", action="append")
    ap.add_argument("--grid", action="append")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("chain_lookahead_sweep.py needs a CUDA device")
    import bench
    from autogptq_b200.chain import DecodeChain

    plan = configs(args)
    facts = gpu_facts()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    hidden, inter, _, M, _ = bench.WORKLOADS["llama2-7b-decode-bs1"]
    model = bench.build_model(hidden, inter, args.blocks, dev, seed=1234)
    nbytes = args.blocks * sum(bench.alg_bytes(M, K, N, bench.GROUP) for (_, K, N) in bench.block_shapes(hidden, inter))
    x_val = torch.randn(M, hidden, dtype=torch.float16, device=dev, generator=torch.Generator(device=dev).manual_seed(4321))
    stream = torch.cuda.Stream(device=dev)
    results = {}
    for rep in range(args.repeat):
        for cfg in plan:
            for k, env in KNOBS.items():
                if k in cfg and cfg[k] != "d":
                    os.environ[env] = cfg[k]
                else:
                    os.environ.pop(env, None)
            with torch.cuda.stream(stream):
                ch, x, y = bench.build_chain(model, M, dev)
                x.copy_(x_val)
                ch.run()
                torch.cuda.synchronize()
                digest = hashlib.sha1(y.cpu().numpy().tobytes()).hexdigest()[:16]
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=stream):
                    ch.run()
                for _ in range(5):
                    g.replay()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record(stream)
                for _ in range(args.reps):
                    g.replay()
                e1.record(stream)
                e1.synchronize()
                us = e0.elapsed_time(e1) / args.reps * 1e3
                ch.run(8)
                torch.cuda.synchronize()
                consumer, producer = profile_summary(ch.profile())
            line = {**facts, "blocks": args.blocks, "rep": rep, "config": cfg, "chain": ch.info(), "us_per_token": round(us, 1),
                    "gbs": round(nbytes / us / 1e3, 1), "y_sha1": digest,
                    "producer_blocked_frac": producer["blocked_full_frac"], "producer": producer, "consumer": consumer}
            print(json.dumps(line), flush=True)
            results.setdefault(json.dumps(cfg, sort_keys=True), []).append(us)
            del g, ch, x, y
            for k, env in KNOBS.items():
                os.environ.pop(env, None)
    if args.repeat > 1:
        for cfg, uss in results.items():
            print(json.dumps({**facts, "summary": json.loads(cfg), "us_per_token_median": round(statistics.median(uss), 1),
                              "us_per_token_range": [round(min(uss), 1), round(max(uss), 1)], "n": len(uss)}), flush=True)


if __name__ == "__main__":
    main()
