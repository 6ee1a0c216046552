#!/usr/bin/env python
"""Ablation timings of the decode chain kernel on synthetic Llama-shaped blocks (measurement aid, not a bench value).

    python tools/chain_probe.py [--model 7b|70b] [--blocks N] [--slots S] [--M 1]

Prints one JSON line per variant: full chain, no dependency waits (weights + math, x ignored), no math (pure TMA
stream + dependency protocol), neither (pure TMA stream) - each as us per token-equivalent and GB/s of algorithmic bytes,
next to the per-layer-launch path (grouped GEMV graph) on the same weights."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

SHAPES = {"7b": (4096, 11008, 4096), "70b": (8192, 28672, 1024), "70b-tp8": (8192, 3584, 128)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="7b")
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--M", type=int, default=1)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--slots", type=int, default=0)
    args = ap.parse_args()
    if args.slots:
        os.environ["AGB200_CHAIN_SLOTS"] = str(args.slots)
    import bench
    from autogptq_b200 import _lib, forward_group
    from autogptq_b200.chain import DecodeChain

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    hidden, inter, kv = SHAPES[args.model]
    gen = torch.Generator(device=dev)
    gen.manual_seed(1)
    tp8 = args.model == "70b-tp8"
    blocks = []
    for _ in range(args.blocks):
        if tp8:      # per-rank shards of a TP-8 70B block (row-parallel layers sliced along K)
            blocks.append({"q": bench.synth_layer(8192, 1024, 128, dev, gen), "k": bench.synth_layer(8192, 128, 128, dev, gen),
                           "v": bench.synth_layer(8192, 128, 128, dev, gen), "o": bench.synth_layer(1024, 8192, 128, dev, gen),
                           "gate": bench.synth_layer(8192, 3584, 128, dev, gen), "up": bench.synth_layer(8192, 3584, 128, dev, gen),
                           "down": bench.synth_layer(3584, 8192, 128, dev, gen)})
        else:
            blocks.append({"q": bench.synth_layer(hidden, hidden, 128, dev, gen), "k": bench.synth_layer(hidden, kv, 128, dev, gen),
                           "v": bench.synth_layer(hidden, kv, 128, dev, gen), "o": bench.synth_layer(hidden, hidden, 128, dev, gen),
                           "gate": bench.synth_layer(hidden, inter, 128, dev, gen), "up": bench.synth_layer(hidden, inter, 128, dev, gen),
                           "down": bench.synth_layer(inter, hidden, 128, dev, gen)})
    M = args.M
    nbytes = sum(bench.alg_bytes(M, l.infeatures, l.outfeatures, 128) for b in blocks for l in b.values())

    ch = DecodeChain(M=M, device=dev)
    x = ch.input(blocks[0]["q"].infeatures)
    t = x
    for b in blocks:
        q, _, _ = ch.stage([b["q"], b["k"], b["v"]], t)
        if tp8:      # shapes only: o reads a 1024-wide slice, down a 3584-wide one
            qs = q
            (o,) = ch.stage([b["o"]], qs)
            gate, _ = ch.stage([b["gate"], b["up"]], o)
            (t,) = ch.stage([b["down"]], gate)
        else:
            (o,) = ch.stage([b["o"]], q)
            gate, _ = ch.stage([b["gate"], b["up"]], o)
            (t,) = ch.stage([b["down"]], gate)
    ch.build()
    x.copy_(torch.randn(M, x.shape[1], device=dev).half())
    info = ch.info()
    stream = torch.cuda.Stream(device=dev)

    def time_graph(fn):
        with torch.cuda.stream(stream):
            fn()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                fn()
            for _ in range(3):
                g.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(stream)
            for _ in range(args.reps):
                g.replay()
            e1.record(stream)
            e1.synchronize()
        return e0.elapsed_time(e1) / args.reps * 1e3

    out = {"model": args.model, "blocks": args.blocks, "M": M, "alg_bytes": nbytes, **info}
    for name, flags in (("full", 0), ("no_deps", 1), ("no_math", 2), ("stream_only", 3), ("no_convert", 4), ("no_deps_no_convert", 5)):
        try:
            us = time_graph(lambda: ch.run(flags))
        except Exception as exc:
            from autogptq_b200.chain import chain_diag
            print(json.dumps({"failed_variant": name, "diag": chain_diag(), "error": str(exc)[:200], **info}), flush=True)
            raise
        print(f"[probe] {name}: {us:.1f} us", file=sys.stderr, flush=True)
        out[name] = {"us": round(us, 1), "gbs": round(nbytes / us / 1e3, 1)}
    # where the consumer warps spend their cycles (one warp per consumer group and CTA), and how long the producer sits
    # on a full ring
    from tools.chain_lookahead_sweep import CONSUMER as cats, profile_summary
    for name, flags in (("full", 8), ("no_deps", 9)):
        with torch.cuda.stream(stream):
            ch.run(flags)
            torch.cuda.synchronize()
        raw = ch.profile()
        pr = raw[:, :3, :].astype("float64")
        tot = pr[:, :, 0].mean()
        out["profile_" + name] = {"total_cycles": round(tot), **{c: round(float(pr[:, :, i].mean() / tot), 3) for i, c in enumerate(cats) if i > 0},
                                  "max_over_ctas": {c: round(float(pr[:, :, i].max() / tot), 3) for i, c in enumerate(cats) if i > 0}}
        out["producer_" + name] = profile_summary(raw)[1]

    def per_layer():
        xx = x
        for b in blocks:
            q, _, _ = forward_group([b["q"], b["k"], b["v"]], xx)
            o = b["o"](q)
            gate, _ = forward_group([b["gate"], b["up"]], o)
            xx = b["down"](gate)
        return xx
    if not tp8:
        us = time_graph(per_layer)
        out["per_layer_launches"] = {"us": round(us, 1), "gbs": round(nbytes / us / 1e3, 1)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
