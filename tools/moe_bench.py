"""Time the grouped mixture-of-experts forward (``QuantExperts``) at Mixtral-8x7B shapes against the per-expert
``QuantLinear`` loop of transformers' ``MixtralExperts.forward``.

    python tools/moe_bench.py [--tokens 1,4,8,64,512,4096] [--blocks 4] [--iters 50]

Seeded random 4-bit experts (H 4096, I 14336, E 8, k 2, group size 128) for ``--blocks`` distinct MoE blocks (4 blocks
= 2.9 GB of experts, far more than the 50 MB L2), seeded routing per block.  Per T: the QuantExperts calls of all
blocks are captured in one CUDA graph and timed with CUDA events over replays; the loop (nonzero() + three
QuantLinear calls per hit expert + index_add_, eager: its host synchronisation cannot be captured) is timed the same
way in the same run.  Reported per block: microseconds, algorithmic bytes of the hit experts (per-layer formula of
``oracle/w4a16_oracle.algorithmic_bytes``) and GB/s against 3.35 TB/s (T <= 8), TFLOP/s against 989 (dense fp16 data
sheet figure).  One JSON line per T, the GPU name and power limit first.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from autogptq_b200 import QuantExperts, QuantLinear  # noqa: E402
from oracle.moe_oracle import active_bytes  # noqa: E402

HBM_GBS = 3350.0
TC_TFLOPS = 989.0


def gpu_facts() -> dict:
    facts = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        facts["power_limit"], facts["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as exc:      # noqa: BLE001 - the facts are informational
        facts["power_limit"] = f"unknown ({exc.__class__.__name__})"
    return facts


def random_layer(K, N, g, gen, dev):
    lin = QuantLinear(4, g, K, N, False)
    lin.qweight = torch.randint(-2 ** 31, 2 ** 31 - 1, (K // 8, N), dtype=torch.int32, device=dev, generator=gen)
    lin.qzeros = torch.randint(-2 ** 31, 2 ** 31 - 1, (K // g, N // 8), dtype=torch.int32, device=dev, generator=gen)
    lin.scales = (torch.rand((K // g, N), device=dev, generator=gen) * 0.01 + 0.001).to(torch.float16)
    lin.g_idx = (torch.arange(K, device=dev, dtype=torch.int32) // g)
    return lin


def loop_forward(qe, x, idx, w):
    """MixtralExperts.forward (modeling_mixtral.py:74-98) over the same QuantLinear modules."""
    E = qe.num_experts
    final = torch.zeros_like(x)
    mask = torch.nn.functional.one_hot(idx, num_classes=E + 1).permute(2, 1, 0)
    for e in torch.greater(mask.sum(dim=(-1, -2)), 0).nonzero().flatten().tolist():
        if e == E:
            continue
        slot, tok = torch.where(mask[e])
        xe = x[tok]
        h = torch.nn.functional.silu(qe.w1[e](xe)) * qe.w3[e](xe)
        y = qe.w2[e](h) * w[tok, slot, None]
        final.index_add_(0, tok, y.to(final.dtype))
    return final


def time_events(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3 / iters       # microseconds per call of fn


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--tokens", default="1,4,8,64,512,4096")
    ap.add_argument("--blocks", type=int, default=4)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--loop-iters", type=int, default=10)
    ap.add_argument("--hidden", type=int, default=4096)
    ap.add_argument("--intermediate", type=int, default=14336)
    ap.add_argument("--experts", type=int, default=8)
    ap.add_argument("--topk", type=int, default=2)
    ap.add_argument("--group-size", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("moe_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    H, I, E, k, g = args.hidden, args.intermediate, args.experts, args.topk, args.group_size
    print(json.dumps(dict(gpu_facts(), shapes=dict(H=H, I=I, E=E, k=k, group_size=g, blocks=args.blocks))), flush=True)

    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    blocks = []
    for _ in range(args.blocks):
        w1 = [random_layer(H, I, g, gen, dev) for _ in range(E)]
        w3 = [random_layer(H, I, g, gen, dev) for _ in range(E)]
        w2 = [random_layer(I, H, g, gen, dev) for _ in range(E)]
        blocks.append(QuantExperts.from_linears(w1, w3, w2))
    expert_bytes = sum(t.numel() * t.element_size() for qe in blocks for lin in qe._layers()
                       for t in (lin.qweight, lin.qzeros, lin.scales))

    for T in [int(t) for t in args.tokens.split(",")]:
        x = (torch.randn((T, H), device=dev, generator=gen) * 0.5).to(torch.float16)
        routes = []
        for _ in blocks:
            idx = torch.argsort(torch.rand((T, E), device=dev, generator=gen), dim=1)[:, :k].contiguous()
            w = torch.softmax(torch.rand((T, k), device=dev, generator=gen), dim=1).to(torch.float16)
            routes.append((idx, w))
        # warm-up (plans, tensor-core copies, workspace), then one graph over all blocks
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for qe, (idx, w) in zip(blocks, routes):
                qe(x, idx, w)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            outs = [qe(x, idx, w) for qe, (idx, w) in zip(blocks, routes)]
        graph.replay()
        torch.cuda.synchronize()
        us = time_events(graph.replay, args.iters) / len(blocks)

        def loop_all():
            return [loop_forward(qe, x, idx, w) for qe, (idx, w) in zip(blocks, routes)]

        ref = loop_all()
        torch.cuda.synchronize()
        loop_us = time_events(loop_all, args.loop_iters) / len(blocks)
        max_rel = max(float((o.float() - r.float()).abs().max() / r.float().abs().max()) for o, r in zip(outs, ref))

        nbytes = sum(active_bytes(idx.cpu().numpy(), E, H, I, g) for idx, _ in routes) / len(blocks)
        flops = 2.0 * T * k * 3 * H * I
        rec = dict(T=T, us_per_block=round(us, 2), loop_us_per_block=round(loop_us, 2),
                   speedup_vs_loop=round(loop_us / us, 2), active_bytes=int(nbytes),
                   tflops=round(flops / us * 1e-6, 2), tflops_frac_of_989=round(flops / us * 1e-6 / TC_TFLOPS, 4),
                   max_rel_diff_vs_loop=round(max_rel, 5))
        if T <= 8:
            rec["gbs"] = round(nbytes / us * 1e-3, 1)
            rec["hbm_frac_of_3350"] = round(nbytes / us * 1e-3 / HBM_GBS, 3)
        print(json.dumps(rec), flush=True)
    print(json.dumps({"expert_bytes_all_blocks": expert_bytes}), flush=True)


if __name__ == "__main__":
    main()
