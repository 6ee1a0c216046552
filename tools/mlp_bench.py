"""Time the Llama MLP with the fused gate/up (``FusedQuantMLP``) against the other ways to run it on the same layers.

    python tools/mlp_bench.py [--tokens 1,4,8,16,64,256,1024,4096,16384] [--copies 4] [--replays 20]

Llama-2-7B MLP shapes (H 4096, I 11008, group size 128), seeded random 4-bit layers, ``--copies`` distinct MLPs
(4 copies = 270 MB of packed weights, far more than the 50 MB L2).  Variants, all computing
``down(silu(gate(x)) * up(x))`` over the same QuantLinear modules:
  fused     FusedQuantMLP: forward_gate_up (one launch for gate, up and silu * mul) + down; above FUSED_MAX_M rows
            this selects the unfused layers
  fused_forced  the fused GEMM forced (only for M > FUSED_MAX_M), to show the other side of that choice
  unfused   the eager module: gate, up, F.silu, *, down (five launches)
  group     forward_group([gate, up]) + F.silu * up + down (gate and up share a launch for M <= 4)
  experts   QuantExperts with one expert and every token routed to it (routing, gather and combine included)
Per M and variant, the calls for all copies are captured in one CUDA graph; every replay is timed with CUDA events and
the per-MLP time reported as median / p10 / p90 in microseconds, with the algorithmic bytes (packed weights, scales,
zeros, x, h and y once) in GB/s against 3.35 TB/s and the dense TFLOP/s against 989 (H100 SXM data sheet figures).
``eager_us`` is the median of the same calls without a graph (the launch cost a non-captured decode loop pays).
One JSON line per M, the GPU name and power limit first.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from autogptq_b200 import FusedQuantMLP, QuantExperts, QuantLinear, _lib, forward_gate_up, forward_group  # noqa: E402
from autogptq_b200.mlp import FUSED_MAX_M  # noqa: E402

HBM_GBS = 3350.0
TC_TFLOPS = 989.0
H, I, G = 4096, 11008, 128


def gpu_facts() -> dict:
    facts = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        facts["power_limit"], facts["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as exc:      # noqa: BLE001 - the facts are informational
        facts["power_limit"] = f"unknown ({exc.__class__.__name__})"
    return facts


def random_layer(K, N, gen, dev):
    lin = QuantLinear(4, G, K, N, False)
    lin.qweight = torch.randint(-2 ** 31, 2 ** 31 - 1, (K // 8, N), dtype=torch.int32, device=dev, generator=gen)
    lin.qzeros = torch.randint(-2 ** 31, 2 ** 31 - 1, (K // G, N // 8), dtype=torch.int32, device=dev, generator=gen)
    lin.scales = (torch.rand((K // G, N), device=dev, generator=gen) * 0.01 + 0.001).to(torch.float16)
    lin.g_idx = torch.arange(K, device=dev, dtype=torch.int32) // G
    return lin


def mlp_bytes(M):
    w = 3 * (H * I // 2 + (H // G) * I * 2 + (H // G) * I // 2)
    return w + M * H * 2 + M * I * 2 + M * H * 2


def timed(calls, replays):
    """Per-call microseconds of one graph over `calls` (median, p10, p90 over replays) and the eager median."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for c in calls:
            c()                                   # warm-up: post_init, tensor-core copies, workspaces, plans
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for c in calls:
            c()
    graph.replay()
    times = []
    for _ in range(replays):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        graph.replay()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / len(calls))
    eager = []
    for _ in range(max(3, replays // 4)):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for c in calls:
            c()
        b.record()
        b.synchronize()
        eager.append(a.elapsed_time(b) * 1e3 / len(calls))
    del graph
    t = torch.tensor(times)
    return {"us": round(float(t.median()), 2), "p10": round(float(t.quantile(0.1)), 2),
            "p90": round(float(t.quantile(0.9)), 2), "eager_us": round(float(torch.tensor(eager).median()), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="1,4,8,16,64,256,1024,4096,16384")
    ap.add_argument("--copies", type=int, default=4)
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--variants", default="fused,unfused,group,experts,fused_forced")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    print(json.dumps(dict(gpu_facts(), shape=f"Llama-2-7B MLP H={H} I={I} g={G}", copies=args.copies,
                          weight_mb=round(args.copies * mlp_bytes(0) / 2 ** 20, 1))), flush=True)
    gen = torch.Generator(device=dev).manual_seed(0)
    mlps = [(random_layer(H, I, gen, dev), random_layer(H, I, gen, dev), random_layer(I, H, gen, dev))
            for _ in range(args.copies)]
    fused = [FusedQuantMLP(g, u, d) for g, u, d in mlps]
    experts = [QuantExperts.from_linears([g], [u], [d]) for g, u, d in mlps]
    variants = args.variants.split(",")
    for M in (int(t) for t in args.tokens.split(",")):
        x = torch.randn(M, H, device=dev, generator=gen).to(torch.float16)
        idx = torch.zeros(M, 1, dtype=torch.int64, device=dev)
        wt = torch.ones(M, 1, device=dev)

        def group_mlp(g, u, d):
            a, b = forward_group([g, u], x)
            return d(F.silu(a) * b)

        calls = {
            "fused": [lambda m=m: m(x) for m in fused],
            "unfused": [lambda g=g, u=u, d=d: d(F.silu(g(x)) * u(x)) for g, u, d in mlps],
            "group": [lambda g=g, u=u, d=d: group_mlp(g, u, d) for g, u, d in mlps],
            "experts": [lambda e=e: e(x, idx, wt) for e in experts],
            # the fused kernel even where FusedQuantMLP selects the unfused layers (M > FUSED_MAX_M)
            "fused_forced": [lambda g=g, u=u, d=d: d(forward_gate_up(g, u, x, kernel=_lib.GATE_UP_GEMM))
                             for g, u, d in mlps],
        }
        row = {"M": M}
        for v in variants:
            if v == "fused_forced" and M <= FUSED_MAX_M:
                continue
            r = timed(calls[v], args.replays)
            r["GBps"] = round(mlp_bytes(M) / r["us"] / 1e3, 1)
            r["pct_hbm"] = round(100 * r["GBps"] / HBM_GBS, 1)
            r["TFLOPs"] = round(6.0 * M * H * I / r["us"] / 1e6, 2)
            r["pct_tc"] = round(100 * r["TFLOPs"] / TC_TFLOPS, 1)
            row[v] = r
        if "fused" in row and "unfused" in row:
            row["fused_speedup_vs_unfused"] = round(row["unfused"]["us"] / row["fused"]["us"], 3)
        print(json.dumps(row), flush=True)
        del x, calls
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
