"""Time the grouped experts' backward (``QuantExperts(input_grad=True)``) at Mixtral-8x7B shapes against autograd through
the per-expert loop of transformers' ``MixtralExperts.forward`` over the same 4-bit ``QuantLinear`` layers, and over
dense 16-bit experts (the upper bound: 4x the weight memory).

    python tools/moe_grad_bench.py [--tokens 16,64,512,2048,4096,8192] [--dtypes float16,bfloat16] [--iters 10]

One block of seeded random experts (H 4096, I 14336, E 8, k 2, group size 128: 0.7 GB of 4-bit weights, far more than
the 50 MB L2), seeded routing.  QuantExperts forward + backward and backward alone are each captured in one CUDA graph
and timed with CUDA events over replays; the loops (nonzero() syncs with the host, so they cannot be captured) are
timed eagerly the same way in the same run.  Backward TFLOP/s counts 6·P·H·I over the valid pairs P (three
reductions of 2·H·I per pair).  One JSON line per (dtype, T), the GPU name and power limit first.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.moe_bench import gpu_facts, random_layer  # noqa: E402
from autogptq_b200 import QuantExperts  # noqa: E402

H, I, E, K_TOP, G = 4096, 14336, 8, 2, 128


def loop(x, idx, w, mlp):
    """MixtralExperts.forward (modeling_mixtral.py) with mlp(e, x_rows) = w2(silu(w1 x) * w3 x) of expert e."""
    final = torch.zeros(x.shape, dtype=torch.float32, device=x.device)
    mask = torch.nn.functional.one_hot(idx, num_classes=E + 1).permute(2, 1, 0)
    for e in torch.greater(mask.sum(dim=(-1, -2)), 0).nonzero().flatten().tolist():
        if e == E:
            continue
        slot, tok = torch.where(mask[e])
        final = final.index_add(0, tok, mlp(e, x[tok]).float() * w[tok, slot, None])
    return final.to(x.dtype)


def time_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def graphed(fn, s):
    """fn captured on stream s (autograd runs a backward on the stream of its forward: a forward run on s outside the
    graph can then be differentiated inside it)."""
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        fn()
    return g.replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="16,64,512,2048,4096,8192")
    ap.add_argument("--dtypes", default="float16,bfloat16")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moe_grad_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    lines = [json.dumps(gpu_facts())]
    print(lines[0], flush=True)
    for dname in args.dtypes.split(","):
        dtype = getattr(torch, dname)
        gen = torch.Generator(device=dev).manual_seed(0)
        layers = {n: [random_layer(K, N, G, gen, dev) for _ in range(E)] for n, K, N in (("w1", H, I), ("w3", H, I), ("w2", I, H))}
        for lins in layers.values():
            for lin in lins:
                lin.scales = lin.scales.to(dtype)
        qe = QuantExperts.from_linears(layers["w1"], layers["w3"], layers["w2"], input_grad=True)
        dense = {n: [torch.randn(K, N, device=dev, dtype=dtype, generator=gen) * 0.02 for _ in range(E)]
                 for n, K, N in (("w1", H, I), ("w3", H, I), ("w2", I, H))}

        def q_mlp(e, xr):
            return qe.w2[e](torch.nn.functional.silu(qe.w1[e](xr)) * qe.w3[e](xr))

        def d_mlp(e, xr):
            return (torch.nn.functional.silu(xr @ dense["w1"][e]) * (xr @ dense["w3"][e])) @ dense["w2"][e]

        for T in (int(t) for t in args.tokens.split(",")):
            g = torch.Generator(device=dev).manual_seed(T)
            idx = torch.stack([torch.randperm(E, device=dev, generator=g)[:K_TOP] for _ in range(T)])
            w = torch.rand(T, K_TOP, device=dev, generator=g)
            w = (w / w.sum(1, keepdim=True)).requires_grad_(True)
            x = (torch.randn(T, H, device=dev, generator=g) * 0.5).to(dtype).requires_grad_(True)
            dy = torch.randn(T, H, device=dev, generator=g).to(dtype)

            def fwd_bwd():
                x.grad, w.grad = None, None
                qe(x, idx, w).backward(dy)

            def loop_fwd_bwd(mlp):
                x.grad, w.grad = None, None
                loop(x, idx, w, mlp).backward(dy)

            s = torch.cuda.Stream()
            t_fb = time_ms(graphed(fwd_bwd, s), args.iters)
            with torch.cuda.stream(s):
                out = qe(x, idx, w)
            torch.cuda.current_stream().wait_stream(s)
            keep = {}

            def bwd():
                keep["g"] = torch.autograd.grad(out, (x, w), dy, retain_graph=True)

            t_b = time_ms(graphed(bwd, s), args.iters)
            t_loop = time_ms(lambda: loop_fwd_bwd(q_mlp), max(2, args.iters // 2))
            t_dense = time_ms(lambda: loop_fwd_bwd(d_mlp), max(2, args.iters // 2))
            P = T * K_TOP
            rec = {"dtype": dname, "T": T, "H": H, "I": I, "E": E, "k": K_TOP, "group_size": G,
                   "fwd_bwd_ms": round(t_fb, 4), "bwd_ms": round(t_b, 4),
                   "loop_quant_fwd_bwd_ms": round(t_loop, 4), "loop_dense_fwd_bwd_ms": round(t_dense, 4),
                   "speedup_vs_quant_loop": round(t_loop / t_fb, 3), "vs_dense_loop": round(t_dense / t_fb, 3),
                   "bwd_tflops": round(6.0 * P * H * I / (t_b * 1e-3) / 1e12, 2)}
            lines.append(json.dumps(rec))
            print(lines[-1], flush=True)
            del out, keep
        del qe, dense, layers
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
