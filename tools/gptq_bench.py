"""Times the GPTQ quantiser on Llama-2-7B layer shapes against a torch restatement of the reference's loop
(auto_gptq/quantization/gptq.py: fp32 matmul Hessian with TF32 off, a column loop of small kernels per block) on the
same GPU.  Prints one JSON line, with the GPU name and power limit read in the same run.

    python tools/gptq_bench.py [--samples 128] [--seqlen 2048] [--group-size 128] [--reps 3]

add_batch is called once per calibration sample ([1, seqlen, K], as the reference's forward hooks do).  Its TFLOP/s
count 2 * T * K^2 per update (the full product X^T X, although the kernel computes only the upper triangle).
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [("q/k/v/o/gate/up 4096->4096", 4096, 4096), ("gate/up 4096->11008", 4096, 11008),
          ("down 11008->4096", 11008, 4096)]


def timed(fn, reps=1):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps, out


def ref_add_batch(H, n, x):
    tmp = 1
    H *= n / (n + tmp)
    n += tmp
    inp = math.sqrt(2 / n) * x.float().t()
    H += inp.matmul(inp.t())
    return n


def ref_quant(x, scale, zero, maxq=15):
    q = torch.clamp(torch.round(x / scale) + zero, 0, maxq)
    return scale * (q - zero)


def ref_find_params(x, maxq=15):
    xmin = torch.minimum(x.min(1)[0], torch.zeros(1, device=x.device))
    xmax = torch.maximum(x.max(1)[0], torch.zeros(1, device=x.device))
    both = (xmin == 0) & (xmax == 0)
    xmin[both], xmax[both] = -1, 1
    scale = (xmax - xmin) / maxq
    return scale.unsqueeze(1), torch.round(-xmin / scale).unsqueeze(1)


def ref_column_loop(W, Hinv, group_size, blocksize=128):
    """The blocked loop of fasterquant (asymmetric, dynamic groups) in torch, one small kernel per operation."""
    K = W.shape[1]
    Q = torch.zeros_like(W)
    scale = zero = None
    for i1 in range(0, K, blocksize):
        i2 = min(i1 + blocksize, K)
        W1 = W[:, i1:i2].clone()
        Err1 = torch.zeros_like(W1)
        Hinv1 = Hinv[i1:i2, i1:i2]
        for i in range(i2 - i1):
            w = W1[:, i]
            d = Hinv1[i, i]
            if (i1 + i) % group_size == 0:
                scale, zero = ref_find_params(W[:, i1 + i:i1 + i + group_size])
            q = ref_quant(w.unsqueeze(1), scale, zero).flatten()
            Q[:, i1 + i] = q
            err1 = (w - q) / d
            W1[:, i:] -= err1.unsqueeze(1).matmul(Hinv1[i, i:].unsqueeze(0))
            Err1[:, i] = err1
        W[:, i2:] -= Err1.matmul(Hinv[i1:i2, i2:])
    return Q


def hinv_steps(H, actorder, percdamp=0.01):
    dead = torch.diag(H) == 0
    H[dead, dead] = 1
    perm = None
    if actorder:
        perm = torch.argsort(torch.diag(H), descending=True, stable=True)
        H = H[perm][:, perm]
    H.diagonal().add_(percdamp * torch.mean(torch.diag(H)))
    H = torch.linalg.cholesky(H)
    H = torch.cholesky_inverse(H)
    return torch.linalg.cholesky(H, upper=True), perm, dead


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--seqlen", type=int, default=2048)
    ap.add_argument("--group-size", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", type=int, default=len(SHAPES), help="run only the first n shapes")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gptq_bench.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False        # as the reference sets it (gptq.py:15)
    from autogptq_b200.gptq import GPTQ, quantize_weight

    dev = torch.device("cuda", 0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    gen = torch.Generator(device=dev).manual_seed(0)
    rows = []
    for name, K, N in SHAPES[:args.shapes]:
        # calibration inputs: correlated fp16 activations
        mix = (torch.randn(K, K, device=dev, generator=gen) / K**0.5 + torch.eye(K, device=dev)).half()
        xs = [(torch.randn(args.seqlen, K, device=dev, generator=gen).half() @ mix) for _ in range(2)]
        lin = torch.nn.Linear(K, N, bias=False, device=dev, dtype=torch.float16)
        W0 = lin.weight.data.clone()
        T = args.samples * args.seqlen
        flop = 2.0 * T * K * K

        g = GPTQ(lin)
        g.add_batch(xs[0][None], None)                      # warm-up
        g.H.zero_()
        g.nsamples = 0
        t_ab, _ = timed(lambda: [g.add_batch(xs[s % 2][None], None) for s in range(args.samples)])
        Href = torch.zeros(K, K, device=dev)
        ref_add_batch(Href, 0, xs[0])                        # warm-up
        Href.zero_()

        def ref_ab():
            nn_ = 0
            for s in range(args.samples):
                nn_ = ref_add_batch(Href, nn_, xs[s % 2])
        t_ab_ref, _ = timed(ref_ab)
        H = g.H
        hinv_steps(H.clone(), False)                        # warm-up (solver initialisation)
        for actorder in (False, True):
            t_chol, (Hinv, perm, dead) = timed(lambda: hinv_steps(H.clone(), actorder))
            Wf = W0.float()
            quantize_weight(Wf.clone(), Hinv, perm=perm, group_size=args.group_size, sym=False)   # warm-up
            t_q, _ = timed(lambda: quantize_weight(Wf.clone(), Hinv, perm=perm, group_size=args.group_size, sym=False),
                           reps=args.reps)
            Wr = Wf[:, perm] if perm is not None else Wf.clone()
            t_q_ref, _ = timed(lambda: ref_column_loop(Wr.clone(), Hinv, args.group_size))
            rows.append({
                "layer": name, "K": K, "N": N, "act_order": actorder,
                "add_batch_ms": round(t_ab * 1e3, 2), "add_batch_tflops": round(flop / t_ab / 1e12, 1),
                "cholesky_ms": round(t_chol * 1e3, 2), "quantize_ms": round(t_q * 1e3, 2),
                "total_ms": round((t_ab + t_chol + t_q) * 1e3, 2),
                "ref_add_batch_ms": round(t_ab_ref * 1e3, 2), "ref_add_batch_tflops": round(flop / t_ab_ref / 1e12, 1),
                "ref_quantize_ms": round(t_q_ref * 1e3, 2), "ref_total_ms": round((t_ab_ref + t_chol + t_q_ref) * 1e3, 2),
                "quantize_speedup": round(t_q_ref / t_q, 1), "add_batch_speedup": round(t_ab_ref / t_ab, 1),
            })
        del g, H, Href, xs, mix
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": smi, "samples": args.samples, "seqlen": args.seqlen, "group_size": args.group_size,
                      "flop_count": "2*T*K^2 per Hessian (full product)", "rows": rows}))


if __name__ == "__main__":
    main()
