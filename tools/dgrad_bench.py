"""Input-gradient benchmark: dx = dy · Wᵀ of 4-bit layers (agb200_w4a16_dgrad) against the alternatives a trainer has.

    python tools/dgrad_bench.py [--dtypes float16,bfloat16] [--ms 16,64,256,1024,4096,16384] [--reps 20] [--out f.json]

Per Llama-2-7B layer shape at group size 128 (4096x4096, 4096->11008, 11008->4096), dtype and batch size M, each
variant runs as one CUDA graph over enough distinct layers to exceed the 50 MB L2, timed with CUDA events (median /
p10 / p90 per layer over the replays):
  dgrad         the dgrad kernel (agb200_w4a16_dgrad, auto selection)
  forward       the forward GEMM at the same (M, K, N): the same FLOPs
  dequant_mm    agb200_w4_dequantize + torch.matmul(dy, W.t()) per call (training without the dgrad kernel)
  cublas        torch.matmul(dy, W.t()) on a pre-dequantised fp16 / bf16 W (4x the weight memory; upper bound)
Then one Llama-2-7B decoder block's seven layers with rank-16 adapters, forward + backward at 4096 tokens, against the
same block on dense weights, and the eager per-call cost of the inference forward (public forward vs the internal
call it dispatches to).  The GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from autogptq_b200 import QuantLinear, _lib  # noqa: E402

SHAPES = [(4096, 4096), (4096, 11008), (11008, 4096)]
L2_BYTES = 50 << 20


def gpu_facts():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def random_layer(K, N, g, dtype, seed):
    """A QuantLinear with random packed weights made on the device (zero nibbles 0..14, scales 0.001..0.011)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    lin = QuantLinear(4, g, K, N, False, weight_dtype=dtype)
    G = K // g
    lin.qweight = torch.randint(-2**31, 2**31 - 1, (K // 8, N), dtype=torch.int32, device="cuda", generator=gen)
    z = torch.randint(0, 15, (G, N), dtype=torch.int32, device="cuda", generator=gen).view(G, N // 8, 8)
    lin.qzeros = sum(z[:, :, j] << (4 * j) for j in range(8)).to(torch.int32)
    lin.scales = (torch.rand((G, N), device="cuda", generator=gen) * 0.01 + 0.001).to(dtype)
    lin.g_idx = (torch.arange(K, device="cuda", dtype=torch.int32) // g)
    lin = lin.cuda()
    lin.post_init()
    return lin


def dequantize(lin, dtype):
    W = torch.empty((lin.infeatures, lin.outfeatures), dtype=dtype, device="cuda")
    scales, _ = lin._run_tensors(dtype)
    _lib.check(_lib.load().agb200_w4_dequantize(lin.qweight.data_ptr(), lin.qzeros.data_ptr(), scales.data_ptr(), None,
                                                W.data_ptr(), lin.infeatures, lin.outfeatures, lin.group_size,
                                                _lib.F16 if dtype == torch.float16 else _lib.BF16,
                                                torch.cuda.current_stream().cuda_stream), "dequantize")
    return W


def time_graph(fn, n_layers, reps):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / n_layers)
    del g
    t = np.asarray(times)
    return dict(median_us=float(np.median(t)), p10_us=float(np.percentile(t, 10)), p90_us=float(np.percentile(t, 90)))


def bench_layers(dtypes, ms, reps):
    rows = []
    for K, N in SHAPES:
        n_layers = max(2, -(-L2_BYTES // (K * N // 2)) + 1)
        for dtype in dtypes:
            layers = [random_layer(K, N, 128, dtype, seed=i) for i in range(n_layers)]
            for lin in layers:
                lin._prepare_tc()
            dense = [dequantize(lin, dtype) for lin in layers]
            for M in ms:
                dy = torch.randn(M, N, device="cuda").to(dtype)
                x = torch.randn(M, K, device="cuda").to(dtype)
                wtmp = torch.empty((K, N), dtype=dtype, device="cuda")
                code = _lib.F16 if dtype == torch.float16 else _lib.BF16
                lib = _lib.load()

                def dgrad():
                    for lin in layers:
                        lin.input_grad(dy)

                def forward():
                    with torch.no_grad():
                        for lin in layers:
                            lin(x)

                def dequant_mm():
                    st = torch.cuda.current_stream().cuda_stream
                    for lin in layers:
                        sc, _ = lin._run_tensors(dtype)
                        lib.agb200_w4_dequantize(lin.qweight.data_ptr(), lin.qzeros.data_ptr(), sc.data_ptr(), None,
                                                 wtmp.data_ptr(), K, N, 128, code, st)
                        torch.matmul(dy, wtmp.t())

                def cublas():
                    for W in dense:
                        torch.matmul(dy, W.t())

                flop = 2.0 * M * K * N
                for name, fn in (("dgrad", dgrad), ("forward", forward), ("dequant_mm", dequant_mm), ("cublas", cublas)):
                    r = time_graph(fn, n_layers, reps)
                    r.update(shape=f"{K}x{N}", dtype=str(dtype).split(".")[-1], M=M, variant=name, layers=n_layers,
                             tflops=flop / r["median_us"] / 1e6)
                    rows.append(r)
                    print(json.dumps(r), flush=True)
                del dy, x, wtmp
            del layers, dense
            torch.cuda.empty_cache()
    return rows


class _Dense(torch.nn.Module):
    def __init__(self, W):
        super().__init__()
        self.W = W                                     # [K, N], frozen

    def forward(self, x):
        return x @ self.W


class _LoRA(torch.nn.Module):
    def __init__(self, base, K, N, r, dtype):
        super().__init__()
        self.base = base
        self.A = torch.nn.Parameter((torch.randn(r, K, device="cuda") / K ** 0.5).to(dtype))
        self.B = torch.nn.Parameter(torch.zeros(N, r, device="cuda", dtype=dtype))

    def forward(self, x):
        return self.base(x) + (x @ self.A.t()) @ self.B.t()


def block_step(make, dtype, T, reps):
    """Seven adapted layers of a Llama-2-7B block (q, k, v, o, gate, up, down).  The attention itself is replaced by
    q + k + v (it is not part of this library); forward + backward of a squared-output loss."""
    H, I, r = 4096, 11008, 16
    q, k, v, o = (_LoRA(make(H, H, i), H, H, r, dtype) for i in range(4))
    gate, up, down = _LoRA(make(H, I, 4), H, I, r, dtype), _LoRA(make(H, I, 5), H, I, r, dtype), _LoRA(make(I, H, 6), I, H, r, dtype)
    x = torch.randn(T, H, device="cuda").to(dtype).requires_grad_(True)

    def step():
        h = x + o(q(x) + k(x) + v(x))
        y = h + down(F.silu(gate(h)) * up(h))
        y.float().pow(2).mean().backward()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    mem = sum(t.numel() * t.element_size() for m in (q, k, v, o, gate, up, down) for t in m.base.state_dict().values()) \
        if isinstance(q.base, torch.nn.Module) else 0
    return dict(median_ms=float(np.median(times)), p10_ms=float(np.percentile(times, 10)),
                p90_ms=float(np.percentile(times, 90)), weight_bytes=mem)


def bench_block(dtype, T, reps):
    def quant(K, N, seed):
        return random_layer(K, N, 128, dtype, seed=100 + seed)

    def dense(K, N, seed):
        return _Dense(dequantize(random_layer(K, N, 128, dtype, seed=100 + seed), dtype))

    out = {}
    for name, make in (("quant_lora", quant), ("dense_lora", dense)):
        r = block_step(make, dtype, T, reps)
        r.update(variant=name, tokens=T, dtype=str(dtype).split(".")[-1])
        print(json.dumps(r), flush=True)
        out[name] = r
        torch.cuda.empty_cache()
    return out


def bench_eager_call(n=3000):
    lin = random_layer(4096, 4096, 128, torch.float16, seed=7)
    x = torch.randn(1, 4096, device="cuda", dtype=torch.float16)
    res = {}
    with torch.no_grad():
        # forward() = the grad-mode check + _forward(), the body it had before it took an autograd path
        for name, fn in (("module_call", lin), ("forward", lin.forward), ("_forward", lin._forward)):
            for _ in range(200):
                fn(x)
            torch.cuda.synchronize()
            import time
            t0 = time.perf_counter()
            for _ in range(n):
                fn(x)
            torch.cuda.synchronize()
            res[name + "_us"] = (time.perf_counter() - t0) / n * 1e6
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtypes", default="float16,bfloat16")
    ap.add_argument("--ms", default="16,64,256,1024,4096,16384")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--tokens", type=int, default=4096)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dgrad_bench needs a CUDA device")
    dtypes = [getattr(torch, d) for d in a.dtypes.split(",")]
    gpu = gpu_facts()
    print(json.dumps({"gpu": gpu}), flush=True)
    res = dict(gpu=gpu, eager=bench_eager_call(), layers=bench_layers(dtypes, [int(m) for m in a.ms.split(",")], a.reps),
               block={str(d).split(".")[-1]: bench_block(d, a.tokens, 10) for d in dtypes}, gpu_after=gpu_facts())
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
