"""Time the fused dense MLP backward (``FusedQuantMLP(fused_backward=True)``) at Llama-2-7B MLP shapes against the
default ``FusedQuantMLP`` in grad mode (autograd through the unfused layers) and a dense 16-bit MLP on cuBLAS.

    python tools/mlp_grad_bench.py [--tokens 16,64,256,1024,2048,4096,8192] [--dtypes float16,bfloat16] [--reps 5]

MLP: H 4096, I 11008, group size 128, seeded random 4-bit layers; COPIES distinct MLPs per graph, so that the weights
(67 MB of 4-bit, 270 MB of 16-bit per MLP) exceed the 50 MB L2.  Per variant and M two CUDA graphs are captured:
forward + backward (``torch.autograd.grad``) and the forward alone in grad mode; backward = their difference.  Graph
replays are timed with CUDA events, the variants alternating within each of ``--reps`` rounds; the median per MLP and
the spread (min..max over rounds) are reported.  Then one Llama-2-7B decoder block (transformers' LlamaDecoderLayer with SDPA
attention, all seven projections 4-bit, rank-16 adapters on q_proj / v_proj) at 4096 tokens, eager, for (a) and (b),
with the memory the forward leaves held for backward and the peak of forward + backward; (a) once with the library's
cut-over (FUSED_BACKWARD_MAX_M) and once with the fused kernels forced at every M.  The MLP table times the module as
built, with FUSED_BACKWARD_MAX_M lifted so that (a) is always the fused path.  One JSON line per result, the GPU name and
power limit first.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.moe_bench import gpu_facts, random_layer  # noqa: E402
import autogptq_b200.mlp as mlp_mod  # noqa: E402
from autogptq_b200 import FusedQuantMLP  # noqa: E402

H, I, G, COPIES = 4096, 11008, 128, 4


class _Dense(torch.nn.Module):
    """The same MLP with 16-bit weights on cuBLAS (what the frozen base costs unquantised)."""

    def __init__(self, dtype, gen, dev):
        super().__init__()
        mk = lambda k, n: (torch.randn((n, k), device=dev, generator=gen) * k ** -0.5).to(dtype)   # noqa: E731
        self.wg, self.wu, self.wd = mk(H, I), mk(H, I), mk(I, H)

    def forward(self, x):
        return F.linear(F.silu(F.linear(x, self.wg)) * F.linear(x, self.wu), self.wd)


def _quant_mlp(dtype, gen, dev, fused):
    layers = []
    for K, N in ((H, I), (H, I), (I, H)):
        lin = random_layer(K, N, G, gen, dev)
        lin.scales = lin.scales.to(dtype)
        layers.append(lin)
    return FusedQuantMLP(*layers, fused_backward=fused)


def _graph(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def _time(g, n=10):
    for _ in range(2):
        g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def bench_mlp(dtype, tokens, reps, dev):
    mlp_mod.FUSED_BACKWARD_MAX_M, cut = 1 << 30, mlp_mod.FUSED_BACKWARD_MAX_M
    try:
        _bench_mlp(dtype, tokens, reps, dev)
    finally:
        mlp_mod.FUSED_BACKWARD_MAX_M = cut


def _bench_mlp(dtype, tokens, reps, dev):
    gen = torch.Generator(device=dev).manual_seed(0)
    variants = {
        "a_fused_backward": [_quant_mlp(dtype, gen, dev, True) for _ in range(COPIES)],
        "b_default": None,
        "c_dense_cublas": [_Dense(dtype, gen, dev) for _ in range(COPIES)],
    }
    variants["b_default"] = [FusedQuantMLP(m.gate_proj, m.up_proj, m.down_proj) for m in variants["a_fused_backward"]]
    for M in tokens:
        x = torch.randn(M, H, device=dev, generator=gen).to(dtype).requires_grad_(True)
        dy = torch.randn(M, H, device=dev, generator=gen).to(dtype)
        graphs = {}
        for name, mlps in variants.items():
            def both(mlps=mlps):
                for m in mlps:
                    torch.autograd.grad(m(x), x, dy)

            def fwd(mlps=mlps):
                for m in mlps:
                    m(x)
            graphs[name] = (_graph(both), _graph(fwd))
        times = {n: ([], []) for n in graphs}
        for _ in range(reps):                       # variants alternate within a round
            for n, (gb, gf) in graphs.items():
                tb, tf = _time(gb) / COPIES, _time(gf) / COPIES
                times[n][0].append(tb)
                times[n][1].append(tb - tf)
        row = {"dtype": str(dtype).replace("torch.", ""), "M": M}
        for n, (tb, tbw) in times.items():
            row[n] = {"fwd_bwd_ms": round(statistics.median(tb), 4), "fwd_bwd_spread": [round(min(tb), 4), round(max(tb), 4)],
                      "bwd_ms": round(statistics.median(tbw), 4), "bwd_spread": [round(min(tbw), 4), round(max(tbw), 4)]}
        a, b = times["a_fused_backward"], times["b_default"]
        row["a_over_b_fwd_bwd"] = round(statistics.median(a[0]) / statistics.median(b[0]), 3)
        row["a_over_b_bwd"] = round(statistics.median(a[1]) / statistics.median(b[1]), 3)
        print(json.dumps(row), flush=True)
        del graphs, x, dy
        torch.cuda.empty_cache()


class _LoRA(torch.nn.Module):
    def __init__(self, base, r, dtype, gen, dev):
        super().__init__()
        self.base = base
        K, N = base.infeatures, base.outfeatures
        self.A = torch.nn.Parameter((torch.randn(r, K, device=dev, generator=gen) / K ** 0.5).to(dtype))
        self.B = torch.nn.Parameter(torch.zeros(N, r, device=dev, dtype=dtype))

    def forward(self, x):
        return self.base(x) + (x @ self.A.t()) @ self.B.t()


def bench_block(dtype, T, reps, dev):
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaDecoderLayer, LlamaRotaryEmbedding

    cfg = LlamaConfig(hidden_size=H, intermediate_size=I, num_attention_heads=32, num_key_value_heads=32,
                      max_position_embeddings=T)
    cfg._attn_implementation = "sdpa"
    gen = torch.Generator(device=dev).manual_seed(1)
    block = LlamaDecoderLayer(cfg, layer_idx=0).to(dtype).to(dev)
    block.requires_grad_(False)
    att = block.self_attn
    for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
        lin = random_layer(H, H, G, gen, dev)
        lin.scales = lin.scales.to(dtype)
        setattr(att, n, _LoRA(lin, 16, dtype, gen, dev) if n in ("q_proj", "v_proj") else lin)
    mlp = _quant_mlp(dtype, gen, dev, True)
    block.mlp = mlp
    x = (torch.randn(1, T, H, device=dev, generator=gen) * 0.1).to(dtype).requires_grad_(True)
    pos = torch.arange(T, device=dev)[None]
    pe = LlamaRotaryEmbedding(config=cfg).to(dev)(x, pos)
    dy = torch.randn(1, T, H, device=dev, generator=gen).to(dtype)
    out = {}
    for fused in (True, False, True, False) * reps:
        mlp.fused_backward = fused
        name = "a_fused_backward" if fused else "b_default"
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        y = block(x, position_embeddings=pe)
        y = y[0] if isinstance(y, tuple) else y
        held = torch.cuda.memory_allocated() - base
        torch.autograd.grad(y, [x] + [p for p in block.parameters() if p.requires_grad], dy)
        b.record()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        r = out.setdefault(name, {"ms": []})
        r["ms"].append(a.elapsed_time(b))
        r["held_MB"], r["peak_MB"] = held / 1e6, peak / 1e6           # the last round's (the first one builds caches)
        del y
    row = {"block": "Llama-2-7B decoder layer, rank-16 adapters on q/v", "dtype": str(dtype).replace("torch.", ""), "T": T,
           "one_MxI_tensor_MB": T * I * 2 / 1e6, "fused_backward_max_m": mlp_mod.FUSED_BACKWARD_MAX_M}
    for n, r in out.items():
        ms = r.pop("ms")[2:]                          # the first round of each warms up
        row[n] = dict(r, fwd_bwd_ms=round(statistics.median(ms), 3), spread=[round(min(ms), 3), round(max(ms), 3)])
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="16,64,256,1024,2048,4096,8192")
    ap.add_argument("--dtypes", default="float16,bfloat16")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--block-tokens", type=int, default=4096)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mlp_grad_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    print(json.dumps(gpu_facts()), flush=True)
    tokens = [int(t) for t in a.tokens.split(",") if t]
    for dt in a.dtypes.split(","):
        if tokens:
            bench_mlp(getattr(torch, dt), tokens, a.reps, dev)
    if a.block_tokens:
        cut = mlp_mod.FUSED_BACKWARD_MAX_M
        for dt in a.dtypes.split(","):
            bench_block(getattr(torch, dt), a.block_tokens, a.reps, dev)
            mlp_mod.FUSED_BACKWARD_MAX_M = 1 << 30        # the fused kernels at every M, past the library's cut-over
            bench_block(getattr(torch, dt), a.block_tokens, a.reps, dev)
            mlp_mod.FUSED_BACKWARD_MAX_M = cut


if __name__ == "__main__":
    main()
