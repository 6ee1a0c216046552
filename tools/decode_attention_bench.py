"""Decode attention per layer: the fused kernel (agb200_decode_attention) against the torch path ChainDecoder runs by
default (rotary_emb + apply_rotary_pos_emb, two index_copy_, SDPA with a length mask over the static cache, the copy
into o_proj's input), both at the same max_length.

    python tools/decode_attention_bench.py [--reps 50] [--contexts 512,2048,4096,16384] [--batches 1,2]
                                           [--kv-cache {dtype,fp8,both}]

Batches above 2 run the per-row entry (agb200_decode_attention_rows) with every row at the same position.
``--kv-cache fp8`` times the kernel over an FP8 cache (E4M3 codes and a power-of-two scale per row, DESIGN §3.19) and
not the torch path; ``both`` alternates the 16-bit and FP8 kernels in one process: 16-bit, FP8, torch, 16-bit, FP8.

Each configuration runs one CUDA graph over enough distinct layers (own caches, q, k, v) that the caches read per
replay exceed the 50 MB L2 several times, so the numbers are HBM numbers, not L2 ones.  The attended context is
`ctx` positions (pos = ctx - 1) in a cache of max_length = ctx + 128.  Bytes per layer are computed from the shapes:
2·B·n_kv·(pos+1)·hd·2 of K and V plus q, k, v and out; for the FP8 cache 2·B·n_kv·(pos+1)·(hd + 4), codes and
scales.  Prints one JSON line with µs per layer and GB/s of each path
and the GPU name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.chain_decoder_bench import gpu_facts, time_graph  # noqa: E402

SHAPES = {"llama2-7b": (32, 32, 128), "mistral-7b": (32, 8, 128)}


def torch_attention(q, k, v, kc, vc, pos, arange, rot, scaling, out, nh, nkv, hd):
    from transformers.models.llama.modeling_llama import apply_rotary_pos_emb

    B = q.shape[0]
    cos, sin = rot(q.view(B, 1, -1), pos.view(1, 1).expand(B, 1))
    mask = (arange <= pos).view(1, 1, 1, -1)
    qh, kh = apply_rotary_pos_emb(q.view(B, 1, nh, hd).transpose(1, 2), k.view(B, 1, nkv, hd).transpose(1, 2), cos, sin)
    kc.index_copy_(2, pos, kh)
    vc.index_copy_(2, pos, v.view(B, 1, nkv, hd).transpose(1, 2))
    o = torch.nn.functional.scaled_dot_product_attention(qh, kc, vc, attn_mask=mask, scale=scaling,
                                                         enable_gqa=nkv != nh)
    out.copy_(o.transpose(1, 2).reshape(B, -1))


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--contexts", default="512,2048,4096,16384")
    ap.add_argument("--batches", default="1,2")
    ap.add_argument("--kv-cache", choices=("dtype", "fp8", "both"), default="dtype")
    args = ap.parse_args()
    dtype_kv, fp8_kv = args.kv_cache in ("dtype", "both"), args.kv_cache in ("fp8", "both")
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding

    from autogptq_b200.attention import (decode_attention, decode_attention_rows, decode_attention_workspace,
                                         quantize_kv)

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power = gpu_facts()
    rec = {"gpu": name, "power_limit": power, "dtype": "float16", "kv_cache": args.kv_cache, "rows": []}
    dt = torch.float16
    for sname, (nh, nkv, hd) in SHAPES.items():
        cfg = LlamaConfig(hidden_size=nh * hd, num_attention_heads=nh, num_key_value_heads=nkv,
                          max_position_embeddings=32768)
        rot = LlamaRotaryEmbedding(cfg, device=dev)
        for B in (int(b) for b in args.batches.split(",")):
            for ctx in (int(c) for c in args.contexts.split(",")):
                L = ctx + 128
                per_layer = 2 * B * nkv * L * hd * 2
                n_layers = max(4, min(64, -(-400 * 2 ** 20 // per_layer)), -(-4 * 50 * 2 ** 20 // per_layer))
                n_layers = min(n_layers, max(1, (24 * 2 ** 30) // per_layer))
                g = torch.Generator(device=dev).manual_seed(ctx + B)
                layers = []
                for _ in range(n_layers):
                    layers.append(dict(
                        q=torch.randn(B, nh * hd, generator=g, device=dev).to(dt),
                        k=torch.randn(B, nkv * hd, generator=g, device=dev).to(dt),
                        v=torch.randn(B, nkv * hd, generator=g, device=dev).to(dt),
                        kc=torch.randn(B, nkv, L, hd, generator=g, device=dev).to(dt),
                        vc=torch.randn(B, nkv, L, hd, generator=g, device=dev).to(dt),
                        out=torch.empty(B, nh * hd, dtype=dt, device=dev)))
                    ly = layers[-1]
                    if fp8_kv:
                        (ly["kc8"], ly["ks"]), (ly["vc8"], ly["vs"]) = quantize_kv(ly["kc"]), quantize_kv(ly["vc"])
                    if not dtype_kv:
                        del ly["kc"], ly["vc"]
                pos = torch.full((1,), ctx - 1, dtype=torch.int64, device=dev)
                pos_rows = torch.full((B,), ctx - 1, dtype=torch.int64, device=dev)
                entry, p_entry = (decode_attention, pos) if B <= 2 else (decode_attention_rows, pos_rows)
                arange = torch.arange(L, device=dev)
                ws = decode_attention_workspace(B, nh, nkv, hd, L, dev)
                sc = hd ** -0.5

                def fused():
                    for ly in layers:
                        entry(ly["q"], ly["k"], ly["v"], ly["kc"], ly["vc"], p_entry, rot.inv_freq,
                              rot.attention_scaling, sc, ly["out"], ws)

                def fused_fp8():
                    for ly in layers:
                        entry(ly["q"], ly["k"], ly["v"], ly["kc8"], ly["vc8"], p_entry, rot.inv_freq,
                              rot.attention_scaling, sc, ly["out"], ws, k_scale=ly["ks"], v_scale=ly["vs"])

                def eager():
                    for ly in layers:
                        torch_attention(ly["q"], ly["k"], ly["v"], ly["kc"], ly["vc"], pos, arange, rot, sc,
                                        ly["out"], nh, nkv, hd)

                io = 2 * B * (2 * nh + 2 * nkv) * hd
                nbytes = 2 * B * nkv * ctx * hd * 2 + io
                nbytes8 = 2 * B * nkv * ctx * (hd + 4) + io
                row = {"shape": sname, "batch": B, "context": ctx, "max_length": L, "layers_per_graph": n_layers,
                       "bytes_per_layer": nbytes, "fp8_bytes_per_layer": nbytes8}
                runs = {"dtype": [("fused", fused, nbytes), ("torch", eager, nbytes), ("fused_again", fused, nbytes)],
                        "fp8": [("fp8", fused_fp8, nbytes8), ("fp8_again", fused_fp8, nbytes8)],
                        "both": [("fused", fused, nbytes), ("fp8", fused_fp8, nbytes8), ("torch", eager, nbytes),
                                 ("fused_again", fused, nbytes), ("fp8_again", fused_fp8, nbytes8)]}[args.kv_cache]
                for what, fn, nb in runs:
                    us = 1000.0 * time_graph(fn, args.reps) / n_layers
                    row[f"{what}_us"] = us
                    row[f"{what}_GBps"] = nb / us / 1e3
                if args.kv_cache == "both":
                    row["fp8_speedup"] = ((row["fused_us"] + row["fused_again_us"]) /
                                          (row["fp8_us"] + row["fp8_again_us"]))
                rec["rows"].append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
                del layers
                torch.cuda.empty_cache()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
