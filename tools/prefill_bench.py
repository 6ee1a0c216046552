"""Prefill on the project's kernels (DESIGN §3.20): ``prefill_attention`` per layer against torch, and
``BatchDecoder.extend`` against the HF ``prefill`` on the Llama-2-7B-shaped synthetic model.  Prints one JSON line.

    python tools/prefill_bench.py [--layers 32] [--reps 20]

* attention: one layer at the Llama-2-7B (32 heads / 32 kv heads / hd 128) and Mistral-7B (32 / 8 / 128) shapes, fp16,
  16-bit and FP8 caches, T in {512, 2048, 8192} from position 0 and T in {1, 16, 256} at position 4096: µs per call
  (CUDA events, mean over --reps after a warm-up) and TFLOP/s of the causal FLOPs (4·hd per attended (query head,
  position) pair).  Beside it, what the HF path runs for the same 16-bit q, k, v: transformers' rotary embedding and
  apply_rotary_pos_emb, the copy into a static cache, and ``F.scaled_dot_product_attention`` on the flash backend
  (k / v repeated to the query heads before the timed window).  From position 0 SDPA runs ``is_causal``; for an
  extend, whose queries see nearly every cached position, it attends over all of them (flash's causal mask is aligned
  top-left, not to the end of the cache).
* whole prefill: ``BatchDecoder.prefill`` (the HF model, then the copy into the static cache) against
  ``BatchDecoder.extend`` on an idle slot, for prompts of 512, 2048 and 8192 tokens, 16-bit and FP8 caches: ms to the
  first token's logits (host clock around work that ends in a synchronise, best of 3 after a warm-up) and the increase
  of ``torch.cuda.max_memory_allocated`` over the memory allocated before the call.
* multi-turn: a 4096-token history plus a 256-token turn; ``extend`` of the turn against re-prefilling all 4352 tokens
  with ``prefill`` and with ``extend``.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.chain_decoder_bench import build_model, gpu_facts  # noqa: E402

FP8 = torch.float8_e4m3fn
MAX_LENGTH = 8448


def causal_flops(start, T, n_heads, hd):
    return 4.0 * hd * n_heads * sum(start + t + 1 for t in range(T))


def time_cuda(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e3          # µs


def attention_rows(reps):
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding, apply_rotary_pos_emb

    from autogptq_b200.attention import prefill_attention, quantize_kv

    dev, dt, hd = "cuda", torch.float16, 128
    cfg = LlamaConfig(hidden_size=4096, num_attention_heads=32, num_key_value_heads=32, head_dim=hd,
                      max_position_embeddings=MAX_LENGTH)
    rot = LlamaRotaryEmbedding(cfg, device=dev)
    rows = []
    g = torch.Generator(device=dev).manual_seed(0)
    for shape, (nh, nkv) in (("llama2_7b", (32, 32)), ("mistral_7b", (32, 8))):
        kc16 = torch.randn(1, nkv, MAX_LENGTH, hd, generator=g, device=dev).to(dt)
        vc16 = torch.randn(1, nkv, MAX_LENGTH, hd, generator=g, device=dev).to(dt)
        (kc8, ks), (vc8, vs) = quantize_kv(kc16), quantize_kv(vc16)
        for start, T in ((0, 512), (0, 2048), (0, 8192), (4096, 1), (4096, 16), (4096, 256)):
            q = torch.randn(1, T, nh * hd, generator=g, device=dev).to(dt)
            k = torch.randn(1, T, nkv * hd, generator=g, device=dev).to(dt)
            v = torch.randn(1, T, nkv * hd, generator=g, device=dev).to(dt)
            out = torch.empty_like(q)
            st = torch.tensor([start], dtype=torch.int64, device=dev)
            fl = causal_flops(start, T, nh, hd)
            row = dict(shape=shape, start=start, T=T, tflop=fl / 1e12)
            for name, kw, caches in (("c16", {}, (kc16, vc16)), ("fp8", dict(k_scale=ks, v_scale=vs), (kc8, vc8))):
                us = time_cuda(lambda: prefill_attention(q, k, v, *caches, st, rot.inv_freq, rot.attention_scaling,
                                                         hd ** -0.5, out, **kw), reps)
                row[f"{name}_us"], row[f"{name}_tflops"] = round(us, 1), round(fl / us / 1e6, 1)
            pid = (start + torch.arange(T, device=dev))[None]
            qv, kv_, vv = (x.view(1, T, -1, hd).transpose(1, 2) for x in (q, k, v))
            G = nh // nkv
            kfull = kc16[:, :, :start + T].repeat_interleave(G, 1).contiguous()
            vfull = vc16[:, :, :start + T].repeat_interleave(G, 1).contiguous()

            def torch_path():
                cos, sin = rot(q, pid)
                qh, kh = apply_rotary_pos_emb(qv, kv_, cos, sin)
                kc16[:, :, start:start + T].copy_(kh)
                vc16[:, :, start:start + T].copy_(vv)
                with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.FLASH_ATTENTION):
                    return torch.nn.functional.scaled_dot_product_attention(qh, kfull, vfull, is_causal=start == 0,
                                                                            scale=hd ** -0.5)

            us = time_cuda(torch_path, reps)
            row["torch_us"] = round(us, 1)
            row["torch_tflops"] = round(fl / us / 1e6, 1)
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
        del kc16, vc16, kc8, vc8, ks, vs
        torch.cuda.empty_cache()
    return rows


def timed_call(fn, reset):
    """(best ms of 3 after a warm-up, peak bytes above what was allocated before the call)."""
    best, peak = float("inf"), 0
    for i in range(4):
        reset()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        if i:
            best = min(best, ms)
            peak = max(peak, torch.cuda.max_memory_allocated() - base)
    return round(best, 2), peak


def model_rows(layers):
    from autogptq_b200 import BatchDecoder

    dev = torch.device("cuda")
    model = build_model(layers, 1, dev)
    g = torch.Generator(device=dev).manual_seed(1)
    prefill, turns = [], []
    for kv in (None, FP8):
        dec = BatchDecoder(model, max_batch=1, max_length=MAX_LENGTH, kv_cache_dtype=kv)
        name = "fp8" if kv else "c16"
        with torch.no_grad():
            for P in (512, 2048, 8192):
                ids = torch.randint(0, 32000, (P,), generator=g, device=dev)
                row = dict(cache=name, prompt=P)
                for what, fn in (("hf_prefill", lambda: dec.prefill(0, ids)), ("extend", lambda: dec.extend(0, ids))):
                    ms, peak = timed_call(fn, lambda: dec.release(0))
                    row[f"{what}_ms"], row[f"{what}_peak_gib"] = ms, round(peak / 2 ** 30, 3)
                prefill.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
            hist = torch.randint(0, 32000, (4096,), generator=g, device=dev)
            turn = torch.randint(0, 32000, (256,), generator=g, device=dev)
            full = torch.cat([hist, turn])

            def set_history():
                dec.release(0)
                dec.extend(0, hist)

            row = dict(cache=name, history=4096, turn=256)
            row["extend_turn_ms"], row["extend_turn_peak_gib"] = timed_call(lambda: dec.extend(0, turn), set_history)
            row["hf_prefill_4352_ms"], _ = timed_call(lambda: dec.prefill(0, full), lambda: dec.release(0))
            row["extend_4352_ms"], _ = timed_call(lambda: dec.extend(0, full), lambda: dec.release(0))
            row["extend_turn_peak_gib"] = round(row["extend_turn_peak_gib"] / 2 ** 30, 3)
            turns.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
        del dec
        torch.cuda.empty_cache()
    return prefill, turns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prefill_bench: needs a CUDA device")
    name, power = gpu_facts()
    attn = attention_rows(args.reps)
    prefill, turns = model_rows(args.layers)
    print(json.dumps(dict(gpu=name, power_limit=power, layers=args.layers, attention=attn, prefill=prefill,
                          multi_turn=turns)))


if __name__ == "__main__":
    main()
