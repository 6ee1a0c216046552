"""Decode tokens/s of a Llama-2-7B-shaped GPTQ model: ChainDecoder (one CUDA graph per token: a decode-chain launch per
decoder block, attention in torch between them) against the HF model's own eager decode step with the same QuantLinears,
with and without inject_fused_mlp.

    python tools/chain_decoder_bench.py [--layers 32] [--prompt 512] [--steps 128] [--batch 1] [--attention torch]

``--attention`` picks ChainDecoder's attention: ``torch`` (the default path; the HF baselines run too), ``fused``
(``fused_attention=True``) or ``both`` (the two decoders alternated, torch / fused / torch / fused, in one run; no HF
baselines).  Each ChainDecoder record has tokens/s and the split of a token between the chain launches, the attentions
and the rest.

Weights are synthetic, packed like bench.py's (uniform nibbles, unit-gain signed scales), with random norm weights, an
fp16 lm_head and embedding.  Prints one JSON line: tokens/s of each path, the split of a ChainDecoder token between the
chain launches and the attentions (each captured in a graph of its own and replayed), the ring slots of a block chain,
and the GPU name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_facts():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # noqa: BLE001 - a missing nvidia-smi leaves the field empty
        pl = f"unknown ({e})"
    return name, pl


def build_model(layers, batch, dev, seed=0):
    from transformers import LlamaConfig, LlamaForCausalLM
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding

    from bench import GROUP, synth_layer

    cfg = LlamaConfig(hidden_size=4096, intermediate_size=11008, num_attention_heads=32, num_key_value_heads=32,
                      num_hidden_layers=layers, vocab_size=32000, max_position_embeddings=4096, rms_norm_eps=1e-5)
    cfg._attn_implementation = "sdpa"
    with torch.device("meta"):
        model = LlamaForCausalLM(cfg)
    model = model.to_empty(device=dev).half()
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    for layer in model.model.layers:
        for mod, names in ((layer.self_attn, ("q_proj", "k_proj", "v_proj", "o_proj")),
                           (layer.mlp, ("gate_proj", "up_proj", "down_proj"))):
            for n in names:
                lin = getattr(mod, n)
                setattr(mod, n, synth_layer(lin.in_features, lin.out_features, GROUP, dev, gen))
        torch.cuda.empty_cache()
    with torch.no_grad():
        model.model.embed_tokens.weight.normal_(0, 1, generator=gen)
        model.lm_head.weight.normal_(0, 4096 ** -0.5, generator=gen)
        for mod in model.modules():
            if type(mod).__name__.endswith("RMSNorm"):
                mod.weight.uniform_(0.5, 1.5, generator=gen)
    model.model.rotary_emb = LlamaRotaryEmbedding(cfg, device=dev)
    return model.eval()


def time_graph(fn, reps, warm=3):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warm):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def timed_steps(step, tok, S):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(S):
        tok = step(tok)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / S


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--prompt", type=int, default=512)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--attention", choices=("torch", "fused", "both"), default="torch")
    args = ap.parse_args()
    from transformers import DynamicCache

    from autogptq_b200 import inject_fused_mlp
    from autogptq_b200.decoder import ChainDecoder

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power = gpu_facts()
    model = build_model(args.layers, args.batch, dev)
    B, T, S = args.batch, args.prompt, args.steps
    prompt = torch.randint(0, 32000, (B, T), device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    rec = {"gpu": name, "power_limit": power, "layers": args.layers, "batch": B, "prompt": T, "steps": S}

    inner = model.model

    def chain_decoder(fused):
        """One ChainDecoder run: (ms per token, split) with one CUDA graph per token."""
        dec = ChainDecoder(model, batch=B, max_length=T + S + 8, fused_attention=fused)
        info = dec.chains[1].info(), dec.chains[0].info()
        logits = dec.prefill(prompt)
        tok = logits.argmax(-1)
        for _ in range(3):                                   # capture + warm replays
            tok = dec.step(tok).argmax(-1)
        dec.position = T
        ms = timed_steps(lambda t: dec.step(t).argmax(-1), tok, S)

        # split: the chains alone and the attentions alone, each as one graph, at the middle of the timed window
        dec.position = T + S // 2
        chains_ms = time_graph(lambda: [c.run() for c in dec.chains], 20)

        def attn_only():
            if fused:
                for i in range(len(dec._attn_in)):
                    dec._fused_attention(i)
                return
            pos_ids = dec._pos.view(1, 1).expand(B, 1)
            cos, sin = inner.rotary_emb(dec._x0.view(B, 1, -1), pos_ids)
            mask = (dec._arange <= dec._pos).view(1, 1, 1, -1)
            for i in range(len(dec._attn_in)):
                dec._attention(i, cos, sin, mask)

        attn_ms = time_graph(attn_only, 20)
        del dec
        torch.cuda.empty_cache()
        return ms, {"chains": chains_ms, "attention": attn_ms, "rest": ms - chains_ms - attn_ms}, info

    if args.attention == "torch":
        ms, split, info = chain_decoder(False)
        rec["block_chain_info"], rec["first_chain_info"] = info
        rec["chain_decoder_ms_per_token"] = ms
        rec["chain_decoder_tokens_per_s"] = 1000.0 * B / ms
        rec["split_ms"] = split
    else:
        order = ["torch", "fused", "torch", "fused"] if args.attention == "both" else ["fused"]
        runs = {m: [] for m in order}
        for m in order:
            ms, split, info = chain_decoder(m == "fused")
            runs[m].append({"ms_per_token": ms, "tokens_per_s": 1000.0 * B / ms, "split_ms": split})
        rec["block_chain_info"], rec["first_chain_info"] = info
        rec["chain_decoder"] = runs
        print(json.dumps(rec))
        return

    def hf_decode(what):
        cache = DynamicCache(config=model.config)
        out = model(input_ids=prompt, past_key_values=cache, use_cache=True)
        t = out.logits[:, -1].argmax(-1, keepdim=True)
        for _ in range(3):
            t = model(input_ids=t, past_key_values=cache, use_cache=True).logits[:, -1].argmax(-1, keepdim=True)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(S):
            t = model(input_ids=t, past_key_values=cache, use_cache=True).logits[:, -1].argmax(-1, keepdim=True)
        b.record()
        torch.cuda.synchronize()
        m = a.elapsed_time(b) / S
        rec[f"{what}_ms_per_token"] = m
        rec[f"{what}_tokens_per_s"] = 1000.0 * B / m

    hf_decode("hf_eager")
    rec["fused_mlps"] = inject_fused_mlp(model)
    hf_decode("hf_eager_fused_mlp")
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
