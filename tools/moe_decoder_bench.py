"""Decode tokens/s of a Mixtral-8x7B-shaped GPTQ model: ChainDecoder (one CUDA graph per token: chains for the
attention projections, the MoE router kernel and the grouped experts) against the HF model's own eager decode step
with the same modules.

    python tools/moe_decoder_bench.py [--layers 32] [--prompts 512,3584] [--batches 1,2] [--steps 64]

Shapes: H 4096, I 14336, 8 experts, top-2, 32/8/128 heads, vocab 32000.  Weights are synthetic, packed like bench.py's
(about 23 GB of experts), with random norm and router weights.  The cache is filled synthetically and ``position`` set
instead of running an HF prefill, so the experts' tensor-core copies are never built; the HF baseline decodes from a
DynamicCache of the same length.  For every batch × prompt length the two attention paths run (torch, then fused),
each record with ms per token, tokens/s, and the split of a token between the chains, the attentions, the routers and
the experts (each part captured in a graph of its own and replayed), the router's µs per layer and the rest.  Prints
one JSON line, with the GPU name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.chain_decoder_bench import gpu_facts, time_graph, timed_steps  # noqa: E402


def build_model(layers, dev, seed=0):
    from transformers import MixtralConfig, MixtralForCausalLM
    from transformers.models.mixtral.modeling_mixtral import MixtralRotaryEmbedding

    from autogptq_b200 import QuantExperts
    from bench import GROUP, synth_layer

    cfg = MixtralConfig(hidden_size=4096, intermediate_size=14336, num_attention_heads=32, num_key_value_heads=8,
                        num_hidden_layers=layers, num_local_experts=8, num_experts_per_tok=2, vocab_size=32000,
                        max_position_embeddings=32768, rms_norm_eps=1e-5)
    cfg._attn_implementation = "sdpa"
    with torch.device("meta"):
        model = MixtralForCausalLM(cfg)
        for layer in model.model.layers:               # never materialise the 16-bit experts
            layer.mlp.experts = torch.nn.Module()
    model = model.to_empty(device=dev).half()
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    H, I, E = cfg.hidden_size, cfg.intermediate_size, cfg.num_local_experts
    for layer in model.model.layers:
        at = layer.self_attn
        for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
            lin = getattr(at, n)
            setattr(at, n, synth_layer(lin.in_features, lin.out_features, GROUP, dev, gen))
        layer.mlp.experts = QuantExperts([synth_layer(H, I, GROUP, dev, gen) for _ in range(E)],
                                         [synth_layer(H, I, GROUP, dev, gen) for _ in range(E)],
                                         [synth_layer(I, H, GROUP, dev, gen) for _ in range(E)])
        torch.cuda.empty_cache()
    with torch.no_grad():
        model.model.embed_tokens.weight.normal_(0, 1, generator=gen)
        model.lm_head.weight.normal_(0, H ** -0.5, generator=gen)
        for mod in model.modules():
            if type(mod).__name__.endswith("RMSNorm"):
                mod.weight.uniform_(0.5, 1.5, generator=gen)
            if type(mod).__name__ == "MixtralTopKRouter":
                mod.weight.normal_(0, 2 * H ** -0.5, generator=gen)
    model.model.rotary_emb = MixtralRotaryEmbedding(cfg, device=dev)
    return model.eval()


@torch.no_grad()
def chain_decoder(model, B, T, S, fused, dev):
    """One ChainDecoder run at a synthetic cache of T positions: (ms per token, split)."""
    from autogptq_b200.decoder import ChainDecoder
    from autogptq_b200.moe import moe_router

    inner = model.model
    dec = ChainDecoder(model, batch=B, max_length=T + S + 8, fused_attention=fused)
    gen = torch.Generator(device=dev).manual_seed(2)
    for k, v in zip(dec.k_cache, dec.v_cache):
        k[:, :, :T].normal_(0, 1, generator=gen)
        v[:, :, :T].normal_(0, 1, generator=gen)
    dec.position = T
    tok = torch.randint(0, 32000, (B,), device=dev, generator=gen)
    for _ in range(3):                                   # capture + warm replays
        tok = dec.step(tok).argmax(-1)
    dec.position = T
    ms = timed_steps(lambda t: dec.step(t).argmax(-1), tok, S)

    # split: each part alone as one graph, at the middle of the timed window
    dec.position = T + S // 2
    L = len(dec._attn_in)
    chains_ms = time_graph(lambda: [c.run() for c in [dec.chains[0]] + dec._o_chains + dec._qkv_chains], 20)

    def routers():
        for m in dec._moe_layers:
            moe_router(m["o"], m["resid"], m["w2"], m["eps2"], m["gate"], m["k"], h=m["h1"], n=m["n2"], idx=m["idx"],
                       w=m["w"])

    def experts():
        for m in dec._moe_layers:
            m["experts"]._forward(m["n2"], m["idx"], m["w"], out=m["out"], plan=m["plan"], ws=m["ws"])

    def attn_only():
        if fused:
            for i in range(L):
                dec._fused_attention(i)
            return
        pos_ids = dec._pos.view(1, 1).expand(B, 1)
        cos, sin = inner.rotary_emb(dec._x0.view(B, 1, -1), pos_ids)
        mask = (dec._arange <= dec._pos).view(1, 1, 1, -1)
        for i in range(L):
            dec._attention(i, cos, sin, mask)

    router_ms = time_graph(routers, 50)
    experts_ms = time_graph(experts, 20)
    attn_ms = time_graph(attn_only, 20)
    del dec
    torch.cuda.empty_cache()
    split = {"chains": chains_ms, "attention": attn_ms, "routers": router_ms, "experts": experts_ms,
             "rest": ms - chains_ms - attn_ms - router_ms - experts_ms}
    return {"ms_per_token": ms, "tokens_per_s": 1000.0 * B / ms, "split_ms": split,
            "router_us_per_layer": 1000.0 * router_ms / L}


@torch.no_grad()
def hf_decode(model, B, T, S, dev):
    """The HF model's eager decode step with the same modules, from a DynamicCache of T synthetic positions."""
    from transformers import DynamicCache

    cfg = model.config
    hd = cfg.hidden_size // cfg.num_attention_heads
    cache = DynamicCache(config=cfg)
    gen = torch.Generator(device=dev).manual_seed(2)
    for i in range(cfg.num_hidden_layers):
        kv = [torch.randn((B, cfg.num_key_value_heads, T, hd), device=dev, generator=gen).half() for _ in range(2)]
        cache.update(kv[0], kv[1], i)
    t = torch.randint(0, 32000, (B, 1), device=dev, generator=gen)
    step = lambda t: model(input_ids=t, past_key_values=cache, use_cache=True).logits[:, -1].argmax(-1, keepdim=True)
    for _ in range(3):
        t = step(t)
    ms = timed_steps(step, t, S)
    return {"ms_per_token": ms, "tokens_per_s": 1000.0 * B / ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--prompts", default="512,3584")
    ap.add_argument("--batches", default="1,2")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--no-hf", action="store_true", help="skip the HF eager baseline")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power = gpu_facts()
    model = build_model(args.layers, dev)
    rec = {"gpu": name, "power_limit": power, "layers": args.layers, "steps": args.steps,
           "experts_gb": sum(sum(t.numel() * t.element_size() for t in (l.qweight, l.qzeros, l.scales))
                             for lay in model.model.layers for l in lay.mlp.experts._layers()) / 1e9,
           "runs": []}
    for B in (int(b) for b in args.batches.split(",")):
        for T in (int(p) for p in args.prompts.split(",")):
            r = {"batch": B, "prompt": T}
            for f in (False, True):
                r["fused_attention" if f else "torch_attention"] = chain_decoder(model, B, T, args.steps, f, dev)
            if not args.no_hf:
                r["hf_eager"] = hf_decode(model, B, T, args.steps // 2, dev)
            rec["runs"].append(r)
            print(f"# {json.dumps(r)}", file=sys.stderr, flush=True)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
