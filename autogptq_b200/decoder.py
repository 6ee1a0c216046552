"""Greedy decoding of a GPTQ Llama / Mistral / Qwen2 model with one decode-chain launch per decoder block.

    dec = ChainDecoder(model, batch=1, max_length=2048)    # model: transformers *ForCausalLM with QuantLinear projections
    tokens = dec.generate(input_ids, max_new_tokens=128)   # prefill on the HF model, then one CUDA graph per token

Between two attentions a decoder layer is QuantLinears, elementwise work and one row reduction:

    o_proj(attn) -> h1 = x + o -> n2 = post_attention_layernorm(h1) -> gate|up -> silu*mul -> down
                 -> x' = h1 + down -> n1' = next input_layernorm(x') -> next q|k|v

The decode chain's norm stage inputs (``x_mode="add_rmsnorm"``) cover the adds and norms, so block i is one chain

    chain_0 = [input_layernorm_0 -> q|k|v_0]
    chain_i = [o_i, add_rmsnorm -> gate|up_i, silu_mul -> down_i, add_rmsnorm(input_layernorm_i+1) -> q|k|v_i+1]

(the last block ends at down_i).  Attention needs the KV cache and runs in torch between two chains: the model's own
rotary embedding and ``apply_rotary_pos_emb``, a static [batch, kv_heads, max_length, head_dim] cache written at a
device-side position, and ``F.scaled_dot_product_attention`` with GQA and a length mask; its output goes straight into
the next chain's o_proj input buffer.  The final add, ``model.model.norm`` and ``lm_head`` run in torch.  One token is
then n_layers + 1 chain launches and n_layers attentions, captured together in one CUDA graph.

``fused_attention=True`` runs each attention as one ``agb200_decode_attention`` launch instead (rotary embedding, cache
write and split-KV attention, ``autogptq_b200.attention``): a token is then 2·n_layers + 1 launches of the project's own
kernels plus the embedding, final norm and lm_head.  It rounds differently from SDPA (fp32 online softmax), so it is
opt-in.  With it, ``kv_cache_dtype=torch.float8_e4m3fn`` keeps the caches as E4M3 codes with a power-of-two scale per
cached row (``autogptq_b200.attention.quantize_kv``, DESIGN §3.19): half the cache bytes; the prompt's keys and values
are quantised at prefill, each step's by the attention kernel.

Mixtral-style models (``MixtralSparseMoeBlock`` MLPs whose ``experts`` are an ``autogptq_b200.QuantExperts``, see
``autogptq_b200.moe``) decode through the same graph with a different block (DESIGN §3.17):

    chain [o_i] -> moe_router: h1 = x + o, n2 = post_attention_layernorm(h1), logits, softmax, top-k, renormalise
                -> QuantExperts on (n2, top_k_index, top_k_weights)
                -> chain [add_rmsnorm(moe_i, h1; input_layernorm_i+1) -> q|k|v_i+1]

so a token is 5 to 8 launches per layer (the experts' forward is several), all in one graph.  Every buffer, the experts'
plans and their workspaces are allocated when the decoder is built.  ``prefill`` runs the HF model: a prompt of more
than 8 tokens (``MOE_DECODE_MAX_T``) makes each ``QuantExperts`` build its tensor-core weight copies on first use, K·N/2
bytes per layer, about 22 GB more for Mixtral-8x7B.  Router variants other than Mixtral's (Qwen2-MoE's shared expert,
DeepSeek, no renormalisation), experts that are not grouped, and models that mix dense and MoE layers are refused.

Scope: batch <= 2 (the chain's M), sequences in lockstep (one prompt length), greedy.  What does not fit raises
NotImplementedError naming the module.  Up to eight independent sequences of any lengths, admitted and retired between
steps: ``autogptq_b200.batch_decoder.BatchDecoder``.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import _lib
from .attention import FP8, attention_supported, decode_attention, decode_attention_workspace, quantize_kv
from .chain import DecodeChain, chain_supported
from .mlp import FusedQuantMLP, _is_silu
from .moe import QuantExperts, moe_router, router_supported
from .qlinear import QuantLinear

_RMSNORMS = ("LlamaRMSNorm", "MistralRMSNorm", "Qwen2RMSNorm", "MixtralRMSNorm")
_MOE_BLOCKS = ("MixtralSparseMoeBlock",)
_ROUTERS = ("MixtralTopKRouter",)


def _norm_of(mod, name: str, who: str = "ChainDecoder"):
    """(weight, eps) of an RMSNorm with transformers' Llama rounding: weight · rnd(h · rsqrt(mean(h²) + eps))."""
    if type(mod).__name__ not in _RMSNORMS or not hasattr(mod, "weight") or not hasattr(mod, "variance_epsilon"):
        raise NotImplementedError(f"{who}: {name} is {type(mod).__name__}; only Llama-style RMSNorm "
                                  f"({', '.join(_RMSNORMS)}) runs inside the decode chain")
    return mod.weight, float(mod.variance_epsilon)


def _plan_moe(i: int, mlp, H: int, batch: int, dtype):
    """(router weight [E, H], top_k, QuantExperts) of a Mixtral sparse MoE block, after checking that they fit."""
    where = f"model.layers.{i}.mlp"
    gate, experts = getattr(mlp, "gate", None), getattr(mlp, "experts", None)
    if type(gate).__name__ not in _ROUTERS:
        raise NotImplementedError(f"ChainDecoder: {where}.gate is {type(gate).__name__}; only {', '.join(_ROUTERS)} "
                                  "(softmax, top-k, renormalised weights) runs in the router kernel")
    w = getattr(gate, "weight", None)
    if getattr(gate, "bias", None) is not None:
        raise NotImplementedError(f"ChainDecoder: {where}.gate has a bias; the router kernel is bias-free")
    if not isinstance(w, torch.Tensor) or w.dim() != 2 or w.shape[1] != H:
        raise NotImplementedError(f"ChainDecoder: {where}.gate.weight has shape "
                                  f"{None if w is None else tuple(w.shape)}, not [num_experts, {H}]")
    if w.dtype != dtype:
        raise NotImplementedError(f"ChainDecoder: {where}.gate.weight is {w.dtype}, the activations {dtype}")
    if not isinstance(experts, QuantExperts):
        raise NotImplementedError(f"ChainDecoder: {where}.experts is {type(experts).__name__}, not "
                                  "autogptq_b200.QuantExperts (build one from the experts' QuantLinear layers with "
                                  "autogptq_b200.group_experts)")
    E, k = w.shape[0], int(getattr(gate, "top_k", 0))
    if experts.hidden_size != H or experts.num_experts != E:
        raise NotImplementedError(f"ChainDecoder: {where}.experts has {experts.num_experts} experts of hidden size "
                                  f"{experts.hidden_size}; the router has {E} of {H}")
    why = router_supported(batch, H, E, k, dtype)
    if why is not None:
        raise NotImplementedError(f"ChainDecoder: {where}.gate: {why}")
    return w.detach().contiguous(), k, experts


def _plan_layer(i: int, layer, batch: int, dtype):
    """The modules of decoder layer i that the chains read, after checking that they fit: (attn, mlp, ln1, ln2, moe)
    with moe = (router weight, top_k, QuantExperts) for a Mixtral sparse MoE block and None for a dense MLP."""
    attn, mlp = getattr(layer, "self_attn", None), getattr(layer, "mlp", None)
    if attn is None or mlp is None:
        raise NotImplementedError(f"ChainDecoder: model.layers.{i} has no self_attn / mlp")
    names = ("q_proj", "k_proj", "v_proj", "o_proj")
    for n in names:
        if not isinstance(getattr(attn, n, None), QuantLinear):
            raise NotImplementedError(f"ChainDecoder: model.layers.{i}.self_attn.{n} is "
                                      f"{type(getattr(attn, n, None)).__name__}, not autogptq_b200.QuantLinear")
    moe = None
    if type(mlp).__name__ in _MOE_BLOCKS:
        moe = _plan_moe(i, mlp, attn.q_proj.infeatures, batch, dtype)
        groups = {"self_attn.q_proj|k_proj|v_proj": [attn.q_proj, attn.k_proj, attn.v_proj],
                  "self_attn.o_proj": [attn.o_proj]}
    elif hasattr(mlp, "experts") or (hasattr(mlp, "gate") and not hasattr(mlp, "gate_proj")):
        raise NotImplementedError(f"ChainDecoder: model.layers.{i}.mlp is {type(mlp).__name__}; the only "
                                  f"mixture-of-experts block ChainDecoder runs is {', '.join(_MOE_BLOCKS)}")
    elif not isinstance(mlp, FusedQuantMLP):
        if not all(hasattr(mlp, n) for n in ("gate_proj", "up_proj", "down_proj")):
            raise NotImplementedError(f"ChainDecoder: model.layers.{i}.mlp ({type(mlp).__name__}) is not a "
                                      "gate/up/down MLP")
        if not _is_silu(getattr(mlp, "act_fn", None)):
            raise NotImplementedError(f"ChainDecoder: model.layers.{i}.mlp.act_fn is "
                                      f"{type(getattr(mlp, 'act_fn', None)).__name__}, not SiLU")
    if moe is None:
        for n in ("gate_proj", "up_proj", "down_proj"):
            if not isinstance(getattr(mlp, n), QuantLinear):
                raise NotImplementedError(f"ChainDecoder: model.layers.{i}.mlp.{n} is "
                                          f"{type(getattr(mlp, n)).__name__}, not autogptq_b200.QuantLinear")
        groups = {"self_attn.q_proj|k_proj|v_proj": [attn.q_proj, attn.k_proj, attn.v_proj],
                  "self_attn.o_proj": [attn.o_proj], "mlp.gate_proj|up_proj": [mlp.gate_proj, mlp.up_proj],
                  "mlp.down_proj": [mlp.down_proj]}
    for n, ls in groups.items():
        if not chain_supported(ls, batch):
            raise NotImplementedError(f"ChainDecoder: model.layers.{i}.{n} cannot run in a decode chain (needs "
                                      "infeatures % 128 == 0, group_size % 128 == 0 or -1, outfeatures % 32 == 0, "
                                      "sibling layers of one shape)")
    ln1 = _norm_of(getattr(layer, "input_layernorm", None), f"model.layers.{i}.input_layernorm")
    ln2 = _norm_of(getattr(layer, "post_attention_layernorm", None), f"model.layers.{i}.post_attention_layernorm")
    for w, n in ((ln1[0], "input_layernorm"), (ln2[0], "post_attention_layernorm")):
        if w.dtype != dtype:
            raise NotImplementedError(f"ChainDecoder: model.layers.{i}.{n}.weight is {w.dtype}, the activations "
                                      f"{dtype}")
    if attn.q_proj.infeatures > _lib.CHAIN_NORM_MAX_K:
        raise NotImplementedError(f"ChainDecoder: model.layers.{i}: hidden size {attn.q_proj.infeatures} > "
                                  f"{_lib.CHAIN_NORM_MAX_K}, the largest a chain norm stage takes")
    return attn, mlp, ln1, ln2, moe


def _is_moe(plans) -> bool:
    """Whether the layers of ``_plan_layer`` are all mixture-of-experts blocks (else all dense)."""
    moe = plans[0][4] is not None
    for i, p in enumerate(plans):
        if (p[4] is not None) != moe:
            raise NotImplementedError(f"ChainDecoder: model.layers.{i}.mlp is {type(p[1]).__name__} but "
                                      f"model.layers.0.mlp is {type(plans[0][1]).__name__}; a model that mixes dense "
                                      "and mixture-of-experts layers is not supported")
    return moe


def _rotary_params(rotary, head_dim: int, who: str = "ChainDecoder(fused_attention=True)"):
    """(inv_freq fp32 [head_dim/2], attention_scaling) of a rotary embedding whose frequencies do not depend on the
    sequence length; default, linear, llama3 and yarn all reduce to these two."""
    rope_type = getattr(rotary, "rope_type", "default")
    if rope_type in ("dynamic", "longrope"):
        raise NotImplementedError(f"{who}: model.model.rotary_emb is {rope_type!r} rope, "
                                  "whose inv_freq changes with the sequence length; a captured graph cannot follow it")
    inv_freq = getattr(rotary, "inv_freq", None)
    if inv_freq is None or inv_freq.dim() != 1 or inv_freq.numel() != head_dim // 2:
        n = None if inv_freq is None else tuple(inv_freq.shape)
        raise NotImplementedError(f"{who}: model.model.rotary_emb.inv_freq has shape {n}, "
                                  f"not [{head_dim // 2}] (partial rotary is not supported)")
    return inv_freq.detach().to(torch.float32).contiguous(), float(getattr(rotary, "attention_scaling", 1.0))


def _check_window(config, max_length: int, who: str = "ChainDecoder"):
    sw = getattr(config, "sliding_window", None)
    if getattr(config, "use_sliding_window", True) is False:
        sw = None
    if sw is not None and sw < max_length:
        raise NotImplementedError(f"{who}: the model attends through a sliding window of {sw} tokens, below "
                                  f"max_length={max_length}; the static cache holds full attention only")


def _kv_fp8(kv_cache_dtype, who: str) -> bool:
    """Whether the KV cache is FP8 (torch.float8_e4m3fn); None keeps it in the activation dtype.  Refuses the rest."""
    if kv_cache_dtype is None:
        return False
    if kv_cache_dtype == FP8:
        return True
    raise NotImplementedError(f"{who}: kv_cache_dtype {kv_cache_dtype}; supported: None (the activation dtype) or "
                              f"{FP8}")


def _kv_caches(n_layers: int, shape, dtype, device, fp8: bool):
    """(k_cache, v_cache, k_scale, v_scale): per-layer static caches of ``shape`` [B, n_kv, max_length, hd] in
    ``dtype``, or E4M3 codes with fp32 scales [B, n_kv, max_length] for ``fp8`` (else the scales are None)."""
    k = [torch.zeros(shape, dtype=FP8 if fp8 else dtype, device=device) for _ in range(n_layers)]
    v = [torch.zeros_like(c) for c in k]
    if not fp8:
        return k, v, None, None
    ks = [torch.ones(shape[:-1], dtype=torch.float32, device=device) for _ in range(n_layers)]
    return k, v, ks, [torch.ones_like(s) for s in ks]


def _store_kv(dec, i: int, index, keys, values):
    """The prompt's keys and values [.., n_kv, T, hd] into layer i's caches at ``index`` (quantised for FP8)."""
    if dec.k_scale is None:
        dec.k_cache[i][index].copy_(keys)
        dec.v_cache[i][index].copy_(values)
        return
    for cache, scale, x in ((dec.k_cache[i], dec.k_scale[i], keys), (dec.v_cache[i], dec.v_scale[i], values)):
        codes, sc = quantize_kv(x)
        cache.view(torch.uint8)[index].copy_(codes.view(torch.uint8))
        scale[index].copy_(sc)


class ChainDecoder:
    """Greedy decoder over a transformers ``LlamaForCausalLM`` / ``MistralForCausalLM`` / ``Qwen2ForCausalLM`` whose
    projections are ``autogptq_b200.QuantLinear`` (``FusedQuantMLP`` MLPs are accepted too), or a
    ``MixtralForCausalLM`` whose experts are ``autogptq_b200.QuantExperts``.  ``fused_attention``:
    run each layer's attention as one CUDA launch (``autogptq_b200.attention.decode_attention``) instead of torch.
    ``kv_cache_dtype``: None (the activation dtype) or ``torch.float8_e4m3fn`` (needs ``fused_attention``)."""

    def __init__(self, model, batch: int = 1, max_length: int = 2048, fused_attention: bool = False,
                 kv_cache_dtype=None):
        if not 1 <= batch <= _lib.CHAIN_MAX_M:
            raise NotImplementedError(f"ChainDecoder: batch {batch}; the decode chain runs 1..{_lib.CHAIN_MAX_M} rows")
        fp8 = _kv_fp8(kv_cache_dtype, "ChainDecoder")
        if fp8 and not fused_attention:
            raise NotImplementedError(f"ChainDecoder: kv_cache_dtype {FP8} needs fused_attention=True; the torch "
                                      "attention reads a 16-bit cache")
        inner = getattr(model, "model", None)
        if inner is None or not hasattr(inner, "layers") or not hasattr(model, "lm_head"):
            raise NotImplementedError(f"ChainDecoder: {type(model).__name__} is not a *ForCausalLM with model.layers "
                                      "and lm_head")
        for n in ("embed_tokens", "rotary_emb", "norm"):
            if not hasattr(inner, n):
                raise NotImplementedError(f"ChainDecoder: model.model has no {n}")
        self.model, self.batch, self.max_length = model, batch, int(max_length)
        cfg = model.config
        _check_window(cfg, self.max_length)
        self.dtype = inner.embed_tokens.weight.dtype
        if self.dtype not in (torch.float16, torch.bfloat16):
            raise NotImplementedError(f"ChainDecoder: activations are {self.dtype}; the chain computes in fp16 / bf16")
        self.fused_attention = bool(fused_attention)
        if self.fused_attention:
            hd = getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads
            n_kv = getattr(cfg, "num_key_value_heads", None) or cfg.num_attention_heads
            why = attention_supported(cfg.num_attention_heads, n_kv, hd, batch, self.max_length, self.dtype)
            if why is not None:
                raise NotImplementedError(f"ChainDecoder(fused_attention=True): model.layers.*.self_attn: {why}")
            self._inv_freq, self._attn_scaling = _rotary_params(inner.rotary_emb, hd)
        self.device = inner.embed_tokens.weight.device
        if self.device.type != "cuda":
            raise RuntimeError("ChainDecoder needs the model on a CUDA device")
        plans = [_plan_layer(i, layer, batch, self.dtype) for i, layer in enumerate(inner.layers)]
        if not plans:
            raise NotImplementedError("ChainDecoder: the model has no decoder layers")
        self.moe = _is_moe(plans)
        fw, feps = _norm_of(inner.norm, "model.norm")
        attn0 = plans[0][0]
        self.head_dim = attn0.head_dim
        self.scaling = attn0.scaling
        self.n_heads = attn0.q_proj.outfeatures // self.head_dim
        self.n_kv = attn0.k_proj.outfeatures // self.head_dim
        H = attn0.q_proj.infeatures

        B, L, dev, dt = batch, len(plans), self.device, self.dtype
        self.k_cache, self.v_cache, self.k_scale, self.v_scale = _kv_caches(
            len(plans), (B, self.n_kv, self.max_length, self.head_dim), dt, dev, fp8)
        self._pos = torch.zeros(1, dtype=torch.int64, device=dev)          # device-side position of the next token
        self._ids = torch.zeros(B, dtype=torch.int64, device=dev)
        self._arange = torch.arange(self.max_length, device=dev)
        self._length = 0                                                    # host copy of the position
        if self.fused_attention:                                            # shared by the layers (one stream)
            self._attn_ws = decode_attention_workspace(B, self.n_heads, self.n_kv, self.head_dim, self.max_length, dev)

        # chain_0 = [input_layernorm_0 -> q|k|v_0]
        self.chains = []
        ch = DecodeChain(M=B, dtype=dt, device=dev)
        self._x0 = ch.input(H)
        w, eps = plans[0][2]
        qkv = ch.stage([attn0.q_proj, attn0.k_proj, attn0.v_proj], self._x0, x_mode="rmsnorm", norm_weight=w, norm_eps=eps)
        self.chains.append(ch.build())
        self._qkv = [qkv]              # q, k, v of block i
        self._attn_in = []             # o_proj input of block i (written by the attention)
        if self.moe:
            self._build_moe(plans, H)
        else:
            self._build_dense(plans)
        self._final_norm = inner.norm
        self._graph = None
        self._logits = None

    def _build_dense(self, plans):
        """chain_i = [o_i, add_rmsnorm -> gate|up_i, silu_mul -> down_i, add_rmsnorm(input_layernorm_i+1) -> q|k|v_i+1]"""
        B, L, dev, dt = self.batch, len(plans), self.device, self.dtype
        resid = self._x0
        for i, (attn, mlp, _, (w2, eps2), _) in enumerate(plans):
            ch = DecodeChain(M=B, dtype=dt, device=dev)
            a_in = ch.input(attn.o_proj.infeatures)
            (o,) = ch.stage([attn.o_proj], a_in)
            gate, up, h1 = ch.stage([mlp.gate_proj, mlp.up_proj], o, x2=resid, x_mode="add_rmsnorm", norm_weight=w2,
                                    norm_eps=eps2)
            (down,) = ch.stage([mlp.down_proj], gate, x2=up, x_mode="silu_mul")
            if i + 1 < L:
                na = plans[i + 1][0]
                w1, eps1 = plans[i + 1][2]
                q, k, v, resid = ch.stage([na.q_proj, na.k_proj, na.v_proj], down, x2=h1, x_mode="add_rmsnorm",
                                          norm_weight=w1, norm_eps=eps1)
                self._qkv.append((q, k, v))
            else:
                self._last = (h1, down)
            self._attn_in.append(a_in)
            self.chains.append(ch.build())

    def _build_moe(self, plans, H: int):
        """Per block i: chain [o_i]; the router (h1 = x + o, n2 = post_attention_layernorm(h1), top-k); the grouped
        experts on n2; then chain [add_rmsnorm(moe_i, h1; input_layernorm_i+1) -> q|k|v_i+1], which publishes the next
        residual.  Every buffer, the experts' plans and their workspaces are allocated here, once."""
        B, L, dev, dt = self.batch, len(plans), self.device, self.dtype
        self._o_chains, self._qkv_chains, self._moe_layers = [], [], []
        resid = self._x0
        for i, (attn, _, _, (w2, eps2), (gate_w, k, experts)) in enumerate(plans):
            ch = DecodeChain(M=B, dtype=dt, device=dev)
            a_in = ch.input(attn.o_proj.infeatures)
            (o,) = ch.stage([attn.o_proj], a_in)
            self._o_chains.append(ch.build())
            self._attn_in.append(a_in)
            h1, n2, out = (torch.zeros((B, H), dtype=dt, device=dev) for _ in range(3))
            idx = torch.zeros((B, k), dtype=torch.int32, device=dev)
            wts = torch.zeros((B, k), dtype=torch.float32, device=dev)
            plan, ws = experts._static_buffers(B, k, dt, dev)
            self._moe_layers.append(dict(o=o, resid=resid, w2=w2, eps2=eps2, gate=gate_w, k=k, experts=experts,
                                         h1=h1, n2=n2, idx=idx, w=wts, out=out, plan=plan, ws=ws))
            if i + 1 < L:
                na = plans[i + 1][0]
                w1, eps1 = plans[i + 1][2]
                ch = DecodeChain(M=B, dtype=dt, device=dev)
                q, kk, v, resid = ch.stage([na.q_proj, na.k_proj, na.v_proj], out, x2=h1, x_mode="add_rmsnorm",
                                           norm_weight=w1, norm_eps=eps1)
                self._qkv.append((q, kk, v))
                self._qkv_chains.append(ch.build())
            else:
                self._last = (h1, out)

    def _moe_block(self, i: int):
        """Block i after its attention: o_proj, the router and the experts, then the next block's q|k|v."""
        m = self._moe_layers[i]
        self._o_chains[i].run()
        moe_router(m["o"], m["resid"], m["w2"], m["eps2"], m["gate"], m["k"], h=m["h1"], n=m["n2"], idx=m["idx"],
                   w=m["w"])
        m["experts"]._forward(m["n2"], m["idx"], m["w"], out=m["out"], plan=m["plan"], ws=m["ws"])
        if i < len(self._qkv_chains):
            self._qkv_chains[i].run()

    # ------------------------------------------------------------------ state
    @property
    def position(self) -> int:
        """Tokens in the cache: the position the next step writes."""
        return self._length

    @position.setter
    def position(self, p: int):
        if not 0 <= p <= self.max_length:
            raise ValueError(f"position {p} outside 0..{self.max_length}")
        self._pos.fill_(p)
        self._length = int(p)

    @torch.no_grad()
    def prefill(self, input_ids: torch.Tensor) -> torch.Tensor:
        """Run the prompt [batch, T] through the HF model (its own prefill kernels), copy its cache into the static one
        and return the logits of the last position [batch, vocab]."""
        from transformers import DynamicCache

        ids = input_ids.to(self.device)
        if ids.dim() != 2 or ids.shape[0] != self.batch:
            raise ValueError(f"input_ids must be [{self.batch}, T] (sequences in lockstep), got {tuple(ids.shape)}")
        T = ids.shape[1]
        if not 1 <= T < self.max_length:
            raise ValueError(f"prompt length {T} must be in 1..{self.max_length - 1}")
        cache = DynamicCache(config=self.model.config)
        out = self.model(input_ids=ids, past_key_values=cache, use_cache=True)
        for i, lay in enumerate(cache.layers):
            _store_kv(self, i, (slice(None), slice(None), slice(0, T)), lay.keys, lay.values)
        self.position = T
        return out.logits[:, -1]

    # ------------------------------------------------------------------ one token
    def _attention(self, i: int, cos, sin, mask):
        from transformers.models.llama.modeling_llama import apply_rotary_pos_emb

        B, hd = self.batch, self.head_dim
        q, k, v = self._qkv[i]
        q = q.view(B, 1, self.n_heads, hd).transpose(1, 2)
        k = k.view(B, 1, self.n_kv, hd).transpose(1, 2)
        v = v.view(B, 1, self.n_kv, hd).transpose(1, 2)
        q, k = apply_rotary_pos_emb(q, k, cos, sin)
        self.k_cache[i].index_copy_(2, self._pos, k)
        self.v_cache[i].index_copy_(2, self._pos, v)
        o = F.scaled_dot_product_attention(q, self.k_cache[i], self.v_cache[i], attn_mask=mask, scale=self.scaling,
                                           enable_gqa=self.n_kv != self.n_heads)
        self._attn_in[i].copy_(o.transpose(1, 2).reshape(B, -1))

    def _fused_attention(self, i: int):
        q, k, v = self._qkv[i]
        fp8 = {} if self.k_scale is None else dict(k_scale=self.k_scale[i], v_scale=self.v_scale[i])
        decode_attention(q, k, v, self.k_cache[i], self.v_cache[i], self._pos, self._inv_freq, self._attn_scaling,
                         self.scaling, self._attn_in[i], self._attn_ws, **fp8)

    def _step_body(self) -> torch.Tensor:
        inner = self.model.model
        self._x0.copy_(inner.embed_tokens(self._ids))
        tail = self._moe_block if self.moe else (lambda i: self.chains[i + 1].run())
        if self.fused_attention:
            self.chains[0].run()
            for i in range(len(self._attn_in)):
                self._fused_attention(i)
                tail(i)
        else:
            pos_ids = self._pos.view(1, 1).expand(self.batch, 1)
            cos, sin = inner.rotary_emb(self._x0.view(self.batch, 1, -1), pos_ids)
            mask = (self._arange <= self._pos).view(1, 1, 1, -1)
            self.chains[0].run()
            for i in range(len(self._attn_in)):
                self._attention(i, cos, sin, mask)
                tail(i)
        h1, down = self._last
        n = self._final_norm(h1 + down)
        logits = self.model.lm_head(n)
        self._pos.add_(1)
        return logits

    @torch.no_grad()
    def step(self, ids: torch.Tensor, use_graph: bool = True) -> torch.Tensor:
        """Decode one token per sequence: ``ids`` [batch] -> logits [batch, vocab] (a buffer the next step overwrites
        when ``use_graph``).  The first graph step captures the whole step in one CUDA graph; later steps replay it."""
        if self._length >= self.max_length:
            raise RuntimeError(f"the static cache is full ({self.max_length} tokens)")
        self._ids.copy_(ids.reshape(-1).to(self._ids.device))
        if not use_graph:
            logits = self._step_body()
        else:
            if self._graph is None:
                p = self._length
                side = torch.cuda.Stream(self.device)
                side.wait_stream(torch.cuda.current_stream(self.device))
                with torch.cuda.stream(side):                 # warm-up outside the graph (library workspaces)
                    self._step_body()
                torch.cuda.current_stream(self.device).wait_stream(side)
                self.position = p
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._logits = self._step_body()
                self._graph = g
                self.position = p
            self._graph.replay()
            logits = self._logits
        self._length += 1
        return logits

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, max_new_tokens: int) -> torch.Tensor:
        """Greedy decoding: prompt [batch, T] -> [batch, T + max_new_tokens]."""
        if input_ids.shape[1] + max_new_tokens > self.max_length:
            raise ValueError(f"prompt + {max_new_tokens} new tokens exceed max_length={self.max_length}")
        logits = self.prefill(input_ids)
        out = [input_ids.to(self.device)]
        for t in range(max_new_tokens):
            tok = logits.argmax(-1)
            out.append(tok.view(-1, 1))
            if t + 1 < max_new_tokens:
                logits = self.step(tok)
        return torch.cat(out, dim=1)


__all__ = ["ChainDecoder"]
