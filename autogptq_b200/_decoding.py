"""The front end ``ChainDecoder`` and ``BatchDecoder`` share (DESIGN §3.18): reading the model, the dense-layer rules and
the Mixtral block's (router, grouped experts, no mixed dense and MoE layers), allocating the KV cache the decoder chose
(``autogptq_b200.kv_cache``), the HF prefill into it, the extend of cache rows on the project's kernels (DESIGN §3.20),
each row's sampling parameters (DESIGN §3.21), and the warm-up, capture and replay of a step's CUDA graphs (the step,
and the step followed by the sampling kernel)."""
from __future__ import annotations

import torch

from . import _lib
from .attention import FP8
from .mlp import FusedQuantMLP, _is_silu
from .moe import QuantExperts, router_supported
from .qlinear import QuantLinear
from .sampling import SamplingState

_RMSNORMS = ("LlamaRMSNorm", "MistralRMSNorm", "Qwen2RMSNorm", "MixtralRMSNorm")
_MOE_BLOCKS = ("MixtralSparseMoeBlock",)
_ROUTERS = ("MixtralTopKRouter",)


def _is_moe_block(mlp) -> bool:
    """Whether a layer's mlp is a mixture-of-experts block: a known one, or any with experts or a router gate."""
    return (type(mlp).__name__ in _MOE_BLOCKS or hasattr(mlp, "experts")
            or (hasattr(mlp, "gate") and not hasattr(mlp, "gate_proj")))


def _norm_of(mod, name: str, who: str = "ChainDecoder"):
    """(weight, eps) of an RMSNorm with transformers' Llama rounding: weight · rnd(h · rsqrt(mean(h²) + eps))."""
    if type(mod).__name__ not in _RMSNORMS or not hasattr(mod, "weight") or not hasattr(mod, "variance_epsilon"):
        raise NotImplementedError(f"{who}: {name} is {type(mod).__name__}; only Llama-style RMSNorm "
                                  f"({', '.join(_RMSNORMS)}) runs inside the decode chain")
    return mod.weight, float(mod.variance_epsilon)


def _quant_linear(who: str, mod, where: str, name: str) -> QuantLinear:
    lin = getattr(mod, name, None)
    if not isinstance(lin, QuantLinear):
        raise NotImplementedError(f"{who}: {where}.{name} is {type(lin).__name__}, not autogptq_b200.QuantLinear")
    return lin


def _rotary_params(rotary, head_dim: int, who: str):
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


def _plan_common(i: int, layer, dtype, who: str):
    """(attn, mlp, ln1, ln2) of decoder layer i after checking the rules every decoder shares: q/k/v/o
    ``QuantLinear``, a SiLU gate/up/down MLP of ``QuantLinear`` (or ``FusedQuantMLP``), Llama-style norms in the
    activation ``dtype``.  A mixture-of-experts mlp (``_is_moe_block``) is left to the caller to plan or refuse."""
    where = f"model.layers.{i}"
    attn, mlp = getattr(layer, "self_attn", None), getattr(layer, "mlp", None)
    if attn is None or mlp is None:
        raise NotImplementedError(f"{who}: {where} has no self_attn / mlp")
    for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
        _quant_linear(who, attn, f"{where}.self_attn", n)
    if not _is_moe_block(mlp):
        if not isinstance(mlp, FusedQuantMLP):
            if not all(hasattr(mlp, n) for n in ("gate_proj", "up_proj", "down_proj")):
                raise NotImplementedError(f"{who}: {where}.mlp ({type(mlp).__name__}) is not a gate/up/down MLP")
            if not _is_silu(getattr(mlp, "act_fn", None)):
                raise NotImplementedError(f"{who}: {where}.mlp.act_fn is "
                                          f"{type(getattr(mlp, 'act_fn', None)).__name__}, not SiLU")
        for n in ("gate_proj", "up_proj", "down_proj"):
            _quant_linear(who, mlp, f"{where}.mlp", n)
    norms = [(n, _norm_of(getattr(layer, n, None), f"{where}.{n}", who))
             for n in ("input_layernorm", "post_attention_layernorm")]
    for n, (w, _) in norms:
        if w.dtype != dtype:
            raise NotImplementedError(f"{who}: {where}.{n}.weight is {w.dtype}, the activations {dtype}")
    return attn, mlp, norms[0][1], norms[1][1]


def _plan_moe(i: int, mlp, H: int, batch: int, dtype, who: str = "ChainDecoder"):
    """(router weight [E, H], top_k, QuantExperts) of a Mixtral sparse MoE block (``_is_moe_block``), after checking
    that they fit the router kernel at ``batch`` rows and the grouped experts."""
    where = f"model.layers.{i}.mlp"
    if type(mlp).__name__ not in _MOE_BLOCKS:
        raise NotImplementedError(f"{who}: {where} is {type(mlp).__name__}; the only mixture-of-experts block {who} "
                                  f"runs is {', '.join(_MOE_BLOCKS)}")
    gate, experts = getattr(mlp, "gate", None), getattr(mlp, "experts", None)
    if type(gate).__name__ not in _ROUTERS:
        raise NotImplementedError(f"{who}: {where}.gate is {type(gate).__name__}; only {', '.join(_ROUTERS)} "
                                  "(softmax, top-k, renormalised weights) runs in the router kernel")
    w = getattr(gate, "weight", None)
    if getattr(gate, "bias", None) is not None:
        raise NotImplementedError(f"{who}: {where}.gate has a bias; the router kernel is bias-free")
    if not isinstance(w, torch.Tensor) or w.dim() != 2 or w.shape[1] != H:
        raise NotImplementedError(f"{who}: {where}.gate.weight has shape "
                                  f"{None if w is None else tuple(w.shape)}, not [num_experts, {H}]")
    if w.dtype != dtype:
        raise NotImplementedError(f"{who}: {where}.gate.weight is {w.dtype}, the activations {dtype}")
    if not isinstance(experts, QuantExperts):
        raise NotImplementedError(f"{who}: {where}.experts is {type(experts).__name__}, not "
                                  "autogptq_b200.QuantExperts (build one from the experts' QuantLinear layers with "
                                  "autogptq_b200.group_experts)")
    E, k = w.shape[0], int(getattr(gate, "top_k", 0))
    if experts.hidden_size != H or experts.num_experts != E:
        raise NotImplementedError(f"{who}: {where}.experts has {experts.num_experts} experts of hidden size "
                                  f"{experts.hidden_size}; the router has {E} of {H}")
    why = router_supported(batch, H, E, k, dtype)
    if why is not None:
        raise NotImplementedError(f"{who}: {where}.gate: {why}")
    return w.detach().contiguous(), k, experts


def _plan_experts(plans, dtype, device, who: str):
    """Create every Mixtral block's expert plan (``QuantExperts._plan``) before the caches exist.  Whether the grouped
    experts' decode kernels fit the device's shared memory is ``agb200_moe_create``'s decision; a block they do not fit
    (ENOSUP) is refused here, naming the layer, instead of failing at the first step.  The plans are cached, so the
    decoder's static buffers reuse them."""
    for i, p in enumerate(plans):
        if p[4] is None:
            continue
        try:
            p[4][2]._plan(dtype, device)
        except _lib.B200KernelError as e:
            if e.code != _lib.ENOSUP:
                raise
            raise NotImplementedError(f"{who}: model.layers.{i}.mlp.experts cannot run on this device: {e}") from None


def _is_moe(plans, who: str = "ChainDecoder") -> bool:
    """Whether the layer plans (attn, mlp, ln1, ln2, moe) are all mixture-of-experts blocks (moe not None), else all
    dense; a model that mixes the two is refused."""
    moe = plans[0][4] is not None
    for i, p in enumerate(plans):
        if (p[4] is not None) != moe:
            raise NotImplementedError(f"{who}: model.layers.{i}.mlp is {type(p[1]).__name__} but "
                                      f"model.layers.0.mlp is {type(plans[0][1]).__name__}; a model that mixes dense "
                                      "and mixture-of-experts layers is not supported")
    return moe


class DecoderBase:
    """Base of a decoder over a KV cache whose step is one captured CUDA graph.  A subclass sets ``_who`` (the prefix
    of its refusals) and ``_plan`` (a layer's plan, starting from ``_plan_common``).  Its constructor calls
    ``_read_model``, sets ``_cache`` (a ``KVCache`` or ``PagedKVCache``, not yet allocated), checks its kernels' limits
    on the geometry, calls ``_read_layers``, checks what spans the layers and calls ``_allocate`` last, so every refusal
    comes before the cache is allocated (a refusal that asks the device, such as a decode chain's shared memory, takes
    ``_cuda_device`` first).  It then sets ``_pos``, the device positions its ``_step_body`` reads and advances."""

    # ------------------------------------------------------------------ reading the model
    def _read_model(self, model, max_length: int, kv_cache_dtype):
        """The model's structure, activation dtype, sliding window and attention geometry (from the config)."""
        who = self._who
        self._fp8 = _kv_fp8(kv_cache_dtype, who)
        inner = getattr(model, "model", None)
        if inner is None or not hasattr(inner, "layers") or not hasattr(model, "lm_head"):
            raise NotImplementedError(f"{who}: {type(model).__name__} is not a *ForCausalLM with model.layers and "
                                      "lm_head")
        for n in ("embed_tokens", "rotary_emb", "norm"):
            if not hasattr(inner, n):
                raise NotImplementedError(f"{who}: model.model has no {n}")
        self.model, self.max_length = model, int(max_length)
        cfg = model.config
        _check_window(cfg, self.max_length, who)
        self.dtype = inner.embed_tokens.weight.dtype
        if self.dtype not in (torch.float16, torch.bfloat16):
            raise NotImplementedError(f"{who}: activations are {self.dtype}; the kernels compute in fp16 / bf16")
        self.hidden_size, self.n_heads = cfg.hidden_size, cfg.num_attention_heads
        self.head_dim = getattr(cfg, "head_dim", None) or self.hidden_size // self.n_heads
        self.n_kv = getattr(cfg, "num_key_value_heads", None) or self.n_heads

    def _read_layers(self):
        """``_plans`` (``_plan`` of each layer, whose q/k/v/o must have the config's geometry), ``scaling`` and
        ``_final``: model.norm's (weight, eps)."""
        inner, who = self.model.model, self._who
        H, q, kv = self.hidden_size, self.n_heads * self.head_dim, self.n_kv * self.head_dim
        self._plans = []
        for i, layer in enumerate(inner.layers):
            plan = self._plan(i, layer)
            for n, shape in (("q_proj", (H, q)), ("k_proj", (H, kv)), ("v_proj", (H, kv)), ("o_proj", (q, H))):
                lin = getattr(plan[0], n)
                if (lin.infeatures, lin.outfeatures) != shape:
                    raise NotImplementedError(
                        f"{who}: model.layers.{i}.self_attn.{n} maps {lin.infeatures} -> {lin.outfeatures} features; "
                        f"the config (hidden_size {H}, {self.n_heads} heads, {self.n_kv} kv heads, head_dim "
                        f"{self.head_dim}) needs {shape[0]} -> {shape[1]}")
            self._plans.append(plan)
        if not self._plans:
            raise NotImplementedError(f"{self._who}: the model has no decoder layers")
        self.scaling = self._plans[0][0].scaling
        self._final = _norm_of(inner.norm, "model.norm", self._who)

    # ------------------------------------------------------------------ the KV cache
    def _cuda_device(self) -> torch.device:
        """``device``: the model's, which must be a CUDA device."""
        self.device = self.model.model.embed_tokens.weight.device
        if self.device.type != "cuda":
            raise RuntimeError(f"{self._who} needs the model on a CUDA device")
        return self.device

    def _allocate(self, rows: int):
        """After every refusal: the CUDA device, the KV cache ``_cache`` the subclass chose (``k_cache`` / ``v_cache`` /
        ``k_scale`` / ``v_scale`` are its tensors) and the step's token ids of ``rows`` rows."""
        self._cuda_device()
        c = self._cache
        c.allocate(len(self._plans), self.device)
        self.k_cache, self.v_cache, self.k_scale, self.v_scale = c.k, c.v, c.k_scale, c.v_scale
        self._ids = torch.zeros(rows, dtype=torch.int64, device=self.device)
        self._graphs = {}                               # step body name -> (CUDA graph, its output buffers)
        self._sampling = SamplingState(rows, self.device)   # each row's sampling parameters, greedy until set

    def _prefill_cache(self, ids: torch.Tensor, rows: slice) -> torch.Tensor:
        """Run ``ids`` [len(rows), T] through the HF model (its own prefill kernels) and store every layer's keys and
        values into the cache at ``rows``, positions :T.  Returns the model's logits [len(rows), T, vocab]."""
        from transformers import DynamicCache

        cache = DynamicCache(config=self.model.config)
        out = self.model(input_ids=ids, past_key_values=cache, use_cache=True)
        for i, lay in enumerate(cache.layers):
            self._cache.store(i, rows, lay.keys, lay.values)
        return out.logits

    def _extend(self, ids: torch.Tensor, rows: slice, starts) -> torch.Tensor:
        """Append ``ids`` [n, T] to cache rows ``rows`` (n of them) at positions ``starts`` (n host ints) .. + T - 1
        on the project's kernels, and return the logits of the last new position [n, vocab].  The model's own modules
        run every layer (its QuantLinear projections at M = n·T, its norms and MLP), so every rounding outside the
        attention is HF's; the cache's prefill attention writes k̂ and v into it and attends causally over it.
        No DynamicCache is built and only the last position reaches model.norm and lm_head."""
        inner = self.model.model
        if not hasattr(self, "_inv_freq"):
            self._inv_freq, self._attn_scaling = _rotary_params(inner.rotary_emb, self.head_dim, self._who)
        n, T = ids.shape
        start = torch.tensor(list(starts), dtype=torch.int64, device=self.device)
        h = inner.embed_tokens(ids)
        out = torch.empty((n, T, self.n_heads * self.head_dim), dtype=self.dtype, device=self.device)
        for i, layer in enumerate(inner.layers):
            attn = self._plans[i][0]
            x = layer.input_layernorm(h)
            self._cache.prefill(i, rows, attn.q_proj(x), attn.k_proj(x), attn.v_proj(x), start, self._inv_freq,
                                self._attn_scaling, self.scaling, out)
            h = h + attn.o_proj(out)
            h = h + layer.mlp(layer.post_attention_layernorm(h))
        return self.model.lm_head(inner.norm(h[:, -1:]))[:, 0]

    # ------------------------------------------------------------------ one step
    def _run_step(self, ids: torch.Tensor, use_graph: bool, body=None):
        """A step body on ``ids``, eagerly or through that body's CUDA graph: the subclass's ``_step_body`` (one step
        on ``_ids`` at the device positions ``_pos``, which it advances: the logits) by default, or another that runs
        it and more (the sampled step).  Each body has its own graph, captured on its first graph step after a warm-up
        outside the graph (library workspaces); both restore ``_pos`` after.  Later steps replay, and the result is a
        buffer the next replay of that graph overwrites."""
        body = self._step_body if body is None else body
        self._ids.copy_(ids.reshape(-1).to(self._ids.device))
        if not use_graph:
            return body()
        name = body.__name__
        if name not in self._graphs:
            saved = self._pos.clone()
            side = torch.cuda.Stream(self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(side):
                body()
            torch.cuda.current_stream(self.device).wait_stream(side)
            self._pos.copy_(saved)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = body()
            self._graphs[name] = (g, out)
            self._pos.copy_(saved)
        g, out = self._graphs[name]
        g.replay()
        return out
