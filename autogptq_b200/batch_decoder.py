"""Greedy decoding of up to eight independent sequences of a GPTQ Llama / Mistral / Qwen2 model, one CUDA graph per step.

    dec = BatchDecoder(model, max_batch=8, max_length=4096)   # model: transformers *ForCausalLM with QuantLinear projections
    logits = dec.prefill(slot, input_ids)      # [T] prompt -> [vocab] logits of its last position; the slot becomes active
    logits = dec.step(ids)                     # ids [max_batch] -> logits [max_batch, vocab]; active slots advance by one
    dec.release(slot)                          # the slot becomes idle
    outs = dec.generate(prompts, max_new_tokens, eos_token_id=None)    # continuous batching over a list of prompts

Each of the ``max_batch`` slots holds one sequence at its own position, or none.  Positions live in a device tensor
``pos`` [max_batch], -1 for an idle slot, so a step is the same launches whatever the slots hold: it is captured once in
a CUDA graph at M = max_batch rows and replayed; admitting or releasing a sequence only changes buffer contents.  A
decoder block runs the project's per-layer kernels on all rows at once (DESIGN §3.18):

    q, k, v = forward_group([q, k, v], n1)       -> decode_attention_rows(pos) -> o_proj
    h1, n2  = add_rmsnorm(o, resid; post_attention_layernorm)
    a       = forward_gate_up(gate, up, n2)      -> down_proj
    resid', n1' = add_rmsnorm(down, h1; next input_layernorm)

The first block's n1 is ``add_rmsnorm`` without a residual; after the last block ``add_rmsnorm(model.norm)`` and the
model's ``lm_head`` (torch) give the logits.  The attention applies each row's rotary embedding at its own position,
writes the row's cache entry and attends over the row's positions only; an idle row writes zeros and touches no cache.
Every kernel computes a row from that row's inputs alone, so what one slot holds never changes another slot's logits.

``prefill`` runs the HF model at batch 1 with a ``DynamicCache`` and copies its keys and values into the slot's row of
the static caches.  ``kv_cache_dtype=torch.float8_e4m3fn`` keeps the caches as E4M3 codes with a power-of-two scale per
cached row (``k_scale`` / ``v_scale``, DESIGN §3.19): half the cache bytes, so twice the positions in the same memory;
prefill quantises the prompt's rows with ``autogptq_b200.attention.quantize_kv``, each step the kernel its own.
Scope: Llama, Mistral and Qwen2 blocks with ``QuantLinear`` projections (``FusedQuantMLP`` MLPs too),
greedy.  Mixture-of-experts blocks, dynamic / longrope rope, a sliding window below max_length and attention shapes the
kernel does not take raise NotImplementedError naming the module.  For batch <= 2 sequences in lockstep,
``ChainDecoder`` runs each block as one decode-chain launch.
"""
from __future__ import annotations

from collections import deque

import torch

from . import _lib
from .attention import attention_rows_supported, decode_attention_rows, decode_attention_workspace
from .decoder import _MOE_BLOCKS, _check_window, _kv_caches, _kv_fp8, _norm_of, _rotary_params, _store_kv
from .mlp import FusedQuantMLP, _is_silu, forward_gate_up
from .moe import add_rmsnorm, add_rmsnorm_supported
from .qlinear import QuantLinear, forward_group

_WHO = "BatchDecoder"


def _plan_layer(i: int, layer, dtype):
    """(attn, mlp, ln1, ln2) of decoder layer i after checking that BatchDecoder runs it."""
    attn, mlp = getattr(layer, "self_attn", None), getattr(layer, "mlp", None)
    if attn is None or mlp is None:
        raise NotImplementedError(f"{_WHO}: model.layers.{i} has no self_attn / mlp")
    if (type(mlp).__name__ in _MOE_BLOCKS or hasattr(mlp, "experts")
            or (hasattr(mlp, "gate") and not hasattr(mlp, "gate_proj"))):
        raise NotImplementedError(f"{_WHO}: model.layers.{i}.mlp is {type(mlp).__name__}; mixture-of-experts blocks "
                                  "are not supported (ChainDecoder decodes Mixtral at batch <= 2)")
    for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
        if not isinstance(getattr(attn, n, None), QuantLinear):
            raise NotImplementedError(f"{_WHO}: model.layers.{i}.self_attn.{n} is "
                                      f"{type(getattr(attn, n, None)).__name__}, not autogptq_b200.QuantLinear")
    if not isinstance(mlp, FusedQuantMLP):
        if not all(hasattr(mlp, n) for n in ("gate_proj", "up_proj", "down_proj")):
            raise NotImplementedError(f"{_WHO}: model.layers.{i}.mlp ({type(mlp).__name__}) is not a gate/up/down MLP")
        if not _is_silu(getattr(mlp, "act_fn", None)):
            raise NotImplementedError(f"{_WHO}: model.layers.{i}.mlp.act_fn is "
                                      f"{type(getattr(mlp, 'act_fn', None)).__name__}, not SiLU")
    for n in ("gate_proj", "up_proj", "down_proj"):
        if not isinstance(getattr(mlp, n), QuantLinear):
            raise NotImplementedError(f"{_WHO}: model.layers.{i}.mlp.{n} is {type(getattr(mlp, n)).__name__}, not "
                                      "autogptq_b200.QuantLinear")
    ln1 = _norm_of(getattr(layer, "input_layernorm", None), f"model.layers.{i}.input_layernorm", _WHO)
    ln2 = _norm_of(getattr(layer, "post_attention_layernorm", None), f"model.layers.{i}.post_attention_layernorm", _WHO)
    for (w, _), n in ((ln1, "input_layernorm"), (ln2, "post_attention_layernorm")):
        if w.dtype != dtype:
            raise NotImplementedError(f"{_WHO}: model.layers.{i}.{n}.weight is {w.dtype}, the activations {dtype}")
    return attn, mlp, ln1, ln2


class BatchDecoder:
    """Greedy decoder of up to ``max_batch`` <= 8 independent sequences over a transformers ``LlamaForCausalLM`` /
    ``MistralForCausalLM`` / ``Qwen2ForCausalLM`` whose projections are ``autogptq_b200.QuantLinear``.
    ``kv_cache_dtype``: None (the activation dtype) or ``torch.float8_e4m3fn``."""

    def __init__(self, model, max_batch: int = 8, max_length: int = 4096, kv_cache_dtype=None):
        if not 1 <= max_batch <= _lib.ATTN_ROWS_MAX_B:
            raise NotImplementedError(f"{_WHO}: max_batch {max_batch}; the decode kernels run 1..{_lib.ATTN_ROWS_MAX_B} "
                                      "rows")
        fp8 = _kv_fp8(kv_cache_dtype, _WHO)
        inner = getattr(model, "model", None)
        if inner is None or not hasattr(inner, "layers") or not hasattr(model, "lm_head"):
            raise NotImplementedError(f"{_WHO}: {type(model).__name__} is not a *ForCausalLM with model.layers and "
                                      "lm_head")
        for n in ("embed_tokens", "rotary_emb", "norm"):
            if not hasattr(inner, n):
                raise NotImplementedError(f"{_WHO}: model.model has no {n}")
        self.model, self.max_batch, self.max_length = model, int(max_batch), int(max_length)
        cfg = model.config
        _check_window(cfg, self.max_length, _WHO)
        self.dtype = inner.embed_tokens.weight.dtype
        if self.dtype not in (torch.float16, torch.bfloat16):
            raise NotImplementedError(f"{_WHO}: activations are {self.dtype}; the kernels compute in fp16 / bf16")
        hd = getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads
        n_kv = getattr(cfg, "num_key_value_heads", None) or cfg.num_attention_heads
        why = attention_rows_supported(cfg.num_attention_heads, n_kv, hd, self.max_batch, self.max_length, self.dtype)
        if why is not None:
            raise NotImplementedError(f"{_WHO}: model.layers.*.self_attn: {why}")
        self._inv_freq, self._attn_scaling = _rotary_params(inner.rotary_emb, hd, _WHO)
        plans = [_plan_layer(i, layer, self.dtype) for i, layer in enumerate(inner.layers)]
        if not plans:
            raise NotImplementedError(f"{_WHO}: the model has no decoder layers")
        self._final = _norm_of(inner.norm, "model.norm", _WHO)
        attn0 = plans[0][0]
        H = attn0.q_proj.infeatures
        why = add_rmsnorm_supported(self.max_batch, H, self.dtype)
        if why is not None:
            raise NotImplementedError(f"{_WHO}: model.layers.*.input_layernorm: {why}")
        self.device = inner.embed_tokens.weight.device
        if self.device.type != "cuda":
            raise RuntimeError(f"{_WHO} needs the model on a CUDA device")
        self.head_dim, self.n_heads, self.n_kv = hd, cfg.num_attention_heads, n_kv
        self.scaling = attn0.scaling
        self._plans = plans

        B, L, dev, dt = self.max_batch, self.max_length, self.device, self.dtype
        self.k_cache, self.v_cache, self.k_scale, self.v_scale = _kv_caches(len(plans), (B, n_kv, L, hd), dt, dev, fp8)
        self._pos = torch.full((B,), -1, dtype=torch.int64, device=dev)   # next position of each slot, -1 idle
        self._host_pos = [-1] * B                                           # its host mirror
        self._ids = torch.zeros(B, dtype=torch.int64, device=dev)
        self._x = torch.zeros((B, H), dtype=dt, device=dev)                # the embedding, block 0's residual
        self._resid = torch.zeros((B, H), dtype=dt, device=dev)            # residual entering block i > 0
        self._h1 = torch.zeros((B, H), dtype=dt, device=dev)
        self._n1 = torch.zeros((B, H), dtype=dt, device=dev)
        self._n2 = torch.zeros((B, H), dtype=dt, device=dev)
        self._attn_out = torch.zeros((B, self.n_heads * hd), dtype=dt, device=dev)
        self._attn_ws = decode_attention_workspace(B, self.n_heads, n_kv, hd, L, dev)
        self._graph = None
        self._logits = None

    # ------------------------------------------------------------------ slots
    @property
    def positions(self) -> list:
        """Tokens in each slot's cache (the position its next step writes), -1 for an idle slot."""
        return list(self._host_pos)

    @positions.setter
    def positions(self, ps):
        ps = [int(p) for p in ps]
        if len(ps) != self.max_batch or any(not -1 <= p <= self.max_length for p in ps):
            raise ValueError(f"positions must be {self.max_batch} values in -1..{self.max_length}, got {ps}")
        self._pos.copy_(torch.tensor(ps, dtype=torch.int64))
        self._host_pos = ps

    def _check_slot(self, slot: int) -> int:
        if not 0 <= int(slot) < self.max_batch:
            raise ValueError(f"slot {slot} outside 0..{self.max_batch - 1}")
        return int(slot)

    @torch.no_grad()
    def prefill(self, slot: int, input_ids: torch.Tensor) -> torch.Tensor:
        """Run the prompt [T] through the HF model at batch 1 (its own prefill kernels), copy its keys and values into
        the slot's row of the static caches and make the slot active at position T.  Other slots are not touched.
        Returns the logits of the last prompt position [vocab]."""
        from transformers import DynamicCache

        slot = self._check_slot(slot)
        ids = input_ids.to(self.device).reshape(1, -1)
        T = ids.shape[1]
        if not 1 <= T < self.max_length:
            raise ValueError(f"prompt length {T} must be in 1..{self.max_length - 1}")
        cache = DynamicCache(config=self.model.config)
        out = self.model(input_ids=ids, past_key_values=cache, use_cache=True)
        for i, lay in enumerate(cache.layers):
            _store_kv(self, i, (slot, slice(None), slice(0, T)), lay.keys[0], lay.values[0])
        self._pos[slot] = T
        self._host_pos[slot] = T
        return out.logits[0, -1]

    def release(self, slot: int):
        """Make the slot idle: its row is skipped by the attention and its cache row is left as it is."""
        slot = self._check_slot(slot)
        self._pos[slot] = -1
        self._host_pos[slot] = -1

    # ------------------------------------------------------------------ one step
    def _step_body(self) -> torch.Tensor:
        inner = self.model.model
        self._x.copy_(inner.embed_tokens(self._ids))
        w, eps = self._plans[0][2]
        add_rmsnorm(self._x, None, w, eps, n=self._n1)
        resid = self._x
        for i, (attn, mlp, _, (w2, eps2)) in enumerate(self._plans):
            q, k, v = forward_group([attn.q_proj, attn.k_proj, attn.v_proj], self._n1)
            fp8 = {} if self.k_scale is None else dict(k_scale=self.k_scale[i], v_scale=self.v_scale[i])
            decode_attention_rows(q, k, v, self.k_cache[i], self.v_cache[i], self._pos, self._inv_freq,
                                  self._attn_scaling, self.scaling, self._attn_out, self._attn_ws, **fp8)
            o = attn.o_proj(self._attn_out)
            add_rmsnorm(o, resid, w2, eps2, h=self._h1, n=self._n2)
            down = mlp.down_proj(forward_gate_up(mlp.gate_proj, mlp.up_proj, self._n2))
            w1, eps1 = self._plans[i + 1][2] if i + 1 < len(self._plans) else self._final
            add_rmsnorm(down, self._h1, w1, eps1, h=self._resid, n=self._n1)
            resid = self._resid
        logits = self.model.lm_head(self._n1)
        self._pos.add_(self._pos >= 0)                  # active slots advance; idle ones stay at -1
        return logits

    @torch.no_grad()
    def step(self, ids: torch.Tensor, use_graph: bool = True) -> torch.Tensor:
        """Decode one token for every active slot: ``ids`` [max_batch] (entries of idle slots are ignored) -> logits
        [max_batch, vocab]; rows of idle slots carry no meaning.  With ``use_graph`` the result is a buffer the next
        step overwrites: the first graph step captures the whole step in one CUDA graph, later steps replay it."""
        active = [p for p in self._host_pos if p >= 0]
        if not active:
            raise RuntimeError(f"{_WHO}.step: no slot is active (prefill one first)")
        if max(active) >= self.max_length:
            raise RuntimeError(f"{_WHO}.step: a slot's static cache is full ({self.max_length} tokens)")
        self._ids.copy_(ids.reshape(-1).to(self._ids.device))
        if not use_graph:
            logits = self._step_body()
        else:
            if self._graph is None:
                saved = self._pos.clone()
                side = torch.cuda.Stream(self.device)
                side.wait_stream(torch.cuda.current_stream(self.device))
                with torch.cuda.stream(side):                 # warm-up outside the graph (library workspaces)
                    self._step_body()
                torch.cuda.current_stream(self.device).wait_stream(side)
                self._pos.copy_(saved)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._logits = self._step_body()
                self._graph = g
                self._pos.copy_(saved)
            self._graph.replay()
            logits = self._logits
        self._host_pos = [p + 1 if p >= 0 else p for p in self._host_pos]
        return logits

    # ------------------------------------------------------------------ continuous batching
    @torch.no_grad()
    def generate(self, prompts, max_new_tokens: int, eos_token_id=None) -> list:
        """Greedy decoding of every prompt (1-D, any lengths) -> a list of 1-D tensors, prompt followed by its new
        tokens: at most ``max_new_tokens``, fewer when ``eos_token_id`` comes first (it is kept).  Prompts fill free
        slots in order; a sequence retires at EOS or after ``max_new_tokens`` and the next prompt takes its slot.  One
        small device-to-host read per step (the greedy tokens)."""
        prompts = [p.reshape(-1) for p in prompts]
        if max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
        for j, p in enumerate(prompts):
            if p.numel() + max_new_tokens > self.max_length:
                raise ValueError(f"prompt {j}: {p.numel()} tokens + {max_new_tokens} new tokens exceed "
                                 f"max_length={self.max_length}")
        for s in range(self.max_batch):
            if self._host_pos[s] >= 0:
                self.release(s)
        queue = deque(range(len(prompts)))
        new = [[] for _ in prompts]
        owner = [None] * self.max_batch              # prompt index held by each slot

        def take(s, tok):
            """Record slot s's next token; retire the sequence when it is done."""
            j = owner[s]
            new[j].append(tok)
            if tok == eos_token_id or len(new[j]) >= max_new_tokens:
                self.release(s)
                owner[s] = None

        while True:
            for s in range(self.max_batch):
                while owner[s] is None and queue:
                    j = queue.popleft()
                    owner[s] = j
                    take(s, int(self.prefill(s, prompts[j]).argmax()))
            live = [s for s in range(self.max_batch) if owner[s] is not None]
            if not live:
                break
            ids = torch.zeros(self.max_batch, dtype=torch.int64)
            for s in live:
                ids[s] = new[owner[s]][-1]
            toks = self.step(ids.to(self.device)).argmax(-1).tolist()
            for s in live:
                take(s, toks[s])
        return [torch.cat([p.to(self.device), torch.tensor(t, dtype=p.dtype, device=self.device)])
                for p, t in zip(prompts, new)]


__all__ = ["BatchDecoder"]
