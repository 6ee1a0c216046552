"""Decoding of a GPTQ Llama / Mistral / Qwen2 model with one decode-chain launch per decoder block.

    dec = ChainDecoder(model, batch=1, max_length=2048)    # model: transformers *ForCausalLM with QuantLinear projections
    tokens = dec.generate(input_ids, max_new_tokens=128)   # prefill on the HF model, then one CUDA graph per token
    tokens = dec.generate(input_ids, 128, sampling=SamplingParams(temperature=0.7, top_p=0.9))   # sampled
    logits = dec.extend(input_ids)                         # or: append [batch, T] tokens on the project's kernels

Between two attentions a decoder layer is QuantLinears, elementwise work and one row reduction:

    o_proj(attn) -> h1 = x + o -> n2 = post_attention_layernorm(h1) -> gate|up -> silu*mul -> down
                 -> x' = h1 + down -> n1' = next input_layernorm(x') -> next q|k|v

The decode chain's norm stage inputs (``x_mode="add_rmsnorm"``) cover the adds and norms, so block i is one chain

    chain_0 = [input_layernorm_0 -> q|k|v_0]
    chain_i = [o_i, add_rmsnorm -> gate|up_i, silu_mul -> down_i, add_rmsnorm(input_layernorm_i+1) -> q|k|v_i+1]

(the last block ends at down_i).  Attention needs the KV cache and runs in torch between two chains: the model's own
rotary embedding and ``apply_rotary_pos_emb``, a static [batch, kv_heads, max_length, head_dim] cache
(``autogptq_b200.kv_cache.KVCache``) written at a device-side position, and ``F.scaled_dot_product_attention`` with
GQA and a length mask; its output goes straight into the next chain's o_proj input buffer.  The final add,
``model.model.norm`` and ``lm_head`` run in torch.  One token is then n_layers + 1 chain launches and n_layers
attentions, captured together in one CUDA graph.

``fused_attention=True`` runs each attention as one ``agb200_decode_attention`` launch instead (rotary embedding, cache
write and split-KV attention, ``autogptq_b200.attention``): a token is then 2·n_layers + 1 launches of the project's own
kernels plus the embedding, final norm and lm_head.  It rounds differently from SDPA (fp32 online softmax), so it is
opt-in, and it is the one that reads an FP8 cache (``kv_cache_dtype=torch.float8_e4m3fn``, DESIGN §3.19).

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

``extend`` appends tokens at ``position`` without the HF model's cache: the model's own modules with the project's
``prefill_attention`` writing the static cache (DESIGN §3.20).  It continues a sequence (a new turn, a prompt in chunks)
or, from position 0, prefills one; Mixtral keeps the HF ``prefill``.

``generate(..., sampling=...)`` samples each token (temperature, top-k, top-p, min-p; DESIGN §3.21) with
``autogptq_b200.sampling``'s kernel inside a second graph of the step; it only reads the logits, so dense and Mixtral
blocks alike take it.

Scope: batch <= 2 (the chain's M), sequences in lockstep (one prompt length), greedy or sampled.  The front end is
``autogptq_b200._decoding``'s, shared with ``autogptq_b200.batch_decoder.BatchDecoder``: up to eight independent
sequences of any lengths, admitted and retired between steps.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import _lib
from ._decoding import DecoderBase, _is_moe, _is_moe_block, _plan_common, _plan_experts, _plan_moe, _rotary_params
from ._decoding import _MOE_BLOCKS, _RMSNORMS, _ROUTERS, _check_window, _norm_of  # noqa: F401 - also importable here
from .attention import FP8, attention_supported, decode_attention, decode_attention_workspace
from .chain import DecodeChain, chain_supported
from .kv_cache import KVCache
from .moe import moe_router
from .sampling import sampling_list

def _plan_layer(i: int, layer, batch: int, dtype):
    """The shared rules, then the chain's: (attn, mlp, ln1, ln2, moe) of decoder layer i with moe = (router weight,
    top_k, QuantExperts) for a Mixtral sparse MoE block and None for a dense MLP."""
    attn, mlp, ln1, ln2 = _plan_common(i, layer, dtype, "ChainDecoder")
    H = attn.q_proj.infeatures
    groups = {"self_attn.q_proj|k_proj|v_proj": [attn.q_proj, attn.k_proj, attn.v_proj],
              "self_attn.o_proj": [attn.o_proj]}
    moe = None
    if not _is_moe_block(mlp):
        groups.update({"mlp.gate_proj|up_proj": [mlp.gate_proj, mlp.up_proj], "mlp.down_proj": [mlp.down_proj]})
    else:
        moe = _plan_moe(i, mlp, H, batch, dtype, "ChainDecoder")
    for n, ls in groups.items():
        if not chain_supported(ls, batch):
            raise NotImplementedError(f"ChainDecoder: model.layers.{i}.{n} cannot run in a decode chain (needs "
                                      "infeatures % 128 == 0, group_size % 128 == 0 or -1, outfeatures % 32 == 0, "
                                      "sibling layers of one shape)")
    if H > _lib.CHAIN_NORM_MAX_K:
        raise NotImplementedError(f"ChainDecoder: model.layers.{i}: hidden size {H} > {_lib.CHAIN_NORM_MAX_K}, the "
                                  "largest a chain norm stage takes")
    return attn, mlp, ln1, ln2, moe


class ChainDecoder(DecoderBase):
    """Greedy or sampling decoder over a transformers ``LlamaForCausalLM`` / ``MistralForCausalLM`` / ``Qwen2ForCausalLM`` whose
    projections are ``autogptq_b200.QuantLinear`` (``FusedQuantMLP`` MLPs are accepted too), or a
    ``MixtralForCausalLM`` whose experts are ``autogptq_b200.QuantExperts``.  ``fused_attention``:
    run each layer's attention as one CUDA launch (``autogptq_b200.attention.decode_attention``) instead of torch.
    ``kv_cache_dtype``: None (the activation dtype) or ``torch.float8_e4m3fn`` (needs ``fused_attention``)."""

    _who = "ChainDecoder"

    def __init__(self, model, batch: int = 1, max_length: int = 2048, fused_attention: bool = False,
                 kv_cache_dtype=None):
        if not 1 <= batch <= _lib.CHAIN_MAX_M:
            raise NotImplementedError(f"ChainDecoder: batch {batch}; the decode chain runs 1..{_lib.CHAIN_MAX_M} rows")
        if kv_cache_dtype == FP8 and not fused_attention:
            raise NotImplementedError(f"ChainDecoder: kv_cache_dtype {FP8} needs fused_attention=True; the torch "
                                      "attention reads a 16-bit cache")
        self.batch, self.fused_attention = batch, bool(fused_attention)
        self._read_model(model, max_length, kv_cache_dtype)
        self._cache = KVCache(batch, self.n_kv, self.max_length, self.head_dim, self.dtype, self._fp8)
        if self.fused_attention:
            why = attention_supported(self.n_heads, self.n_kv, self.head_dim, batch, self.max_length, self.dtype)
            if why is not None:
                raise NotImplementedError(f"ChainDecoder(fused_attention=True): model.layers.*.self_attn: {why}")
            self._inv_freq, self._attn_scaling = _rotary_params(model.model.rotary_emb, self.head_dim,
                                                                "ChainDecoder(fused_attention=True)")
        self._read_layers()
        self.moe = _is_moe(self._plans, "ChainDecoder")

        # the chains are built before the caches: whether a block's chain fits the device's shared memory is the
        # library's decision (DESIGN §3.5), and a block that does not fit is refused before the caches are allocated
        plans, attn0, H = self._plans, self._plans[0][0], self.hidden_size
        B, dev, dt = batch, self._cuda_device(), self.dtype
        if self.moe:
            _plan_experts(plans, dt, dev, "ChainDecoder")
        self._pos =torch.zeros(1, dtype=torch.int64, device=dev)          # device-side position of the next token
        self._counter = torch.zeros(B, dtype=torch.int64, device=dev)      # its copy per row, the sampler's counter
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
        self.chains.append(self._build(ch, 0))
        self._qkv = [qkv]              # q, k, v of block i
        self._attn_in = []             # o_proj input of block i (written by the attention)
        if self.moe:
            self._build_moe(plans, H)
        else:
            self._build_dense(plans)
        self._allocate(batch)

    def _plan(self, i: int, layer):
        return _plan_layer(i, layer, self.batch, self.dtype)

    def _build(self, ch: DecodeChain, i: int) -> DecodeChain:
        """``ch.build()`` of a chain that starts in block i; a chain the device cannot hold (ENOSUP: the digits of its
        widest x leave no room for the smallest ring) is a refusal."""
        try:
            return ch.build()
        except _lib.B200KernelError as e:
            if e.code != _lib.ENOSUP:
                raise
            raise NotImplementedError(f"ChainDecoder: model.layers.{i} at batch {self.batch} does not fit in one decode "
                                      f"chain launch: {e}") from None

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
            self.chains.append(self._build(ch, i))

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
            self._o_chains.append(self._build(ch, i))
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
                self._qkv_chains.append(self._build(ch, i + 1))
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
        ids = input_ids.to(self.device)
        if ids.dim() != 2 or ids.shape[0] != self.batch:
            raise ValueError(f"input_ids must be [{self.batch}, T] (sequences in lockstep), got {tuple(ids.shape)}")
        T = ids.shape[1]
        if not 1 <= T < self.max_length:
            raise ValueError(f"prompt length {T} must be in 1..{self.max_length - 1}")
        logits = self._prefill_cache(ids, slice(None))
        self.position = T
        return logits[:, -1]

    @torch.no_grad()
    def extend(self, input_ids: torch.Tensor) -> torch.Tensor:
        """Append ``input_ids`` [batch, T] in lockstep at ``position`` on the project's kernels (DESIGN §3.20) and
        return the logits of the last new position [batch, vocab]; ``position`` advances by T.  The cache layout is
        the same for both ``fused_attention`` settings, so steps of either kind follow.  Mixture-of-experts models
        are refused: use ``prefill``."""
        if self.moe:
            raise NotImplementedError("ChainDecoder.extend: mixture-of-experts blocks are not supported (the router "
                                      f"kernel takes at most {_lib.MOE_DECODE_MAX_T} rows); use prefill")
        if input_ids.dim() != 2 or input_ids.shape[0] != self.batch:
            raise ValueError(f"ChainDecoder.extend: input_ids must be [{self.batch}, T] (sequences in lockstep), got "
                             f"{tuple(input_ids.shape)}")
        T = input_ids.shape[1]
        if T < 1:
            raise ValueError("ChainDecoder.extend: input_ids is empty")
        p = self._length
        if p + T >= self.max_length:
            raise ValueError(f"ChainDecoder.extend: position {p} + {T} tokens must stay below "
                             f"max_length={self.max_length}")
        logits = self._extend(input_ids.to(self.device), slice(None), [p] * self.batch)
        self.position = p + T
        return logits

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
        decode_attention(q, k, v, self.k_cache[i], self.v_cache[i], self._pos, self._inv_freq, self._attn_scaling,
                         self.scaling, self._attn_in[i], self._attn_ws, **self._cache.scales(i))

    def _step_body(self) -> torch.Tensor:
        inner = self.model.model
        self._x0.copy_(inner.embed_tokens(self._ids))
        if self.fused_attention:
            attention = self._fused_attention
        else:
            pos_ids = self._pos.view(1, 1).expand(self.batch, 1)
            cos, sin = inner.rotary_emb(self._x0.view(self.batch, 1, -1), pos_ids)
            mask = (self._arange <= self._pos).view(1, 1, 1, -1)
            attention = lambda i: self._attention(i, cos, sin, mask)  # noqa: E731
        tail = self._moe_block if self.moe else (lambda i: self.chains[i + 1].run())
        self.chains[0].run()
        for i in range(len(self._attn_in)):
            attention(i)
            tail(i)
        h1, down = self._last
        logits = self.model.lm_head(inner.norm(h1 + down))
        self._pos.add_(1)
        return logits

    def _sampled_step_body(self):
        """The step, then every row's token sampled at the advanced position."""
        logits = self._step_body()
        self._counter.copy_(self._pos.expand(self.batch))
        return self._sampling.sample(logits, self._counter), logits

    @torch.no_grad()
    def step(self, ids: torch.Tensor, use_graph: bool = True) -> torch.Tensor:
        """Decode one token per sequence: ``ids`` [batch] -> logits [batch, vocab] (a buffer the next step overwrites
        when ``use_graph``).  The first graph step captures the whole step in one CUDA graph; later steps replay it."""
        if self._length >= self.max_length:
            raise RuntimeError(f"the static cache is full ({self.max_length} tokens)")
        logits = self._run_step(ids, use_graph)
        self._length += 1
        return logits

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, max_new_tokens: int, sampling=None) -> torch.Tensor:
        """Decoding: prompt [batch, T] -> [batch, T + max_new_tokens].  ``sampling``: None is greedy (the argmax of the
        logits); a ``SamplingParams``, or a list of ``batch`` of them, samples row b with its parameters at counter =
        the token's position: the first token from the prefill's logits, the later ones in the step's sampled graph."""
        params = None if sampling is None else sampling_list(sampling, self.batch, "ChainDecoder.generate")
        if input_ids.shape[1] + max_new_tokens > self.max_length:
            raise ValueError(f"prompt + {max_new_tokens} new tokens exceed max_length={self.max_length}")
        if params is not None:
            return self._generate_sampled(input_ids, max_new_tokens, params)
        logits = self.prefill(input_ids)
        out = [input_ids.to(self.device)]
        for t in range(max_new_tokens):
            tok = logits.argmax(-1)
            out.append(tok.view(-1, 1))
            if t + 1 < max_new_tokens:
                logits = self.step(tok)
        return torch.cat(out, dim=1)

    def _generate_sampled(self, input_ids: torch.Tensor, max_new_tokens: int, params: list) -> torch.Tensor:
        for b, sp in enumerate(params):
            self._sampling.set(b, sp)
        logits = self.prefill(input_ids)
        out = [input_ids.to(self.device)]
        for t in range(max_new_tokens):
            if t == 0:                                  # the prefill's logits, sampled at the first new position
                self._counter.fill_(self._length)
                tok = self._sampling.sample(logits, self._counter).clone()
            else:                                       # the step and the sampler in one graph
                tok = self._run_step(tok, True, self._sampled_step_body)[0].clone()
                self._length += 1
            out.append(tok.view(-1, 1))
        return torch.cat(out, dim=1)


__all__ = ["ChainDecoder"]
