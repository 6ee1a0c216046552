"""Decoding of up to eight independent sequences of a GPTQ Llama / Mistral / Qwen2 / Mixtral model, one CUDA graph per
step.

    dec = BatchDecoder(model, max_batch=8, max_length=4096)   # model: transformers *ForCausalLM with QuantLinear projections
    logits = dec.prefill(slot, input_ids)      # [T] prompt -> [vocab] logits of its last position; the slot becomes active
    logits = dec.extend(slot, input_ids)       # [T] more tokens at the slot's position (0 when idle) -> [vocab]
    logits = dec.step(ids)                     # ids [max_batch] -> logits [max_batch, vocab]; active slots advance by one
    dec.release(slot)                          # the slot becomes idle
    outs = dec.generate(prompts, max_new_tokens, eos_token_id=None)    # continuous batching over a list of prompts
    dec.set_sampling(slot, SamplingParams(temperature=0.7, top_p=0.9))  # the slot's sampling parameters (None: greedy)
    token = dec.sample(slot, logits)           # sample prefill's / extend's logits with them
    tokens, logits = dec.step_sample(ids)      # the step and the sampling kernel in one CUDA graph
    outs = dec.generate(prompts, max_new_tokens, sampling=SamplingParams(...))     # sampled continuous batching

Each of the ``max_batch`` slots holds one sequence at its own position, or none.  Positions live in a device tensor
``pos`` [max_batch], -1 for an idle slot, so a step is the same launches whatever the slots hold: it is captured once in
a CUDA graph at M = max_batch rows and replayed; admitting or releasing a sequence only changes buffer contents.  A
decoder block runs the project's per-layer kernels on all rows at once (DESIGN §3.18):

    q, k, v = forward_group([q, k, v], n1)       -> decode_attention_rows(pos) -> o_proj
    h1, n2  = add_rmsnorm(o, resid; post_attention_layernorm)
    a       = forward_gate_up(gate, up, n2)      -> down_proj
    resid', n1' = add_rmsnorm(down, h1; next input_layernorm)

A Mixtral block (``MixtralSparseMoeBlock`` whose ``experts`` are an ``autogptq_b200.QuantExperts``) replaces the MLP by
the router and the grouped 4-bit experts (DESIGN §3.23):

    h1, n2, idx, w = moe_router(o, resid; post_attention_layernorm, gate, top_k, pos)
    moe     = experts._forward(n2, idx, w)
    resid', n1' = add_rmsnorm(moe, h1; next input_layernorm)

The router reads the same ``pos`` as the attention: an idle row gets expert index -1 and weight 0, so the experts give it
a zero row and stream no expert's weights for it, and a step's expert bytes follow the active rows alone.  Every
buffer, the experts' plans and their workspaces are allocated when the decoder is built.

The first block's n1 is ``add_rmsnorm`` without a residual; after the last block ``add_rmsnorm(model.norm)`` and the
model's ``lm_head`` (torch) give the logits.  The attention applies each row's rotary embedding at its own position,
writes the row's cache entry and attends over the row's positions only; an idle row writes zeros and touches no cache.
Every kernel computes a row from that row's inputs alone, so what one slot holds never changes another slot's logits.

``prefill`` runs the HF model at batch 1 and stores its keys and values in the slot's cache rows; with
``kv_cache_dtype=torch.float8_e4m3fn`` they are FP8 (DESIGN §3.19), half the cache bytes.  ``extend(slot, ids)``
appends T tokens at the slot's position on the project's kernels instead (DESIGN §3.20): the model's own modules for
everything but attention, and ``prefill_attention`` writing the cache and attending causally over it, with no
second cache and lm_head on the last position only.  On an idle slot it is a prompt prefill; on an active one it
continues the sequence (a new conversation turn, or the next chunk of a long prompt).  For Mixtral both run the model's
own MoE blocks, so a prompt of more than 8 tokens (``MOE_DECODE_MAX_T``) makes each ``QuantExperts`` build its
tensor-core weight copies on first use, K·N/2 bytes per layer, about 22 GB more for Mixtral-8x7B.

Tokens are greedy, or sampled (temperature, top-k, top-p, min-p; DESIGN §3.21) by ``autogptq_b200.sampling``'s kernel,
which runs in the step's graph: each slot's parameters and seed live in device tensors [max_batch], so one graph serves
any mix of greedy and sampled slots, and a slot's token depends only on its own logits, parameters, seed and position.
With ``kv_block_size`` the KV cache is paged (DESIGN §3.22): one pool of ``kv_blocks`` blocks per layer, a block table
per slot, and blocks shared by reference.  The memory then follows the tokens held, not ``max_batch × max_length``;
``fork(src, dst)`` gives an idle slot another slot's prefix without recomputing or copying its full blocks, and
``generate(..., n=k)`` prefills each prompt once and samples k continuations from it.  The step, its graph and its
results are the static cache's, bit for bit; only where a cache row lives changes.  Both layouts are
``autogptq_b200.kv_cache``'s ``KVCache`` and ``PagedKVCache``.

Scope: Llama, Mistral and Qwen2 blocks with ``QuantLinear`` projections (``FusedQuantMLP`` MLPs too), and Mixtral blocks
with ``QuantLinear`` attention projections and ``QuantExperts``.  Router variants other than Mixtral's (Qwen2-MoE's
shared expert, DeepSeek, a router bias), experts that are not grouped, and models that mix dense and MoE layers are
refused.  The model checks, the prefill and the graph capture are ``autogptq_b200._decoding``'s, shared with
``ChainDecoder``, which runs each block of batch <= 2 sequences in lockstep as one decode-chain launch.
"""
from __future__ import annotations

import dataclasses
from collections import deque

import torch

from . import _lib
from ._decoding import (_MOE_BLOCKS, DecoderBase, _is_moe, _is_moe_block, _plan_common, _plan_experts, _plan_moe,
                        _rotary_params)
from .attention import decode_attention_workspace
from .kv_cache import KVCache, PagedKVCache
from .mlp import forward_gate_up
from .moe import QuantExperts, add_rmsnorm, add_rmsnorm_supported, moe_router
from .qlinear import forward_group
from .sampling import SamplingParams, sampling_list

_WHO = "BatchDecoder"


class BatchDecoder(DecoderBase):
    """Greedy or sampling decoder of up to ``max_batch`` <= 8 independent sequences over a transformers ``LlamaForCausalLM`` /
    ``MistralForCausalLM`` / ``Qwen2ForCausalLM`` whose projections are ``autogptq_b200.QuantLinear``, or a
    ``MixtralForCausalLM`` whose attention projections are ``QuantLinear`` and whose experts are
    ``autogptq_b200.QuantExperts``.
    ``kv_cache_dtype``: None (the activation dtype) or ``torch.float8_e4m3fn``.  ``kv_block_size``: None (a static
    cache, ``k_cache[i]`` [max_batch, n_kv, max_length, head_dim]) or a power of two in 16..256: a paged cache of
    ``kv_blocks`` blocks per layer (default max_batch·ceil(max_length / kv_block_size), the static capacity), whose
    pools are ``k_cache[i]`` [kv_blocks, n_kv, kv_block_size, head_dim] (FP8 scales ``k_scale[i]``
    [kv_blocks, n_kv, kv_block_size])."""

    _who = _WHO

    def __init__(self, model, max_batch: int = 8, max_length: int = 4096, kv_cache_dtype=None, kv_block_size=None,
                 kv_blocks=None):
        if not 1 <= max_batch <= _lib.ATTN_ROWS_MAX_B:
            raise NotImplementedError(f"{_WHO}: max_batch {max_batch}; the decode kernels run 1..{_lib.ATTN_ROWS_MAX_B} "
                                      "rows")
        self.max_batch = int(max_batch)
        self._read_model(model, max_length, kv_cache_dtype)
        B, H, hd, dt = self.max_batch, self.hidden_size, self.head_dim, self.dtype
        self.kv_block_size = None if kv_block_size is None else int(kv_block_size)
        if self.kv_block_size is None:
            if kv_blocks is not None:
                raise ValueError(f"{_WHO}: kv_blocks goes with kv_block_size (a paged cache)")
            self._cache = KVCache(B, self.n_kv, self.max_length, hd, dt, self._fp8)
        else:
            self._cache = PagedKVCache(B, self.n_kv, self.max_length, hd, dt, self._fp8, self.kv_block_size, kv_blocks)
            self.kv_blocks = self._cache.num_blocks
        why = self._cache.unsupported(self.n_heads)
        if why is not None:
            raise NotImplementedError(f"{_WHO}: model.layers.*.self_attn: {why}")
        self._inv_freq, self._attn_scaling = _rotary_params(model.model.rotary_emb, hd, _WHO)
        self._read_layers()
        self.moe = _is_moe(self._plans, _WHO)
        why = add_rmsnorm_supported(B, H, dt)
        if why is not None:
            raise NotImplementedError(f"{_WHO}: model.layers.*.input_layernorm: {why}")
        if self._final[0].dtype != dt:                  # the last add_rmsnorm reads it
            raise NotImplementedError(f"{_WHO}: model.norm.weight is {self._final[0].dtype}, the activations {dt}")
        if self.moe:
            _plan_experts(self._plans, dt, self._cuda_device(), _WHO)
        self._allocate(B)

        dev = self.device
        self._pos = torch.full((B,), -1, dtype=torch.int64, device=dev)   # next position of each slot, -1 idle
        self._host_pos = [-1] * B                                           # its host mirror
        self._x = torch.zeros((B, H), dtype=dt, device=dev)                # the embedding, block 0's residual
        self._resid = torch.zeros((B, H), dtype=dt, device=dev)            # residual entering block i > 0
        self._h1 = torch.zeros((B, H), dtype=dt, device=dev)
        self._n1 = torch.zeros((B, H), dtype=dt, device=dev)
        self._n2 = torch.zeros((B, H), dtype=dt, device=dev)
        self._attn_out = torch.zeros((B, self.n_heads * hd), dtype=dt, device=dev)
        self._attn_ws = decode_attention_workspace(B, self.n_heads, self.n_kv, hd, self._cache.length, dev)
        self._moe_layers = []                       # per Mixtral block: the router's outputs and the experts' buffers
        for *_, (w2, eps2), moe in (self._plans if self.moe else []):
            gate, k, experts = moe
            plan, ws = experts._static_buffers(B, k, dt, dev)
            self._moe_layers.append(dict(
                gate=gate, k=k, w2=w2, eps2=eps2, experts=experts, plan=plan, ws=ws,
                h1=torch.zeros((B, H), dtype=dt, device=dev), n2=torch.zeros((B, H), dtype=dt, device=dev),
                idx=torch.zeros((B, k), dtype=torch.int32, device=dev),
                w=torch.zeros((B, k), dtype=torch.float32, device=dev),
                out=torch.zeros((B, H), dtype=dt, device=dev)))

    @property
    def kv_cache_bytes(self) -> int:
        """Bytes of the KV cache: every layer's caches (static) or pools (paged), scales included."""
        return self._cache.nbytes

    @property
    def kv_blocks_free(self):
        """Free blocks of the paged cache's pool (None for a static cache)."""
        return self._cache.blocks_free

    def _need_paged(self, what: str):
        """The refusal of ``fork`` and ``generate(n > 1)`` on a static cache, before their arguments are checked."""
        if self.kv_block_size is None:
            raise NotImplementedError(f"{_WHO}.{what} needs the paged KV cache (BatchDecoder(..., kv_block_size=...))")

    def _plan(self, i: int, layer):
        """(attn, mlp, ln1, ln2, moe): ``_plan_common``'s, with moe = (router weight, top_k, QuantExperts) of a
        Mixtral block and None for a dense MLP.  A Mixtral block's experts are checked first: an unquantised model's
        block is named for what it lacks, the grouped 4-bit experts."""
        mlp = getattr(layer, "mlp", None)
        if type(mlp).__name__ in _MOE_BLOCKS and not isinstance(getattr(mlp, "experts", None), QuantExperts):
            raise NotImplementedError(f"{_WHO}: model.layers.{i}.mlp is {type(mlp).__name__} whose experts are "
                                      f"{type(getattr(mlp, 'experts', None)).__name__}, not autogptq_b200.QuantExperts "
                                      "(build them with autogptq_b200.group_experts)")
        attn, mlp, ln1, ln2 = _plan_common(i, layer, self.dtype, _WHO)
        moe = None
        if _is_moe_block(mlp):
            moe = _plan_moe(i, mlp, self.hidden_size, self.max_batch, self.dtype, _WHO)
        return attn, mlp, ln1, ln2, moe

    # ------------------------------------------------------------------ slots
    @property
    def positions(self) -> list:
        """Tokens in each slot's cache (the position its next step writes), -1 for an idle slot."""
        return list(self._host_pos)

    @positions.setter
    def positions(self, ps):
        if self.kv_block_size is not None:
            raise RuntimeError(f"{_WHO}: positions cannot be set with a paged KV cache (a position needs its blocks); "
                               "use release, prefill or extend")
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
        the slot's cache rows and make the slot active at position T.  Other slots are not touched.
        Returns the logits of the last prompt position [vocab]."""
        slot = self._check_slot(slot)
        ids = input_ids.to(self.device).reshape(1, -1)
        T = ids.shape[1]
        if not 1 <= T < self.max_length:
            raise ValueError(f"prompt length {T} must be in 1..{self.max_length - 1}")
        if not self._cache.fits(slot, T):
            raise RuntimeError(f"{_WHO}.prefill: the KV cache pool cannot hold {T} tokens ({self.kv_blocks_free} "
                               "blocks free)")
        self.release(slot)
        self._cache.reserve({slot: T})
        logits = self._prefill_cache(ids, slice(slot, slot + 1))
        self._pos[slot] = T
        self._host_pos[slot] = T
        return logits[0, -1]

    @torch.no_grad()
    def extend(self, slot: int, input_ids: torch.Tensor) -> torch.Tensor:
        """Append the tokens ``input_ids`` [T] to the slot at its position p (0 for an idle slot, so this is a prompt
        prefill) on the project's kernels (DESIGN §3.20) and make the slot active at p + T.  Other slots' cache rows
        and positions are not touched.  Returns the logits of the last new position [vocab].  Calling it several times
        feeds a prompt in chunks, or continues a conversation without re-reading its history."""
        slot = self._check_slot(slot)
        if input_ids.dim() != 1:
            raise ValueError(f"{_WHO}.extend: input_ids must be 1-D [T] (one slot), got {tuple(input_ids.shape)}")
        T = input_ids.numel()
        if T < 1:
            raise ValueError(f"{_WHO}.extend: input_ids is empty")
        p = max(self._host_pos[slot], 0)
        if p + T >= self.max_length:
            raise ValueError(f"{_WHO}.extend: slot {slot} at position {p} + {T} tokens must stay below "
                             f"max_length={self.max_length}")
        self._cache.reserve({slot: p + T})
        logits = self._extend(input_ids.to(self.device).view(1, T), slice(slot, slot + 1), [p])
        self._pos[slot] = p + T
        self._host_pos[slot] = p + T
        return logits[0]

    def set_sampling(self, slot: int, params: SamplingParams | None):
        """The slot's sampling parameters for ``sample`` and ``step_sample`` (None: greedy); a ``seed=None`` draws its
        seed from torch's default CPU generator now.  They stay until set again, across release and prefill."""
        slot = self._check_slot(slot)
        if params is not None and not isinstance(params, SamplingParams):
            raise TypeError(f"{_WHO}.set_sampling: params must be a SamplingParams or None, got {type(params).__name__}")
        self._sampling.set(slot, params)

    @torch.no_grad()
    def sample(self, slot: int, logits: torch.Tensor) -> int:
        """Sample the [vocab] logits ``prefill`` / ``extend`` returned for an active slot with the slot's parameters,
        at counter = the slot's position (where the token will go).  One device-to-host read."""
        slot = self._check_slot(slot)
        p = self._host_pos[slot]
        if p < 0:
            raise RuntimeError(f"{_WHO}.sample: slot {slot} is idle")
        counter = torch.full((1,), p, dtype=torch.int64, device=self.device)
        return int(self._sampling.sample(logits.reshape(1, -1), counter, slice(slot, slot + 1))[0])

    def release(self, slot: int):
        """Make the slot idle: its row is skipped by the attention and its cache row is left as it is (paged: the slot
        drops its blocks; a block no slot holds is free)."""
        slot = self._check_slot(slot)
        self._pos[slot] = -1
        self._host_pos[slot] = -1
        self._cache.release(slot)

    @torch.no_grad()
    def fork(self, src: int, dst: int):
        """Make the idle slot ``dst`` continue the active slot ``src``'s sequence (paged cache only): ``dst`` takes
        ``src``'s position and its full blocks by reference, and a copy of its partially filled last block (every
        layer, FP8 scales included).  Sampling parameters are not copied.  Raises RuntimeError, with nothing changed,
        when no block is free for the copy."""
        self._need_paged("fork")
        src, dst = self._check_slot(src), self._check_slot(dst)
        p = self._host_pos[src]
        if p < 0:
            raise RuntimeError(f"{_WHO}.fork: slot {src} is idle")
        if self._host_pos[dst] >= 0 or src == dst:
            raise RuntimeError(f"{_WHO}.fork: slot {dst} must be idle")
        self._cache.fork(src, dst, p)
        self._pos[dst] = p
        self._host_pos[dst] = p

    # ------------------------------------------------------------------ one step
    def _step_body(self) -> torch.Tensor:
        inner = self.model.model
        self._x.copy_(inner.embed_tokens(self._ids))
        w, eps = self._plans[0][2]
        add_rmsnorm(self._x, None, w, eps, n=self._n1)
        resid = self._x
        for i, (attn, mlp, _, (w2, eps2), moe) in enumerate(self._plans):
            q, k, v = forward_group([attn.q_proj, attn.k_proj, attn.v_proj], self._n1)
            self._cache.decode(i, q, k, v, self._pos, self._inv_freq, self._attn_scaling, self.scaling, self._attn_out,
                               self._attn_ws)
            o = attn.o_proj(self._attn_out)
            w1, eps1 = self._plans[i + 1][2] if i + 1 < len(self._plans) else self._final
            if moe is None:
                add_rmsnorm(o, resid, w2, eps2, h=self._h1, n=self._n2)
                down = mlp.down_proj(forward_gate_up(mlp.gate_proj, mlp.up_proj, self._n2))
                add_rmsnorm(down, self._h1, w1, eps1, h=self._resid, n=self._n1)
            else:                                       # idle rows (pos -1) route to no expert: a zero output row
                m = self._moe_layers[i]
                moe_router(o, resid, w2, eps2, m["gate"], m["k"], h=m["h1"], n=m["n2"], idx=m["idx"], w=m["w"],
                           pos=self._pos)
                m["experts"]._forward(m["n2"], m["idx"], m["w"], out=m["out"], plan=m["plan"], ws=m["ws"])
                add_rmsnorm(m["out"], m["h1"], w1, eps1, h=self._resid, n=self._n1)
            resid = self._resid
        logits = self.model.lm_head(self._n1)
        self._pos.add_(self._pos >= 0)                  # active slots advance; idle ones stay at -1
        return logits

    def _sampled_step_body(self):
        """The step, then every slot's token sampled at its advanced position (idle slots: -1, token 0)."""
        logits = self._step_body()
        return self._sampling.sample(logits, self._pos), logits

    def _check_step(self, what: str):
        active = [p for p in self._host_pos if p >= 0]
        if not active:
            raise RuntimeError(f"{_WHO}.{what}: no slot is active (prefill one first)")
        if max(active) >= self.max_length:
            raise RuntimeError(f"{_WHO}.{what}: a slot's static cache is full ({self.max_length} tokens)")
        self._cache.reserve({s: p + 1 for s, p in enumerate(self._host_pos) if p >= 0})   # the blocks the step writes

    @torch.no_grad()
    def step(self, ids: torch.Tensor, use_graph: bool = True) -> torch.Tensor:
        """Decode one token for every active slot: ``ids`` [max_batch] (entries of idle slots are ignored) -> logits
        [max_batch, vocab]; rows of idle slots carry no meaning.  With ``use_graph`` the result is a buffer the next
        step overwrites: the first graph step captures the whole step in one CUDA graph, later steps replay it."""
        self._check_step("step")
        logits = self._run_step(ids, use_graph)
        self._host_pos = [p + 1 if p >= 0 else p for p in self._host_pos]
        return logits

    @torch.no_grad()
    def step_sample(self, ids: torch.Tensor, use_graph: bool = True):
        """``step`` followed by the sampling kernel with each slot's parameters (``set_sampling``) at counter = the
        slot's advanced position: ``ids`` [max_batch] -> (tokens int64 [max_batch], logits [max_batch, vocab]); idle
        slots get token 0.  With ``use_graph`` both run in one CUDA graph, captured apart from ``step``'s, and the
        results are buffers the next sampled step overwrites."""
        self._check_step("step_sample")
        out = self._run_step(ids, use_graph, self._sampled_step_body)
        self._host_pos = [p + 1 if p >= 0 else p for p in self._host_pos]
        return out

    # ------------------------------------------------------------------ continuous batching
    @torch.no_grad()
    def generate(self, prompts, max_new_tokens: int, eos_token_id=None, sampling=None, n: int = 1) -> list:
        """Decoding of every prompt (1-D, any lengths) -> a list of 1-D tensors, prompt followed by its new tokens: at
        most ``max_new_tokens``, fewer when ``eos_token_id`` comes first (it is kept).  Prompts fill free slots in
        order; a sequence retires at EOS or after ``max_new_tokens`` and the next prompt takes its slot.  One small
        device-to-host read per step (the tokens).  ``sampling``: None is greedy (the argmax of the logits); a
        ``SamplingParams``, or a list of one per prompt, samples: each admitted prompt's parameters go to its slot, the
        first token comes from ``sample`` and the later ones from ``step_sample``.

        ``n`` > 1 (paged cache and ``sampling`` only): each prompt is prefilled once and forked into ``n`` slots, and the
        result lists its ``n`` samples prompt-major (prompt j's copy i at j·n + i).  Copy i of a prompt whose seed is s
        samples with seed (s + i) mod 2^64, so it equals an ``n=1`` run with that seed; ``seed=None`` draws a seed per
        copy.  With a paged cache a prompt is admitted only when the pool's uncommitted blocks cover its worst case
        (``paged_kv.worst_case_blocks``), so no step runs out of blocks; one that could never fit is a ValueError."""
        prompts = list(prompts)
        n = int(n)
        if n != 1:
            self._need_paged("generate(n > 1)")
            if not 1 <= n <= self.max_batch:
                raise ValueError(f"{_WHO}.generate: n={n} samples per prompt; 1..max_batch={self.max_batch}")
            if sampling is None:
                raise ValueError(f"{_WHO}.generate: n > 1 needs sampling (greedy copies would be identical)")
        params = None if sampling is None else sampling_list(sampling, len(prompts), f"{_WHO}.generate")
        prompts = [p.reshape(-1) for p in prompts]
        if max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
        for j, p in enumerate(prompts):
            if p.numel() + max_new_tokens > self.max_length:
                raise ValueError(f"prompt {j}: {p.numel()} tokens + {max_new_tokens} new tokens exceed "
                                 f"max_length={self.max_length}")
        pool = self._cache.num_blocks                # 0 for a static cache, whose prompts need no blocks
        worst = [self._cache.worst_case_blocks(p.numel(), max_new_tokens, n) for p in prompts]
        for j, w in enumerate(worst):
            if w > pool:
                raise ValueError(f"prompt {j}: {prompts[j].numel()} tokens + {max_new_tokens} new tokens, {n} "
                                 f"sample(s), may need {w} blocks; the pool has {pool}")
        for s in range(self.max_batch):
            if self._host_pos[s] >= 0:
                self.release(s)
        queue = deque(range(len(prompts)))
        new = [[] for _ in range(len(prompts) * n)]
        owner = [None] * self.max_batch              # output index (prompt j's copy i: j·n + i) held by each slot
        live = [0] * len(prompts)                    # copies of each prompt still decoding
        committed = 0                                # worst-case blocks of the prompts with live copies

        def take(s, tok):
            """Record slot s's next token; retire the sequence when it is done."""
            nonlocal committed
            o = owner[s]
            new[o].append(tok)
            if tok == eos_token_id or len(new[o]) >= max_new_tokens:
                self.release(s)
                owner[s] = None
                live[o // n] -= 1
                if live[o // n] == 0:
                    committed -= worst[o // n]

        def admit(j, slots):
            nonlocal committed
            committed += worst[j]
            live[j] = n
            for i, s in enumerate(slots):
                owner[s] = j * n + i
                if params is not None:
                    seed = params[j].seed
                    self.set_sampling(s, params[j] if seed is None or i == 0 else
                                      dataclasses.replace(params[j], seed=(seed + i) % 2 ** 64))
            logits = self.prefill(slots[0], prompts[j])
            for s in slots[1:]:
                self.fork(slots[0], s)
            for s in slots:
                take(s, int(logits.argmax()) if params is None else self.sample(s, logits))

        while True:
            while queue:
                free = [s for s in range(self.max_batch) if owner[s] is None]
                j = queue[0]
                if len(free) < n or committed + worst[j] > pool:
                    break
                queue.popleft()
                admit(j, free[:n])
            active = [s for s in range(self.max_batch) if owner[s] is not None]
            if not active:
                break
            ids = torch.zeros(self.max_batch, dtype=torch.int64)
            for s in active:
                ids[s] = new[owner[s]][-1]
            if params is None:
                toks = self.step(ids.to(self.device)).argmax(-1).tolist()
            else:
                toks = self.step_sample(ids.to(self.device))[0].tolist()
            for s in active:
                take(s, toks[s])
        return [torch.cat([prompts[o // n].to(self.device), torch.tensor(t, dtype=prompts[o // n].dtype,
                                                                         device=self.device)])
                for o, t in enumerate(new)]

__all__ = ["BatchDecoder"]
