"""GPTQ checkpoint -> ``autogptq_b200.QuantLinear`` modules, without the reference's modelling stack (SURVEY.md 8f rank 1).

What the reference does for this step: ``AutoGPTQForCausalLM.from_quantized`` builds the HF model skeleton, swaps every
``nn.Linear`` for a ``QuantLinear`` (``modeling/_utils.py:92-148``), then fills the buffers by name from a single
``.safetensors`` / ``.bin`` file (``modeling/_base.py:1114-1121``) whose quantisation settings come from
``quantize_config.json`` (``quantization/config.py:20,58-72``) or from the safetensors metadata
(``modeling/_base.py:557-566``: ``gptq_bits``, ``gptq_group_size``, ``gptq_desc_act``).

Here the packed tensors are all that is needed: every ``<prefix>.qweight`` in the checkpoint (one file or HF-style
shards with ``*.safetensors.index.json``) becomes one ``QuantLinear`` keyed by ``<prefix>``, its shapes read off the
tensors.  Nothing is repacked (the kernels read the checkpoint layout); with ``tp_world > 1`` each layer is cut for this
rank right after it has been read (``sharding.py``: q/k/v/gate/up by columns, o/down by rows): one FULL layer is in host
memory at a time, a rank keeps only its share; tensors that are not packed-layer buffers (embeddings, norms, lm_head)
are never read.  Host-side only: works on CPU tensors; moving to the GPU is ``device=``.

AutoAWQ "GEMM" checkpoints (``quant_config.json``, or ``quantization_config`` in an HF ``config.json``) load the same
way: each layer is rewritten exactly into the GPTQ layout (``awq.awq_to_gptq``) as it is read, before any TP slicing, so
the modules are ordinary GPTQ-layout ``QuantLinear``s (the reference converts in a slow fp16 round trip, writes a cache
file and refuses sharded checkpoints, ``modeling/_base.py:974-1062``).
"""
from __future__ import annotations

import json
import os
import re
from dataclasses import dataclass
from typing import Callable, Dict, Iterator, Mapping, Optional, Tuple, Union

import torch

from .awq import awq_to_gptq
from .qlinear import QuantLinear
from .sharding import shard_column_parallel, shard_row_parallel, shard_to_module

QUANT_CONFIG_FILENAME = "quantize_config.json"            # quantization/config.py:20
AWQ_CONFIG_FILENAME = "quant_config.json"                 # AutoAWQ
HF_CONFIG_FILENAME = "config.json"                        # transformers: its "quantization_config" entry
_PACKED_SUFFIXES = ("qweight", "qzeros", "scales", "g_idx", "bias")
# Megatron-style plan for Llama-family decoder blocks (SURVEY.md 8e)
LLAMA_TP_PLAN = {
    r"\.(q_proj|k_proj|v_proj|gate_proj|up_proj)$": "column",
    r"\.(o_proj|down_proj)$": "row",
}


@dataclass
class QuantSettings:
    bits: int = 4
    group_size: int = -1
    desc_act: bool = False
    sym: bool = True
    checkpoint_format: str = "gptq"

    @classmethod
    def from_mapping(cls, d: Mapping) -> "QuantSettings":
        g = lambda *names, default=None: next((d[n] for n in names if n in d), default)   # noqa: E731
        truthy = lambda v: str(v).lower() in ("true", "1")                                # noqa: E731
        # synonyms accepted by the reference (quantization/config.py:51-55) and its safetensors metadata keys; AWQ
        # configs say zero_point instead of sym
        sym = g("sym", default=None)
        out = cls(bits=int(g("bits", "w_bit", "gptq_bits", default=4)),
                  group_size=int(g("group_size", "q_group_size", "gptq_group_size", default=-1)),
                  desc_act=truthy(g("desc_act", "gptq_desc_act", default=False)),
                  sym=truthy(sym) if sym is not None else not truthy(g("zero_point", default=False)),
                  checkpoint_format=str(g("checkpoint_format", "gptq_checkpoint_format", default="gptq")).lower())
        if truthy(g("is_marlin_format", default=False)):
            out.checkpoint_format = "marlin"
        # AWQ: quant_method "awq" (HF) or a bare "version" (AutoAWQ's quant_config.json) names the layout
        # (quantization/config.py:141-143); AWQ does not reorder rows (:152-154)
        method = str(g("quant_method", default="")).lower()
        if method == "awq" or (method == "" and "version" in d):
            version = str(g("version", default="gemm")).lower()
            if version != "gemm":
                raise NotImplementedError(f"AWQ version {version!r}: only AutoAWQ's GEMM layout is read "
                                          "(GEMV / Marlin / exllama AWQ checkpoints are not)")
            out.checkpoint_format = "gemm"
        if out.checkpoint_format == "gemm":
            out.desc_act = False
        return out


def read_quant_settings(path: str) -> Optional[QuantSettings]:
    """``quantize_config.json`` next to the weights, else the ``gptq_*`` metadata of the first safetensors file, else
    AutoAWQ's ``quant_config.json``, else the ``quantization_config`` of an HF ``config.json``."""
    d = path if os.path.isdir(path) else os.path.dirname(path)
    cfg = os.path.join(d, QUANT_CONFIG_FILENAME)
    if os.path.exists(cfg):
        return QuantSettings.from_mapping(json.load(open(cfg)))
    for f in _weight_files(path):
        from safetensors import safe_open

        with safe_open(f, framework="pt", device="cpu") as fh:
            meta = fh.metadata() or {}
        if any(k.startswith("gptq_") for k in meta):
            return QuantSettings.from_mapping(meta)
        break
    for name, key in ((AWQ_CONFIG_FILENAME, None), (HF_CONFIG_FILENAME, "quantization_config")):
        cfg = os.path.join(d, name)
        if os.path.exists(cfg):
            with open(cfg) as fh:
                m = json.load(fh)
            m = m.get(key) if key is not None else m
            if m:
                return QuantSettings.from_mapping(m)
    return None


def _weight_files(path: str) -> list:
    if os.path.isfile(path):
        return [path]
    idx = [f for f in sorted(os.listdir(path)) if f.endswith(".safetensors.index.json")]
    if idx:
        weight_map = json.load(open(os.path.join(path, idx[0])))["weight_map"]
        return [os.path.join(path, f) for f in sorted(set(weight_map.values()))]
    return [os.path.join(path, f) for f in sorted(os.listdir(path)) if f.endswith(".safetensors")]


def iter_packed_layers(source: Union[str, Mapping[str, torch.Tensor]]) -> Iterator[Tuple[str, Dict[str, torch.Tensor]]]:
    """Yield ``(prefix, {qweight, qzeros, scales, g_idx?, bias?})`` for every packed layer of a checkpoint directory /
    file (one shard in memory at a time) or of an in-memory state dict.  A layer split over two shards is completed
    when its last tensor arrives."""
    pending: Dict[str, Dict[str, torch.Tensor]] = {}

    def feed(name: str, tensor: torch.Tensor):
        prefix, _, leaf = name.rpartition(".")
        if leaf not in _PACKED_SUFFIXES:
            return None
        pending.setdefault(prefix, {})[leaf] = tensor
        return prefix

    def ready(names_left: set, prefix: str) -> bool:
        have = pending[prefix]
        if not all(k in have for k in ("qweight", "qzeros", "scales")):
            return False
        return not any(f"{prefix}.{leaf}" in names_left for leaf in _PACKED_SUFFIXES if leaf not in have)

    if isinstance(source, Mapping):
        for name in source:
            feed(name, source[name])
        for prefix in sorted(pending):
            if ready(set(), prefix):
                yield prefix, pending[prefix]
        return

    from safetensors import safe_open

    files = _weight_files(source)
    # names first (cheap: the safetensors header), tensors only for the packed leaves - embeddings, norms and lm_head
    # are never materialised
    names_of = {}
    for f in files:
        with safe_open(f, framework="pt", device="cpu") as fh:
            names_of[f] = sorted(k for k in fh.keys() if k.rpartition(".")[2] in _PACKED_SUFFIXES)
    left = set(n for ns in names_of.values() for n in ns)
    # a stray `*.bias` of an ordinary nn.Linear shares the suffix: only prefixes that have a qweight are packed layers
    packed_prefixes = set(n.rpartition(".")[0] for n in left if n.endswith(".qweight"))
    for f in files:
        with safe_open(f, framework="pt", device="cpu") as fh:
            for name in names_of[f]:
                left.discard(name)
                if name.rpartition(".")[0] not in packed_prefixes:
                    continue
                prefix = feed(name, fh.get_tensor(name))
                if prefix is not None and ready(left, prefix):
                    yield prefix, pending.pop(prefix)


def build_quant_linear(tensors: Mapping[str, torch.Tensor], settings: QuantSettings, device=None,
                       tp: Optional[Tuple[str, int, int]] = None, allow_gathered_input: bool = False) -> QuantLinear:
    """One ``QuantLinear`` from the packed tensors of a layer; ``tp = (mode, rank, world)`` slices it first (the module
    then carries ``tp_mode / tp_rank / tp_world / tp_n_range / tp_k_range / tp_x_index``; a row-parallel shard's bias lives
    on rank 0 only and its outputs are PARTIAL sums - wrap it in ``autogptq_b200.tp.RowParallelQuantLinear`` or run it in a
    ``TPDecodeChain``).  ``settings.checkpoint_format == "gemm"`` (AWQ) converts the layer to the GPTQ layout first, on
    ``device`` when that is a CUDA device."""
    if settings.bits != 4:
        raise NotImplementedError(f"{settings.bits}-bit GPTQ checkpoints are outside the H100 hot path (4-bit only)")
    if settings.checkpoint_format not in ("gptq", "gemm"):
        raise NotImplementedError(f"checkpoint_format={settings.checkpoint_format!r}: only the GPTQ and AWQ GEMM pack "
                                  "layouts are read (Marlin checkpoints must be converted back, cf. marlin_utils.py:118-198)")
    qweight, qzeros, scales = tensors["qweight"], tensors["qzeros"], tensors["scales"]
    awq = settings.checkpoint_format == "gemm"
    if awq:
        if device is not None and torch.device(device).type == "cuda":
            qweight, qzeros, scales = (t.to(device) for t in (qweight, qzeros, scales))
        qweight, qzeros = awq_to_gptq(qweight, qzeros, scales)
    K, N = qweight.shape[0] * 8, qweight.shape[1]
    G = scales.shape[0]
    group_size = settings.group_size if settings.group_size != -1 else K
    if G != -(-K // group_size) or qzeros.shape != (G, N // 8) or scales.shape != (G, N):
        hint = ""
        if not awq and qweight.dim() == 2 and scales.dim() == 2 and scales.shape[1] == 8 * qweight.shape[1]:
            hint = (" - these are the shapes of an AWQ GEMM layer (qweight [K, N/8], packed along N): load it with "
                    "checkpoint_format='gemm'")
        raise ValueError(f"packed tensor shapes do not match group_size={settings.group_size}: qweight {tuple(qweight.shape)}, "
                         f"qzeros {tuple(qzeros.shape)}, scales {tuple(scales.shape)}{hint}")
    g_idx = None if awq else tensors.get("g_idx")     # AWQ has no act-order: groups are sequential
    if g_idx is None:
        g_idx = torch.arange(K, dtype=torch.int32) // group_size
    bias = tensors.get("bias")
    if tp is not None and tp[2] > 1:
        mode, rank, world = tp
        fn = shard_column_parallel if mode == "column" else shard_row_parallel
        shard = fn(qweight, qzeros, scales, g_idx.to(torch.int32), bias, group_size, rank, world)
        if shard.x_index is not None and not allow_gathered_input:
            # a row-parallel act-order shard multiplies the columns x_index of the FULL activation, not the contiguous
            # K-slice a plain Megatron row-parallel layer gets: feeding it the local slice is silently wrong
            raise NotImplementedError(
                "row-parallel shard of an act-order layer: its input is x_full[..., shard.x_index] (an all-gather of the "
                "column-parallel producer), see autogptq_b200.tp.RowParallelQuantLinear; pass allow_gathered_input=True "
                "to get the bare module with .tp_x_index attached")
        lin = shard_to_module(shard, device if device is not None else qweight.device, dtype=scales.dtype)
        # what the caller needs to wire the shard: how it was cut and which inputs it consumes
        lin.tp_mode, lin.tp_rank, lin.tp_world = mode, rank, world
        lin.tp_n_range, lin.tp_k_range, lin.tp_x_index = shard.n_range, shard.k_range, shard.x_index
        return lin
    lin = QuantLinear(4, settings.group_size, K, N, bias is not None, weight_dtype=scales.dtype)
    lin.qweight, lin.qzeros, lin.scales = qweight.contiguous(), qzeros.contiguous(), scales.contiguous()
    lin.g_idx = g_idx.to(torch.int32).contiguous()
    if bias is not None:
        lin.bias = bias.contiguous()
    return lin.to(device) if device is not None else lin


def load_quant_linears(source: Union[str, Mapping[str, torch.Tensor]], settings: Optional[QuantSettings] = None, device=None,
                       tp_rank: int = 0, tp_world: int = 1, tp_plan: Optional[Mapping[str, str]] = None,
                       select: Optional[Callable[[str], bool]] = None, allow_gathered_input: bool = False) -> Dict[str, QuantLinear]:
    """All packed layers of a GPTQ or AWQ GEMM checkpoint as ``{prefix: QuantLinear}`` (GPTQ layout either way).

    ``tp_world > 1``: layers whose prefix matches a pattern of ``tp_plan`` (default: the Llama plan) are sliced for
    ``tp_rank`` ("column" / "row"); the others are replicated.  ``select(prefix)`` filters layers (e.g. one decoder
    block).  The modules are ready for ``forward`` once on a CUDA device (``post_init`` runs lazily)."""
    if settings is None:
        settings = read_quant_settings(source) if isinstance(source, str) else None
        if settings is None:
            raise ValueError("quantisation settings not found: pass settings=QuantSettings(...) "
                             f"or put {QUANT_CONFIG_FILENAME} next to the weights")
    plan = [(re.compile(p), m) for p, m in (tp_plan or LLAMA_TP_PLAN).items()]
    out: Dict[str, QuantLinear] = {}
    for prefix, tensors in iter_packed_layers(source):
        if select is not None and not select(prefix):
            continue
        tp = None
        if tp_world > 1:
            mode = next((m for rx, m in plan if rx.search(prefix)), None)
            if mode is not None:
                tp = (mode, tp_rank, tp_world)
        out[prefix] = build_quant_linear(tensors, settings, device=device, tp=tp, allow_gathered_input=allow_gathered_input)
    return out


def packed_state_dict(layers: Mapping[str, QuantLinear]) -> Dict[str, torch.Tensor]:
    """The inverse: checkpoint tensors of a set of (unsharded) modules, named like the reference saves them."""
    sd = {}
    for prefix, lin in layers.items():
        for leaf in _PACKED_SUFFIXES:
            t = getattr(lin, leaf, None)
            if t is not None:
                sd[f"{prefix}.{leaf}"] = t.detach().cpu().contiguous()
    return sd


__all__ = ["QuantSettings", "read_quant_settings", "iter_packed_layers", "build_quant_linear", "load_quant_linears",
           "packed_state_dict", "LLAMA_TP_PLAN"]
