"""Next-token sampling on the GPU: temperature, top-k, top-p and min-p in one seeded kernel (DESIGN §3.21).

    params = SamplingParams(temperature=0.7, top_k=50, top_p=0.9, seed=1234)
    tokens = sample(logits, temperature, top_k, top_p, min_p, seed, counter)    # device tensors, one entry per row

The semantics are transformers' ``TemperatureLogitsWarper``, ``TopKLogitsWarper``, ``TopPLogitsWarper`` and
``MinPLogitsWarper`` in that order, made exact (``include/autogptq_b200.h``, ``agb200_sample``); the draw is a
Gumbel-max over the kept tokens with Philox4x32-10 keyed by the row's seed at its counter, the position the token will
occupy.  A row's token therefore depends only on its own logits, parameters, seed and counter: not on the row's index,
on the other rows, or on whether the call runs eagerly or in a CUDA graph.  ``BatchDecoder`` and ``ChainDecoder`` run
the kernel inside their step graphs.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from . import _lib

_DTYPE_CODE = {torch.float16: _lib.F16, torch.bfloat16: _lib.BF16, torch.float32: _lib.F32}


@dataclass(frozen=True)
class SamplingParams:
    """One sequence's sampling parameters.  ``temperature == 0`` is greedy (the argmax); ``top_k == 0``,
    ``top_p == 1`` and ``min_p == 0`` turn their filter off.  ``seed=None`` draws a seed from torch's default CPU
    generator when the parameters are given to a decoder, so ``torch.manual_seed`` reproduces a run."""

    temperature: float = 1.0
    top_k: int = 0
    top_p: float = 1.0
    min_p: float = 0.0
    seed: int | None = None

    def __post_init__(self):
        t, k, p, m = self.temperature, self.top_k, self.top_p, self.min_p
        if isinstance(t, bool) or not isinstance(t, (int, float)) or not math.isfinite(t) or t < 0:
            raise ValueError(f"SamplingParams: temperature must be a finite number >= 0, got {t!r}")
        if isinstance(k, bool) or not isinstance(k, int) or k < 0:
            raise ValueError(f"SamplingParams: top_k must be an int >= 0 (0: off), got {k!r}")
        if isinstance(p, bool) or not isinstance(p, (int, float)) or not 0 < p <= 1:
            raise ValueError(f"SamplingParams: top_p must be in (0, 1] (1: off), got {p!r}")
        if isinstance(m, bool) or not isinstance(m, (int, float)) or not 0 <= m <= 1:
            raise ValueError(f"SamplingParams: min_p must be in [0, 1] (0: off), got {m!r}")
        s = self.seed
        if s is not None and (isinstance(s, bool) or not isinstance(s, int) or not 0 <= s < 2 ** 64):
            raise ValueError(f"SamplingParams: seed must be None or an int in [0, 2^64), got {s!r}")

    def resolved_seed(self) -> int:
        """The seed, or a fresh one from torch's default CPU generator when it is None."""
        if self.seed is not None:
            return int(self.seed)
        lo, hi = torch.randint(0, 2 ** 32, (2,), dtype=torch.int64).tolist()
        return lo | hi << 32


GREEDY = SamplingParams(temperature=0.0)


def sampling_list(sampling, n: int, who: str) -> list:
    """``sampling`` (one ``SamplingParams`` for all, or a list of ``n``) as a list of ``n``; refuses anything else."""
    if isinstance(sampling, SamplingParams):
        return [sampling] * n
    if not isinstance(sampling, (list, tuple)) or not all(isinstance(s, SamplingParams) for s in sampling):
        raise TypeError(f"{who}: sampling must be a SamplingParams or a list of them, got {type(sampling).__name__}")
    if len(sampling) != n:
        raise ValueError(f"{who}: sampling has {len(sampling)} entries for {n} sequences")
    return list(sampling)


def _signed(seed: int) -> int:
    """A 64-bit seed as the int64 with the same bits (the device tensors hold the bits as int64)."""
    return seed - 2 ** 64 if seed >= 2 ** 63 else seed


class SamplingState:
    """Device parameters of ``rows`` sequences ([rows] tensors the kernel reads), so one captured graph serves any mix
    of greedy and sampled rows: changing a row's parameters only changes buffer contents.  Every row starts greedy."""

    def __init__(self, rows: int, device):
        dev = torch.device(device)
        self.temperature = torch.zeros(rows, dtype=torch.float32, device=dev)
        self.top_k = torch.zeros(rows, dtype=torch.int32, device=dev)
        self.top_p = torch.ones(rows, dtype=torch.float32, device=dev)
        self.min_p = torch.zeros(rows, dtype=torch.float32, device=dev)
        self.seed = torch.zeros(rows, dtype=torch.int64, device=dev)
        self.tokens = torch.zeros(rows, dtype=torch.int64, device=dev)

    def set(self, row: int, params: SamplingParams | None):
        """Row ``row``'s parameters (None: greedy); draws the seed of ``seed=None`` now."""
        params = GREEDY if params is None else params
        self.temperature[row] = float(params.temperature)
        self.top_p[row] = float(params.top_p)
        self.min_p[row] = float(params.min_p)
        self.top_k[row] = min(int(params.top_k), 2 ** 31 - 1)
        self.seed[row] = _signed(params.resolved_seed())

    def sample(self, logits: torch.Tensor, counter: torch.Tensor, rows: slice = slice(None)) -> torch.Tensor:
        """The kernel on ``logits`` [n, V] with the parameters of ``rows`` and ``counter`` [n], into ``tokens[rows]``."""
        return sample(logits, self.temperature[rows], self.top_k[rows], self.top_p[rows], self.min_p[rows],
                      self.seed[rows], counter, out=self.tokens[rows])


def sample_supported(B: int, V: int, dtype) -> str | None:
    """None when ``sample`` takes [B, V] logits of ``dtype``, else the reason it does not."""
    if dtype not in _DTYPE_CODE:
        return f"dtype {dtype}; the sampler reads fp16, bf16 or fp32 logits"
    if not 1 <= V <= _lib.SAMPLE_MAX_V:
        return f"vocabulary {V}; the sampler takes 1..{_lib.SAMPLE_MAX_V} logits per row"
    if not 1 <= B <= 65535:
        return f"{B} rows; the sampler takes 1..65535"
    return None


def sample(logits: torch.Tensor, temperature: torch.Tensor, top_k: torch.Tensor, top_p: torch.Tensor,
           min_p: torch.Tensor, seed: torch.Tensor, counter: torch.Tensor, out: torch.Tensor | None = None):
    """Sample one token per row of ``logits`` [B, V] (fp16 / bf16 / fp32, any row stride, contiguous last dimension)
    in one launch (``agb200_sample``).  Per-row device tensors [B]: ``temperature`` fp32 (0: greedy), ``top_k`` int32
    (0: off), ``top_p`` fp32 (1: off), ``min_p`` fp32 (0: off), ``seed`` int64 (the bits of a 64-bit seed),
    ``counter`` int64 (the position the token will occupy; < 0: an idle row, token 0).  Returns ``out`` int64 [B].
    No host synchronisation."""
    if logits.dim() != 2:
        raise ValueError(f"sample: logits must be [B, V], got {tuple(logits.shape)}")
    B, V = logits.shape
    dev = logits.device
    if dev.type != "cuda":
        raise RuntimeError("sample needs CUDA tensors (there is no CPU fallback)")
    why = sample_supported(B, V, logits.dtype)
    if why is not None:
        raise NotImplementedError(f"sample: {why}")
    if logits.stride(1) != 1 or logits.stride(0) < V:
        raise ValueError(f"sample: logits need a contiguous last dimension and a row stride >= V, got strides "
                         f"{tuple(logits.stride())}")
    out = torch.empty(B, dtype=torch.int64, device=dev) if out is None else out
    for name, t, dt in (("temperature", temperature, torch.float32), ("top_k", top_k, torch.int32),
                        ("top_p", top_p, torch.float32), ("min_p", min_p, torch.float32),
                        ("seed", seed, torch.int64), ("counter", counter, torch.int64), ("out", out, torch.int64)):
        if tuple(t.shape) != (B,) or t.dtype != dt:
            raise ValueError(f"sample: {name} must be {dt} [{B}], got {t.dtype} {list(t.shape)}")
        if t.device != dev:
            raise ValueError(f"sample: {name} is on {t.device}, logits on {dev}")
        if not t.is_contiguous():
            raise ValueError(f"sample: {name} must be contiguous")
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.agb200_sample(logits.data_ptr(), logits.stride(0), _DTYPE_CODE[logits.dtype], B, V,
                               temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(), min_p.data_ptr(),
                               seed.data_ptr(), counter.data_ptr(), out.data_ptr(),
                               torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(rc, "agb200_sample")
    return out


__all__ = ["SamplingParams", "sample", "sample_supported"]
