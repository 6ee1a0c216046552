"""One decode step of one attention layer in one launch (``agb200_decode_attention``, DESIGN §3.16).

    ws = decode_attention_workspace(B, n_heads, n_kv, head_dim, max_length, device)
    decode_attention(q, k, v, k_cache, v_cache, pos, inv_freq, attention_scaling, scaling, out, ws)

applies transformers' rotary embedding to q and k (the same roundings as ``apply_rotary_pos_emb``), writes k̂ and v to
position ``pos`` of the static caches, and attends every query head over positions 0..pos (GQA: query head h reads kv
head h // (n_heads / n_kv)).  ``pos`` is an int64 device scalar, so the call can be captured once in a CUDA graph and
replayed as the position advances.  No host synchronisation.

``decode_attention_rows`` (``agb200_decode_attention_rows``, DESIGN §3.18) runs the same kernel for up to
``ATTN_ROWS_MAX_B`` = 8 independent sequences: ``pos`` is an int64 device tensor [B], row b attends over 0..pos[b], and a
row with pos[b] = -1 is idle (zeros out, its cache row untouched).  The workspace is ``decode_attention_workspace``'s.
"""
from __future__ import annotations

import torch

from . import _lib

_DT = {torch.float16: _lib.F16, torch.bfloat16: _lib.BF16}


def attention_supported(n_heads: int, n_kv: int, head_dim: int, batch: int, max_length: int, dtype) -> str | None:
    """None when the kernel takes this shape, else the reason it does not."""
    if dtype not in _DT:
        return f"dtype {dtype}; the kernel computes in fp16 / bf16"
    if head_dim not in _lib.ATTN_HEAD_DIMS:
        return f"head_dim {head_dim}; the kernel takes {' or '.join(map(str, _lib.ATTN_HEAD_DIMS))}"
    if n_kv <= 0 or n_heads % n_kv != 0:
        return f"{n_heads} query heads over {n_kv} kv heads"
    if n_heads // n_kv > _lib.ATTN_MAX_G:
        return f"{n_heads // n_kv} query heads per kv head; the kernel takes at most {_lib.ATTN_MAX_G}"
    if not 1 <= batch <= _lib.ATTN_MAX_B:
        return f"batch {batch}; the kernel takes 1..{_lib.ATTN_MAX_B}"
    if batch * n_kv * max_length * head_dim >= 2 ** 31:
        return "the cache has 2^31 elements or more"
    return None


def attention_rows_supported(n_heads: int, n_kv: int, head_dim: int, batch: int, max_length: int, dtype) -> str | None:
    """None when ``decode_attention_rows`` takes this shape, else the reason it does not."""
    why = attention_supported(n_heads, n_kv, head_dim, 1, max_length, dtype)
    if why is None and not 1 <= batch <= _lib.ATTN_ROWS_MAX_B:
        why = f"batch {batch}; the kernel takes 1..{_lib.ATTN_ROWS_MAX_B} independent rows"
    if why is None and batch * n_kv * max_length * head_dim >= 2 ** 31:
        why = "the cache has 2^31 elements or more"
    return why


def decode_attention_workspace(batch: int, n_heads: int, n_kv: int, head_dim: int, max_length: int,
                               device) -> torch.Tensor:
    """A zeroed workspace for ``decode_attention`` of this shape on ``device``.  Calls leave it ready for the next
    call, so one workspace serves every layer of a model that runs them one after another on one stream."""
    device = torch.device(device)
    with torch.cuda.device(device):
        n = int(_lib.load().agb200_decode_attention_workspace_bytes(batch, n_heads, n_kv, head_dim, max_length))
    if n == 0:
        raise ValueError(f"decode_attention: invalid shape batch={batch}, n_heads={n_heads}, n_kv={n_kv}, "
                         f"head_dim={head_dim}, max_length={max_length}")
    return torch.zeros(n, dtype=torch.uint8, device=device)


def decode_attention(q, k, v, k_cache, v_cache, pos, inv_freq, attention_scaling: float, scaling: float, out,
                     workspace=None):
    """q [B, n_heads·hd], k / v [B, n_kv·hd], caches [B, n_kv, max_length, hd], pos int64 [1] (device), inv_freq fp32
    [hd/2], out [B, n_heads·hd] written in place and returned.  Raises NotImplementedError outside the kernel's limits."""
    return _launch("decode_attention", attention_supported, 1, q, k, v, k_cache, v_cache, pos, inv_freq,
                   attention_scaling, scaling, out, workspace)


def decode_attention_rows(q, k, v, k_cache, v_cache, pos, inv_freq, attention_scaling: float, scaling: float, out,
                          workspace=None):
    """``decode_attention`` for independent sequences: pos int64 [B] (device), one position per row, -1 for an idle
    row (zeros out, cache row untouched).  B <= ``ATTN_ROWS_MAX_B``."""
    return _launch("decode_attention_rows", attention_rows_supported, None, q, k, v, k_cache, v_cache, pos, inv_freq,
                   attention_scaling, scaling, out, workspace)


def _launch(entry, supported, n_pos, q, k, v, k_cache, v_cache, pos, inv_freq, attention_scaling, scaling, out,
            workspace):
    """Checks and the call of agb200_<entry>; ``n_pos`` elements of pos (None: one per row)."""
    if k_cache.dim() != 4:
        raise ValueError(f"k_cache must be [B, n_kv, max_length, head_dim], got {tuple(k_cache.shape)}")
    B, n_kv, L, hd = k_cache.shape
    dev = k_cache.device
    if dev.type != "cuda":
        raise RuntimeError(f"{entry} needs CUDA tensors (there is no CPU fallback)")
    dt = k_cache.dtype
    if q.dim() != 2 or q.shape[0] != B or q.shape[1] % hd != 0:
        raise ValueError(f"q must be [{B}, n_heads·{hd}], got {tuple(q.shape)}")
    n_heads = q.shape[1] // hd
    why = supported(n_heads, n_kv, hd, B, L, dt)
    if why is not None:
        raise NotImplementedError(f"{entry}: {why}")
    for name, t, shape in (("q", q, (B, n_heads * hd)), ("k", k, (B, n_kv * hd)), ("v", v, (B, n_kv * hd)),
                           ("v_cache", v_cache, (B, n_kv, L, hd)), ("out", out, (B, n_heads * hd))):
        if tuple(t.shape) != shape:
            raise ValueError(f"{name} must be {list(shape)}, got {list(t.shape)}")
        if t.dtype != dt:
            raise ValueError(f"{name} is {t.dtype}, the cache {dt}")
    for name, t in (("q", q), ("k", k), ("v", v), ("k_cache", k_cache), ("v_cache", v_cache), ("out", out),
                    ("pos", pos), ("inv_freq", inv_freq)):
        if t.device != dev:
            raise ValueError(f"{name} is on {t.device}, the cache on {dev}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
    n_pos = B if n_pos is None else n_pos
    if pos.dtype != torch.int64 or pos.numel() != n_pos:
        raise ValueError(f"pos must be {n_pos} int64 element(s), got {pos.dtype} with {pos.numel()} elements")
    if inv_freq.dtype != torch.float32 or tuple(inv_freq.shape) != (hd // 2,):
        raise ValueError(f"inv_freq must be float32 [{hd // 2}], got {inv_freq.dtype} {list(inv_freq.shape)}")
    lib = _lib.load()
    with torch.cuda.device(dev):
        need = int(lib.agb200_decode_attention_workspace_bytes(B, n_heads, n_kv, hd, L))
        if workspace is None:
            workspace = decode_attention_workspace(B, n_heads, n_kv, hd, L, dev)
        elif workspace.device != dev or workspace.numel() * workspace.element_size() < need:
            raise ValueError(f"workspace must hold {need} bytes on {dev}")
        rc = getattr(lib, f"agb200_{entry}")(
            q.data_ptr(), k.data_ptr(), v.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), pos.data_ptr(),
            inv_freq.data_ptr(), float(attention_scaling), float(scaling), out.data_ptr(), B, n_heads, n_kv, hd, L,
            _DT[dt], workspace.data_ptr(), workspace.numel() * workspace.element_size(),
            torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(rc, f"agb200_{entry}")
    return out


__all__ = ["decode_attention", "decode_attention_rows", "decode_attention_workspace", "attention_supported",
           "attention_rows_supported"]
