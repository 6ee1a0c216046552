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

FP8 cache (``agb200_decode_attention_fp8`` / ``agb200_decode_attention_rows_fp8``, DESIGN §3.19): caches of
``torch.float8_e4m3fn`` codes [B, n_kv, max_length, head_dim] with ``k_scale=`` / ``v_scale=`` fp32
[B, n_kv, max_length], one power-of-two scale per cached row, select the FP8 entries.  The step quantises the new k̂ and v with
``quantize_kv``'s rule, writes codes and scales at the position and attends through them.  q, k, v and out stay in
the activation dtype.  Half the cache bytes (hd + 4 per row instead of 2·hd).

``prefill_attention`` (``agb200_prefill_attention`` / ``agb200_prefill_attention_fp8``, DESIGN §3.20) appends T new
tokens to each of up to eight rows at their own ``start`` positions and attends them causally over the cache: the
cache rows it writes are bit-equal to the decode step's for the same token, whatever T, and the attention runs on the
tensor cores (mma.sync, fp32 softmax).  Feeding a prompt in chunks gives the same cache bytes as one call.

Paged cache (``decode_attention_rows_paged`` / ``prefill_attention_paged``, DESIGN §3.22): per layer, pools
[num_blocks, n_kv, block_size, hd] (and for FP8 scale pools [num_blocks, n_kv, block_size]) and an int32 block table
[B, max_blocks]; position t of row b is row t % block_size of block table[b, t // block_size].  block_size is a power of
two in 16..256.  For the same contents the outputs and every cache byte written are bit-equal to the static entries'
with max_length = max_blocks·block_size.  A table entry outside [0, num_blocks) is no block: it is never dereferenced,
and the row it belongs to gets NaN (decode: if it holds pos, or any position below it; prefill: any position of
0 .. start + T - 1), with no write to the pools at pos (decode) or at all (prefill).
"""
from __future__ import annotations

import functools

import torch

from . import _lib

_DT = {torch.float16: _lib.F16, torch.bfloat16: _lib.BF16}
FP8 = torch.float8_e4m3fn
E4M3_MAX = 448.0


def quantize_kv(x: torch.Tensor):
    """Rows x [..., hd] (fp16 / bf16) -> (codes float8_e4m3fn [..., hd], scale fp32 [...]), the FP8 cache's format:
    scale = 2^e with e the smallest integer such that max|x| <= 448·2^e (at least -126), codes = e4m3(x·2^-e) rounded
    to nearest even; a row of zeros gets scale 1 and codes 0.  Every code·scale is exact in fp32 (and in the dtype for
    bf16, and for fp16 when 448·2^-16 < max|x| <= 448·2^7).  The kernel quantises the new token by the same rule."""
    if x.dtype not in _DT:
        raise ValueError(f"quantize_kv: x is {x.dtype}; the cache rows are fp16 / bf16")
    a = x.abs().amax(dim=-1).float()                  # exact
    f, E = torch.frexp(a)                             # a = f·2^E, f in [0.5, 1)
    e = torch.where(f <= E4M3_MAX / 512, E - 9, E - 8).clamp(min=-126)
    e = torch.where(a == 0, torch.zeros_like(e), e).to(torch.int32)
    pow2 = lambda n: ((n + 127) << 23).view(torch.float32)                 # 2^n for -126 <= n <= 127, exactly
    codes = (x.float() * pow2(-e).unsqueeze(-1)).to(FP8)                  # exact scaling, then one rounding
    codes.view(torch.uint8).masked_fill_((a == 0).unsqueeze(-1), 0)
    return codes, pow2(e)


def dequantize_kv(codes: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """codes [..., hd], scale [...] -> the fp32 values the FP8 cache holds (exact)."""
    return codes.float() * scale.unsqueeze(-1)


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


def paged_attention_supported(n_heads: int, n_kv: int, head_dim: int, batch: int, block_size: int, num_blocks: int,
                              dtype) -> str | None:
    """None when the paged entries take this shape (pools of ``num_blocks`` blocks of ``block_size`` rows), else the
    reason they do not: the per-row decode limits, with the pool in place of the static cache."""
    if block_size not in _lib.KV_BLOCK_SIZES:
        return f"block_size {block_size}; a power of two in {_lib.KV_BLOCK_SIZES[0]}..{_lib.KV_BLOCK_SIZES[-1]}"
    if num_blocks < 1:
        return f"num_blocks {num_blocks}; at least 1"
    why = attention_rows_supported(n_heads, n_kv, head_dim, batch, 1, dtype)
    if why is None and num_blocks * n_kv * block_size * head_dim >= 2 ** 31:
        why = "the pool has 2^31 elements or more"
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
                     workspace=None, *, k_scale=None, v_scale=None):
    """q [B, n_heads·hd], k / v [B, n_kv·hd], caches [B, n_kv, max_length, hd], pos int64 [1] (device), inv_freq fp32
    [hd/2], out [B, n_heads·hd] written in place and returned.  Raises NotImplementedError outside the kernel's limits.
    float8_e4m3fn caches with ``k_scale`` / ``v_scale`` fp32 [B, n_kv, max_length]: the FP8 cache (module docstring)."""
    return _launch("decode_attention", attention_supported, q, k, v, k_cache, v_cache, pos, inv_freq,
                   attention_scaling, scaling, out, k_scale, v_scale, workspace=workspace, n_pos=1)


def decode_attention_rows(q, k, v, k_cache, v_cache, pos, inv_freq, attention_scaling: float, scaling: float, out,
                          workspace=None, *, k_scale=None, v_scale=None):
    """``decode_attention`` for independent sequences: pos int64 [B] (device), one position per row, -1 for an idle
    row (zeros out, cache row untouched).  B <= ``ATTN_ROWS_MAX_B``.  FP8 caches as ``decode_attention``."""
    return _launch("decode_attention_rows", attention_rows_supported, q, k, v, k_cache, v_cache, pos, inv_freq,
                   attention_scaling, scaling, out, k_scale, v_scale, workspace=workspace)


def prefill_attention_supported(n_heads: int, n_kv: int, head_dim: int, batch: int, max_length: int,
                                dtype) -> str | None:
    """None when ``prefill_attention`` takes this shape, else the reason it does not (the per-row decode limits)."""
    return attention_rows_supported(n_heads, n_kv, head_dim, batch, max_length, dtype)


def prefill_attention(q, k, v, k_cache, v_cache, start, inv_freq, attention_scaling: float, scaling: float, out, *,
                      k_scale=None, v_scale=None):
    """Causal attention of T new tokens per row over the static caches (``agb200_prefill_attention``, DESIGN §3.20):
    q [B, T, n_heads·hd], k / v [B, T, n_kv·hd], caches [B, n_kv, max_length, hd], start int64 [B] (device), inv_freq
    fp32 [hd/2], out [B, T, n_heads·hd] written in place and returned.  Row b's tokens are written to the caches at
    positions start[b] .. start[b] + T - 1 (k̂ with the rotary embedding, as ``decode_attention`` writes one token), then
    token t attends positions 0 .. start[b] + t.  A row whose tokens do not fit gets NaN and no cache write.
    float8_e4m3fn caches with ``k_scale`` / ``v_scale``: the FP8 cache, as ``decode_attention``.  Raises
    NotImplementedError outside the kernel's limits.  No workspace, no host synchronisation."""
    return _launch("prefill_attention", prefill_attention_supported, q, k, v, k_cache, v_cache, start, inv_freq,
                   attention_scaling, scaling, out, k_scale, v_scale, prefill=True)


def decode_attention_rows_paged(q, k, v, k_pool, v_pool, block_table, pos, inv_freq, attention_scaling: float,
                                scaling: float, out, workspace=None, *, k_scale=None, v_scale=None):
    """``decode_attention_rows`` over a paged cache (module docstring): pools [num_blocks, n_kv, block_size, hd] (the
    block size is the pools'), block_table int32 [B, max_blocks] (device), pos int64 [B].  float8_e4m3fn pools with
    ``k_scale`` / ``v_scale`` fp32 [num_blocks, n_kv, block_size]: the FP8 cache.  The workspace is
    ``decode_attention_workspace(B, n_heads, n_kv, hd, max_blocks·block_size)``.  Raises NotImplementedError outside
    the kernel's limits."""
    return _launch("decode_attention_rows_paged", paged_attention_supported, q, k, v, k_pool, v_pool, pos, inv_freq,
                   attention_scaling, scaling, out, k_scale, v_scale, workspace=workspace, table=block_table)


def prefill_attention_paged(q, k, v, k_pool, v_pool, block_table, start, inv_freq, attention_scaling: float,
                            scaling: float, out, *, k_scale=None, v_scale=None):
    """``prefill_attention`` over a paged cache (module docstring): q [B, T, n_heads·hd], pools and block_table as
    ``decode_attention_rows_paged``, start int64 [B].  A row with a position 0 .. start + T - 1 outside the table or
    without a block gets NaN and no write.  Raises NotImplementedError outside the kernel's limits."""
    return _launch("prefill_attention_paged", paged_attention_supported, q, k, v, k_pool, v_pool, start, inv_freq,
                   attention_scaling, scaling, out, k_scale, v_scale, prefill=True, table=block_table)


def _launch(entry, supported, q, k, v, k_cache, v_cache, pos, inv_freq, attention_scaling, scaling, out, k_scale,
            v_scale, *, workspace=None, n_pos=None, prefill=False, table=None):
    """Checks, the workspace (decode) and the call of agb200_<entry>[_fp8]: ``n_pos`` elements of pos (None: one per
    row); ``prefill``: activations [B, T, features] from start positions; ``table``: the caches are pools read through
    this block table.  The activation dtype is the 16-bit cache's, or q's for an FP8 cache."""
    paging = ()
    if table is not None:
        if k_cache.dim() != 4:
            raise ValueError(f"k_pool must be [num_blocks, n_kv, block_size, head_dim], got {tuple(k_cache.shape)}")
        num_blocks, _, bs, _ = k_cache.shape
        if table.dtype != torch.int32 or table.dim() != 2:
            raise ValueError(f"{entry}: block_table must be int32 [B, max_blocks], got {table.dtype} "
                             f"{list(table.shape)}")
        rows, max_blocks = table.shape
        if q.dim() != (3 if prefill else 2) or q.shape[0] != rows:
            raise ValueError(f"{entry}: q must have {rows} rows (block_table's), got {tuple(q.shape)}")
        if max_blocks < 1 or max_blocks * bs > 2 ** 30:
            raise ValueError(f"{entry}: block_table has {max_blocks} blocks per row of {bs}; need 1..2^30 positions")
        if table.device != k_cache.device or not table.is_contiguous():
            raise ValueError(f"{entry}: block_table must be contiguous on {k_cache.device}")
        supported = functools.partial(supported, num_blocks=num_blocks)
        paging = (table.data_ptr(), bs, num_blocks, max_blocks)
    lead = ()
    if prefill:
        if q.dim() != 3:
            raise ValueError(f"q must be [B, T, n_heads·head_dim], got {tuple(q.shape)}")
        lead = (q.shape[1],)
        if lead[0] < 1:
            raise ValueError(f"{entry}: T must be at least 1")
    if k_cache.dim() != 4:
        raise ValueError(f"k_cache must be [B, n_kv, max_length, head_dim], got {tuple(k_cache.shape)}")
    nb, n_kv, L, hd = k_cache.shape
    B = rows if paging else nb
    dev = k_cache.device
    if dev.type != "cuda":
        raise RuntimeError(f"{entry} needs CUDA tensors (there is no CPU fallback)")
    fp8 = k_cache.dtype == FP8
    if not fp8 and (k_scale is not None or v_scale is not None):
        raise ValueError(f"{entry}: k_scale / v_scale go with a {FP8} cache, not {k_cache.dtype}")
    if fp8 and (k_scale is None or v_scale is None):
        raise ValueError(f"{entry}: a {FP8} cache needs k_scale and v_scale (fp32 [B, n_kv, max_length])")
    dt = q.dtype if fp8 else k_cache.dtype
    lead = (B,) + lead                              # [B, features], or [B, T, features] for prefill
    if q.dim() != len(lead) + 1 or tuple(q.shape[:-1]) != lead or q.shape[-1] % hd != 0:
        raise ValueError(f"q must be [{', '.join(map(str, lead))}, n_heads·{hd}], got {tuple(q.shape)}")
    n_heads = q.shape[-1] // hd
    why = supported(n_heads, n_kv, hd, B, L, dtype=dt)
    if why is not None:
        raise NotImplementedError(f"{entry}: {why}")
    checks = [("q", q, lead + (n_heads * hd,), dt), ("k", k, lead + (n_kv * hd,), dt),
              ("v", v, lead + (n_kv * hd,), dt), ("v_cache", v_cache, (nb, n_kv, L, hd), k_cache.dtype),
              ("out", out, lead + (n_heads * hd,), dt)]
    if fp8:
        checks += [("k_scale", k_scale, (nb, n_kv, L), torch.float32),
                   ("v_scale", v_scale, (nb, n_kv, L), torch.float32)]
    for name, t, shape, want in checks:
        if tuple(t.shape) != shape:
            raise ValueError(f"{name} must be {list(shape)}, got {list(t.shape)}")
        if t.dtype != want:
            if not fp8:
                raise ValueError(f"{name} is {t.dtype}, the cache {dt}")
            raise ValueError(f"{name} is {t.dtype}, the activations (q) {dt}" if want == dt else
                             f"{name} is {t.dtype}, not {want}")
    pos_name = "start" if prefill else "pos"
    tensors = [("q", q), ("k", k), ("v", v), ("k_cache", k_cache), ("v_cache", v_cache), ("out", out),
               (pos_name, pos), ("inv_freq", inv_freq)] + ([("k_scale", k_scale), ("v_scale", v_scale)] if fp8 else [])
    for name, t in tensors:
        if t.device != dev:
            raise ValueError(f"{name} is on {t.device}, the cache on {dev}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
    n_pos = B if n_pos is None else n_pos
    if pos.dtype != torch.int64 or pos.numel() != n_pos:
        raise ValueError(f"{pos_name} must be {n_pos} int64 element(s), got {pos.dtype} with {pos.numel()} elements")
    if inv_freq.dtype != torch.float32 or tuple(inv_freq.shape) != (hd // 2,):
        raise ValueError(f"inv_freq must be float32 [{hd // 2}], got {inv_freq.dtype} {list(inv_freq.shape)}")
    caches = (k_cache.data_ptr(), v_cache.data_ptr())
    if fp8:
        entry, caches = entry + "_fp8", caches + (k_scale.data_ptr(), v_scale.data_ptr())
    if paging:
        L = max_blocks * bs                         # the positions a row can address
    lib = _lib.load()
    with torch.cuda.device(dev):
        ws = ()
        if not prefill:
            need = int(lib.agb200_decode_attention_workspace_bytes(B, n_heads, n_kv, hd, L))
            if workspace is None:
                workspace = decode_attention_workspace(B, n_heads, n_kv, hd, L, dev)
            elif workspace.device != dev or workspace.numel() * workspace.element_size() < need:
                raise ValueError(f"workspace must hold {need} bytes on {dev}")
            ws = (workspace.data_ptr(), workspace.numel() * workspace.element_size())
        rc = getattr(lib, f"agb200_{entry}")(
            q.data_ptr(), k.data_ptr(), v.data_ptr(), *caches, *paging, pos.data_ptr(), inv_freq.data_ptr(),
            float(attention_scaling), float(scaling), out.data_ptr(), *lead, n_heads, n_kv, hd,
            *(() if paging else (L,)), _DT[dt], *ws, torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(rc, f"agb200_{entry}")
    return out


__all__ = ["decode_attention", "decode_attention_rows", "decode_attention_workspace", "attention_supported",
           "attention_rows_supported", "prefill_attention", "prefill_attention_supported", "quantize_kv",
           "dequantize_kv", "decode_attention_rows_paged", "prefill_attention_paged", "paged_attention_supported"]
