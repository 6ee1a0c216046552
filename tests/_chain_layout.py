"""The decode chain's shared-memory layout restated in Python: ``ChainSmem<M>::fixed`` / ``total`` (chain.cuh) and the
ring-depth rule of ``agb200_chain_create_norm`` (chain.cu), for the tests to hold ``DecodeChain.info()`` to.

A chain's shared memory is a ring of 17 KB weight slots plus a fixed part sized by its widest x:

    fixed = digits (rows_pad · 4M · 8, to 128 B) + digit-sum table (rows_pad / 16 · 32) + staged x + reductions
            (2 · 12 warps · 2M · 32 · 4) + descriptors (6 · 96 · 4) + 64 + mbarriers ((3 · 13 + 2 · 2 + 32) · 8) + 1024

with rows_pad = 128 k8-rows per started 1024-k chunk of the widest K, and the staged x M·K·2 bytes (to 128 B) of the
widest stage that is a norm stage or gathers x (act-order).  The ring takes what the device's opt-in leaves, at most
13 slots; fewer than 3 is refused (``AGB200_ENOSUP``).  Without ``AGB200_CHAIN_SMEM_KB`` / ``AGB200_CHAIN_SLOTS``."""
from __future__ import annotations

H100_SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100: 227 KB
SLOT_BYTES = 17 * 1024
MAX_SLOTS, MIN_SLOTS = 13, 3


def _align(n: int, a: int = 128) -> int:
    return (n + a - 1) // a * a


def fixed_bytes(M: int, rows_pad: int, xs_bytes: int) -> int:
    """``ChainSmem<M>::fixed(rows_pad, xs_bytes)``."""
    digits = _align(rows_pad * 4 * M * 8)
    dsum = rows_pad // 16 * 4 * 8
    red = 2 * 12 * (2 * M) * 32 * 4
    desc = 6 * 96 * 4
    bars = (3 * MAX_SLOTS + 2 * 2 + 32) * 8
    return digits + dsum + xs_bytes + red + desc + 64 + bars + 1024


def layout(M: int, stages, smem_optin: int = H100_SMEM_OPTIN):
    """(ring slots, dynamic shared memory bytes) of a chain whose stages are (K, staged) pairs, ``staged`` for a norm
    stage or an act-order one; None when the chain is refused."""
    rows_pad = max(-(-K // 1024) * 128 for K, _ in stages)
    xs = max([_align(M * K * 2) for K, staged in stages if staged] or [0])
    fixed = fixed_bytes(M, rows_pad, xs)
    if fixed + MIN_SLOTS * SLOT_BYTES > smem_optin:
        return None
    slots = min((smem_optin - fixed) // SLOT_BYTES, MAX_SLOTS)
    return slots, slots * SLOT_BYTES + fixed


def block_stages(H: int, I: int, act_order: bool, q_dim: int | None = None):
    """The stages of one dense decoder block as ChainDecoder chains it (o, add_rmsnorm gate|up, silu_mul down,
    add_rmsnorm next q|k|v), with act-order on every projection or on none."""
    return [(q_dim or H, act_order), (H, True), (I, act_order), (H, True)]


def block_layout(H: int, I: int, M: int, act_order: bool, smem_optin: int = H100_SMEM_OPTIN):
    return layout(M, block_stages(H, I, act_order), smem_optin)


# (H, I) of real GPTQ checkpoints, and what ChainDecoder takes on an H100 at batch 1 and 2 (DESIGN §3.5): ring slots,
# None where the block's chain is refused.  Keys: (M, act_order).
WIDTHS = {
    "llama2_7b": (4096, 11008),
    "llama2_13b": (5120, 13824),
    "mistral_7b": (4096, 14336),
    "qwen2_1.5b": (1536, 8960),
    "qwen2_7b": (3584, 18944),
    "llama_70b": (8192, 28672),
    "qwen2_72b": (8192, 29568),
}
H100_SLOTS = {
    "llama2_7b": {(1, False): 9, (1, True): 8, (2, False): 6, (2, True): 4},
    "llama2_13b": {(1, False): 8, (1, True): 7, (2, False): 4, (2, True): None},
    "mistral_7b": {(1, False): 8, (1, True): 7, (2, False): 4, (2, True): None},
    "qwen2_1.5b": {(1, False): 10, (1, True): 9, (2, False): 7, (2, True): 5},
    "qwen2_7b": {(1, False): 7, (1, True): 5, (2, False): None, (2, True): None},
    "llama_70b": {(1, False): 4, (1, True): None, (2, False): None, (2, True): None},
    "qwen2_72b": {(1, False): 4, (1, True): None, (2, False): None, (2, True): None},
}
