"""The grouped experts' decode layout restated in Python: what ``agb200_moe_create`` (moe.cu) plans for the decode path
(T <= 8) from the constants of moe.cuh and moe.cu, and ``agb200_moe_plan_bytes``, for the tests to hold the library to.

    up stage (w1|w3):  up_rps = round_up(H / 8, 32) k8-rows of x per work item (all of H: h needs the full K)
                       up_smem = up_rps · kMdRows · 16 + kMdRedBytes          kMdRows = 8, kMdRedBytes = 8 · 8 · 32 · 4
    down stage (w2):   split I in 2, 4 or 8 (at most 8) until down_rps · kMdRows · 16 <= kDownXsCap (64 KB, 3 CTAs/SM),
                       down_rps = round_up(ceil(I / 8 / down_split), 32)
                       down_smem = down_rps · kMdRows · 16 + kMdRedBytes

A plan whose up_smem exceeds the device's opt-in is refused (``AGB200_ENOSUP``); the down stage always fits once split."""
from __future__ import annotations

H100_SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100: 227 KB
MD_ROWS = 8                       # kMdRows: x rows per pass (the n = 8 of mma.m16n8k16)
MD_RED_BYTES = 8 * MD_ROWS * 32 * 4   # kMdRedBytes = kMdWarps · kMdRows · kMdTN · 4
DOWN_XS_CAP = 64 * 1024           # kDownXsCap
MAX_DOWN_SPLIT = 8
TENSOR_MAP_BYTES = 128            # sizeof(CUtensorMap)
EXPERT_DESC_BYTES = 4 * 3 * 8 + 2 * 8   # sizeof(agb::MoeExpertDev): 4 arrays of 3 pointers, perm13, inv2


def _round_up(v: int, a: int) -> int:
    return (v + a - 1) // a * a


def decode_layout(H: int, I: int, smem_optin: int = H100_SMEM_OPTIN):
    """dict(up_rps, up_smem, down_split, down_rps, down_smem) of ``agb200_moe_create``'s decode path, or None when it
    refuses H (8 rows of x do not fit the opt-in)."""
    up_rps = _round_up(H // 8, 32)
    up_smem = up_rps * MD_ROWS * 16 + MD_RED_BYTES
    if up_smem > smem_optin:
        return None
    down_split, down_rps = 1, _round_up(I // 8, 32)
    while down_split < MAX_DOWN_SPLIT and down_rps * MD_ROWS * 16 > DOWN_XS_CAP:
        down_split *= 2
        down_rps = _round_up(-(-(I // 8) // down_split), 32)
    return dict(up_rps=up_rps, up_smem=up_smem, down_split=down_split, down_rps=down_rps,
                down_smem=down_rps * MD_ROWS * 16 + MD_RED_BYTES)


def max_hidden(smem_optin: int = H100_SMEM_OPTIN) -> int:
    """The largest H (a multiple of 128) whose up stage fits ``smem_optin``."""
    return max(H for H in range(128, 65536 + 1, 128) if decode_layout(H, 128, smem_optin) is not None)


def plan_bytes(E: int, I: int) -> int:
    """``agb200_moe_plan_bytes``: 9 tensor maps and one descriptor per expert, and each expert's inverse w2
    permutation (I int32), each part 256-byte aligned."""
    return (_round_up(E * 9 * TENSOR_MAP_BYTES, 256) + _round_up(E * EXPERT_DESC_BYTES, 256)
            + _round_up(E * I * 4, 256))


# (E, k, H, I) of the experts of real checkpoints
WIDTHS = {
    "mixtral_8x7b": (8, 2, 4096, 14336),
    "mixtral_8x22b": (8, 2, 6144, 16384),
    "qwen1.5_moe_a2.7b": (60, 4, 2048, 1408),
    "qwen3_30b_a3b": (128, 8, 2048, 768),
}
# What the decode path plans for them on an H100: (up_smem, down_split, down_smem); None where H is refused.  H = 16384
# is the largest hidden size the router kernel takes (AGB200_CHAIN_NORM_MAX_K) and needs 264 KB for 8 rows of x.
H100_DECODE = {
    "mixtral_8x7b": (73728, 4, 65536),
    "mixtral_8x22b": (106496, 4, 73728),         # 104 KB: two up-stage CTAs per SM instead of three
    "qwen1.5_moe_a2.7b": (40960, 1, 32768),
    "qwen3_30b_a3b": (40960, 1, 20480),
}
REFUSED_H = 16384
