"""Input-gradient oracle for the dgrad tests: dx = dy · dequant(W)ᵀ in fp32 (NumPy, built on the W4A16 oracle)."""
import os

import numpy as np

from oracle import moe_oracle as MO
from oracle import w4a16_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DGRAD_GOLDENS = ["seq_g128", "seq_g32_bias", "seq_gfull", "act_g128", "act_g32_bias"]


def dgrad(d, dy, round_to=None, rows=None):
    """dx[M, K] = dy[M, N] · Wᵀ in fp32, W = s·(q − z) with the wrap rule and g_idx (so act-order layers come out in
    the original column order of x).  ``round_to`` ("float16" / "bfloat16") rounds the scales and then every weight to
    that dtype, as the kernels do; None keeps them exact.  ``rows`` = (k0, k1), multiples of 8: those dx columns only."""
    k0, k1 = rows or (0, d["K"])
    s = np.asarray(d["scales"], dtype=np.float32)
    if round_to is not None:
        s = MO.round_to(s, round_to)
    W = O.dequantize(d["qweight"][k0 // 8:k1 // 8], d["qzeros"], s, g_idx=np.asarray(d["g_idx"])[k0:k1])
    if round_to is not None:
        W = MO.round_to(W, round_to)
    return np.asarray(dy, dtype=np.float32).reshape(-1, W.shape[1]) @ W.T


def load_golden(name):
    z = dict(np.load(os.path.join(GOLDEN, f"dgrad_{name}.npz")))
    K = z["x"].shape[1]
    d = dict(qweight=z["qweight"], qzeros=z["qzeros"], scales=z["scales"], g_idx=z["g_idx"],
             bias=z["bias"] if z["bias"].size else None, K=K, N=z["qweight"].shape[1], group_size=int(z["group_size"]))
    return d, z
