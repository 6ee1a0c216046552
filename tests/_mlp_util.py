"""Oracle and helpers of the fused gate/up tests (autogptq_b200.forward_gate_up / FusedQuantMLP)."""
import numpy as np
import torch

from oracle import w4a16_oracle as O
from oracle.mlp_oracle import gate_up
from tests._util import assert_parity, make_layer

TOL = {torch.float16: dict(rtol=1e-3, atol_rms=1.6e-3), torch.bfloat16: dict(rtol=8e-3, atol_rms=4e-3)}   # as the MoE tests
DT = {torch.float16: "float16", torch.bfloat16: "bfloat16"}
ULP = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}
# Share of h elements allowed to differ from the oracle at all.  A difference needs g or u to land on the other side of a
# rounding boundary (the fp32 sums differ only in their last bits), which is rare; breaking the rounding rule (silu(g)
# or g / u left unrounded before the product) moves a fifth or more of all elements.
MAX_MISMATCH = 0.05

def make_pair(K, I, g, desc_act=False, bias=False, dtype=torch.float16, seed=0):
    """(gate QuantLinear, up QuantLinear, oracle dicts with the scales / bias the device uses); up shares gate's g_idx."""
    mods, ref = [], []
    for j in range(2):
        d = O.random_packed(K, I, g, seed=seed + j, desc_act=desc_act, bias=bias)
        if j == 1 and desc_act:
            d["g_idx"] = ref[0]["g_idx"]              # gate and up see the same inputs: one act-order permutation
        lin = make_layer(d, device="cuda", dtype=dtype)
        mods.append(lin)
        ref.append(dict(d, scales=lin.scales.float().cpu().numpy(),
                        bias=None if lin.bias is None else lin.bias.float().cpu().numpy()))
    return mods[0], mods[1], ref[0], ref[1]


def x_rows(M, K, dtype, seed=1):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((M, K)).astype(np.float32)).to(dtype).cuda()


def assert_gate_up(h, x, gref, uref, dtype, exact_w, what):
    """assert_parity of h against the oracle (exact weights for the decode kernel, weights rounded to the dtype for the
    tensor-core GEMM), after excusing two ulps of every h: g and u are rounded to the dtype before the product, so a
    last-bit difference in either fp32 sum moves h by up to one ulp each.  Such differences must stay rare:
    at most MAX_MISMATCH of the elements may differ at all."""
    h_ref = gate_up(x.float().cpu().numpy(), gref, uref, DT[dtype], weight_dtype=None if exact_w else DT[dtype])
    h = np.asarray(h.float().cpu().numpy(), dtype=np.float32).reshape(h_ref.shape)
    err = h - h_ref
    mismatch = float(np.mean(err != 0))
    assert mismatch <= MAX_MISMATCH, f"{what}: {mismatch:.2%} of h differ from the oracle (rounding rule?)"
    excused = np.sign(err) * np.maximum(np.abs(err) - 2 * ULP[dtype] * np.abs(h_ref), 0)
    assert_parity(h_ref + excused, h_ref, what=what, **TOL[dtype])
