"""Generate the input-gradient fixtures ``tests/golden/dgrad_*.npz`` from the REFERENCE itself.

Run in the authoring container only (needs /root/reference; the GPU box has no reference tree):

    python tests/golden/make_golden_dgrad.py

The reference's Python QuantLinear classes (``qlinear_cuda_old.py``: wrap rule, sequential groups;
``qlinear_cuda.py``: g_idx gather) are loaded by file path and run on their differentiable CPU path
(dequantise + ``torch.matmul``, qlinear_cuda_old.py:291-355 / qlinear_cuda.py:300-314) with ``x.requires_grad``;
``y.backward(dy)`` then gives ``x.grad = dy · Wᵀ``, which is stored.  Zero nibbles stay in [0, 14] as in the other
goldens: ``qlinear_cuda.py`` does not wrap zeros, this project and ``qlinear_cuda_old.py`` do.  Nothing here is imported
by the product.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import w4a16_oracle as O  # noqa: E402  (only for the synthetic generator)


def load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


old = load("qlinear_cuda_old", f"{REF}/auto_gptq/nn_modules/qlinear/qlinear_cuda_old.py")
new = load("qlinear_cuda", f"{REF}/auto_gptq/nn_modules/qlinear/qlinear_cuda.py")


def ref_dgrad(cls_mod, d, x, dy):
    K, N, gs = d["K"], d["N"], d["group_size"]
    lin = cls_mod.QuantLinear(bits=4, group_size=gs, infeatures=K, outfeatures=N, bias=d["bias"] is not None,
                              weight_dtype=torch.float32)
    lin.qweight = torch.from_numpy(d["qweight"].copy())
    lin.qzeros = torch.from_numpy(d["qzeros"].copy())
    lin.scales = torch.from_numpy(d["scales"].astype(np.float32))
    lin.g_idx = torch.from_numpy(d["g_idx"].copy())
    if d["bias"] is not None:
        lin.bias = torch.from_numpy(d["bias"].astype(np.float32))
    xt = torch.from_numpy(x.astype(np.float32)).requires_grad_(True)
    y = lin(xt)
    y.backward(torch.from_numpy(dy.astype(np.float32)))
    return xt.grad.numpy().copy()


cases = [
    # name,         K,    N,   g,   desc_act, bias,  M
    ("seq_g128",    512,  256, 128, False,    False, 5),
    ("seq_g32_bias", 256, 384, 32,  False,    True,  3),
    ("seq_gfull",   384,  128, -1,  False,    False, 7),
    ("act_g128",    512,  256, 128, True,     False, 4),
    ("act_g32_bias", 256, 384, 32,  True,     True,  2),
]
for i, (name, K, N, g, act, bias, M) in enumerate(cases):
    d = O.random_packed(K, N, g, seed=300 + i, desc_act=act, zero_max=14, bias=bias)
    rng = np.random.default_rng(400 + i)
    x = rng.standard_normal((M, K)).astype(np.float16)
    dy = rng.standard_normal((M, N)).astype(np.float16)
    out = {"dx_new": ref_dgrad(new, d, x, dy)}
    if not act:
        out["dx_old"] = ref_dgrad(old, d, x, dy)
    np.savez_compressed(os.path.join(HERE, f"dgrad_{name}.npz"), qweight=d["qweight"], qzeros=d["qzeros"],
                        scales=d["scales"], g_idx=d["g_idx"], bias=(d["bias"] if bias else np.zeros(0, np.float16)),
                        x=x, dy=dy, group_size=np.int32(d["group_size"]), desc_act=np.bool_(act), **out)
    print("wrote", f"dgrad_{name}.npz", sorted(out))
print("done")
