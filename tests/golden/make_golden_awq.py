"""Writes tests/golden/awq_*.npz: AutoAWQ GEMM layers converted by the reference's own AWQ -> GPTQ repack
(``unpack_awq`` + ``pack_from_tensors``, auto_gptq/modeling/_utils.py:525-701) on the CPU.

    python tests/golden/make_golden_awq.py /path/to/AutoGPTQ

_utils.py cannot be imported by path (relative imports, the whole modelling stack), so only the three functions are
taken from its syntax tree and executed with torch and numpy; Tensor.cuda is the identity while the fixtures are made.
The AWQ inputs are packed here the way AutoAWQ's WQLinear_GEMM.from_linear packs them (nibble i of a word holds column
8c + [0, 2, 4, 6, 1, 3, 5, 7][i]), independently of oracle/awq_oracle.py.  Each file holds:
  intweight [K, N] uint8, zeros [G, N] uint8     the integers of the layer
  awq_qweight, awq_qzeros, scales, bias          the AWQ checkpoint tensors
  ref_zeros [G, N]                               the zeros the reference's unpack_awq recovers
  ref_weight [N, K] fp16                         the fp16 weight it dequantises to
  ref_qweight, ref_qzeros                        the GPTQ tensors pack_from_tensors writes
The reference's unpack_awq reshapes by group_size along N (N % group_size == 0) and re-quantises by dividing by the
scale (no zero scales).
"""
import ast
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

# (name, K, N, group_size).  pack_from_tensors sizes qweight as K // 32 * 4 rows (_utils.py:672) and so drops the last
# K % 32 rows: every K is a multiple of 32, and g = 64 and 128 leave a partial last group.
LAYERS = [("awq_g32", 224, 128, 32), ("awq_g64", 352, 192, 64), ("awq_g128", 416, 256, 128)]
ORDER = [0, 2, 4, 6, 1, 3, 5, 7]


def load_reference_awq(ref_root):
    path = os.path.join(ref_root, "auto_gptq", "modeling", "_utils.py")
    tree = ast.parse(open(path).read(), filename=path)
    wanted = {"awq_reverse_reorder_int_tensor", "unpack_awq", "pack_from_tensors"}
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in wanted]
    assert {n.name for n in body} == wanted
    ns = {"torch": torch, "np": np}
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns["unpack_awq"], ns["pack_from_tensors"]


def autoawq_pack(v):
    """uint8 [R, N] -> int32 [R, N/8], AutoAWQ's GEMM order."""
    v = v.astype(np.uint32)
    out = np.zeros((v.shape[0], v.shape[1] // 8), dtype=np.uint32)
    for c in range(out.shape[1]):
        for i in range(8):
            out[:, c] |= v[:, 8 * c + ORDER[i]] << np.uint32(4 * i)
    return out.view(np.int32)


def make_layer(unpack_awq, pack_from_tensors, name, K, N, g, seed):
    rng = np.random.default_rng(seed)
    G = -(-K // g)
    q = rng.integers(0, 16, size=(K, N), dtype=np.uint8)
    z = rng.integers(0, 16, size=(G, N), dtype=np.uint8)
    z.reshape(-1)[:16] = np.arange(16)                      # every zero value, 0 included
    scales = (rng.random((G, N), dtype=np.float32) * 0.01 + 0.001).astype(np.float16)
    bias = (rng.standard_normal(N) * 0.1).astype(np.float16)
    qweight, qzeros = autoawq_pack(q), autoawq_pack(z)
    weight, zeros = unpack_awq(torch.from_numpy(qweight), torch.from_numpy(qzeros), torch.from_numpy(scales),
                               bits=4, group_size=g)
    gq, gz = pack_from_tensors(weight, zeros, torch.from_numpy(scales), bits=4, group_size=g)
    data = dict(intweight=q, zeros=z, awq_qweight=qweight, awq_qzeros=qzeros, scales=scales, bias=bias,
                group_size=np.int32(g), ref_zeros=zeros.numpy().astype(np.int32), ref_weight=weight.numpy(),
                ref_qweight=gq.numpy(), ref_qzeros=gz.numpy())
    assert data["ref_weight"].dtype == np.float16 and data["ref_weight"].shape == (N, K)
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **data)
    print(f"{path}: {os.path.getsize(path)} bytes")


def main():
    if len(sys.argv) != 2:
        sys.exit("usage: make_golden_awq.py <AutoGPTQ source tree>")
    unpack_awq, pack_from_tensors = load_reference_awq(sys.argv[1])
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        for i, (name, K, N, g) in enumerate(LAYERS):
            make_layer(unpack_awq, pack_from_tensors, name, K, N, g, seed=300 + i)
    finally:
        torch.Tensor.cuda = cuda


if __name__ == "__main__":
    main()
