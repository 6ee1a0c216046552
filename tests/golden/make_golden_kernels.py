"""Store outputs of the reference's compiled kernels (oracle/_ref) for the tests that compare with them:
`python tests/golden/make_golden_kernels.py qigen|exllamav2 [OUT_DIR]` (exllamav2 needs a GPU).  Inputs are seeded."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from oracle import w4a16_oracle as O  # noqa: E402

# (K, N, M) of tests/test_oracle_qigen.py; layer seed K + N + M, x seed M
QIGEN_CASES = [(4096, 4096, 1), (4096, 11008, 1), (11008, 4096, 3), (1024, 512, 8)]
# tests/test_gpu_2b_skinny.py::test_reference_exllamav2_kernel_agrees: one layer, x seed M
EXL_K, EXL_N, EXL_G, EXL_SEED, EXL_MS = 1024, 1024, 128, 43, (1, 8, 64)


def qigen_inputs(K, N, M):
    d = O.random_packed(K, N, 128, seed=K + N + M, zero_max=14, scale_dtype=np.float32)
    x = np.random.default_rng(M).standard_normal((M, K)).astype(np.float32)
    return d, x


def make_qigen(out):
    from oracle import qigen_ref

    assert qigen_ref.available(), "oracle/_ref/cQIGen not built"
    ys = {}
    for K, N, M in QIGEN_CASES:
        d, x = qigen_inputs(K, N, M)
        ys[f"y_{K}_{N}_{M}"] = qigen_ref.QigenLinear(d["qweight"], d["qzeros"], d["scales"], 128).forward(x).numpy()
    np.savez_compressed(os.path.join(out, "kernel_qigen.npz"), **ys)


def make_exllamav2(out):
    import torch

    from oracle import ref_kernels
    from tests._util import make_layer, rand_x

    assert ref_kernels.exllamav2() is not None, "oracle/_ref/exllamav2_kernels not built"
    d = O.random_packed(EXL_K, EXL_N, EXL_G, seed=EXL_SEED)
    lin = make_layer(d)
    ref = ref_kernels.ExllamaV2Layer(lin.qweight, lin.qzeros, lin.scales, EXL_K, EXL_N)
    ys = {}
    for M in EXL_MS:
        x = torch.from_numpy(rand_x(M, EXL_K, seed=M)).cuda()
        ys[f"y_{M}"] = ref(x).half().cpu().numpy()
    np.savez_compressed(os.path.join(out, "kernel_exllamav2.npz"), **ys)


if __name__ == "__main__":
    what = sys.argv[1]
    out = sys.argv[2] if len(sys.argv) > 2 else HERE
    os.makedirs(out, exist_ok=True)
    {"qigen": make_qigen, "exllamav2": make_exllamav2}[what](out)
    print("wrote", os.path.join(out, f"kernel_{what}.npz"))
