"""The reference's compiled qigen CPU kernel agrees with the NumPy oracle: pins the timed CPU baseline of bench.py to the
same arithmetic contract (zero nibbles <= 14: qigen does not wrap).  The kernel's outputs are stored in
tests/golden/kernel_qigen.npz (written by tests/golden/make_golden_kernels.py from oracle/_ref/cQIGen)."""
import os

import numpy as np
import pytest

from oracle import w4a16_oracle as O
from tests.golden.make_golden_kernels import QIGEN_CASES, qigen_inputs


@pytest.mark.parametrize("K,N,M", QIGEN_CASES)
def test_qigen_matches_oracle(golden_dir, K, N, M):
    d, x = qigen_inputs(K, N, M)
    y = np.load(os.path.join(golden_dir, "kernel_qigen.npz"))[f"y_{K}_{N}_{M}"]
    ref = O.forward(x, d["qweight"], d["qzeros"], d["scales"], g_idx=d["g_idx"], group_size=128, bias=None, out_dtype=np.float32)
    rms = float(np.sqrt(np.mean(ref ** 2)))
    assert np.abs(y - ref).max() <= 2e-4 * rms + 1e-4 * np.abs(ref).max()
