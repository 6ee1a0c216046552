"""The decode chain's shared-memory layout restated (``tests/_chain_layout.py``) against what an H100 measured, and the
blocks of real checkpoints it accepts or refuses at batch 1 and 2 (DESIGN §3.5)."""
import pytest

from tests import _chain_layout as L
from tests.test_gpu_21_chain_norm import BASE_INFO


def test_restatement_reproduces_the_measured_bench_chain():
    """test_chain_without_norm_stages_keeps_its_shape's chain: q|k|v, o, gate|up, silu_mul down of a Llama-2-7B block,
    no norm stage, no act-order; (ring slots, shared memory bytes) measured on an H100 80GB HBM3."""
    stages = [(4096, False), (4096, False), (4096, False), (11008, False)] * 2
    for M in (1, 2):
        assert L.layout(M, stages) == BASE_INFO[M]
    # with the block's two norm stages the fixed part grows by the staged x, M * 4096 * 2 bytes
    for M in (1, 2):
        with_norm = L.layout(M, [(4096, True), (4096, False), (4096, True), (11008, False)])
        fixed = with_norm[1] - with_norm[0] * L.SLOT_BYTES
        assert fixed == BASE_INFO[M][1] - BASE_INFO[M][0] * L.SLOT_BYTES + M * 4096 * 2


@pytest.mark.parametrize("name", sorted(L.WIDTHS))
def test_dense_block_accept_refuse_table(name):
    H, I = L.WIDTHS[name]
    for (M, act), slots in L.H100_SLOTS[name].items():
        got = L.block_layout(H, I, M, act)
        assert (got and got[0]) == slots, (name, M, act, got)
        if got is not None:
            assert got[1] <= L.H100_SMEM_OPTIN and got[0] >= L.MIN_SLOTS


def test_limits():
    # K = 32768 (32 chunks, the most a stage takes) fits at M = 1 with a 4-slot ring, not at M = 2
    assert L.layout(1, [(32768, False)]) == (4, 4 * L.SLOT_BYTES + L.fixed_bytes(1, 4096, 0))
    assert L.layout(2, [(32768, False)]) is None
    # a 1024-k chunk is the unit: K = 1152 costs two chunks of digits, as K = 2048 does
    assert L.layout(1, [(1152, False)]) == L.layout(1, [(2048, False)])
    # the smallest chain leaves room for 12 slots on an H100; the ring never exceeds 13 slots whatever the opt-in
    assert L.layout(1, [(128, False)])[0] == 12
    assert L.layout(1, [(128, False)], smem_optin=1 << 20)[0] == L.MAX_SLOTS
    # a smaller opt-in only shortens the ring, until fewer than 3 slots are left
    fx = L.fixed_bytes(1, 1408, 0)
    assert L.layout(1, [(11008, False)], smem_optin=fx + 3 * L.SLOT_BYTES) == (3, fx + 3 * L.SLOT_BYTES)
    assert L.layout(1, [(11008, False)], smem_optin=fx + 3 * L.SLOT_BYTES - 1) is None
