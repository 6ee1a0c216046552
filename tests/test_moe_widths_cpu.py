"""The grouped experts' decode layout restated (``tests/_moe_layout.py``): the experts of real MoE checkpoints that
``agb200_moe_create`` accepts on an H100 and the shared memory it plans for them, the hidden sizes it refuses although
the router kernel takes them, and ``agb200_moe_plan_bytes``."""
import pytest

from tests import _moe_layout as L


@pytest.mark.parametrize("name", sorted(L.WIDTHS))
def test_real_widths_accept_table(name):
    E, k, H, I = L.WIDTHS[name]
    got = L.decode_layout(H, I)
    assert got is not None, name
    assert (got["up_smem"], got["down_split"], got["down_smem"]) == L.H100_DECODE[name]
    assert got["up_smem"] <= L.H100_SMEM_OPTIN and got["down_smem"] <= L.H100_SMEM_OPTIN
    # the down stage's split covers I: every work item's rows are k8-rows of its share, 32-row aligned
    assert got["down_split"] * got["down_rps"] * 8 >= I and got["down_rps"] % 32 == 0
    assert got["down_rps"] * L.MD_ROWS * 16 <= L.DOWN_XS_CAP


def test_refused_hidden_sizes():
    """8 rows of x fit the H100's 227 KB opt-in up to H = 13824; the router kernel takes H up to 16384, so
    14336 ... 16384 pass the router's check and are refused by the experts."""
    assert L.max_hidden() == 13824
    assert L.decode_layout(13824, 128)["up_smem"] == 229376
    for H in (13952, 14336, 15360, L.REFUSED_H):
        assert L.decode_layout(H, 128) is None, H
    assert L.decode_layout(L.REFUSED_H, 128, smem_optin=1 << 20)["up_smem"] == 270336


def test_down_split_rule():
    # I <= 4096: one split; up to 8192: two; up to 16384: four; beyond, eight at most (the x may then exceed 64 KB)
    assert [L.decode_layout(128, I)["down_split"] for I in (4096, 4224, 8192, 8320, 16384, 16512, 65536)] == \
        [1, 2, 2, 4, 4, 8, 8]
    assert L.decode_layout(128, 65536)["down_rps"] * L.MD_ROWS * 16 > L.DOWN_XS_CAP
    # the I of tests/test_gpu_20_silu_mul_precision.py::test_moe_decode_down_split split in 2 and 4
    assert [L.decode_layout(256, I)["down_split"] for I in (4224, 8320)] == [2, 4]


@pytest.mark.parametrize("name", sorted(L.WIDTHS))
def test_plan_bytes_match_the_library(name):
    from autogptq_b200 import _lib

    E, _, H, I = L.WIDTHS[name]
    lib = _lib.load()
    for g in (128, -1):
        assert int(lib.agb200_moe_plan_bytes(E, H, I, g)) == L.plan_bytes(E, I)
