"""Single arithmetic decisions of the kernels that random rigs rarely reach (tests/kernel_edges.py), through the emulation
build, bit for bit against the oracle: the float weight pyrDown's summation orders on gray masks (also through the
shuffle pyrDown under SB_EMU_LANES), a gain product of exactly 2^31 and rays with z == 0."""
import pytest

import kernel_edges

_CASES = kernel_edges.emu_cases()


@pytest.mark.parametrize("k", range(len(_CASES)), ids=[c for c, _ in _CASES])
def test_edge_against_oracle(use_emu, oracle, monkeypatch, k):
    _CASES[k][1](oracle, monkeypatch)


def test_order_cases_cover_every_width_residue():
    """The padded rects of the order cases give float-pyrDown levels with every width0 % 4 and every dw % 4, levels whose
    SIMD body is empty; every one is checked on the int16 and on the uint8-only result."""
    cases = [kernel_edges.orders_case(s) for s, _ in kernel_edges.ORDER_SEEDS]
    widths = set().union(*(kernel_edges.order_widths(c) for c in cases))
    assert {w0 for w0, _, _ in widths} == {0, 1, 2, 3}, widths
    assert {dw for _, dw, _ in widths} == {0, 1, 2, 3}, widths
    assert {empty for _, _, empty in widths} == {False, True}, widths
    ids = [c for c, _ in _CASES if c.startswith("orders_")]
    assert sum(c.count("_u8") for c in ids) == sum(c.count("_s16") for c in ids) > 0
    assert any(lanes for _, lanes in kernel_edges.ORDER_SEEDS), "the shuffle pyrDown must run some of them"
