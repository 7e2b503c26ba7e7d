"""tests/kernel_edges.py's cases on the GPU, bit for bit against the oracle: the weight pyramid's summation orders on gray
masks (the shuffle pyrDown; uint8-only results take the tile kernel's level 0), a gain product of exactly 2^31, rays
with z == 0, and binary-mask rigs whose level 3 needs the reference's summation orders."""
import pytest

import kernel_edges

pytestmark = pytest.mark.gpu

_CASES = kernel_edges.gpu_cases()


@pytest.mark.parametrize("k", range(len(_CASES)), ids=[c for c, _ in _CASES])
def test_edge_against_oracle(cuda_lib, oracle, k):
    _CASES[k][1](oracle)
