"""The drop-in classes on the GPU (tests/dropin_fuzz.py): the GPU rig and crop sets and the drop-in-only draws, bit for bit
against the CPU oracle, and every panorama equal to the fused Compositor's for the same case."""
import numpy as np
import pytest

import dropin_fuzz
import fuzz_chain
import rig_fuzz

pytestmark = pytest.mark.gpu

SEED = dropin_fuzz.seed_from_env()


@pytest.mark.parametrize("k", range(dropin_fuzz.gpu_count()))
def test_dropin_fuzz_against_oracle_and_compositor(cuda_lib, oracle, k):
    dc = dropin_fuzz.gpu_set(SEED)[k]
    imgs, ex, got = dropin_fuzz.run_and_check(oracle, dc, SEED)
    fused = fuzz_chain.compositor_run(dc.case, imgs, ex, crop=dc.crop.crop if dc.crop is not None else None)
    assert np.array_equal(fused["pano"], got["pano"]) and np.array_equal(fused["pmask"], got["pmask"]), \
        f"{dc.describe()}: the drop-in panorama differs from the compositor's"


def test_dropin_fuzz_coverage_on_the_gpu(oracle):
    cs = dropin_fuzz.gpu_set(SEED)
    assert len(cs) == dropin_fuzz.gpu_count()
    # the k_warp_wide paths from the maps for the drop-in-only draws (the ones drawn for them), the rest from the draw
    rows = [(c, dropin_fuzz.coverage(c, oracle if c.name.startswith("own_") else None)) for c in cs]
    print(f"\ndrop-in fuzz coverage, GPU set (seed {SEED}, {len(cs)} cases):\n" + rig_fuzz.coverage_table(rows))
    reached = set().union(*(t for _, t in rows))
    assert dropin_fuzz.WANT <= reached, f"not reached: {sorted(dropin_fuzz.WANT - reached)}"
