"""Seeded random rigs (tests/rig_fuzz.py) through the compositor on the GPU, bit for bit against the CPU oracle, and the
A/B environment switches of the library, each of which must give the same bytes as the defaults."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import rig_fuzz
from stitching_b200 import Compositor

pytestmark = pytest.mark.gpu

SEED = rig_fuzz.seed_from_env()


@pytest.mark.parametrize("k", range(len(rig_fuzz.gpu_ids())), ids=rig_fuzz.gpu_ids())
def test_rig_fuzz_against_oracle(cuda_lib, oracle, k):
    case = rig_fuzz.gpu_set(SEED)[k]
    imgs, ex = rig_fuzz.images(case), rig_fuzz.extras(case)
    ref = rig_fuzz.oracle_run(oracle, case, imgs, ex)
    got = rig_fuzz.compositor_run(Compositor, case, imgs, ex)
    rig_fuzz.check(case, got, ref, SEED)


def test_rig_fuzz_coverage_on_the_gpu(oracle):
    """The GPU fuzz set reaches every kernel variant and launch-time branch listed here, by the launchers' own
    predicates (restated in rig_fuzz.coverage)."""
    cs = rig_fuzz.gpu_set(SEED)
    rows = [(c, rig_fuzz.coverage(c)) for c in cs]
    print(f"\nrig fuzz coverage, GPU set (seed {SEED}, {len(cs)} cases):\n" + rig_fuzz.coverage_table(rows))
    reached = set().union(*(t for _, t in rows))
    want = set(rig_fuzz.PYRDOWN_INSTANCES) | {
        "tile l0 yes", "tile l0 no", "tile l1 yes", "nb=0", "nb=1", "nb>=2", "feather", "no", "blend width < 1", "n>32",
        "odd pano width", "z<=0", "map projection", "mixed extras", "feather w>8192", "k_dt_rows_warp",
        "k_warp_rgbm<HAS_BM=0>", "k_warp_rgbm<HAS_BM=1>", "k_warp_wide", "2-px source"}
    assert want <= reached, f"not reached: {sorted(want - reached)}"
    assert rig_fuzz.redraw_share(cs) < 0.5, f"{rig_fuzz.redraw_share(cs):.2f} rejected draws per case"


# A/B switches: each is read once per process, so every setting runs in a child process
SWITCHES = [("SB_TILE", "0"), ("SB_TILE_MAXL", "3"), ("SB_GRAPH", "0"), ("SB_PDL", "0"), ("SB_DT", "0"), ("SB_PD_BIN", "0"),
            ("SB_SRC4", "0")]

_CHILD = """
import sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import rig_fuzz
from stitching_b200 import Compositor, _lib
_lib.check(_lib.lib().sb_init(0), "sb_init")
cs = rig_fuzz.gpu_set(int(sys.argv[3]))
out = {}
for k in map(int, sys.argv[4].split(",")):
    c = cs[k]
    got = rig_fuzz.compositor_run(Compositor, c, rig_fuzz.images(c), rig_fuzz.extras(c))
    out[f"{k}_pano"], out[f"{k}_pmask"] = got["pano"], got["pmask"]
    for i in range(c.n):
        out[f"{k}_w{i}"], out[f"{k}_m{i}"] = got["warped"][i], got["masks"][i]
np.savez(sys.argv[2], **out)
"""


def _ab_cases(cs):
    """About six cases for the switches: multiband with at least 4 bands (tile levels 2 and 3 under SB_TILE_MAXL=3) with
    and without gray masks, feather (the distance-transform kernels, the wide row kernel), and more than 32 images."""
    def first(pred, skip=()):
        return next(k for k, c in enumerate(cs) if k not in skip and pred(c))

    picked = []
    mb = lambda c: rig_fuzz.plan(c)[0] == "multiband" and rig_fuzz.plan(c)[1] >= 4  # noqa: E731
    picked.append(first(lambda c: mb(c) and all(m == "none" for m in c.masks)))
    picked.append(first(lambda c: mb(c) and all(m == "none" for m in c.masks) and c.wtype != cs[picked[0]].wtype))
    picked.append(first(lambda c: mb(c) and any(m in ("ramp", "random") for m in c.masks)))
    picked.append(first(lambda c: rig_fuzz.plan(c)[0] == "feather" and c.n >= 3))
    picked.append(next(k for k, c in enumerate(cs) if c.name == "wide_feather"))
    picked.append(first(lambda c: c.n > rig_fuzz.WARP_BATCH and rig_fuzz.plan(c)[0] == "multiband", picked))
    return picked


def test_ab_switches_give_identical_bytes(cuda_lib):
    from conftest import ROOT

    cs = rig_fuzz.gpu_set(SEED)
    picked = _ab_cases(cs)
    print("A/B cases: " + "; ".join(cs[k].describe() for k in picked))
    res = {}
    with tempfile.TemporaryDirectory() as d:
        for key, val in [(None, None)] + SWITCHES:
            env = {k: v for k, v in os.environ.items() if not (k.startswith("SB_") and k != "SB_RIG_FUZZ_SEED")}
            if key:
                env[key] = val
            out = os.path.join(d, f"{key or 'defaults'}.npz")
            subprocess.check_call([sys.executable, "-c", _CHILD, ROOT, out, str(SEED), ",".join(map(str, picked))], env=env)
            with np.load(out) as z:
                res[key] = {k: z[k] for k in z.files}
    base = res.pop(None)
    for key, arrays in res.items():
        assert arrays.keys() == base.keys()
        for name, a in arrays.items():
            k = int(name.split("_")[0])
            assert np.array_equal(a, base[name]), f"{key}={dict(SWITCHES)[key]}: {name} differs ({cs[k].describe()})"
