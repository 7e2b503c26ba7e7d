"""The compositor with a crop (Stitcher's default Cropper) on the GPU: seeded crops bit for bit against the CPU oracle,
the full crop against no crop, submit / wait against composite(), the A/B switches, and the sharded roles on one GPU."""
import os

import numpy as np
import pytest

import crop_fuzz
import fuzz_chain
import rig_fuzz

pytestmark = pytest.mark.gpu

SEED = crop_fuzz.seed_from_env()
GPU_COUNT = 40
NAMED = ["many", "full"]

_sets = {}


def gpu_set():
    if "gpu" not in _sets:
        _sets["gpu"] = crop_fuzz.cases(SEED, GPU_COUNT, rig_fuzz.GPU) + [crop_fuzz.named(n, rig_fuzz.GPU) for n in NAMED]
    return _sets["gpu"]


@pytest.mark.parametrize("k", range(GPU_COUNT + len(NAMED)))
def test_crop_fuzz_against_oracle(cuda_lib, oracle, k):
    crop_fuzz.run_and_check(oracle, gpu_set()[k], SEED)


def test_crop_fuzz_coverage_on_the_gpu():
    rows = [(c, crop_fuzz.coverage(c)) for c in gpu_set()]
    print("\ncrop fuzz coverage, GPU set:\n" + rig_fuzz.coverage_table(rows))
    reached = set().union(*(t for _, t in rows))
    want = {"multiband", "feather", "no", "nb=0", "nb=1", "nb>=2", "affine", "spherical", "cylindrical", "map projection",
            "n>32", "tile l0 yes", "tile l0 no", "crop changes num_bands", "fed smaller than prepared",
            "placement off by rounding", "extras"}
    assert want <= reached, f"not reached: {sorted(want - reached)}"
    assert len(gpu_set()) == GPU_COUNT + len(NAMED)


def test_full_crop_equals_no_crop(cuda_lib):
    cc = crop_fuzz.named("full", rig_fuzz.GPU)
    imgs, ex = rig_fuzz.images(cc.case), rig_fuzz.extras(cc.case)
    got = fuzz_chain.compositor_run(cc.case, imgs, ex, crop=cc.crop)
    plain = fuzz_chain.compositor_run(cc.case, imgs, ex)
    assert np.array_equal(got["pano"], plain["pano"]) and np.array_equal(got["pmask"], plain["pmask"])


def _multiband_crop(cs):
    return next(c for c in cs if rig_fuzz.plan(c.cropped_case())[0] == "multiband" and
                any((f[2], f[3]) != tuple(s) for f, s in zip(c.fed(), c.crop.sizes)))


def test_submit_wait_with_a_crop_equals_composite(cuda_lib):
    cc = _multiband_crop(gpu_set())
    imgs = rig_fuzz.images(cc.case)
    c = crop_fuzz.compositor(cc)
    try:
        ref, ref_mask = c.composite(imgs)
        srcs = []
        for im in imgs:
            p = c.pinned_empty(im.shape)
            p[...] = im
            srcs.append(p)
        outs = [(c.pinned_empty(ref.shape), c.pinned_empty(ref_mask.shape)) for _ in range(4)]
        tickets = [c.submit(srcs, o, m) for o, m in outs[:3]]
        c.wait(tickets[0])
        tickets.append(c.submit(srcs, *outs[3]))
        for t in tickets[1:]:
            c.wait(t)
        for o, m in outs:
            assert np.array_equal(o, ref) and np.array_equal(m, ref_mask)
    finally:
        c.close()


def test_ab_switches_with_a_crop_give_identical_bytes(cuda_lib):
    cs = gpu_set()[:GPU_COUNT]
    picked = sorted({cs.index(_multiband_crop(cs)),
                     next(k for k, c in enumerate(cs) if rig_fuzz.plan(c.cropped_case())[1] >= 3),
                     next(k for k, c in enumerate(cs) if any(m in ("ramp", "random", "seam") for m in c.case.masks)),
                     next(k for k, c in enumerate(cs) if rig_fuzz.plan(c.cropped_case())[0] == "feather")})
    fuzz_chain.ab_run("crop_fuzz:ab_arrays", [SEED, GPU_COUNT, picked],
                      [("SB_TILE", "0"), ("SB_PD_BIN", "0"), ("SB_SRC4", "0"), ("SB_GRAPH", "0")], "SB_CROP_FUZZ_SEED")


def test_sharded_crop_roles_on_one_gpu(cuda_lib, oracle):
    """All ranks of a cropped sharded composite on one GPU, the slabs moved with device copies: every strip equals the
    grouped oracle fed with the cropped images."""
    cs = crop_fuzz.sharded_cases(SEED, 6, rig_fuzz.GPU)
    ran = set()
    for cc in cs:
        for world in (2, 3):
            if cc.n >= world and crop_fuzz.sharded_check(oracle, cc, world, fuzz_chain.device_copy, SEED):
                ran.add(world)
    assert ran == {2, 3}, f"worlds run: {sorted(ran)} of {len(cs)} cases"


def test_reference_stitcher_with_crop(cuda_lib):
    """The recorded crop=True Stitcher run (tests/golden/golden_crop.npz) through the compositor on the GPU."""
    from conftest import ROOT

    pytest.importorskip("cv2")
    got, ref = crop_fuzz.stitch_replay(os.path.join(ROOT, "tests", "golden", "golden_crop.npz"))
    assert got == ref
