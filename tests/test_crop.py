"""The compositor with a crop (Stitcher's default Cropper), in the emulation build: bit for bit against the oracle that
slices the warped images as Stitcher.crop_final_resolution does, and the refusals of a cropped sb_compositor_create."""
import os
import types

import numpy as np
import pytest

import crop_fuzz
import fuzz_chain
import rig_fuzz
from conftest import ROOT
from stitching_b200 import Crop, StitchingError

SEED = crop_fuzz.seed_from_env()
EMU_COUNT = 24
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_crop.npz")

_sets = {}


def emu_set():
    if "emu" not in _sets:
        _sets["emu"] = crop_fuzz.cases(SEED, EMU_COUNT, rig_fuzz.EMU) + [crop_fuzz.named("many", rig_fuzz.EMU)]
    return _sets["emu"]


@pytest.mark.parametrize("k", range(EMU_COUNT + 1))
def test_crop_fuzz_against_oracle(use_emu, oracle, k):
    """Rects (feed corner and fed size), pano roi, num_bands, every cropped warped image and mask, the panorama and its
    mask equal the oracle's, with set_mask / set_seam_mask / set_gain sized to the cropped images."""
    crop_fuzz.run_and_check(oracle, emu_set()[k], SEED)


def test_crop_fuzz_coverage():
    rows = [(c, crop_fuzz.coverage(c)) for c in emu_set()]
    print("\ncrop fuzz coverage, emulation set:\n" + rig_fuzz.coverage_table(rows))
    reached = set().union(*(t for _, t in rows))
    want = {"multiband", "feather", "no", "nb=0", "nb=1", "nb>=2", "affine", "spherical", "cylindrical", "map projection",
            "n>32", "tile l0 yes", "tile l0 no", "crop changes num_bands", "fed smaller than prepared",
            "placement off by rounding", "extras"}
    assert want <= reached, f"not reached: {sorted(want - reached)}"
    assert len(emu_set()) == EMU_COUNT + 1


def test_full_crop_equals_no_crop(use_emu, oracle):
    """Every image whole, placed at its warped corner shifted by a constant: the same bytes as the uncropped compositor."""
    cc = crop_fuzz.named("full", rig_fuzz.EMU)
    imgs, ex = rig_fuzz.images(cc.case), rig_fuzz.extras(cc.case)
    got = crop_fuzz.run_and_check(oracle, cc, SEED)
    plain = fuzz_chain.compositor_run(cc.case, imgs, ex)
    assert got["num_bands"] == plain["num_bands"]
    assert np.array_equal(got["pano"], plain["pano"]) and np.array_equal(got["pmask"], plain["pmask"])


def test_from_cropper_matches_the_reference_cropper():
    """golden_crop.npz holds what the reference Cropper's crop_images / crop_rois return for random rect sets, LIRs and
    aspects (including products on .5, slices clipped at the bottom and right, and a zero-width overlap): Crop plus the
    library's numpy-slice clipping must give every slice, corner and size."""
    z = np.load(GOLDEN)
    for k in range(int(z["count"])):
        p = f"c{k}_"
        ns = types.SimpleNamespace(do_crop=True, overlapping_rectangles=[tuple(map(int, r)) for r in z[p + "overlaps"]],
                                   intersection_rectangles=[tuple(map(int, r)) for r in z[p + "inters"]])
        crop = Crop.from_cropper(ns, float(z[p + "aspect"]))
        assert [list(c) for c in crop.corners] == z[p + "corners"].tolist(), k
        assert [list(s) for s in crop.sizes] == z[p + "sizes"].tolist(), k
        warped = z[p + "warped_sizes"]   # (w, h) of each FINAL warped image
        cropped = z[p + "slices"]        # x, y, w, h of what crop_img returned, as found in the image
        for (x, y, w, h), (W, H), ref in zip(crop.rects, warped, cropped):
            got = (x, y, max(0, min(w, W - x)), max(0, min(h, H - y)))
            if ref[2] and ref[3]:
                assert got == tuple(ref), (k, got, tuple(ref))
            else:
                assert got[2] * got[3] == 0, (k, got)
    assert Crop.from_cropper(types.SimpleNamespace(do_crop=False), 2.0) is None


def test_empty_crop_is_refused(use_emu):
    """A zero-width overlap gets through the reference Cropper; its blenders then cannot feed the empty image (feed
    asserts for "no" and feather and does not return for multiband), so the compositor refuses it at creation."""
    cc = crop_fuzz.named("full", rig_fuzz.EMU)
    rects = list(cc.crop.rects)
    rects[1] = (rects[1][0], 0, 0, rects[1][3])
    with pytest.raises(StitchingError, match="image 1 is empty"):
        crop_fuzz.compositor(crop_fuzz.CropCase(cc.case, Crop(rects, cc.crop.corners, cc.crop.sizes), 1.0))
    rects = list(cc.crop.rects)
    rects[2] = (cc.case.rects[2][2], 0, 4, 4)  # starts at the right edge: numpy gives an empty slice
    with pytest.raises(StitchingError, match="image 2 is empty"):
        crop_fuzz.compositor(crop_fuzz.CropCase(cc.case, Crop(rects, cc.crop.corners, cc.crop.sizes), 1.0))


def test_bad_crops_are_refused(use_emu):
    cc = crop_fuzz.named("full", rig_fuzz.EMU)
    c = cc.crop
    with pytest.raises(StitchingError, match="rects for"):
        crop_fuzz.compositor(crop_fuzz.CropCase(cc.case, Crop(c.rects[1:], c.corners[1:], c.sizes[1:]), 1.0))
    rects = list(c.rects)
    rects[0] = (-1, 0, 5, 5)
    with pytest.raises(StitchingError, match="image 0 has a negative offset"):
        crop_fuzz.compositor(crop_fuzz.CropCase(cc.case, Crop(rects, c.corners, c.sizes), 1.0))
    sizes = list(c.sizes)
    sizes[1] = (sizes[1][0] - 1, sizes[1][1])
    with pytest.raises(StitchingError, match="more than its prepared size"):
        crop_fuzz.compositor(crop_fuzz.CropCase(cc.case, Crop(c.rects, c.corners, sizes), 1.0))


def _memmove(d, s, n):
    import ctypes

    ctypes.memmove(d, s, n)


def test_sharded_crop_equals_grouped_oracle(use_emu, oracle):
    """World 2 and 3: every rank's own cropped warped images and its strip of the panorama equal the grouped oracle
    (tests/shard_fuzz.py) fed with the cropped images, through the transport hooks."""
    cs = crop_fuzz.sharded_cases(SEED, 6, rig_fuzz.EMU)
    ran = set()
    for cc in cs:
        for world in (2, 3):
            if cc.n >= world and crop_fuzz.sharded_check(oracle, cc, world, _memmove, SEED):
                ran.add(world)
    assert ran == {2, 3}, f"worlds run: {sorted(ran)} of {len(cs)} cases"


def test_reference_stitcher_with_crop(use_emu):
    """The recorded run of the unmodified reference Stitcher with crop=True: the compositor built from its cameras,
    Cropper rectangles, LOW seam masks and gains returns the panorama Stitcher.stitch returned, bit for bit."""
    pytest.importorskip("cv2")
    got, ref = crop_fuzz.stitch_replay(GOLDEN)
    assert got == ref
