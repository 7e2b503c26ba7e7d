"""The default Stitcher at camera resolution without a GPU: the recorded crop=True runs of the reference
(tests/golden/golden_fullres_*.npz) against the rebuilt views, Crop.from_cropper and the CPU oracle stage by stage, and
small ratio draws through the emulation build."""
import pytest

import fullres

SEED = fullres.seed_from_env()
EMU_COUNT = 4


@pytest.mark.parametrize("name", fullres.RECORDS)
def test_rebuilt_views_are_the_recorded_inputs(name):
    """reference_cases.camera_views rebuilds, from the seed alone, the bytes the reference Stitcher was fed."""
    fullres.views(fullres.record(name))


@pytest.mark.parametrize("name", fullres.RECORDS)
def test_from_cropper_gives_the_prepared_rois(name):
    """Crop.from_cropper over the recorded Cropper rectangles at the recorded LOW -> FINAL ratio gives the corners and
    sizes the reference's Blender.prepare received, and slices of the recorded cropped shapes."""
    z = fullres.record(name)
    crop = fullres.crop(z)
    assert [list(c) for c in crop.corners] == z["corners"].tolist()
    assert [list(s) for s in crop.sizes] == z["sizes"].tolist()
    for i, ((x, y, w, h), d, dm) in enumerate(zip(crop.rects, z["cropped"], z["warped"])):
        H, W = fullres.shape_of(str(dm))[:2]
        assert fullres.shape_of(str(d)) == (max(0, min(h, H - y)), max(0, min(w, W - x)), 3), i


def test_oracle_pinned_at_camera_resolution(oracle):
    """Record A (4 x 12 MP, LOW -> FINAL about 11): the oracle's warp, numpy slice, gain_apply and seam_resize of every
    image equal the reference's stages bit for bit (the blend is left to the GPU tests)."""
    z = fullres.record("a")
    imgs = fullres.views(z)
    for i in range(int(z["n"])):
        fullres.oracle_stages(oracle, z, imgs, i)


def emu_set():
    return fullres.cases(SEED, EMU_COUNT, 100, 220, 40_000)


@pytest.mark.parametrize("k", range(EMU_COUNT))
def test_ratio_draws_against_oracle(use_emu, oracle, k):
    """The GPU file's ratio draws at reduced sizes: the same aspects, so LOW images of a few pixels stretched 5-22x."""
    fullres.run_and_check(oracle, emu_set()[k], SEED)
