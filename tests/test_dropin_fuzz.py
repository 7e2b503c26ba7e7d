"""The drop-in classes (what install() puts under the reference Stitcher) on seeded random rigs and crops in the emulation
build, bit for bit against the oracle (tests/dropin_fuzz.py); the blend strength in double in the compositor; the warp's
refusal of sides cv::remap refuses; and the device-mask form of sb_blender_feed_dev."""
import ctypes as C

import numpy as np
import pytest

import dropin_fuzz
import fuzz_chain
import rig_fuzz
from stitching_b200 import Compositor, StitchingError, _lib, rigs

SEED = dropin_fuzz.seed_from_env()


@pytest.mark.parametrize("k", range(len(dropin_fuzz.EMU_RIG) + dropin_fuzz.EMU_CROP + dropin_fuzz.EMU_OWN))
def test_dropin_fuzz_against_oracle(use_emu, oracle, monkeypatch, k):
    """Warp, crop, compensate, resize the seam mask, blend (and the timelapse frames) through the drop-ins, fed as device
    twins, host copies, int16 or a mix: every intermediate and the panorama equal the oracle's."""
    dc = dropin_fuzz.emu_set(SEED)[k]
    for key, v in dc.env.items():
        monkeypatch.setenv(key, v)
    dropin_fuzz.run_and_check(oracle, dc, SEED)


def test_dropin_fuzz_coverage(oracle):
    cs = dropin_fuzz.emu_set(SEED)
    rows = [(c, dropin_fuzz.emu_coverage(c, oracle)) for c in cs]
    print(f"\ndrop-in fuzz coverage, emulation set (seed {SEED}, {len(cs)} cases):\n" + rig_fuzz.coverage_table(rows))
    reached = set().union(*(t for _, t in rows))
    assert dropin_fuzz.WANT <= reached, f"not reached: {sorted(dropin_fuzz.WANT - reached)}"
    own = [c for c in cs if c.name.startswith("own_")]
    assert rig_fuzz.redraw_share([c.case for c in own]) < 0.5


# -- the blend strength in double -----------------------------------------------------------------------------------------
def _compositor_vs_oracle(oracle, case):
    imgs, ex = rig_fuzz.images(case), rig_fuzz.extras(case)
    ref = rig_fuzz.oracle_run(oracle, case, imgs, ex)
    got = fuzz_chain.compositor_run(case, imgs, ex)
    rig_fuzz.check(case, got, ref, "strength")


def test_strength_that_float32_rounds(use_emu, oracle):
    """A feather rig at strength 2.9: in float32 the blend width, hence the sharpness, moves and one panorama value
    differs from the reference's."""
    case = list(rig_fuzz.cases(7, 3, rig_fuzz.EMU))[2]
    assert (case.wtype, case.n, case.blender) == ("cylindrical", 4, "feather")
    case.strength = 2.9
    _compositor_vs_oracle(oracle, case)


def test_strength_sweep_not_float32_exact(use_emu, oracle):
    """Feather and multiband rigs at strengths float32 cannot hold, through the compositor against the oracle."""
    picked = [c for c in rig_fuzz.cases(7, 40, rig_fuzz.EMU) if c.blender in ("feather", "multiband") and c.n <= 4][:8]
    assert len(picked) == 8
    for k, case in enumerate(picked):
        for s in (0.3, 2.9, 5.3, 7.7, 13.1)[k % 2::2]:
            case.strength = s
            _compositor_vs_oracle(oracle, case)


def test_num_bands_at_a_strength_float32_rounds(use_emu, oracle):
    """A 68x64 pano at strength 388.057: 6 bands in double (the reference), 7 in float32."""
    cams = [rigs.Camera(1, 1, 0, 0, np.eye(3, dtype=np.float32))]
    c = Compositor(cams, [(68, 64)], "affine", "multiband", 388.057)
    try:
        assert tuple(c.roi) == (0, 0, 68, 64)
        b = oracle.Blender("multiband", 388.057)
        b.prepare([(0, 0)], [(68, 64)])
        assert c.num_bands == b.num_bands == 6
        pano, mask = c.composite([rigs.noise_image(64, 68, 5)])
        bo = oracle.Blender("multiband", 388.057)
        bo.prepare([(0, 0)], [(68, 64)])
        _, wi, wm = oracle.warp("affine", 1.0, np.eye(3, dtype=np.float32), np.eye(3, dtype=np.float32), rigs.noise_image(64, 68, 5))
        bo.feed(wi, wm, (0, 0))
        ref = bo.blend()
        assert np.array_equal(pano, ref[0]) and np.array_equal(mask, ref[1])
    finally:
        c.close()


# -- sides of 32767 px and more: cv::remap asserts -------------------------------------------------------------------------
def _affine(sx=1.0, sy=1.0):
    return rigs.Camera(1, 1, 0, 0, np.array([[sx, 0, 0], [0, sy, 0], [0, 0, 1]], np.float32))


def _warper():
    from stitching_b200 import Warper

    w = Warper("affine")
    w.set_scale([_affine()])
    return w


def test_warp_of_sides_below_32767_matches_the_oracle(use_emu, oracle):
    w = _warper()
    for size in ((32766, 2), (2, 32766)):
        img = rigs.noise_image(size[1], size[0], 3)
        wi, wm = w.warp_image(img, _affine()), w.create_and_warp_mask(size, _affine())
        rect, ri, rm = oracle.warp("affine", 1.0, np.eye(3, dtype=np.float32), _affine().R, img)
        assert w.warp_roi(size, _affine()) == rect and wi.shape[:2] == (size[1], size[0])
        assert np.array_equal(wi, ri) and np.array_equal(wm, rm)


@pytest.mark.parametrize("what", ["source width", "source height", "result width", "result height"])
def test_warp_refuses_sides_of_32767(use_emu, what):
    """What cv.PyRotationWarper.warp raises on (remap asserts every side below SHRT_MAX): the image and the mask warp
    refuse it with an error catchable as cv2.error; warp_roi (warpRoi does not assert) still answers."""
    size, cam = {"source width": ((32767, 2), _affine()), "source height": ((2, 32767), _affine()),
                 "result width": ((16384, 2), _affine(sx=2)), "result height": ((2, 16384), _affine(sy=2))}[what]
    w = _warper()
    rect = w.warp_roi(size, cam)
    assert max(rect[2], rect[3]) == 32767 or max(size) == 32767
    try:
        import cv2

        errors = (StitchingError, cv2.error)
    except ImportError:
        errors = (StitchingError,)
    for err in errors:
        with pytest.raises(err, match="32767"):
            w.warp_image(np.zeros((size[1], size[0], 3), np.uint8), cam)
        with pytest.raises(err, match="32767"):
            w.create_and_warp_mask(size, cam)


def test_compositor_refuses_sides_of_32767(use_emu):
    cams = [_affine(), _affine(sx=2)]
    with pytest.raises(StitchingError, match="image 1"):
        Compositor(cams, [(40, 30), (16384, 2)], "affine", "multiband", 5)
    with pytest.raises(StitchingError, match="image 0"):
        Compositor(cams[:1], [(2, 32767)], "affine", "no", 5)
    Compositor(cams, [(40, 30), (16383, 2)], "affine", "multiband", 5).close()


# -- sb_blender_feed_dev with the mask from a device twin -------------------------------------------------------------------
def test_feed_dev_with_a_mask_twin_equals_the_host_mask(use_emu):
    """sb_warp_keep keeps the image and the mask; feeding both twins (at a crop offset) gives the blend of the host
    mask feed, for the byte and the multiband layouts alike."""
    L = _lib.lib()
    fp = lambda a: a.ctypes.data_as(_lib.c_float_p)  # noqa: E731
    cfg = rigs.config("cfg2", 25)
    cams = cfg["cameras"][2:5]
    scale = np.float32(cams[0].focal)
    from stitching_b200 import Warper

    keep = []
    try:
        twins = []
        for i, cam in enumerate(cams):
            img = rigs.noise_image(cfg["h"], cfg["w"], 40 + i)
            K = np.ascontiguousarray(Warper.get_K(cam))
            rect = (C.c_int * 4)()
            assert L.sb_warp_roi(0, scale, fp(K), fp(cam.R), cfg["w"], cfg["h"], rect) == 0
            w, h = rect[2], rect[3]
            wi, wm = np.empty((h, w, 3), np.uint8), np.empty((h, w), np.uint8)
            ki, km = C.c_void_p(), C.c_void_p()
            _lib.check(L.sb_warp_keep(0, scale, fp(K), fp(cam.R), img.ctypes.data_as(C.c_void_p), cfg["w"], cfg["h"], cfg["w"] * 3,
                                      wi.ctypes.data_as(C.c_void_p), w * 3, wm.ctypes.data_as(C.c_void_p), w, rect,
                                      C.byref(ki), C.byref(km)), "sb_warp_keep")
            keep += [ki.value, km.value]
            twins.append((tuple(rect), wi, wm, ki.value, km.value))
        x0, y0 = 3, 2  # the crop: the rectangle (x0, y0) .. (w - 4, h - 1) of every warped image
        corners = [(r[0] + x0, r[1] + y0) for r, *_ in twins]
        sizes = [(r[2] - x0 - 4, r[3] - y0 - 1) for r, *_ in twins]
        roi = (min(c[0] for c in corners), min(c[1] for c in corners),
               max(c[0] + s[0] for c, s in zip(corners, sizes)) - min(c[0] for c in corners),
               max(c[1] + s[1] for c, s in zip(corners, sizes)) - min(c[1] for c in corners))
        for kind, nb in ((2, 3), (1, 0), (0, 0)):
            res = []
            for from_twin in (True, False):
                b = L.sb_blender_create(kind, nb, C.c_float(0.02))
                try:
                    _lib.check(L.sb_blender_prepare(b, *roi), "sb_blender_prepare")
                    for (r, wi, wm, ki, km), c, (w, h) in zip(twins, corners, sizes):
                        m = np.ascontiguousarray(wm[y0:y0 + h, x0:x0 + w])
                        _lib.check(L.sb_blender_feed_dev(b, ki, x0, y0, km if from_twin else None, x0, y0,
                                                         None if from_twin else m.ctypes.data_as(C.c_void_p), w, w, h, c[0], c[1]),
                                   "sb_blender_feed_dev")
                    pano, mask = np.empty((roi[3], roi[2], 3), np.uint8), np.empty((roi[3], roi[2]), np.uint8)
                    _lib.check(L.sb_blender_blend(b, pano.ctypes.data_as(C.c_void_p), roi[2] * 3, mask.ctypes.data_as(C.c_void_p),
                                                  roi[2], None, 0), "sb_blender_blend")
                    res.append((pano, mask))
                finally:
                    L.sb_blender_destroy(b)
            assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1]), f"kind {kind}"
            assert res[0][1].any()
    finally:
        for p in keep:
            L.sb_devimg_release(p)
