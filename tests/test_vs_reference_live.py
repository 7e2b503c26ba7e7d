"""The oracle and the drop-in classes against the UNMODIFIED reference classes on seeded random cases.

The committed goldens (tests/golden/*.npz) were written by the reference once; this file adds a wider pin on random inputs
(tests/reference_cases.py, what the reference returned for them in tests/golden/golden_reference.npz):
every projection of Warper.WARP_TYPE_CHOICES (roi, warped image, warped mask), the three blenders with gray and binary masks,
the Timelapser, the FINAL-resolution steps, and the product's own classes side by side with the reference's.
"""
import numpy as np
import pytest

import reference_cases as rc
from stitching_b200 import Warper


@pytest.fixture(scope="module")
def pins():
    return rc.Pins()


def test_every_projection_against_the_reference_warper(pins, oracle):
    checked = 0
    for key, wtype, cam, scale, aspect, img in rc.warp_cases():
        K = Warper.get_K(cam, aspect)
        size = (img.shape[1], img.shape[0])
        roi = tuple(int(v) for v in pins.value(key + ".roi"))
        got_roi = oracle.warp_roi(wtype, scale * aspect, K, cam.R, size)
        assert tuple(got_roi) == roi, (key, got_roi, roi)
        if roi[2] * roi[3] > 4_000_000:
            continue  # a degenerate draw (horizon in view): the rect is exact, the pixels would take minutes
        rect, gimg, gmask = oracle.warp(wtype, scale * aspect, K, cam.R, img)
        pins.array(key + ".img", gimg, f"{key}: warped image")
        pins.array(key + ".mask", gmask, f"{key}: warped mask")
        checked += 1
    assert checked >= 40


def test_blenders_and_timelapser_against_the_reference(pins, oracle):
    for trial, kind, strength, corners, sizes, imgs, masks in rc.blend_cases():
        b = oracle.Blender(kind, strength)
        b.prepare(corners, sizes)
        for img, m, c in zip(imgs, masks, corners):
            b.feed(img, m, c)
        pb, mb = b.blend()
        pins.array(f"blend.{trial}.pano", np.asarray(pb), f"{kind} strength {strength}: panorama")
        pins.array(f"blend.{trial}.mask", np.asarray(mb), f"{kind} strength {strength}: mask")
        for tl_kind in ("as_is", "crop"):
            tb = oracle.Timelapser(tl_kind)
            tb.initialize(corners, sizes)
            for i, (img, c) in enumerate(zip(imgs, corners)):
                tb.process_frame(img, c)
                key = f"timelapse.{trial}.{tl_kind}.{i}"
                if tb.roi[2] == 0 or tb.roi[3] == 0:  # rects that touch in a line: the reference's get_frame raises on the empty canvas
                    assert str(pins.value(key)) == "raises cv2.error", key
                    continue
                pins.array(key, tb.get_frame(), f"timelapse {tl_kind}")


def test_final_resolution_steps_against_the_reference(pins, oracle):
    """SeamFinder.resize (seam_finder.py:38-43) and Images.resize_img_by_scaler (images.py:120-123) on random shapes;
    ExposureErrorCompensator.apply (exposure_error_compensator.py:43-45) with gains the reference's own feed() estimated."""
    for case in rc.final_resolution_cases():
        if case[0] == "seam":
            _, t, seam, mask = case
            pins.array(f"seam.{t}", oracle.seam_resize(seam, mask), f"SeamFinder.resize {seam.shape} -> {mask.shape}")
        elif case[0] == "resize":
            _, t, img, size = case
            pins.array(f"resize.{t}", oracle.resize_linear_exact(img, size), f"Images.resize {img.shape} -> {size}")
        else:
            _, kind, corners, imgs, masks = case
            for i in range(len(imgs)):
                if kind == "no":
                    pins.array(f"gain.no.{i}", imgs[i], "compensator no: identity")
                    continue
                gain = pins.value(f"gain.{kind}.{i}.gains")
                pins.array(f"gain.{kind}.{i}", oracle.gain_apply(imgs[i], gain), f"compensator {kind} image {i}")


def test_drop_in_classes_against_the_reference_classes(pins, use_emu):
    """The product's own classes (their kernels through tests/emu) against the reference's, same calls, same inputs:
    Warper (set_scale, warp_rois, warp_images, create_and_warp_masks) -> Blender (prepare, feed, blend) for random rigs of every
    blender type and a handful of projections, and Timelapser frames of the same warped images."""
    import stitching_b200

    for trial, wtype, btype, cams, imgs in rc.dropin_cases():
        key = f"dropin.{trial}"
        sizes = [(img.shape[1], img.shape[0]) for img in imgs]
        w = stitching_b200.Warper(wtype)
        w.set_scale(cams)
        warped = list(w.warp_images(imgs, cams))
        masks = list(w.create_and_warp_masks(sizes, cams))
        corners, wsizes = w.warp_rois(sizes, cams)
        b = stitching_b200.Blender(btype, 5)
        b.prepare(corners, wsizes)
        for img, m, c in zip(warped, masks, corners):
            b.feed(img, m, c)
        pano, pmask = b.blend()
        t = stitching_b200.Timelapser("as_is")
        t.initialize(corners, wsizes)
        t.process_frame(warped[1], corners[1])
        got = [[tuple(int(v) for v in c) for c in corners], [tuple(int(v) for v in s) for s in wsizes]]
        want = [[tuple(int(v) for v in c) for c in pins.value(key + ".corners")], [tuple(int(v) for v in s) for s in pins.value(key + ".sizes")]]
        assert got == want, (wtype, got, want)
        for i in range(len(imgs)):
            pins.array(f"{key}.warped.{i}", warped[i], f"{wtype}: warped image {i}")
            pins.array(f"{key}.mask.{i}", masks[i], f"{wtype}: warped mask {i}")
        pins.array(key + ".pano", pano, f"{wtype} + {btype}: panorama")
        pins.array(key + ".pmask", pmask, f"{wtype} + {btype}: panorama mask")
        pins.array(key + ".frame", t.get_frame(), f"{wtype}: timelapse frame")
