"""Writes tests/golden/golden_crop.npz: what the reference Cropper (OpenStitching/stitching, cropper.py) returns for
random LOW-resolution rect sets, LIRs and LOW -> FINAL aspects.  Only this file is written; no other golden moves.

    python tests/golden/gen_crop_golden.py <path to a checkout of the reference>

Per case: the overlap and intersection rectangles (LOW pixels) that Cropper.prepare derives from the rects and the LIR,
the aspect, the FINAL warped sizes, and what crop_images returns for FINAL warped images of those sizes (the slice origin,
read back from pixel values, and its shape) and what crop_rois returns.  The cases include aspects whose products end
in .5, slices clipped at the bottom and right, and a zero-width overlap (which get_overlap lets through).
"""
import os
import sys

import numpy as np


def main(ref):
    sys.path.insert(0, ref)
    from stitching.cropper import Cropper, Rectangle

    rng = np.random.default_rng(20261015)
    aspects = [1.0, 1.5, 2.5, 0.5, 3.0, 1.25, 2.0, 0.75]
    out = {}
    k = 0
    while k < 60:
        n = int(rng.integers(1, 7))
        aspect = aspects[k % len(aspects)] if k < 40 else float(rng.uniform(0.4, 3.5))
        corners = [(int(rng.integers(-50, 50)), int(rng.integers(-30, 30))) for _ in range(n)]
        sizes = [(int(rng.integers(1, 60)), int(rng.integers(1, 40))) for _ in range(n)]
        zc = Cropper.get_zero_center_corners(corners)
        rects = Cropper.get_rectangles(zc, sizes)
        W = max(r.x2 for r in rects)
        H = max(r.y2 for r in rects)
        if k == 0:  # a zero-width overlap: the LIR starts where image 0 ends
            lir = Rectangle(rects[0].x2, 0, max(1, W - rects[0].x2), H)
        else:
            lx, ly = int(rng.integers(0, max(1, W // 3))), int(rng.integers(0, max(1, H // 3)))
            lir = Rectangle(lx, ly, max(1, int(rng.integers((W - lx) // 2, W - lx + 1))), max(1, int(rng.integers((H - ly) // 2, H - ly + 1))))
        try:
            overlaps = Cropper.get_overlaps(rects, lir)
        except Exception:
            continue
        cr = Cropper(True)
        cr.overlapping_rectangles = overlaps
        cr.intersection_rectangles = Cropper.get_intersections(rects, overlaps)
        # FINAL warped images: the LOW sizes scaled, sometimes a pixel short, so that the scaled slice is clipped
        warped = [(max(1, int(round(w * aspect)) - int(rng.integers(0, 2))), max(1, int(round(h * aspect)) - int(rng.integers(0, 2))))
                  for w, h in sizes]
        imgs = [np.arange(h * w, dtype=np.int64).reshape(h, w) for w, h in warped]
        slices = []
        for img, (w, h) in zip(cr.crop_images(imgs, aspect), warped):
            if img.size:
                v = int(img[0, 0])
                slices.append((v % w, v // w, img.shape[1], img.shape[0]))
            else:
                slices.append((0, 0, img.shape[1], img.shape[0]))
        final_corners = [(int(round(x * aspect)), int(round(y * aspect))) for x, y in corners]
        cc, cs = cr.crop_rois(final_corners, warped, aspect)
        p = f"c{k}_"
        out[p + "overlaps"] = np.array([tuple(r) for r in overlaps], np.int64)
        out[p + "inters"] = np.array([tuple(r) for r in cr.intersection_rectangles], np.int64)
        out[p + "aspect"] = np.float64(aspect)
        out[p + "warped_sizes"] = np.array(warped, np.int64)
        out[p + "slices"] = np.array(slices, np.int64)
        out[p + "corners"] = np.array(cc, np.int64)
        out[p + "sizes"] = np.array(cs, np.int64)
        k += 1
    out["count"] = np.int64(k)
    out.update(record_stitch())
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_crop.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {k} cases")


def maximal_interior_rectangle(mask, contour=None):
    """(x, y, w, h) of a largest axis-parallel rectangle of True pixels (histogram stack per row).  It stands in for the
    `largestinteriorrectangle` package, which is not installed here: the rectangle only decides which rectangles the
    reference's own Cropper derives, and those are recorded."""
    h, w = mask.shape
    heights = np.zeros(w + 1, np.int64)
    best = (0, 0, 0, 0)
    for y in range(h):
        heights[:w] = np.where(mask[y], heights[:w] + 1, 0)
        stack = []
        for x in range(w + 1):
            start = x
            while stack and stack[-1][1] >= heights[x]:
                start, hh = stack.pop()
                if hh * (x - start) > best[2] * best[3]:
                    best = (start, y - hh + 1, x - start, hh)
            stack.append((start, heights[x]))
    return np.array(best)


def record_stitch():
    """One run of the unmodified reference Stitcher with crop=True on reference_cases.synthetic_views (otherwise
    PIPELINE_SETTINGS): cameras, warper scale, the MEDIUM -> FINAL and LOW -> FINAL ratios, the Cropper's rectangles, the
    LOW seam masks, getMatGains(), the digest of the FINAL inputs and of the panorama."""
    import types

    import cv2 as cv

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
    import reference_cases as RC
    from stitching import Stitcher
    from stitching.images import Images

    sys.modules["largestinteriorrectangle"] = types.SimpleNamespace(lir=maximal_interior_rectangle)
    views = RC.synthetic_views(cv)
    st = Stitcher(**dict(RC.PIPELINE_SETTINGS, crop=True))
    seen = {}
    wave, seams = st.perform_wave_correction, st.find_seam_masks

    def keep_cameras(cameras):
        seen["cameras"] = wave(cameras)
        return seen["cameras"]

    def keep_seams(*a):
        seen["seams"] = [np.asarray(s.get() if hasattr(s, "get") else s) for s in seams(*a)]
        return seen["seams"]

    st.perform_wave_correction, st.find_seam_masks = keep_cameras, keep_seams
    pano = st.stitch(views)
    out = {"stitch_cameras": np.stack([RC.camera_value(c) for c in seen["cameras"]]),
           "stitch_scale": np.float64(st.warper.scale),
           "stitch_medium_to_final": np.float64(st.images.get_ratio(Images.Resolution.MEDIUM, Images.Resolution.FINAL)),
           "stitch_low_to_final": np.float64(st.images.get_ratio(Images.Resolution.LOW, Images.Resolution.FINAL)),
           "stitch_overlaps": np.array([tuple(r) for r in st.cropper.overlapping_rectangles], np.int64),
           "stitch_inters": np.array([tuple(r) for r in st.cropper.intersection_rectangles], np.int64),
           "stitch_inputs": np.array([RC.digest(v) for v in views]),
           "stitch_pano": np.array(RC.digest(pano))}
    for i, s in enumerate(seen["seams"]):
        out[f"stitch_seam{i}"] = s
    for i, g in enumerate(st.compensator.compensator.getMatGains()):
        out[f"stitch_gain{i}"] = np.asarray(g)
    out["stitch_n"] = np.int64(len(seen["seams"]))
    print(f"stitch: pano {pano.shape}, overlaps {out['stitch_overlaps'].tolist()}, low->final {out['stitch_low_to_final']}")
    return out


if __name__ == "__main__":
    main(sys.argv[1])
