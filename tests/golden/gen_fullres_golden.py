"""Writes tests/golden/golden_fullres_a.npz and golden_fullres_b*.npz: runs of the unmodified reference Stitcher
(OpenStitching/stitching) with crop=True, otherwise reference_cases.PIPELINE_SETTINGS, on camera-resolution views.  Only
these files are written; no other golden moves, and a second run writes the same bytes.

    python tests/golden/gen_fullres_golden.py <path to a checkout of the reference>

Record A: 4 views of 4000 x 3000 (12 MP, LOW -> FINAL about 11); record B: 3 views of 8000 x 6000 (48 MP, about 21.9).
The views are reference_cases.camera_views, rebuilt from the seed by the tests; the record holds their digests.

Per record: the cameras after wave correction, the warper scale, the MEDIUM / LOW -> FINAL ratios, the Cropper's
rectangles, the LOW seam masks, getMatGains(), the corners and sizes Blender.prepare receives, num_bands, the digest
of the panorama and, per image, the digest of every FINAL-resolution stage: the warped image and mask
(warp_final_resolution), the cropped image and mask (crop_final_resolution), the compensated image
(compensate_exposure_errors) and the blend mask (resize_seam_masks).  Each digest is taken as the stage hands its
result on, before the next stage can write into it (the compensator applies its gain in place).
"""
import os
import sys
import time
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# name -> (views, width, height, seed)
RECORDS = {"a": (4, 4000, 3000, 403), "b": (3, 8000, 6000, 402)}
STAGES = ("warped", "warped_mask", "cropped", "cropped_mask", "compensated", "blend_mask")


def record(name):
    import cv2 as cv

    import reference_cases as RC
    from gen_crop_golden import maximal_interior_rectangle
    from stitching import Stitcher
    from stitching.images import Images

    n, w, h, seed = RECORDS[name]
    sys.modules["largestinteriorrectangle"] = types.SimpleNamespace(lir=maximal_interior_rectangle)
    views = RC.camera_views(w, h, n, seed)
    st = Stitcher(**dict(RC.PIPELINE_SETTINGS, crop=True))
    seen = {s: [] for s in STAGES}

    def tap(gen, stage):
        for a in gen:
            seen[stage].append(RC.digest(a))
            yield a

    wave, seams, warp_final, crop_final = st.perform_wave_correction, st.find_seam_masks, st.warp_final_resolution, st.crop_final_resolution
    compensate, resize_seams, init = st.compensate_exposure_errors, st.resize_seam_masks, st.initialize_composition

    def keep_cameras(cameras):
        seen["cameras"] = wave(cameras)
        return seen["cameras"]

    def keep_seams(*a):
        seen["seams"] = [np.asarray(s.get() if hasattr(s, "get") else s) for s in seams(*a)]
        return seen["seams"]

    def keep_warp(imgs, cameras):
        imgs, masks, corners, sizes = warp_final(imgs, cameras)
        return tap(imgs, "warped"), tap(masks, "warped_mask"), corners, sizes

    def keep_crop(imgs, masks, corners, sizes):
        imgs, masks, corners, sizes = crop_final(imgs, masks, corners, sizes)
        return tap(imgs, "cropped"), tap(masks, "cropped_mask"), corners, sizes

    def keep_prepared(corners, sizes):
        seen["corners"], seen["sizes"] = [tuple(c) for c in corners], [tuple(s) for s in sizes]
        return init(corners, sizes)

    st.perform_wave_correction, st.find_seam_masks = keep_cameras, keep_seams
    st.warp_final_resolution, st.crop_final_resolution = keep_warp, keep_crop
    st.compensate_exposure_errors = lambda corners, imgs: tap(compensate(corners, imgs), "compensated")
    st.resize_seam_masks = lambda seam_masks: tap(resize_seams(seam_masks), "blend_mask")
    st.initialize_composition = keep_prepared
    t0 = time.time()
    pano = st.stitch(views)
    k = len(seen["seams"])
    assert k == n, f"record {name}: the Stitcher kept {k} of {n} views"
    assert all(len(seen[s]) == n for s in STAGES), {s: len(seen[s]) for s in STAGES}
    out = {"views": np.array([n, w, h, seed], np.int64),
           "inputs": np.array([RC.digest(v) for v in views]),
           "cameras": np.stack([RC.camera_value(c) for c in seen["cameras"]]),
           "scale": np.float64(st.warper.scale),
           "medium_to_final": np.float64(st.images.get_ratio(Images.Resolution.MEDIUM, Images.Resolution.FINAL)),
           "low_to_final": np.float64(st.images.get_ratio(Images.Resolution.LOW, Images.Resolution.FINAL)),
           "overlaps": np.array([tuple(r) for r in st.cropper.overlapping_rectangles], np.int64),
           "inters": np.array([tuple(r) for r in st.cropper.intersection_rectangles], np.int64),
           "corners": np.array(seen["corners"], np.int64),
           "sizes": np.array(seen["sizes"], np.int64),
           "num_bands": np.int64(st.blender.blender.numBands()),
           "pano": np.array(RC.digest(pano)),
           "n": np.int64(n)}
    for s in STAGES:
        out[s] = np.array(seen[s])
    for i, s in enumerate(seen["seams"]):
        out[f"seam{i}"] = s
    for i, g in enumerate(st.compensator.compensator.getMatGains()):
        out[f"gain{i}"] = np.asarray(g)
    print(f"record {name}: {n} x {w}x{h}, LOW -> FINAL {out['low_to_final']:.4f}, MEDIUM -> FINAL {out['medium_to_final']:.4f}, "
          f"pano {pano.shape}, num_bands {int(out['num_bands'])}, seams {[s.shape for s in seen['seams']]}, "
          f"gains {[np.asarray(g).shape for g in st.compensator.compensator.getMatGains()]}, {time.time() - t0:.0f} s")
    return out


def main(ref):
    sys.path.insert(0, ref)
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    import replay

    for name in RECORDS:
        replay.save(f"golden_fullres_{name}.npz", record(name))


if __name__ == "__main__":
    main(sys.argv[1])
