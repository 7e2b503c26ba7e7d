"""Writes tests/golden/golden_timelapse_stitcher_as_is.npz and golden_timelapse_stitcher_crop.npz: runs of the unmodified
reference Stitcher (OpenStitching/stitching) with timelapse="as_is" and "crop", crop=True and final_megapix=3, otherwise
reference_cases.PIPELINE_SETTINGS, on the 4 camera views of 4000 x 3000 of tests/golden/gen_fullres_golden.py's record
"a".  Only these files are written; no other golden moves, and a second run writes the same bytes.

    python tests/golden/gen_timelapse_stitcher_golden.py <path to a checkout of the reference>

A record holds what a gen_final_scale_golden.py record holds minus the blend (no panorama, no num_bands: the Stitcher
prepares no blender in timelapse mode) plus "frames", the digest of every frame the Timelapser produced.  The frames are
captured by wrapping Timelapser.process_and_save_frame (process_frame, then get_frame); no file is written.
"canvas_gap" is 1 when the canvas of "crop" is a gap rectangle: resultRoiIntersection of images that do not all
overlap, which cv::Rect(tl, br) returns as the positive-size gap between them.
"""
import os
import sys
import time
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# name -> (timelapse, final_megapix, views, width, height, seed): the views of gen_fullres_golden.py's record "a"
RECORDS = {"as_is": ("as_is", 3, 4, 4000, 3000, 403), "crop": ("crop", 3, 4, 4000, 3000, 403)}
STAGES = ("resized", "warped", "warped_mask", "cropped", "cropped_mask", "compensated", "blend_mask")


def canvas_gap(corners, sizes):
    return int(max(c[0] for c in corners) > min(c[0] + s[0] for c, s in zip(corners, sizes)) or
               max(c[1] for c in corners) > min(c[1] + s[1] for c, s in zip(corners, sizes)))


def record(name):
    import reference_cases as RC
    from gen_crop_golden import maximal_interior_rectangle
    from stitching import Stitcher
    from stitching.images import Images

    kind, megapix, n, w, h, seed = RECORDS[name]
    sys.modules["largestinteriorrectangle"] = types.SimpleNamespace(lir=maximal_interior_rectangle)
    views = RC.camera_views(w, h, n, seed)
    st = Stitcher(**dict(RC.PIPELINE_SETTINGS, crop=True, final_megapix=megapix, timelapse=kind))
    seen = {s: [] for s in STAGES}
    seen["frames"] = []

    def tap(gen, stage):
        for a in gen:
            seen[stage].append(RC.digest(a))
            yield a

    wave, seams, resize_final = st.perform_wave_correction, st.find_seam_masks, st.resize_final_resolution
    warp_final, crop_final = st.warp_final_resolution, st.crop_final_resolution
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

    def keep_frame(img_name, img, corner):
        # process_and_save_frame without the cv.imwrite (timelapser.py:38-39)
        st.timelapser.process_frame(img, corner)
        seen["frames"].append(RC.digest(st.timelapser.get_frame()))

    st.perform_wave_correction, st.find_seam_masks = keep_cameras, keep_seams
    st.resize_final_resolution = lambda: tap(resize_final(), "resized")
    st.warp_final_resolution, st.crop_final_resolution = keep_warp, keep_crop
    st.compensate_exposure_errors = lambda corners, imgs: tap(compensate(corners, imgs), "compensated")
    st.resize_seam_masks = lambda seam_masks: tap(resize_seams(seam_masks), "blend_mask")
    st.initialize_composition = keep_prepared
    st.timelapser.process_and_save_frame = keep_frame
    t0 = time.time()
    assert st.stitch(views) is None  # create_final_panorama blends nothing in timelapse mode
    k = len(seen["seams"])
    assert k == n, f"record {name}: the Stitcher kept {k} of {n} views"
    assert all(len(seen[s]) == n for s in STAGES + ("frames",)), {s: len(seen[s]) for s in STAGES + ("frames",)}
    out = {"views": np.array([n, w, h, seed], np.int64),
           "timelapse": np.array(kind),
           "final_megapix": np.float64(megapix),
           "final_sizes": np.array(st.images.get_scaled_img_sizes(Images.Resolution.FINAL), np.int64),
           "inputs": np.array([RC.digest(v) for v in views]),
           "cameras": np.stack([RC.camera_value(c) for c in seen["cameras"]]),
           "scale": np.float64(st.warper.scale),
           "medium_to_final": np.float64(st.images.get_ratio(Images.Resolution.MEDIUM, Images.Resolution.FINAL)),
           "low_to_final": np.float64(st.images.get_ratio(Images.Resolution.LOW, Images.Resolution.FINAL)),
           "overlaps": np.array([tuple(r) for r in st.cropper.overlapping_rectangles], np.int64),
           "inters": np.array([tuple(r) for r in st.cropper.intersection_rectangles], np.int64),
           "corners": np.array(seen["corners"], np.int64),
           "sizes": np.array(seen["sizes"], np.int64),
           "canvas_gap": np.int64(canvas_gap(seen["corners"], seen["sizes"]) if kind == "crop" else 0),
           "frames": np.array(seen["frames"]),
           "n": np.int64(n)}
    for s in STAGES:
        out[s] = np.array(seen[s])
    for i, s in enumerate(seen["seams"]):
        out[f"seam{i}"] = s
    for i, g in enumerate(st.compensator.compensator.getMatGains()):
        out[f"gain{i}"] = np.asarray(g)
    print(f"record {name}: {n} x {w}x{h} -> FINAL {out['final_sizes'].tolist()}, timelapse {kind}, frames "
          f"{[str(d).split(' ')[0] for d in seen['frames']]}, canvas_gap {int(out['canvas_gap'])}, {time.time() - t0:.0f} s")
    return out


def main(ref):
    sys.path.insert(0, ref)
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    import replay

    for name in RECORDS:
        replay.save(f"golden_timelapse_stitcher_{name}.npz", record(name))


if __name__ == "__main__":
    main(sys.argv[1])
