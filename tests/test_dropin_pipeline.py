"""Drop-in check against the real reference pipeline.

The reference's stitching.Stitcher (crop=False) ran unmodified on synthetic views of a textured plane
(tests/reference_cases.py: synthetic_views, synthetic_scans) -- stitch, stitch_verbose, two other warper types, a
timelapse run, one Stitcher for two image sets and AffineStitcher -- and every call that crossed the hot-path boundary
at the bindings stitching_b200.install() replaces (Warper, Images.resize_img_by_scaler, ExposureErrorCompensator.apply,
SeamFinder.resize, Blender, Timelapser) was RECORDED (tests/golden/gen_golden.py: record_pipeline): the exact
cv.detail.CameraParams, numpy-float aspect, cv.UMat blend masks and corner tuples it handed over, and digests of what cv2
returned.  The reference's registration is not deterministic from run to run (RANSAC), so the record, not a fresh run, is
the pin.  Here each record is REPLAYED through the product's classes (on the emulation build, tests/emu), every call fed
with what the replay itself produced before it: every resized and warped image, mask, roi, compensated image, resized seam
mask, timelapse frame and panorama must be identical.
"""
import importlib
import sys

import numpy as np
import pytest

import reference_cases as rc


def replay(cv, name, sources):
    """Replay the recorded run `name` through the product's classes; returns the kinds of the calls, the panoramas and the
    timelapse frames it produced."""
    import stitching_b200

    pins = rc.Pins()
    log = []
    for k in range(int(pins.value(f"pipe.{name}.n"))):
        prefix = f"pipe.{name}.{k}."
        log.append({key[len(prefix):]: v for key, v in pins.data.items() if key.startswith(prefix)})
    # what the replay has produced so far (and the inputs it started from), by digest: the next call's inputs
    made = {rc.digest(v): v for v in sources}

    def produced(e, key, k):
        if key + "_value" in e:  # made by the reference's own code outside the boundary, stored as it was
            v = e[key + "_value"]
            return cv.UMat(v) if key == "mask" and str(e["mask_type"]) == "UMat" else v
        d = str(e[key])
        assert d in made, f"{name} call {k}: input {d} is nothing the replay produced"
        return made[d]

    def check(e, got, what):
        d = rc.digest(got)
        assert d == str(e["out"]), f"{name} {what}: got {d}, the reference {e['out']}"
        made[d] = got

    blender = timelapser = None
    panos, frames, kinds = [], [], []
    for k, e in enumerate(log):
        kind = str(e["kind"])
        kinds.append(kind)
        if kind in ("warp_image", "warp_mask", "warp_roi"):
            w = stitching_b200.Warper(str(e["type"]))
            w.scale = float(e["scale"])
            cam, aspect = rc.camera_from_value(cv, e["camera"]), np.float64(e["aspect"])
            if kind == "warp_image":
                check(e, w.warp_image(produced(e, "input", k), cam, aspect), f"call {k} warp_image")
            elif kind == "warp_mask":
                check(e, w.create_and_warp_mask(tuple(int(v) for v in e["size"]), cam, aspect), f"call {k} create_and_warp_mask")
            else:
                assert tuple(w.warp_roi(tuple(int(v) for v in e["size"]), cam, aspect)) == tuple(int(v) for v in e["roi"]), f"{name} call {k} warp_roi"
        elif kind == "img_resize":  # images.py:120-123: the MEDIUM / LOW / FINAL resolution inputs
            check(e, stitching_b200.images.resize_exact(produced(e, "input", k), tuple(int(v) for v in e["size"])), f"call {k} Images.resize")
        elif kind == "gain_apply":  # with the gains the reference compensator's own feed() estimated ("no": none, identity)
            check(e, stitching_b200.exposure_error_compensator.apply_gain(produced(e, "input", k).copy(), e.get("gain")),
                  f"call {k} ExposureErrorCompensator.apply")
        elif kind == "seam_resize":  # the LOW-resolution seam mask arrives as cv.UMat, the warped mask as ndarray
            seam = cv.UMat(e["seam"]) if str(e["seam_type"]) == "UMat" else e["seam"]
            got = stitching_b200.seam_finder.resize(seam, produced(e, "mask", k))
            # same container type as the reference's cv2 chain (cv.UMat in the pipeline): seam_finder.py:47 and
            # verbose.py:149-156 call cv.UMat.get on it
            assert type(got).__name__ == str(e["out_type"]), f"SeamFinder.resize returned {type(got).__name__}, the reference {e['out_type']}"
            check(e, got, f"call {k} SeamFinder.resize")
        elif kind == "prepare":
            blender = stitching_b200.Blender(str(e["type"]), float(e["strength"]))
            blender.prepare([tuple(int(v) for v in c) for c in e["corners"]], [tuple(int(v) for v in s) for s in e["sizes"]])
        elif kind == "feed":
            mask = produced(e, "mask", k)
            assert type(mask).__name__ == str(e["mask_type"]), f"{name} call {k}: feed mask {type(mask).__name__}, the reference {e['mask_type']}"
            blender.feed(produced(e, "input", k), mask, tuple(int(v) for v in e["corner"]))
        elif kind == "blend":
            pano, mask = blender.blend()
            assert rc.digest(mask) == str(e["mask"]), f"{name} call {k}: panorama mask"
            assert rc.digest(pano) == str(e["pano"]), f"{name} call {k} panorama: {rc.digest(pano)}, the reference {e['pano']}"
            panos.append(pano)
        elif kind == "tl_init":
            timelapser = stitching_b200.Timelapser(str(e["type"]))
            timelapser.initialize([tuple(int(v) for v in c) for c in e["corners"]], [tuple(int(v) for v in s) for s in e["sizes"]])
        elif kind == "tl_frame":
            timelapser.process_frame(produced(e, "input", k), tuple(int(v) for v in e["corner"]))
            frame = timelapser.get_frame()
            check(e, frame, f"call {k} Timelapser frame")
            frames.append(frame)
        else:
            raise AssertionError(f"{name} call {k}: unknown kind {kind}")
    return kinds, panos, frames


@pytest.fixture()
def cv(use_emu):
    return pytest.importorskip("cv2")


def test_recorded_boundary_calls_replay_identically(cv):
    kinds, panos, _ = replay(cv, "stitch", rc.synthetic_views(cv))
    assert kinds.count("warp_image") >= 6 and kinds.count("feed") == 3 and kinds.count("blend") == 1
    assert kinds.count("seam_resize") == 3, "stitcher.py:223-225 resizes one seam mask per image"
    assert kinds.count("img_resize") >= 6, "images.py:120-123 resamples every image to the working resolutions"
    assert kinds.count("gain_apply") == 3, "stitcher.py:219-221 compensates every image"
    pins = rc.Pins()
    applied = [k for k, kind in enumerate(kinds) if kind == "gain_apply"]
    assert any(str(pins.value(f"pipe.stitch.{k}.input")) != str(pins.value(f"pipe.stitch.{k}.out")) for k in applied), "compensation changed nothing"
    assert any(str(pins.value(f"pipe.stitch.{k}.mask_type")) == "UMat" for k, kind in enumerate(kinds) if kind == "feed"), \
        "the pipeline hands cv.UMat masks to feed"


def _stand_in_package(tmp_path):
    """A package laid out like the reference (module names and the names each module binds), to see what install() patches."""
    pkg = tmp_path / "stitching_layout"
    pkg.mkdir()
    files = {
        "__init__.py": "",
        "warper.py": "class Warper:\n    pass\n",
        "blender.py": "class Blender:\n    pass\n",
        "timelapser.py": "class Timelapser:\n    pass\n",
        "images.py": "class Images:\n    @staticmethod\n    def resize_img_by_scaler(scaler, size, img):\n        return img\n",
        "exposure_error_compensator.py": "class ExposureErrorCompensator:\n    def apply(self, *args):\n        return args[2]\n",
        "seam_finder.py": "from .blender import Blender\n\nclass SeamFinder:\n    @staticmethod\n    def resize(seam_mask, mask):\n        return mask\n",
        "stitcher.py": "from .warper import Warper\nfrom .blender import Blender\nfrom .timelapser import Timelapser\n",
        "cropper.py": "from .blender import Blender\n",
        "verbose.py": "from .warper import Warper\nfrom .blender import Blender\nfrom .timelapser import Timelapser\n",
    }
    for name, text in files.items():
        (pkg / name).write_text(text)
    sys.path.insert(0, str(tmp_path))
    try:
        return importlib.import_module("stitching_layout")
    finally:
        sys.path.remove(str(tmp_path))


def test_stitcher_runs_end_to_end_on_the_swapped_classes(cv, tmp_path):
    """install() rebinds every name the reference's modules import, and the recorded Stitcher.stitch runs end to end on
    the swapped classes with the reference's panorama as result."""
    import stitching_b200

    pkg = _stand_in_package(tmp_path)
    assert stitching_b200.install(pkg) is pkg and stitching_b200.install(pkg) is pkg
    for mod, names in (("warper", ("Warper",)), ("blender", ("Blender",)), ("timelapser", ("Timelapser",)),
                       ("stitcher", ("Warper", "Blender", "Timelapser")), ("cropper", ("Blender",)), ("seam_finder", ("Blender",)),
                       ("verbose", ("Warper", "Blender", "Timelapser"))):
        m = importlib.import_module(f"stitching_layout.{mod}")
        for name in names:
            assert getattr(m, name) is getattr(stitching_b200, name), f"{mod}.{name} not patched"
    assert pkg.seam_finder.SeamFinder.resize is stitching_b200.seam_finder.resize
    assert pkg.images.Images.resize_img_by_scaler is stitching_b200.images.resize_img_by_scaler
    assert pkg.exposure_error_compensator.ExposureErrorCompensator.apply.__name__ == "_apply"
    for name in [m for m in sys.modules if m == "stitching_layout" or m.startswith("stitching_layout.")]:
        del sys.modules[name]

    _, panos, _ = replay(cv, "stitch", rc.synthetic_views(cv))
    pano = panos[-1]
    assert pano.ndim == 3 and pano.dtype == np.uint8
    assert (pano.sum(axis=2) > 0).mean() > 0.5


def test_stitch_verbose_runs_after_install(cv):
    """Stitcher.stitch_verbose (verbose.py) draws the FINAL-resolution seam masks with SeamFinder.draw_seam_mask, i.e.
    cv.UMat.get(seam_mask) (seam_finder.py:47, verbose.py:149-156): the drop-in SeamFinder.resize has to hand out what the
    reference hands out (a cv.UMat) -- checked call for call by the replay of the recorded verbose run."""
    kinds, panos, frames = replay(cv, "verbose", rc.synthetic_views(cv))
    pins = rc.Pins()
    resized = [k for k, kind in enumerate(kinds) if kind == "seam_resize"]
    assert len(resized) == 3 and all(str(pins.value(f"pipe.verbose.{k}.out_type")) == "UMat" for k in resized), \
        "verbose.py:149-156 resizes one seam mask per image and draws it through cv.UMat.get"
    assert frames, "verbose.py's timelapse excursion"
    pano = panos[-1]
    assert pano.ndim == 3 and pano.dtype == np.uint8 and (pano.sum(axis=2) > 0).mean() > 0.5


@pytest.mark.parametrize("warper_type", ["fisheye", "compressedPlaneA2B1"])  # the two the reference's own tests use (tests/test_stitcher.py:85,110)
def test_stitcher_with_other_warper_types_after_install(cv, warper_type):
    kinds, panos, _ = replay(cv, warper_type, rc.synthetic_views(cv))
    pins = rc.Pins()
    assert {str(pins.value(f"pipe.{warper_type}.{k}.type")) for k, kind in enumerate(kinds) if kind == "warp_image"} == {warper_type}
    pano = panos[-1]
    assert pano.ndim == 3 and pano.dtype == np.uint8 and (pano.sum(axis=2) > 0).mean() > 0.3


def test_timelapse_run_after_install(cv):
    """Stitcher(timelapse="as_is"): the warped FINAL-resolution frames go to the Timelapser (stitcher.py:242-252) instead of
    the blender; one frame per input, each the frame of the whole panorama roi with one image in it."""
    kinds, panos, frames = replay(cv, "timelapse", rc.synthetic_views(cv))
    assert not panos and kinds.count("tl_init") == 1  # create_final_panorama blends nothing in timelapse mode (stitcher.py:257-260)
    assert len(frames) == 3 and all(f.shape == frames[0].shape for f in frames)
    cover = [(f.sum(axis=2) > 0) for f in frames]
    assert all(0.1 < c.mean() < 0.9 for c in cover)                     # one image per frame, not the panorama
    centres = [np.nonzero(c.any(axis=0))[0].mean() for c in cover]
    assert min(abs(a - b) for i, a in enumerate(centres) for b in centres[i + 1:]) > 100  # three different places on the canvas


def test_one_stitcher_for_two_image_sets_and_affine_stitcher_after_install(cv):
    """tests/test_stitcher.py:283-290 of the reference re-uses one Stitcher for two image sets, :173-185 runs AffineStitcher
    (affine warper, no compensator): both recorded, both replayed on the drop-in classes."""
    views = rc.synthetic_views(cv)
    _, panos, _ = replay(cv, "two_sets", views)
    assert len(panos) == 3
    first, second, again = panos
    assert first.ndim == 3 and second.ndim == 3 and second.shape[1] < first.shape[1]
    assert abs(again.shape[0] - first.shape[0]) <= 30 and abs(again.shape[1] - first.shape[1]) <= 30

    kinds, panos, _ = replay(cv, "affine", rc.synthetic_scans(cv))
    pins = rc.Pins()
    assert {str(pins.value(f"pipe.affine.{k}.type")) for k, kind in enumerate(kinds) if kind == "warp_image"} == {"affine"}
    pano = panos[-1]
    assert pano.ndim == 3 and pano.dtype == np.uint8
    assert pano.shape[1] > 1200 and (pano.sum(axis=2) > 0).mean() > 0.5  # wider than one scan: the scans were composed
