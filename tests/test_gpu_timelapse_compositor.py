"""Timelapse frames from the fused compositor on the H100: the reference Stitcher's recorded timelapse run replayed from
its camera views, random rigs / crops / resized inputs / gains against the oracle, the A/B switches in child processes,
and the drop-in chain (Warper.warp_image -> slice -> apply_gain -> Timelapser) on the same rig."""
import numpy as np
import pytest

import fuzz_chain
import reference_cases as RC
import replay
import rig_fuzz
import timelapse_fuzz as TF
from stitching_b200 import Compositor

pytestmark = pytest.mark.gpu

SEED = TF.seed_from_env()
COUNT = 150

_sets = {}


def _cases():
    if SEED not in _sets:
        _sets[SEED] = TF.cases(SEED, COUNT, rig_fuzz.GPU)
    return _sets[SEED]


@pytest.mark.parametrize("k", range(COUNT + 2))
def test_fuzz_against_oracle(cuda_lib, oracle, k):
    TF.run_and_check(oracle, _cases()[k], SEED)


def test_fuzz_coverage():
    tags = set()
    for tc in _cases():
        tags |= TF.coverage(tc)
    assert TF.WANT <= tags, f"not reached: {sorted(TF.WANT - tags)}"


def _recorded_run(cv, name="timelapse"):
    """The recorded Stitcher(timelapse="as_is") run of golden_reference.npz: per fed image the FINAL warp call, its gain,
    the camera view it was resized from, and the frame digest; plus the recorded Timelapser.initialize."""
    pins = RC.Pins()
    log = []
    for k in range(int(pins.value(f"pipe.{name}.n"))):
        prefix = f"pipe.{name}.{k}."
        log.append({key[len(prefix):]: v for key, v in pins.data.items() if key.startswith(prefix)})
    views = {RC.digest(v): v for v in RC.synthetic_views(cv)}
    by_out = {str(e["out"]): e for e in log if "out" in e and str(e["kind"]) in ("warp_image", "gain_apply", "img_resize")}
    init = next(e for e in log if str(e["kind"]) == "tl_init")
    images = []
    for e in log:
        if str(e["kind"]) != "tl_frame":
            continue
        g = by_out[str(e["input"])]
        assert str(g["kind"]) == "gain_apply"
        w = by_out[str(g["input"])]
        assert str(w["kind"]) == "warp_image"
        r = by_out[str(w["input"])]
        assert str(r["kind"]) == "img_resize" and str(r["input"]) in views, "the FINAL input is a resize of a camera view"
        images.append(dict(warp=w, gain=g.get("gain"), view=views[str(r["input"])], size=tuple(int(v) for v in r["size"]),
                           corner=tuple(int(v) for v in e["corner"]), frame=str(e["out"])))
    return init, images


def test_replays_recorded_timelapse_stitcher(cuda_lib):
    """golden_reference.npz's Stitcher(timelapse="as_is") run, from the camera views: the compositor resizes them to
    FINAL, warps with the recorded cameras, scale and ratio, applies the recorded gains, and every frame equals the
    reference's byte for byte."""
    cv = pytest.importorskip("cv2")
    init, images = _recorded_run(cv)
    assert str(init["type"]) == "as_is" and len(images) == 3
    w0 = images[0]["warp"]
    assert all(float(im["warp"]["scale"]) == float(w0["scale"]) and float(im["warp"]["aspect"]) == float(w0["aspect"]) for im in images)
    cams = [RC.camera_from_value(cv, im["warp"]["camera"]) for im in images]
    views = [im["view"] for im in images]
    c = Compositor(cams, [im["size"] for im in images], str(w0["type"]), scale=float(w0["scale"]), aspect=float(w0["aspect"]),
                   timelapse="as_is", input_sizes=[(v.shape[1], v.shape[0]) for v in views])
    try:
        corners = [tuple(int(v) for v in x) for x in init["corners"]]
        sizes = [tuple(int(v) for v in x) for x in init["sizes"]]
        assert [tuple(r[:2]) for r in c.rects] == [im["corner"] for im in images] == corners
        assert [tuple(r[2:]) for r in c.rects] == sizes
        x0, y0 = min(x for x, _ in corners), min(y for _, y in corners)
        assert tuple(c.roi) == (x0, y0, max(x + w for (x, _), (w, _) in zip(corners, sizes)) - x0,
                                max(y + h for (_, y), (_, h) in zip(corners, sizes)) - y0)
        for i, im in enumerate(images):
            c.set_gain(i, im["gain"])
        for k in range(2):  # the first step and a replay of the captured one
            frames = c.timelapse(views)
            for i, (f, im) in enumerate(zip(frames, images)):
                assert RC.digest(f) == im["frame"], f"step {k} frame {i}: {RC.digest(f)}, the reference {im['frame']}"
    finally:
        c.close()


AB_CASES = list(range(0, 24, 3)) + [COUNT, COUNT + 1]


@pytest.mark.parametrize("env", [{"SB_GRAPH": "0"}, {"SB_SRC4": "0"}], ids=["SB_GRAPH=0", "SB_SRC4=0"])
def test_ab_switches_give_identical_frames(cuda_lib, env):
    fuzz_chain.ab_run("timelapse_fuzz:frame_digests", [SEED, COUNT, AB_CASES, rig_fuzz.GPU], list(env.items()),
                      "SB_TIMELAPSE_FUZZ_SEED")


def test_equals_dropin_chain(cuda_lib):
    """The drop-in classes in the Stitcher's call order -- Warper.warp_image, the crop's slice, apply_gain, Timelapser
    initialize / process_frame / get_frame -- give the compositor's frames on the same rigs."""
    import stitching_b200
    from stitching_b200.exposure_error_compensator import apply_gain

    done = 0
    for tc in _cases()[:40]:
        if 0 in TF.canvas(tc)[2:] or tc.input_sizes is not None:
            continue
        imgs, gs = TF.frames_in(tc), TF.gains(tc)
        got = TF.compositor_run(tc, imgs, gs)
        w = stitching_b200.Warper(tc.case.wtype)
        w.scale = float(tc.case.scale())
        t = stitching_b200.Timelapser(tc.kind)
        t.initialize(*tc.prepared())
        fed = tc.fed()
        for i, (img, cam, g) in enumerate(zip(imgs, tc.case.cams, gs)):
            wi = np.asarray(w.warp_image(img, cam, 1))
            if tc.crop is not None:
                x, y, cw, ch = tc.crop.rects[i]
                wi = np.ascontiguousarray(wi[y:y + ch, x:x + cw])
            if g is not None:
                wi = apply_gain(wi.copy(), g)
            t.process_frame(wi, fed[i][:2])
            replay.assert_exact(got["frames"][i], np.asarray(t.get_frame()), f"{tc.describe()}: frame {i} vs the drop-in chain")
        done += 1
    assert done >= 10


@pytest.mark.parametrize("name", TF.RECORDS)
def test_replays_recorded_timelapse_records(cuda_lib, name):
    """golden_timelapse_stitcher_{as_is,crop}.npz (the reference Stitcher with crop=True, final_megapix=3 and the
    timelapse setting) replayed from the camera views: rects, canvas and every frame, also from pipelined steps."""
    TF.record_replay(TF.record(name))
