"""Timelapse frames from the fused compositor (Compositor(..., timelapse="as_is" | "crop")), in the emulation build:
random rigs, crops, resized inputs and gains against the oracle's warp -> slice -> gain -> Timelapser, the pipelined
path over every buffer set, set_gain between steps, the refusals and the canvas with a zero side."""
import ctypes

import numpy as np
import pytest

import crop_fuzz
import rig_fuzz
import timelapse_fuzz as TF
from stitching_b200 import Compositor, Crop, StitchingError, _lib, rigs

SEED = TF.seed_from_env()
COUNT = 25


def _cases():
    return TF.cases(SEED, COUNT, rig_fuzz.EMU)


@pytest.mark.parametrize("k", range(COUNT + 2))
def test_fuzz_against_oracle(use_emu, oracle, k):
    TF.run_and_check(oracle, _cases()[k], SEED)


def test_fuzz_coverage():
    tags = set()
    for tc in _cases():
        tags |= TF.coverage(tc)
    assert TF.WANT <= tags, f"not reached: {sorted(TF.WANT - tags)}"


def _pinned(c, batch):
    out = []
    for img in batch:
        p = c.pinned_empty(img.shape)
        p[...] = img
        out.append(p)
    return out


@pytest.mark.parametrize("kind", TF.KINDS)
def test_pipelined_steps(use_emu, oracle, kind):
    """Six submits over the three buffer sets, new frames each step: every ticket's frames equal timelapse() of its batch
    and the oracle's frames; the frames are read-only."""
    cc = crop_fuzz.named("many", rig_fuzz.EMU)
    tc = TF.TLCase(cc.case, kind, cc.crop)
    steps = 6
    c = TF.compositor(tc)
    try:
        batches = [[rigs.noise_image(h, w, 9000 + 100 * k + i) for i, (w, h) in enumerate(tc.case.sizes)] for k in range(steps)]
        srcs = [_pinned(c, b) for b in batches]
        tickets, got = [], {}
        for k in range(steps):
            if len(tickets) == 3:
                t = tickets.pop(0)
                c.wait(t)
                got[t] = [f.copy() for f in c.frames(t)]
            tickets.append(c.submit_timelapse(srcs[k]))
        for t in tickets:
            c.wait(t)
            got[t] = [f.copy() for f in c.frames(t)]
        fr = c.frames(tickets[-1])
        assert not fr[0].flags.writeable
        with pytest.raises(ValueError):
            fr[0][0, 0, 0] = 1
        for k in range(steps):
            once = c.timelapse(batches[k])
            ref = TF.oracle_run(oracle, tc, batches[k], [None] * tc.n)
            for i in range(tc.n):
                assert np.array_equal(got[k][i], once[i]), f"step {k} frame {i}: pipelined != timelapse()"
                assert np.array_equal(got[k][i], ref["frames"][i]), f"step {k} frame {i} != oracle"
    finally:
        c.close()


def test_set_gain_between_submits(use_emu, oracle):
    """set_gain after a step changes the next step only (the captured step is rebuilt)."""
    tc = next(t for t in _cases() if t.crop is not None and t.kind == "crop" and any(p is not None for p in TF.parts(t)))
    imgs = TF.frames_in(tc)
    gs = TF.gains(tc)
    fed = tc.fed()
    g2 = [np.full((3, 2), 1.3 + 0.05 * i, np.float32) for i in range(tc.n)]
    c = TF.compositor(tc)
    try:
        before = c.timelapse(imgs)
        for i, g in enumerate(g2):
            c.set_gain(i, g)
        after = c.timelapse(imgs)
        for i in range(tc.n):
            c.set_gain(i, None)
        plain = c.timelapse(imgs)
    finally:
        c.close()
    for got, want_g in ((before, [None] * tc.n), (after, g2), (plain, [None] * tc.n)):
        ref = TF.oracle_run(oracle, tc, imgs, want_g)
        TF.check(tc, dict(rects=fed, roi=ref["roi"], frames=got), ref, SEED)
    assert gs is not None


def _refusal_compositor():
    case = rig_fuzz.named("odd_origins", rig_fuzz.EMU)
    return case, Compositor(case.cams, case.sizes, case.wtype, timelapse="as_is")


def test_refusals(use_emu):
    case, c = _refusal_compositor()
    other = Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength)
    L = use_emu
    try:
        assert c.num_bands == -1
        imgs = rig_fuzz.images(case)
        h, w = c.roi[3], c.roi[2]
        calls = [
            ("sb_compositor_upload", lambda: c.upload(imgs)),
            ("sb_compositor_run", c.run),
            ("sb_compositor_download", c.download),
            ("sb_compositor_download_warped", lambda: c.download_warped(0)),
            ("sb_compositor_submit", lambda: c.submit(imgs, np.empty((h, w, 3), np.uint8), np.empty((h, w), np.uint8))),
            ("sb_compositor_set_mask", lambda: c.set_mask(0, np.zeros(c.rects[0][:1:-1], np.uint8))),
            ("sb_compositor_set_seam_mask", lambda: c.set_seam_mask(0, np.zeros((4, 4), np.uint8))),
            ("sb_compositor_shard_phase", lambda: c.shard_phase(0)),
            ("sb_compositor_shard_slab", lambda: c.shard_slab(1, True)),
        ]
        for name, call in calls:
            with pytest.raises(StitchingError, match=rf"{name} failed \(-4\).*timelapse"):
                call()
        from stitching_b200.compositor import time_multi
        with pytest.raises(StitchingError, match=r"\(-4\).*timelapse"):
            time_multi([other, c], 1)
        # a ticket that was never submitted, a compositor without frames, frames of the wrong size
        with pytest.raises(StitchingError, match="not in flight"):
            c.frames(0)
        with pytest.raises(StitchingError, match=r"sb_compositor_submit_timelapse failed \(-4\)"):
            other.submit_timelapse(imgs)
        with pytest.raises(StitchingError, match="image 0: expected a uint8"):
            c.submit_timelapse([np.zeros((2, 2, 3), np.uint8)] + imgs[1:])
        with pytest.raises(StitchingError, match="expected 3 images"):
            c.submit_timelapse(imgs[1:])
        t = c.submit_timelapse(imgs)
        c.wait(t)
        c.frames(t)
        for _ in range(3):
            c.submit_timelapse(imgs)
        with pytest.raises(StitchingError, match=f"ticket {t} is not in flight"):
            c.frames(t)
        # what works: timing, model bytes, sync
        ms, stages = c.time(2)
        assert [n for n, _ in stages] == ["warp", "paste"]
        tot, per = c.model_bytes()
        assert len(per) == 2 and tot == sum(per)
        c.sync()
    finally:
        c.close()
        other.close()
    with pytest.raises(StitchingError, match="unknown timelapse kind"):
        Compositor(case.cams, case.sizes, case.wtype, timelapse="no")
    with pytest.raises(StitchingError, match="one GPU"):
        Compositor(case.cams, case.sizes, case.wtype, timelapse="crop", rank=0, world=2)
    # the C ABI refuses a kind outside the enum, a timelapse over two GPUs and in_w without in_h
    w = (ctypes.c_int * case.n)(*[s[0] for s in case.sizes])
    rig = _lib.Rig(case.n, 0, 1.0, 0, 5.0, w, (ctypes.c_int * case.n)(*[s[1] for s in case.sizes]),
                   (ctypes.c_float * (9 * case.n))(), (ctypes.c_float * (9 * case.n))())
    for kind in (3, -1):
        assert not L.sb_compositor_create(ctypes.byref(rig), ctypes.byref(_lib.CompositorOpts(world=1, timelapse=kind)))
        assert b"unknown timelapse kind" in L.sb_last_error()
    assert not L.sb_compositor_create(ctypes.byref(rig), ctypes.byref(_lib.CompositorOpts(rank=0, world=2, timelapse=1)))
    assert b"one GPU" in L.sb_last_error()
    assert not L.sb_compositor_create(ctypes.byref(rig), ctypes.byref(_lib.CompositorOpts(in_w=w, world=1, timelapse=1)))
    assert b"invalid argument" in L.sb_last_error()


def test_frames_out_of_pinned_memory(use_emu, oracle, monkeypatch):
    """The frames cannot be allocated (SB_PINNED_MAX_BYTES below their size): every submit fails with SB_ERR_NOMEM and
    the byte count, no ticket exists, and once the memory is there the next submit allocates them and runs."""
    case, c = _refusal_compositor()
    try:
        imgs = rig_fuzz.images(case)
        need = 3 * case.n * c.roi[2] * c.roi[3] * 3
        monkeypatch.setenv("SB_PINNED_MAX_BYTES", str(need // 3 - 1))
        for _ in range(2):
            with pytest.raises(StitchingError, match=rf"submit_timelapse failed \(-5\).*: {need} bytes of page-locked memory"):
                c.submit_timelapse(imgs)
            with pytest.raises(StitchingError, match="not in flight"):
                c.frames(0)
            with pytest.raises(StitchingError, match="not in flight"):
                c.wait(0)
        monkeypatch.delenv("SB_PINNED_MAX_BYTES")
        tc = TF.TLCase(case, "as_is")
        ref = TF.oracle_run(oracle, tc, imgs, [None] * case.n)
        t = c.submit_timelapse(imgs)
        assert t == 0
        c.wait(t)
        for i, f in enumerate(c.frames(t)):
            assert np.array_equal(f, ref["frames"][i]), f"frame {i}"
    finally:
        c.close()


def test_frame_views_keep_the_compositor(use_emu):
    """A view from frames() holds the compositor: dropping the last other reference frees nothing under it."""
    import gc
    import weakref

    case, c = _refusal_compositor()
    imgs = rig_fuzz.images(case)
    t = c.submit_timelapse(imgs)
    c.wait(t)
    views = c.frames(t)
    want = [v.copy() for v in views]
    ref = weakref.ref(c)
    del c
    gc.collect()
    assert ref() is not None
    assert all(np.array_equal(v, w) for v, w in zip(views, want))
    del views
    gc.collect()
    assert ref() is None


def _touching(O, kind, gap):
    """Two affine images side by side, their warped rects `gap` px apart (0: touching, negative: overlapping)."""
    sizes = [(20, 12), (16, 12)]
    cam0 = rigs.Camera(1, 1, 0, 0, np.eye(3, dtype=np.float32))
    r0 = O.warp_roi("affine", 1.0, cam0.K(), cam0.R, sizes[0])
    # the warp maps back through R: a translation by -t places the image at t
    cam1 = rigs.Camera(1, 1, 0, 0, np.array([[1, 0, -(r0[0] + r0[2] + gap)], [0, 1, 0], [0, 0, 1]], np.float32))
    r1 = O.warp_roi("affine", 1.0, cam1.K(), cam1.R, sizes[1])
    assert r1[0] - (r0[0] + r0[2]) == gap and r0[1] == r1[1] and r0[3] == r1[3], (r0, r1)
    return [cam0, cam1], sizes, r0, r1


def test_zero_side_canvas(use_emu, oracle):
    """Images that touch: the "crop" canvas has width 0, which the reference cannot show either; refused at creation with
    its extent.  Apart or overlapping, the canvas is the gap or the overlap."""
    cams, sizes, r0, r1 = _touching(oracle, "crop", 0)
    with pytest.raises(StitchingError, match=rf"timelapse canvas \({r1[0]},{r1[1]} 0x{r1[3]}\) has a zero side"):
        Compositor(cams, sizes, "affine", timelapse="crop")
    Compositor(cams, sizes, "affine", timelapse="as_is").close()
    for gap in (3, -4):
        cams, sizes, r0, r1 = _touching(oracle, "crop", gap)
        c = Compositor(cams, sizes, "affine", timelapse="crop")
        try:
            assert tuple(c.roi) == (min(r1[0], r0[0] + r0[2]), r0[1], abs(gap), r0[3]), (gap, c.roi, r0, r1)
        finally:
            c.close()


def test_empty_slice_refused(use_emu):
    """A crop slice that is empty stays refused: the reference Stitcher fails on it before any frame (SeamFinder.resize
    of the empty slice's mask raises in cv.resize)."""
    case = rig_fuzz.named("odd_origins", rig_fuzz.EMU)
    rects = [(0, 0, r[2], r[3]) for r in case.rects]
    rects[1] = (case.rects[1][2], 0, 5, 5)  # starts at the warped image's right edge
    crop = Crop(rects, [r[:2] for r in case.rects], [r[2:] for r in case.rects])
    with pytest.raises(StitchingError, match="crop of image 1 is empty"):
        Compositor(case.cams, case.sizes, case.wtype, timelapse="crop", crop=crop)


def test_records_hold_what_the_replay_needs():
    """The two recorded reference runs: four frames each, the "crop" canvas as resultRoiIntersection of the prepared
    rects (those views all overlap, so no gap rectangle: the fuzz draws reach that case)."""
    for name in TF.RECORDS:
        z = TF.record(name)
        assert str(z["timelapse"]) == name and len(z["frames"]) == int(z["n"]) == 4
        corners, sizes = [tuple(map(int, v)) for v in z["corners"]], [tuple(map(int, v)) for v in z["sizes"]]
        x, y, w, h = TF.canvas_of(name, corners, sizes)
        assert all(str(f).startswith(f"|u1[{h}, {w}, 3]") for f in z["frames"]), (name, (w, h), z["frames"])
        assert int(z["canvas_gap"]) == 0


@pytest.mark.parametrize("name", TF.RECORDS)
def test_record_replays_in_emulation(use_emu, name):
    TF.record_replay(TF.record(name))
