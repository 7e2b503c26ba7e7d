"""Host logic of the product (plans, geometry, error behaviour, Python drop-ins) on a GPU-less box.

These tests compile the PRODUCT sources against tests/emu's serial CUDA stand-in -- test infrastructure
that lets the plan / index arithmetic run without a device.  The CUDA build itself is covered by
tests/test_gpu_parity.py (-m gpu).
"""
import ctypes as C

import numpy as np
import pytest

import replay
import rig_fuzz
from stitching_b200 import Blender, Compositor, StitchingError, Warper, rigs


def test_interface_constants_match_the_reference_boundary():
    # warper.py:10-29, blender.py:8-14 (what stitcher.py / cli/stitch.py read)
    assert Warper.DEFAULT_WARP_TYPE == "spherical"
    assert len(Warper.WARP_TYPE_CHOICES) == 16 and Warper.WARP_TYPE_CHOICES[:4] == ("spherical", "plane", "affine", "cylindrical")
    assert Blender.BLENDER_CHOICES == ("multiband", "feather", "no")
    assert Blender.DEFAULT_BLENDER == "multiband" and Blender.DEFAULT_BLEND_STRENGTH == 5


def test_warper_goldens_through_emulated_library(use_emu):
    replay.run_warper_goldens(Warper)


def test_blender_goldens_through_emulated_library(use_emu):
    replay.run_blender_goldens(Blender)


def test_e2e_goldens_through_emulated_library(use_emu):
    replay.run_e2e_goldens(Warper, Blender)


def test_compositor_matches_oracle(use_emu, oracle):
    for name, sd, ncap in (("cfg2", 25, None), ("cfg3", 25, 5), ("cfg5", 12, None)):
        cfg = rigs.config(name, sd)
        cams = cfg["cameras"][:ncap] if ncap else cfg["cameras"]
        imgs = [rigs.noise_image(cfg["h"], cfg["w"], 1000 + i) for i in range(len(cams))]
        ref = replay.oracle_composite(oracle, cfg, cams, imgs)
        c = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), cfg["warper"], cfg["blender"], cfg["strength"])
        assert [r[:2] for r in c.rects] == [tuple(x) for x in ref["corners"]]
        assert [r[2:] for r in c.rects] == [tuple(x) for x in ref["sizes"]]
        if cfg["blender"] == "multiband":
            assert c.num_bands == ref["num_bands"]
        pano, mask = c.composite(imgs)
        replay.assert_exact(pano, ref["pano"], f"{name} pano")
        replay.assert_exact(mask, ref["pmask"], f"{name} mask")
        wi, wm = c.download_warped(1)
        replay.assert_exact(wi, ref["warped"][1], f"{name} warped image 1")
        replay.assert_exact(wm, ref["masks"][1], f"{name} warped mask 1")
        total, per_launch = c.model_bytes()
        assert total > 0 and abs(sum(per_launch) - total) < 1e-6 * total
        ms, launches = c.time(1)
        assert len(launches) == len(per_launch) and launches[0][0] == "warp"
        c.close()


def test_source_layouts_of_the_warp_kernel_agree(use_emu, monkeypatch):
    """The compositor repacks every uploaded source to one word per pixel for the warp kernel (SB_SRC4, default on); the
    packed 3-byte path (SB_SRC4=0) is the same arithmetic on the same pixels: identical panoramas, masks and warped images."""
    cfg = rigs.config("cfg2", 16)
    cams = cfg["cameras"][:4]
    sizes = [(cfg["w"], cfg["h"])] * len(cams)
    imgs = [rigs.noise_image(cfg["h"], cfg["w"], 40 + i) for i in range(len(cams))]
    out = []
    for flag in ("1", "0"):
        monkeypatch.setenv("SB_SRC4", flag)
        c = Compositor(cams, sizes, cfg["warper"], cfg["blender"], cfg["strength"])
        pano, mask = c.composite(imgs)
        out.append((pano.copy(), mask.copy(), [np.concatenate([a.ravel(), b.ravel()]) for a, b in (c.download_warped(i) for i in range(len(cams)))]))
        c.close()
    replay.assert_exact(out[0][0], out[1][0], "pano, word-per-pixel vs packed sources")
    replay.assert_exact(out[0][1], out[1][1], "mask, word-per-pixel vs packed sources")
    for a, b in zip(out[0][2], out[1][2]):
        assert np.array_equal(a, b)


def test_host_pool_reuses_and_bounds_page_locked_memory(use_emu, monkeypatch):
    """The drop-ins' result arrays come from pooled page-locked buffers (stitching_b200/host_pool.py): a buffer goes back to the
    pool when its last view dies, the next array of that size class takes it, small arrays and an exhausted pool fall back to
    np.empty, and the arrays are ordinary writable ndarrays."""
    import gc

    from stitching_b200 import host_pool

    host_pool.trim()
    a = host_pool.empty((300, 400, 3), np.uint8)
    assert a.shape == (300, 400, 3) and a.dtype == np.uint8 and a.flags.writeable and a.flags.c_contiguous
    a[...] = 7
    addr = a.ctypes.data
    view = a[10:20]
    del a
    gc.collect()
    assert sum(len(v) for v in host_pool._free.values()) == 0  # a view keeps the buffer out of the pool
    del view
    gc.collect()
    assert sum(len(v) for v in host_pool._free.values()) == 1
    b = host_pool.empty((350, 400, 3), np.int16)                 # same 1 MiB size class: the cached buffer is reused
    assert b.ctypes.data == addr and b.dtype == np.int16
    small = host_pool.empty((10, 10), np.uint8)                   # not worth pinning
    assert small.base is None
    monkeypatch.setenv("SB_PINNED_LIMIT_MB", "1")
    c = host_pool.empty((2000, 2000), np.uint8)                   # over the limit: pageable
    assert c.shape == (2000, 2000) and c.base is None
    del b, c
    gc.collect()
    host_pool.trim()
    assert host_pool._total == 0 and not any(host_pool._free.values())


def test_unit_weight_shortcuts_are_exact():
    """The two identities the fast collapse kernel uses instead of float work (sb_collapse_fast.cu):
    (short)trunc(L * 1.0f) == L, and (short)trunc(a / fl(1 + 1e-5f)) == a - sign(a) for every int16 a."""
    a = np.arange(-32768, 32768, dtype=np.int32)
    den = np.float32(1.0) + np.float32(1e-5)
    q = (a.astype(np.float32) / den).astype(np.float32)
    assert np.array_equal(np.trunc(q).astype(np.int32), a - np.sign(a))
    # weight sum exactly 2: (short)trunc(a / fl(2 + 1e-5f)) == (|a| - 1) / 2 toward zero, signed
    den2 = np.float32(2.0) + np.float32(1e-5)
    q2 = (a.astype(np.float32) / den2).astype(np.float32)
    t = a - np.sign(a)
    assert np.array_equal(np.trunc(q2).astype(np.int32), (t + (t < 0)) >> 1)
    assert np.float32(255.0) * np.float32(1.0 / 255.0) == np.float32(1.0)  # a 255 mask byte is weight exactly 1
    assert np.array_equal(np.trunc(a.astype(np.float32) * np.float32(1.0)).astype(np.int32), a)


def test_compositor_with_seam_like_blend_masks(use_emu, oracle):
    """Mask set B (gray ramps, 256 levels) through Compositor.set_mask == oracle fed with the same masks."""
    for name, sd in (("cfg2", 25), ("cfg5", 12)):
        cfg = rigs.config(name, sd)
        cams = cfg["cameras"]
        imgs = [rigs.synth_image(cfg["h"], cfg["w"], 40 + i) for i in range(len(cams))]
        ref = replay.oracle_composite(oracle, cfg, cams, imgs, mask_fn=lambda ms: replay.ramp_masks(ms, 16))
        c = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), cfg["warper"], cfg["blender"], cfg["strength"])
        for i, m in enumerate(ref["masks"]):
            c.set_mask(i, m)
        pano, mask = c.composite(imgs)
        replay.assert_exact(pano, ref["pano"], f"{name} pano with ramp masks")
        replay.assert_exact(mask, ref["pmask"], f"{name} mask with ramp masks")
        c.close()


def test_pipelined_submit_wait_equals_composite(use_emu):
    cfg = rigs.config("cfg2", 25)
    cams = cfg["cameras"]
    sizes = [(cfg["w"], cfg["h"])] * len(cams)
    c = Compositor(cams, sizes, cfg["warper"], cfg["blender"], cfg["strength"])
    batches = [[rigs.noise_image(cfg["h"], cfg["w"], 10 * b + i) for i in range(len(cams))] for b in range(5)]
    expected = [c.composite(b) for b in batches]
    _, _, pw, ph = c.roi
    outs = [(c.pinned_empty((ph, pw, 3)), c.pinned_empty((ph, pw))) for _ in range(2)]
    tickets = []
    for k, b in enumerate(batches):
        if k >= 2:
            c.wait(tickets[k - 2])
            assert np.array_equal(outs[k & 1][0], expected[k - 2][0]) and np.array_equal(outs[k & 1][1], expected[k - 2][1])
        tickets.append(c.submit(b, *outs[k & 1]))
    for k in (3, 4):
        c.wait(tickets[k])
        assert np.array_equal(outs[k & 1][0], expected[k][0])
    with pytest.raises(StitchingError):
        c.wait(tickets[0])  # long gone
    c.close()


def test_band_clipping_matches_oracle(use_emu, oracle):
    """MultiBandBlender::prepare's band clipping -- product plan vs oracle restatement."""
    rng = np.random.default_rng(3)
    L = oracle.lib()
    for _ in range(200):
        n = int(rng.integers(1, 5))
        sizes = [(int(rng.integers(5, 400)), int(rng.integers(5, 300))) for _ in range(n)]
        corners = [(int(rng.integers(-500, 500)), int(rng.integers(-300, 300))) for _ in range(n)]
        roi = oracle.result_roi(corners, sizes)
        nbr = int(rng.integers(0, 12))
        h = L.so_mb_create(nbr, *roi)
        b = use_emu.sb_blender_create(2, nbr, C.c_float(0))
        assert use_emu.sb_blender_prepare(b, *roi) == 0
        assert use_emu.sb_blender_num_bands(b) == L.so_mb_num_bands(h)
        use_emu.sb_blender_destroy(b)
        L.so_mb_destroy(h)


def test_generators_and_fused_extension(use_emu):
    cams = rigs.yaw_ring(3, 80, 60, 90, 25)
    w = Warper("cylindrical")
    w.set_scale(cams)
    imgs = [rigs.noise_image(60, 80, i) for i in range(3)]
    gen = w.warp_images(imgs, cams)
    assert hasattr(gen, "__next__")  # stitcher.py:185-189 relies on laziness
    first = next(gen)
    both = w.warp_image_and_mask(imgs[0], cams[0])
    assert np.array_equal(first, both[0])
    assert np.array_equal(w.create_and_warp_mask((80, 60), cams[0]), both[1])
    corners, sizes = w.warp_rois([(80, 60)] * 3, cams)
    assert len(corners) == 3 and all(len(c) == 2 for c in corners) and first.shape[:2] == (sizes[0][1], sizes[0][0])
    # a cropped (non-contiguous) view is accepted, like the reference after cropper.py:150-151
    big = rigs.noise_image(70, 100, 9)
    view = big[5:65, 10:90]
    assert np.array_equal(w.warp_image(view, cams[0]), w.warp_image(np.ascontiguousarray(view), cams[0]))


def test_error_behaviour(use_emu):
    cams = rigs.yaw_ring(2, 64, 48, 70, 20)
    w = Warper()
    with pytest.raises(TypeError):  # scale is None until set_scale (warper.py:44)
        w.warp_roi((64, 48), cams[0])
    w.set_scale(cams)
    bad = rigs.Camera(70, 1, 32, 24, np.eye(3))
    bad.R = np.eye(3, dtype=np.float64)  # cv2 asserts CV_32F
    with pytest.raises(StitchingError):
        w.warp_roi((64, 48), bad)
    f = Warper("fisheye")  # every reference choice is served (warper.py:10-27) ...
    f.scale = 70.0
    assert len(f.warp_roi((64, 48), cams[0])) == 4
    g = Warper("equirectangular")  # ... and a name the reference does not know fails on use, like cv.PyRotationWarper
    g.scale = 1.0
    with pytest.raises(StitchingError):
        g.warp_roi((64, 48), cams[0])
    b = Blender("multiband", 5)
    with pytest.raises(AttributeError):  # blender.py:41 before prepare: self.blender is None
        b.feed(np.zeros((4, 4, 3), np.uint8), np.zeros((4, 4), np.uint8), (0, 0))
    b.prepare([(0, 0), (30, 0)], [(40, 30), (40, 30)])
    with pytest.raises(StitchingError):  # leaves the prepared roi
        b.feed(np.zeros((30, 40, 3), np.uint8), np.full((30, 40), 255, np.uint8), (500, 0))
    with pytest.raises(StitchingError):  # mask / image size mismatch
        b.feed(np.zeros((30, 40, 3), np.uint8), np.full((30, 41), 255, np.uint8), (0, 0))
    b.feed(np.zeros((30, 40, 3), np.uint8), np.full((30, 40), 255, np.uint8), (0, 0))
    pano, mask = b.blend()
    assert pano.shape == (30, 70, 3) and mask.shape == (30, 70) and pano.dtype == np.uint8
    with pytest.raises(StitchingError):  # blend() consumed the state, like OpenCV
        b.blender.blend()
    # blend width < 1 silently selects the NO blender (blender.py:27)
    tiny = Blender("multiband", 0.1)
    tiny.prepare([(0, 0)], [(8, 8)])
    assert tiny.blender.kind == "no"


def test_umat_like_mask_and_create_panorama(use_emu, oracle):
    class FakeUMat:  # cv.UMat exposes .get() -> ndarray (seam_finder.py:38-43 hands UMats to Blender.feed)
        def __init__(self, a):
            self._a = a

        def get(self):
            return self._a

    rng = np.random.default_rng(4)
    imgs = [rng.integers(0, 256, (20, 30, 3), dtype=np.uint8) for _ in range(2)]
    masks = [rng.integers(0, 2, (20, 30), dtype=np.uint8) * 255 for _ in range(2)]
    corners, sizes = [(0, 0), (12, 5)], [(30, 20), (30, 20)]
    pano, pmask = Blender.create_panorama(imgs, [FakeUMat(m) for m in masks], corners, sizes)
    o = oracle.Blender("no")
    o.prepare(corners, sizes)
    for i, m, c in zip(imgs, masks, corners):
        o.feed(i, m, c)
    ep, em = o.blend()
    assert np.array_equal(pano, ep) and np.array_equal(pmask, em)


def test_seam_resize_drop_in_and_fused(use_emu, oracle):
    """SeamFinder.resize through the C ABI (host buffers) == the reference's goldens == the oracle; the fused
    Compositor.set_seam_mask == set_mask(SeamFinder.resize(seam, warped mask))."""
    from stitching_b200 import seam_finder

    replay.run_seam_goldens(seam_finder.resize)
    rng = np.random.default_rng(11)
    for t in range(12):
        sh, sw = int(rng.integers(3, 60)), int(rng.integers(3, 80))
        h, w = max(2, int(sh * rng.uniform(0.5, 6))), max(2, int(sw * rng.uniform(0.5, 6)))
        seam = rng.integers(0, 256, (sh, sw), dtype=np.uint8) if t % 2 else (rng.random((sh, sw)) < 0.5).astype(np.uint8) * 255
        mask = (rng.random((h, w)) < 0.9).astype(np.uint8) * 255
        replay.assert_exact(seam_finder.resize(seam, mask), oracle.seam_resize(seam, mask), f"seam resize fuzz {t}")
    cfg = rigs.config("cfg2", 25)
    cams = cfg["cameras"]
    sizes = [(cfg["w"], cfg["h"])] * len(cams)
    imgs = [rigs.synth_image(cfg["h"], cfg["w"], 60 + i) for i in range(len(cams))]
    a = Compositor(cams, sizes, cfg["warper"], cfg["blender"], cfg["strength"])
    b = Compositor(cams, sizes, cfg["warper"], cfg["blender"], cfg["strength"])
    plain, _ = a.composite(imgs)  # also yields the warped validity masks of the rig
    valid = [a.download_warped(i)[1] for i in range(len(cams))]
    seams = replay.seam_masks_low(valid)
    for i, s in enumerate(seams):
        a.set_mask(i, oracle.seam_resize(s, valid[i]))
        b.set_seam_mask(i, s)
    pa, ma = a.composite(imgs)
    pb, mb = b.composite(imgs)
    replay.assert_exact(pb, pa, "pano with fused seam masks")
    replay.assert_exact(mb, ma, "mask with fused seam masks")
    assert not np.array_equal(pb, plain), "the seam masks must change the blend"
    a.close()
    b.close()


def test_warp_collective_kernels_under_lane_emulation(use_emu, oracle, monkeypatch):
    """The kernels whose lanes talk to each other -- the warp-shuffle pyrDown (sb_pyrdown_fast.cu) and the ballot-based
    distance transform (sb_feather_fast.cu) -- themselves on the CPU: tests/emu plays the 32 lanes of a warp with 32 host
    threads that meet at every collective.  Slow, hence small rigs (level-0 and level->=1 variants, virtual halo lanes,
    border-rule templates; feather weights) against the oracle."""
    monkeypatch.setenv("SB_EMU_LANES", "1")
    # (the compositor's masks are the validity test's 0 / 255: level 0 takes the integer weight shortcut; the last case
    # switches it off so that the generic float weight path of level 0 runs under the lane emulation as well)
    for name, sd, ncap, strength in (("cfg2", 50, 3, 5), ("cfg3", 60, 3, 20), ("cfg5", 20, 4, 5), ("cfg2-generic", 50, 3, 5)):  # cfg5: ballot-based feather DT
        if name.endswith("-generic"):
            monkeypatch.setenv("SB_PD_BIN", "0")
            name = name[:-8]
        cfg = rigs.config(name, sd)
        cams = cfg["cameras"][:ncap]
        imgs = [rigs.noise_image(cfg["h"], cfg["w"], 500 + i) for i in range(len(cams))]
        cfg = dict(cfg, strength=strength)
        ref = replay.oracle_composite(oracle, cfg, cams, imgs)
        c = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), cfg["warper"], cfg["blender"], strength)
        pano, mask = c.composite(imgs)
        c.close()
        replay.assert_exact(pano, ref["pano"], f"{name} pano through the shuffle pyrDown")
        replay.assert_exact(mask, ref["pmask"], f"{name} mask through the shuffle pyrDown")


def test_shared_memory_tile_kernels_under_block_emulation(use_emu, oracle, monkeypatch):
    """k_collapse_tile (levels 0 and 1 on staged shared-memory tiles, sb_collapse_tile.cu) itself on the CPU: tests/emu plays a
    CTA with one host thread per thread (256), __syncthreads is their rendezvous, the asynchronous copies are plain copies.
    Slow, hence small rigs: single-GPU composites against the oracle (rect origins at every alignment the run-time window
    shifts have to handle, tiles on the pano border, several images per tile), and a three-rank sharded composite whose
    strips take slabs of partial sums as items from both sides."""
    import test_sharded

    monkeypatch.setenv("SB_EMU_BLOCKS", "1")
    launches0 = _launches()
    for name, sd, ncap, strength in (("cfg2", 25, 4, 5), ("cfg3", 40, 5, 20), ("cfg2", 20, 3, 60)):
        cfg = dict(rigs.config(name, sd), strength=strength)
        cams = cfg["cameras"][:ncap]
        imgs = [rigs.noise_image(cfg["h"], cfg["w"], 600 + i) if i % 2 else rigs.synth_image(cfg["h"], cfg["w"], 600 + i) for i in range(len(cams))]
        ref = replay.oracle_composite(oracle, cfg, cams, imgs)
        c = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), cfg["warper"], cfg["blender"], strength)
        assert c.num_bands >= 2, "the tile kernel serves levels 0 and 1 below the top level"
        pano, mask = c.composite(imgs)
        c.close()
        replay.assert_exact(pano, ref["pano"], f"{name}/{sd} pano through the tile kernels")
        replay.assert_exact(mask, ref["pmask"], f"{name}/{sd} mask through the tile kernels")
    cfg = rigs.config("cfg2", 20)
    cams = cfg["cameras"][:6]
    imgs = [rigs.noise_image(cfg["h"], cfg["w"], 70 + i) for i in range(len(cams))]
    single = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), cfg["warper"], cfg["blender"], cfg["strength"])
    ref_pano, ref_mask = single.composite(imgs)
    single.close()
    pano, mask, moved = test_sharded.run_sharded(cfg, cams, imgs, 3, lambda d, s, n: C.memmove(d, s, n))
    assert moved > 0 and np.array_equal(mask, ref_mask)
    assert np.abs(pano.astype(np.int32) - ref_pano.astype(np.int32)).max() <= 1
    assert _launches() > launches0


def _launches():
    from stitching_b200 import _lib

    return _lib.lib().sb_launch_count()


def test_parallel_distance_transform_under_lane_emulation(use_emu, oracle, monkeypatch):
    """The feather weights' L1 distance transform in its parallel form -- ballot words + warp scans along the rows (several
    words per lane for wide rows), chunked prefix minima along the columns -- against the oracle's FeatherBlender on mask
    shapes that stress the carries: no zero at all, a single zero pixel, zero rows / columns, rows wider than 1024, fewer
    rows than chunks, ragged last chunks."""
    monkeypatch.setenv("SB_EMU_LANES", "1")
    # (the lane emulation pays a 32-thread rendezvous per shuffle: small cases; tests/test_zz_gpu_gain.py runs larger ones)
    _distance_transform_stress(oracle, [(12, 1100), (150, 37), (5, 70)])


def _distance_transform_stress(oracle, shapes):
    rng = np.random.default_rng(99)
    for t, (h, w) in enumerate(shapes):
        masks = []
        m = np.full((h, w), 255, np.uint8)                       # no zero anywhere: weight 1 everywhere
        masks.append(m.copy())
        m[rng.integers(0, h), rng.integers(0, w)] = 0            # one zero pixel
        masks.append(m.copy())
        m = np.full((h, w), 255, np.uint8)
        m[:, : w // 3] = 0                                       # zero columns on the left, none in the rows' right part
        m[h // 2] = 0
        masks.append(m.copy())
        m = (rng.random((h, w)) > 0.002).astype(np.uint8) * 255  # sparse zeros
        m[rng.integers(0, h)] = 255                              # ... and one row without any
        masks.append(m)
        for k, mask in enumerate(masks):
            img = rigs.noise_image(h, w, 10 * t + k)
            strength = 100 if k % 2 else 5  # soft (never saturates) and sharp (saturates after a few pixels)
            a, b = Blender("feather", strength), oracle.Blender("feather", strength)
            for bl in (a, b):
                bl.prepare([(0, 0), (3, 2)], [(w, h), (w, h)])
                bl.feed(img, mask, (0, 0))
                bl.feed(img[::-1].copy(), mask[:, ::-1].copy(), (3, 2))
            (pa, ma), (pb, mb) = a.blend(), b.blend()
            replay.assert_exact(pa, pb, f"feather {h}x{w} mask {k} strength {strength}")
            replay.assert_exact(ma, mb, f"feather mask {h}x{w} mask {k} strength {strength}")


def test_fused_final_resolution_chain(use_emu, oracle):
    """Gains and seam masks together (some images with neither): compositor == warp -> apply -> SeamFinder.resize -> feed."""
    got, ref = replay.fused_chain_case(oracle, Warper, Blender, Compositor, rigs, 25)
    replay.assert_exact(got[0], ref[0], "pano of the fused chain")
    replay.assert_exact(got[1], ref[1], "mask of the fused chain")


def test_image_resize_drop_in(use_emu, oracle):
    """Images.resize_img_by_scaler through the C ABI == the reference's goldens == the oracle."""
    from stitching_b200 import images

    replay.run_resize_goldens(images.resize_exact)
    rng = np.random.default_rng(31)
    for t in range(10):
        sh, sw = int(rng.integers(2, 120)), int(rng.integers(2, 160))
        sc = rng.uniform(0.1, 1.0) if t % 3 else rng.uniform(1.0, 3.0)
        size = (max(1, int(round(sw * sc))), max(1, int(round(sh * sc))))
        src = rng.integers(0, 256, (sh, sw, 3) if t % 2 else (sh, sw), dtype=np.uint8)
        replay.assert_exact(images.resize_exact(src, size), oracle.resize_linear_exact(src, size), f"resize fuzz {t}")

    class Scaler:  # what megapix_scaler.py's scalers offer to images.py:120-123
        def get_scaled_img_size(self, size):
            return (size[0] // 3, size[1] // 3)

    img = rigs.synth_image(90, 120, 1)
    assert images.resize_img_by_scaler(Scaler(), (120, 90), img).shape == (30, 40, 3)


def test_timelapser_drop_in(use_emu, oracle):
    """Timelapser (the other sink of the warped frames) through the C ABI == the reference's goldens == the oracle, from host
    arrays and from device twins; interface constants and file naming as the reference's."""
    from stitching_b200 import Timelapser

    replay.run_timelapse_goldens(Timelapser)
    replay.timelapse_fuzz(oracle, Timelapser, Warper, rigs, 25)
    t = Timelapser("crop", "x_")
    assert (Timelapser.TIMELAPSE_CHOICES, Timelapser.DEFAULT_TIMELAPSE, Timelapser.DEFAULT_TIMELAPSE_PREFIX) == (("no", "as_is", "crop"), "no", "fixed_")
    assert t.do_timelapse and t.get_fixed_filename("/a/b/c.jpg") == "/a/b/x_c.jpg"
    off = Timelapser()
    assert not off.do_timelapse and off.timelapser is None
    with pytest.raises(AttributeError):
        off.initialize([(0, 0)], [(4, 4)])
    touching = Timelapser("crop")  # rects that share only an edge: empty intersection canvas, get_frame fails like the reference's
    touching.initialize([(0, 0), (40, 0)], [(40, 30), (40, 30)])
    touching.process_frame(rigs.noise_image(30, 40, 1), (0, 0))
    with pytest.raises(StitchingError):
        touching.get_frame()


def test_exposure_gain_drop_in_and_fused(use_emu, oracle):
    """ExposureErrorCompensator.apply through the C ABI == the reference's goldens == the oracle; the fused
    Compositor.set_gain == warp -> apply -> feed."""
    from stitching_b200 import exposure_error_compensator as ec

    replay.run_gain_goldens(lambda img, gain: ec.apply_gain(img.copy(), gain))
    rng = np.random.default_rng(21)
    for t in range(8):
        h, w = int(rng.integers(20, 160)), int(rng.integers(20, 200))
        img = rigs.noise_image(h, w, 300 + t)
        gain = rng.uniform(0.5, 2.5, (int(rng.integers(1, 9)), int(rng.integers(1, 9))) + ((3,) if t % 2 else ())).astype(np.float32)
        replay.assert_exact(ec.apply_gain(img.copy(), gain), oracle.gain_apply(img, gain), f"gain map fuzz {t}")
    got, ref, pano0 = replay.fused_gain_case(oracle, Warper, Blender, Compositor, rigs, 25)
    replay.assert_exact(got[0], ref[0], "pano with fused exposure gains")
    replay.assert_exact(got[1], ref[1], "mask with fused exposure gains")
    assert not np.array_equal(got[0], pano0), "removing a gain must change the panorama back"


def _twin_chain(oracle):
    """warp -> crop (slicing, cropper.py:150-151) -> ExposureErrorCompensator.apply -> Blender.feed / blend with the warped
    images' device twins, against the same chain on plain host copies of the same arrays."""
    from stitching_b200 import Blender, Warper, device_array, exposure_error_compensator, rigs

    cfg = rigs.config("cfg2", 20)
    cams = cfg["cameras"][:3]
    imgs = [rigs.synth_image(cfg["h"], cfg["w"], 5 + i) for i in range(3)]
    sizes = [(cfg["w"], cfg["h"])] * 3
    warper = Warper("spherical")
    warper.set_scale(cams)
    warped = list(warper.warp_images(imgs, cams))
    masks = list(warper.create_and_warp_masks(sizes, cams))
    corners, wsizes = warper.warp_rois(sizes, cams)
    assert all(isinstance(w, device_array.DeviceBacked) and device_array.twin(w) is not None and not w.flags.writeable for w in warped)
    assert all(type(m) is np.ndarray and m.flags.writeable for m in masks), "masks stay plain ndarrays (cv2 writes into them)"
    # what leaves the twin: copies and conversions; what keeps it: plain 2-D slices
    assert device_array.twin(warped[0].astype(np.int16)) is None and device_array.twin(warped[0].copy()) is None
    assert device_array.twin(warped[0][::2]) is None and device_array.twin(warped[0] + 1) is None
    crop = (slice(3, -5), slice(7, -2))
    cropped = [w[crop] for w in warped]
    cmasks = [m[crop] for m in masks]
    ccorners = [(c[0] + 7, c[1] + 3) for c in corners]
    csizes = [(w.shape[1], w.shape[0]) for w in cropped]
    for w in cropped:
        tw = device_array.twin(w)
        assert tw is not None and tw[1:] == (7, 3, w.shape[1], w.shape[0])
    rng = np.random.default_rng(3)
    gains = [rng.uniform(0.8, 1.2, (4, 5)).astype(np.float32), np.float64(1.07), None]
    plain = [np.array(w) for w in cropped]  # host copies without twins: the reference path of the same drop-ins
    for w, p, g in zip(cropped, plain, gains):
        out = exposure_error_compensator.apply_gain(w, g)
        assert out is w and device_array.twin(out) is not None, "apply modifies its argument in place and returns it"
        exposure_error_compensator.apply_gain(p, g)
        assert np.array_equal(np.asarray(w), p)
    res = []
    for feed_imgs in (cropped, plain):
        b = Blender("multiband", 5)
        b.prepare(ccorners, csizes)
        for im, m, c in zip(feed_imgs, cmasks, ccorners):
            b.feed(im, m, c)
        res.append(b.blend())
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
    assert res[0][1].any()
    return res[0]


def test_device_twins_through_warp_crop_compensate_feed(use_emu, oracle):
    _twin_chain(oracle)


def _compositor_other_projections(oracle, names):
    """The fused compositor with the projections whose maps the library's host code builds (and mercator, which runs from
    tables): a small yaw ring per projection against the oracle's warp + blend."""
    for k, name in enumerate(names):
        cfg = rigs.config("cfg2", 25)
        cfg = dict(cfg, warper=name)
        cams = cfg["cameras"][2:5]
        imgs = [rigs.noise_image(cfg["h"], cfg["w"], 2000 + 10 * k + i) for i in range(len(cams))]
        ref = replay.oracle_composite(oracle, cfg, cams, imgs)
        c = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), name, "multiband", 5)
        assert [r[:2] for r in c.rects] == [tuple(x) for x in ref["corners"]], name
        pano, mask = c.composite(imgs)
        replay.assert_exact(pano, ref["pano"], f"{name} pano")
        replay.assert_exact(mask, ref["pmask"], f"{name} mask")
        c.close()


def test_compositor_with_the_other_projections(use_emu, oracle):
    _compositor_other_projections(oracle, ["fisheye", "compressedPlaneA2B1", "paniniPortraitA1.5B1", "mercator", "transverseMercator", "stereographic"])


# -- seeded random rigs (tests/rig_fuzz.py) through the emulation build, bit for bit against the oracle -------------------
_EMU_SEED = rig_fuzz.seed_from_env()


@pytest.mark.parametrize("k", range(len(rig_fuzz.emu_ids())), ids=rig_fuzz.emu_ids())
def test_rig_fuzz_against_oracle(use_emu, oracle, monkeypatch, k):
    """One random rig (or one named rig that aims at a branch): rects, pano roi, num_bands, every warped image and mask,
    the panorama and its mask equal the oracle's.  The named cases run the shuffle pyrDown (SB_EMU_LANES) or the tile
    collapse (SB_EMU_BLOCKS) of the emulation build."""
    case = rig_fuzz.emu_set(_EMU_SEED)[k]
    for key, v in case.env.items():
        monkeypatch.setenv(key, v)
    imgs, ex = rig_fuzz.images(case), rig_fuzz.extras(case)
    ref = rig_fuzz.oracle_run(oracle, case, imgs, ex)
    got = rig_fuzz.compositor_run(Compositor, case, imgs, ex)
    rig_fuzz.check(case, got, ref, _EMU_SEED)


def test_rig_fuzz_coverage_under_emulation(oracle):
    """The emulated fuzz set reaches the branches the emulation build can run, by the launchers' own predicates."""
    cs = rig_fuzz.emu_set(_EMU_SEED)
    rows = [(c, rig_fuzz.emu_coverage(c)) for c in cs]
    print(f"\nrig fuzz coverage, emulation set (seed {_EMU_SEED}, {len(cs)} cases):\n" + rig_fuzz.coverage_table(rows))
    reached = set().union(*(t for _, t in rows))
    want = {"nb=0", "nb=1", "nb>=2", "feather", "no", "n>32", "odd pano width", "map projection", "mixed extras",
            "gray blend mask", "k_warp_rgbm<HAS_BM=1>", "k_warp_rgbm<HAS_BM=0>", "tile l0 yes", "tile l0 no",
            "k_pyrdown_walk<1,0,1>", "k_pyrdown_walk<0,1,1>", "k_pyrdown_walk<0,0,0>", "k_pyrdown_walk<1,1,0>"}
    assert want <= reached, f"not reached: {sorted(want - reached)}"
    lanes_gray = [c for c in cs if "SB_EMU_LANES" in c.env and c.blender == "multiband" and
                  any(m in ("ramp", "random") for m in c.masks)]
    assert lanes_gray, "a gray set_mask must run through the shuffle pyrDown (BIN off)"
    assert rig_fuzz.redraw_share(cs) < 0.5, f"{rig_fuzz.redraw_share(cs):.2f} rejected draws per case"
