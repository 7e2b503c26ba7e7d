"""Parity of the CUDA path (through the C ABI / Python drop-ins) against the CPU oracle and the golden vectors.

Bar (BASELINE.json north_star): final uint8 panorama within +-1 LSB per channel, roi / corners / sizes /
num_bands / masks exact.  The tests assert the stronger property the design aims at -- bit-exact -- and
print the mismatch histogram when that fails, so a +-1 result is visible as such.
"""
import os
import time

import numpy as np
import pytest

import replay
from stitching_b200 import Blender, Compositor, Warper, rigs

pytestmark = pytest.mark.gpu


def histogram(got, exp):
    d = np.abs(got.astype(np.int64) - exp.astype(np.int64)).ravel()
    vals, counts = np.unique(d, return_counts=True)
    return {int(v): int(c) for v, c in zip(vals, counts)}


def assert_parity(got, exp, what):
    assert got.shape == exp.shape, f"{what}: shape {got.shape} vs {exp.shape}"
    if not np.array_equal(got, exp):
        h = histogram(got, exp)
        assert max(h) <= 1, f"{what}: beyond +-1 LSB, |diff| histogram {h}"
        pytest.fail(f"{what}: within +-1 LSB but not bit-exact, |diff| histogram {h}")


def test_native_library_is_the_one_running(cuda_lib):
    import ctypes as C

    name = C.create_string_buffer(128)
    sm, maj, mnr = C.c_int(), C.c_int(), C.c_int()
    assert cuda_lib.sb_device_info(name, 128, C.byref(sm), C.byref(maj), C.byref(mnr)) == 0
    assert (maj.value, mnr.value) == (9, 0), f"not an sm_90 device: {name.value} sm_{maj.value}{mnr.value}"
    before = cuda_lib.sb_launch_count()
    cams = rigs.yaw_ring(1, 64, 48, 70, 0)
    w = Warper()
    w.set_scale(cams)
    w.warp_image(rigs.noise_image(48, 64, 0), cams[0])
    assert cuda_lib.sb_launch_count() > before, "no kernel was launched"
    with open(f"/proc/{os.getpid()}/maps") as f:
        assert "libstitch_b200.so" in f.read()


@pytest.mark.parametrize("mode", [0, 1])
def test_shared_reciprocal_division_is_the_ieee_division(cuda_lib, mode):
    """The warp and collapse kernels divide through one refined reciprocal per pixel (sb_device.cuh); over the operand
    ranges they guarantee it must be the IEEE quotient bit for bit: 2^32 pseudo-random pairs per mode on the device."""
    import ctypes as C

    bad = C.c_ulonglong(123)
    assert cuda_lib.sb_selftest_division(1 << 32, 2026 + mode, mode, C.byref(bad)) == 0
    assert bad.value == 0, f"mode {mode}: {bad.value} of 2^32 quotients differ from __fdiv_rn"


def test_seam_resize_goldens_fuzz_and_fused(cuda_lib, oracle):
    """SeamFinder.resize on the device: the reference's goldens, fuzz against the oracle, and the fused
    Compositor.set_seam_mask against set_mask(SeamFinder.resize(..)) -- all bit-exact."""
    from stitching_b200 import seam_finder

    replay.run_seam_goldens(seam_finder.resize)
    rng = np.random.default_rng(12)
    for t in range(16):
        sh, sw = int(rng.integers(3, 200)), int(rng.integers(3, 260))
        h, w = max(2, int(sh * rng.uniform(0.5, 8))), max(2, int(sw * rng.uniform(0.5, 8)))
        seam = rng.integers(0, 256, (sh, sw), dtype=np.uint8) if t % 2 else (rng.random((sh, sw)) < 0.5).astype(np.uint8) * 255
        mask = (rng.random((h, w)) < 0.9).astype(np.uint8) * 255
        assert_parity(seam_finder.resize(seam, mask), oracle.seam_resize(seam, mask), f"seam resize fuzz {t}")
    cfg = rigs.config("cfg2", 4)
    cams = cfg["cameras"]
    sizes = [(cfg["w"], cfg["h"])] * len(cams)
    imgs = [rigs.synth_image(cfg["h"], cfg["w"], 60 + i) for i in range(len(cams))]
    a = Compositor(cams, sizes, cfg["warper"], cfg["blender"], cfg["strength"])
    b = Compositor(cams, sizes, cfg["warper"], cfg["blender"], cfg["strength"])
    a.composite(imgs)
    valid = [a.download_warped(i)[1] for i in range(len(cams))]
    seams = replay.seam_masks_low(valid)
    for i, s in enumerate(seams):
        a.set_mask(i, oracle.seam_resize(s, valid[i]))
        b.set_seam_mask(i, s)
    pa, ma = a.composite(imgs)
    pb, mb = b.composite(imgs)
    assert_parity(pb, pa, "pano with fused seam masks")
    assert_parity(mb, ma, "mask with fused seam masks")
    a.close()
    b.close()


def test_warper_goldens(cuda_lib):
    replay.run_warper_goldens(Warper)


def test_blender_goldens(cuda_lib):
    replay.run_blender_goldens(Blender)


def test_e2e_goldens(cuda_lib):
    replay.run_e2e_goldens(Warper, Blender)


def test_warp_fuzz_against_oracle(cuda_lib, oracle):
    rng = np.random.default_rng(42)
    for t in range(24):
        wtype = ["spherical", "cylindrical", "plane", "affine"][t % 4]
        w, h = int(rng.integers(60, 700)), int(rng.integers(60, 500))
        img = rigs.noise_image(h, w, 500 + t)
        if wtype == "affine":
            th, s = rng.uniform(-0.2, 0.2), rng.uniform(0.8, 1.2)
            R = np.array([[s * np.cos(th), -s * np.sin(th), rng.uniform(-300, 300)],
                          [s * np.sin(th), s * np.cos(th), rng.uniform(-200, 200)], [0, 0, 1]], np.float32)
            cam, scale = rigs.Camera(1.0, 1.0, 0.0, 0.0, R), 1.0
        else:
            f = float(rng.uniform(0.5, 2.0) * max(w, h))
            if wtype == "plane":
                R = rigs.rot_y(rng.uniform(-0.6, 0.6)) @ rigs.rot_x(rng.uniform(-0.4, 0.4))
            elif t % 8 == 0:
                R = rigs.rot_y(rng.uniform(-3, 3)) @ rigs.rot_x(rng.uniform(1.0, 1.8))  # pole in view
            else:
                R = rigs.rot_y(rng.uniform(-3.1, 3.1)) @ rigs.rot_x(rng.uniform(-0.5, 0.5))
            cam = rigs.Camera(f, float(rng.uniform(0.95, 1.05)), w / 2 + rng.uniform(-10, 10), h / 2 + rng.uniform(-10, 10), R)
            scale = float(f * rng.uniform(0.6, 1.4))
        wr = Warper(wtype)
        wr.scale = scale
        rect, oi, om = oracle.warp(wtype, scale, Warper.get_K(cam, 1), cam.R, img)
        assert tuple(wr.warp_roi((w, h), cam)) == rect
        gi, gm = wr.warp_image_and_mask(img, cam)
        assert_parity(gi, oi, f"warp fuzz {t} {wtype} image")
        assert np.array_equal(gm, om), f"warp fuzz {t} {wtype} mask"
        assert np.array_equal(wr.warp_image(img, cam), gi) and np.array_equal(wr.create_and_warp_mask((w, h), cam), gm)


def test_blend_fuzz_against_oracle(cuda_lib, oracle):
    rng = np.random.default_rng(43)
    for t in range(30):
        btype = ["multiband", "feather", "no"][t % 3]
        n = int(rng.integers(2, 6))
        imgs, masks, corners = [], [], []
        for i in range(n):
            w, h = int(rng.integers(17, 420)), int(rng.integers(17, 330))
            img = rigs.noise_image(h, w, 900 + 10 * t + i) if t % 2 else rigs.synth_image(h, w, 900 + 10 * t + i)
            kind = t % 5
            if kind == 0:
                m = np.full((h, w), 255, np.uint8)
            elif kind == 1:
                m = (rng.random((h, w)) > 0.3).astype(np.uint8) * 255
            elif kind == 2:
                m = rng.integers(0, 256, (h, w), dtype=np.uint8)
            elif kind == 3:
                m = np.zeros((h, w), np.uint8)
                m[h // 5: h - h // 6, w // 7: w - w // 5] = 255
            else:
                m = np.clip(np.add.outer(np.arange(h), np.arange(w)) * 2, 0, 255).astype(np.uint8)
            if t % 4 == 3:
                img = img.astype(np.int16) * 3 - 200
            imgs.append(img)
            masks.append(m)
            corners.append((int(rng.integers(-300, 300)), int(rng.integers(-200, 200))))
        strength = float(rng.choice([1, 5, 20, 60, 100]))
        sizes = [(m.shape[1], m.shape[0]) for m in masks]
        o = oracle.Blender(btype, strength)
        o.prepare(corners, sizes)
        b = Blender(btype, strength)
        b.prepare(corners, sizes)
        if o.num_bands is not None:
            assert b.blender.num_bands == o.num_bands
        for img, m, c in zip(imgs, masks, corners):
            o.feed(img, m, c)
            b.feed(img, m, c)
        os16, om = o.blend_s16()
        if t % 4 in (0, 3):
            pano, pmask, s16 = b.blender.blend(want_s16=True)
            assert_parity(s16, os16, f"blend fuzz {t} {btype} int16 result")
        else:  # uint8 result only: level 0 of the collapse may run in the tile kernel (it never writes int16)
            pano, pmask = b.blender.blend()
        assert_parity(pano, oracle.convert_scale_abs(os16), f"blend fuzz {t} {btype} uint8 result")
        assert np.array_equal(pmask, om), f"blend fuzz {t} {btype} mask"


@pytest.mark.parametrize("name,scale_down,ncap", [("cfg2", 4, None), ("cfg3", 8, 8), ("cfg4", 8, None), ("cfg5", 2, None)])
def test_compositor_against_oracle(cuda_lib, oracle, name, scale_down, ncap):
    cfg = rigs.config(name, scale_down)
    cams = cfg["cameras"][:ncap] if ncap else cfg["cameras"]
    imgs = [rigs.noise_image(cfg["h"], cfg["w"], 1000 + i) if i % 2 else rigs.synth_image(cfg["h"], cfg["w"], i)
            for i in range(len(cams))]
    ref = replay.oracle_composite(oracle, cfg, cams, imgs)
    c = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), cfg["warper"], cfg["blender"], cfg["strength"])
    assert [r[:2] for r in c.rects] == [tuple(x) for x in ref["corners"]]
    assert [r[2:] for r in c.rects] == [tuple(x) for x in ref["sizes"]]
    if cfg["blender"] == "multiband":
        assert c.num_bands == ref["num_bands"]
    pano, mask = c.composite(imgs)
    for i in range(len(cams)):
        wi, wm = c.download_warped(i)
        assert_parity(wi, ref["warped"][i], f"{name} warped image {i}")
        assert np.array_equal(wm, ref["masks"][i]), f"{name} warped mask {i}"
    assert_parity(pano, ref["pano"], f"{name} pano")
    assert np.array_equal(mask, ref["pmask"]), f"{name} pano mask"
    c.close()


def test_drop_in_classes_equal_compositor(cuda_lib):
    """The per-call drop-in path (host round trips) and the fused resident path give the same panorama."""
    cfg = rigs.config("cfg2", 4)
    cams = cfg["cameras"]
    imgs = [rigs.synth_image(cfg["h"], cfg["w"], i) for i in range(len(cams))]
    w = Warper(cfg["warper"])
    w.set_scale(cams)
    sizes_in = [(cfg["w"], cfg["h"])] * len(cams)
    corners, sizes = w.warp_rois(sizes_in, cams)
    b = Blender(cfg["blender"], cfg["strength"])
    b.prepare(corners, sizes)
    for img, m, corner in zip(w.warp_images(imgs, cams), w.create_and_warp_masks(sizes_in, cams), corners):
        b.feed(img, m, corner)
    pano, mask = b.blend()
    c = Compositor(cams, sizes_in, cfg["warper"], cfg["blender"], cfg["strength"])
    p2, m2 = c.composite(imgs)
    assert np.array_equal(pano, p2) and np.array_equal(mask, m2)


@pytest.mark.parametrize("name,scale_down", [("cfg2", 4), ("cfg5", 2)])
def test_compositor_with_seam_like_blend_masks(cuda_lib, oracle, name, scale_down):
    """Mask set B of SURVEY 8(d): gray-ramp blend masks (what SeamFinder.resize produces) instead of validity masks."""
    cfg = rigs.config(name, scale_down)
    cams = cfg["cameras"]
    imgs = [rigs.noise_image(cfg["h"], cfg["w"], 40 + i) for i in range(len(cams))]
    ref = replay.oracle_composite(oracle, cfg, cams, imgs, mask_fn=lambda ms: replay.ramp_masks(ms, 64))
    c = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), cfg["warper"], cfg["blender"], cfg["strength"])
    for i, m in enumerate(ref["masks"]):
        c.set_mask(i, m)
    pano, mask = c.composite(imgs)
    assert_parity(pano, ref["pano"], f"{name} pano with ramp masks")
    assert np.array_equal(mask, ref["pmask"])
    c.close()


@pytest.mark.parametrize("name,scale_down,world", [("cfg2", 4, 2), ("cfg3", 8, 8)])
def test_sharded_roles_on_one_gpu(cuda_lib, name, scale_down, world):
    """The kernels' multi-GPU roles (partial sums out, slabs in, strips) with all ranks on ONE device and the slabs
    moved by device copies instead of NCCL (tests/test_gpu_sharded.py covers NCCL itself when 2 GPUs are there)."""
    import test_sharded

    cfg = rigs.config(name, scale_down)
    cams = cfg["cameras"]
    imgs = [rigs.noise_image(cfg["h"], cfg["w"], 70 + i) if i % 2 else rigs.synth_image(cfg["h"], cfg["w"], 70 + i)
            for i in range(len(cams))]
    single = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), cfg["warper"], cfg["blender"], cfg["strength"])
    ref_pano, ref_mask = single.composite(imgs)
    single.close()

    def copy(dst, src, n):
        from stitching_b200 import _lib

        _lib.check(cuda_lib.sb_device_copy(dst, src, n), "sb_device_copy")

    pano, mask, moved = test_sharded.run_sharded(cfg, cams, imgs, world, copy)
    assert moved > 0 and np.array_equal(mask, ref_mask)
    d = np.abs(pano.astype(np.int32) - ref_pano.astype(np.int32))
    assert d.max() <= 1, histogram(pano, ref_pano)
    print(f"{name} x{world}: {int((d != 0).sum())} of {d.size} values differ by 1, {moved / 1e6:.1f} MB of slabs")


def test_pipelined_submit_wait(cuda_lib):
    """The 2-deep pipelined end-to-end path returns exactly what the synchronous path returns, batch by batch."""
    cfg = rigs.config("cfg2", 4)
    cams = cfg["cameras"]
    sizes = [(cfg["w"], cfg["h"])] * len(cams)
    c = Compositor(cams, sizes, cfg["warper"], cfg["blender"], cfg["strength"])
    batches = []
    for b in range(6):
        pinned = [c.pinned_empty((cfg["h"], cfg["w"], 3)) for _ in cams]
        for i, p in enumerate(pinned):
            p[...] = rigs.noise_image(cfg["h"], cfg["w"], 10 * b + i)
        batches.append(pinned)
    expected = [tuple(a.copy() for a in c.composite(b)) for b in batches]
    _, _, pw, ph = c.roi
    outs = [(c.pinned_empty((ph, pw, 3)), c.pinned_empty((ph, pw))) for _ in range(2)]
    tickets = []
    for k, b in enumerate(batches):
        if k >= 2:
            c.wait(tickets[k - 2])
            assert np.array_equal(outs[k & 1][0], expected[k - 2][0]) and np.array_equal(outs[k & 1][1], expected[k - 2][1])
        tickets.append(c.submit(b, *outs[k & 1]))
    for k in (4, 5):
        c.wait(tickets[k])
        assert np.array_equal(outs[k & 1][0], expected[k][0]) and np.array_equal(outs[k & 1][1], expected[k][1])
    c.close()


def test_simple_and_fast_kernels_agree(cuda_lib):
    """A/B inside one process is not possible (the variant is chosen once per process): run the other variant in
    a child process and compare panoramas byte for byte."""
    import subprocess
    import sys
    import tempfile

    code = (
        "import sys, numpy as np; sys.path.insert(0, sys.argv[1]);"
        "from stitching_b200 import Compositor, rigs;"
        "cfg = rigs.config('cfg2', 4); cams = cfg['cameras'];"
        "imgs = [rigs.noise_image(cfg['h'], cfg['w'], 300 + i) for i in range(len(cams))];"
        "c = Compositor(cams, [(cfg['w'], cfg['h'])] * len(cams), cfg['warper'], cfg['blender'], cfg['strength']);"
        "p, m = c.composite(imgs); np.savez(sys.argv[2], p=p, m=m)"
    )
    from conftest import ROOT

    res = {}
    with tempfile.TemporaryDirectory() as d:
        for variant in ("simple", "fast"):
            env = dict(os.environ)
            env["SB_KERNELS"] = variant
            out = os.path.join(d, variant + ".npz")
            subprocess.check_call([sys.executable, "-c", code, ROOT, out], env=env)
            z = np.load(out)
            res[variant] = (z["p"], z["m"])
    assert np.array_equal(res["simple"][0], res["fast"][0]) and np.array_equal(res["simple"][1], res["fast"][1])


def test_full_size_properties(cuda_lib, oracle):
    """BASELINE cfg 2 at full size (8 x 4000x3000, spherical, multiband): size-independent properties."""
    cfg = rigs.config("cfg2", 1)
    cams = cfg["cameras"]
    n = len(cams)
    sizes_in = [(cfg["w"], cfg["h"])] * n
    c = Compositor(cams, sizes_in, cfg["warper"], cfg["blender"], cfg["strength"])
    assert c.num_bands == 7 and c.roi[2:] == (18376, 2950), (c.num_bands, c.roi)  # SURVEY 8(d)
    # (1) a constant image blends to that constant wherever the mask is set (partition of unity up to the
    #     per-image truncation of (short)(L*w): at most one count per contributing image and level)
    const = [np.full((cfg["h"], cfg["w"], 3), (200, 90, 17), np.uint8)] * n
    pano, mask = c.composite(const)
    assert mask.any() and set(np.unique(mask)) <= {0, 255}
    inside = mask == 255
    for ch, v in enumerate((200, 90, 17)):
        d = np.abs(pano[..., ch][inside].astype(np.int32) - v)
        assert d.max() <= 2 * (c.num_bands + 1), int(d.max())
    assert not pano[~inside].any()
    # (2) determinism, and (3) one full-size warped image against the oracle
    imgs = [rigs.synth_image(cfg["h"], cfg["w"], i) for i in range(n)]
    p1, m1 = c.composite(imgs)
    p2, m2 = c.composite(imgs)
    assert np.array_equal(p1, p2) and np.array_equal(m1, m2)
    t0 = time.time()
    rect, oi, om = oracle.warp(cfg["warper"], c.scale, Warper.get_K(cams[3], 1), cams[3].R, imgs[3])
    wi, wm = c.download_warped(3)
    assert rect == c.rects[3]
    assert_parity(wi, oi, "full-size warped image 3")
    assert np.array_equal(wm, om)
    print(f"oracle full-size warp: {time.time() - t0:.1f}s")
    # (4) the mask of the panorama is the union of the warped masks placed at their corners
    union = np.zeros(mask.shape, bool)
    for i in range(n):
        _, wm = c.download_warped(i)
        x, y = c.rects[i][0] - c.roi[0], c.rects[i][1] - c.roi[1]
        union[y: y + wm.shape[0], x: x + wm.shape[1]] |= wm > 0
    assert np.array_equal(union, m1 == 255)
    c.close()


def test_against_cv2_directly_when_available(cuda_lib):
    """Same-process cross-check with the reference's numeric backend (cv2 ships in the image)."""
    cv = pytest.importorskip("cv2")
    cfg = rigs.config("cfg2", 8)
    cams = cfg["cameras"][:4]
    imgs = [rigs.noise_image(cfg["h"], cfg["w"], 77 + i) for i in range(4)]
    w = Warper("spherical")
    w.set_scale(cams)
    warped, masks, corners, sizes = [], [], [], []
    for img, cam in zip(imgs, cams):
        pw = cv.PyRotationWarper("spherical", w.scale)  # the calls of stitching/warper.py:44-51, 59-67, 80-82
        K = Warper.get_K(cam, 1)
        _, ref_img = pw.warp(img, K, cam.R, cv.INTER_LINEAR, cv.BORDER_REFLECT)
        _, ref_mask = pw.warp(255 * np.ones(img.shape[:2], np.uint8), K, cam.R, cv.INTER_NEAREST, cv.BORDER_CONSTANT)
        roi = pw.warpRoi((cfg["w"], cfg["h"]), K, cam.R)
        gi, gm = w.warp_image_and_mask(img, cam)
        assert tuple(w.warp_roi((cfg["w"], cfg["h"]), cam)) == tuple(roi)
        assert_parity(gi, ref_img, "cv2 warp image")
        assert np.array_equal(gm, ref_mask)
        warped.append(gi); masks.append(gm); corners.append(roi[0:2]); sizes.append(roi[2:4])
    dst = cv.detail.resultRoi(corners=corners, sizes=sizes)
    bw = np.sqrt(dst[2] * dst[3]) * 5 / 100
    mb = cv.detail_MultiBandBlender()  # the calls of stitching/blender.py:31-32, 38, 41, 46-47
    mb.setNumBands(int(np.log(bw) / np.log(2.0) - 1.0))
    mb.prepare(dst)
    b = Blender("multiband", 5)
    b.prepare(corners, sizes)
    for img, m, c in zip(warped, masks, corners):
        mb.feed(cv.UMat(img.astype(np.int16)), m, c)
        b.feed(img, m, c)
    ref, ref_mask = mb.blend(None, None)
    pano, pmask = b.blend()
    assert_parity(pano, cv.convertScaleAbs(ref), "cv2 multiband pano")
    assert np.array_equal(pmask, ref_mask)


def _full_size_case(name, n_images=None, noise=False):
    """GPU composite vs the reference's cv2 call sequence (oracle/cv_path.py) on the same full-size inputs."""
    pytest.importorskip("cv2")
    from oracle import cv_path

    cfg = rigs.config(name, 1)
    cams = cfg["cameras"][: n_images or cfg["n"]]
    n = len(cams)
    gen = rigs.noise_image if noise else rigs.synth_image
    imgs = [gen(cfg["h"], cfg["w"], 40 + i) for i in range(n)]
    c = Compositor(cams, [(cfg["w"], cfg["h"])] * n, cfg["warper"], cfg["blender"], cfg["strength"])
    pano, mask = c.composite(imgs)
    nb = c.num_bands
    c.close()
    t0 = time.time()
    ref_pano, ref_mask, _ = cv_path.composite(cfg, cams, imgs, os.cpu_count())
    if hasattr(ref_mask, "get"):
        ref_mask = ref_mask.get()
    print(f"{name}/{n}: cv2 reference path {time.time() - t0:.1f} s, pano {pano.shape}, {nb} bands")
    assert_parity(pano, ref_pano, f"{name}/{n} full-size panorama vs cv2")
    assert np.array_equal(mask, ref_mask), f"{name}/{n}: {int((mask != ref_mask).sum())} mask values differ"
    return nb


def test_benchmarked_configuration_at_full_size_against_cv2(cuda_lib):
    """EXACTLY what bench.py times at N = 1 -- BASELINE configs[1]: 8 x 4000x3000, spherical, multiband, 7 bands -- end to
    end against the reference's CPU path: panorama and mask bit for bit (the reference's own tests pin only the shape,
    tests/test_stitcher.py:229-231)."""
    assert _full_size_case("cfg2") == 7


def test_other_configurations_at_full_size_against_cv2(cuda_lib):
    """configs[4] (16 x 2000x1500 affine + feather) whole; configs[2] (cylindrical, f = 8000) and configs[3]
    (8000x6000 spherical) at full image size on the first images of their rings (what cv2 finishes in about a minute);
    cfg 2 once more on pure noise, the adversarial input for rounding."""
    _full_size_case("cfg5")
    _full_size_case("cfg3", 12)
    _full_size_case("cfg4", 3)
    _full_size_case("cfg2", 4, noise=True)
