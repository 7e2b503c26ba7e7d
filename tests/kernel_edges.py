"""Cases aimed at single arithmetic decisions of the kernels that random rigs rarely or never reach (helper module: no
tests in here; tests/test_kernel_edges.py runs them in the emulation build, tests/test_gpu_kernel_edges.py on the GPU,
tests/mutants.py names them as the killers of its faults).

* Weight-pyramid orders: Blender cases with gray masks, so that the binary-mask shortcut is off and the float weight
  pyrDown runs in OpenCV's position-dependent summation orders (sb_pyramid.cuh).  The padded rects' level widths cover
  every residue of width0 and dw mod 4, and widths whose SIMD body is empty.  A weight one ulp off reaches the uint8
  panorama only when it flips a truncation, so the seeds in ORDER_SEEDS were searched (`python tests/kernel_edges.py
  --search`): for each order fault of tests/mutants.py, the first seeds of `orders_case` whose result the faulty library
  gets wrong.  Every seed runs twice: once comparing the int16 result, once the uint8 one only (level 0 then runs in
  the tile kernel on the GPU).
* A gain product of exactly 2^31 (value 128, gain 2^24): cvRound gives INT_MIN, which saturates to 0.
* A ray with z == 0 exactly: a camera turned by exactly 90 degrees whose warped rect starts at the column u == 0.
* Binary masks with four to six bands (GPU): the shuffle pyrDown's single summation order is exact up to level 2 only.
"""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from stitching_b200 import rigs  # noqa: E402

# (seed, SB_EMU_LANES?) of orders_case, from --search: 18 kills gather_h_simd_x0 (and walk_h_simd_x0 under the lanes),
# 120 tap5h_order, 576 gather_v_simd_le (walk_v_simd_le), 808 tap5v_order, 17527 hs_end_late
ORDER_SEEDS = [(18, False), (120, False), (576, False), (808, False), (17527, False),
               (18, True), (120, True), (576, True), (808, True)]


# -- weight-pyramid orders ------------------------------------------------------------------------------------------------
def orders_case(seed):
    """A gray-mask multiband Blender case: images (uint8), masks, corners, the strength and whether the int16 result is
    compared.  Narrow images piled on one spot: the border and tail columns, whose order differs from the SIMD body's,
    are a large share of every level, and several weights meet in every pixel's normalisation."""
    rng = np.random.default_rng(seed)
    nb = int(rng.choice([1, 2, 2, 3, 3]))
    n = int(rng.integers(2, 6))
    imgs, masks, corners = [], [], []
    for i in range(n):
        w, h = int(rng.integers(2, 24)), int(rng.integers(6, 28))
        corners.append((int(rng.integers(-8, 8)), int(rng.integers(-6, 6))))
        imgs.append(rigs.noise_image(h, w, seed * 10 + i))
        kind = rng.random()
        if kind < 0.3:
            m = rng.integers(0, 256, (h, w))
        elif kind < 0.7:  # mostly full weight with gray specks: sums near integers
            m = np.where(rng.random((h, w)) < 0.2, rng.integers(1, 255, (h, w)), 255)
        else:  # a ramp
            m = np.minimum(np.arange(w)[None, :] * 255 // max(1, w - 1) + rng.integers(0, 40), 255) * np.ones((h, 1), np.int64)
        masks.append(m.astype(np.uint8))
    x0 = min(c[0] for c in corners)
    y0 = min(c[1] for c in corners)
    W = max(c[0] + im.shape[1] for c, im in zip(corners, imgs)) - x0
    H = max(c[1] + im.shape[0] for c, im in zip(corners, imgs)) - y0
    strength = 2.0 ** (nb + 1.5) * 100 / math.sqrt(W * H)
    return dict(imgs=imgs, masks=masks, corners=corners, strength=strength)


def order_widths(case):
    """(width0 % 4, dw % 4, SIMD body empty) of every level the float pyrDown filters, from the padded rects (restated
    from BlendPlan::set_geometry / add_feed, as rig_fuzz.plan does)."""
    sizes = [(im.shape[1], im.shape[0]) for im in case["imgs"]]
    x0 = min(c[0] for c in case["corners"])
    y0 = min(c[1] for c in case["corners"])
    w = max(c[0] + s[0] for c, s in zip(case["corners"], sizes)) - x0
    h = max(c[1] + s[1] for c, s in zip(case["corners"], sizes)) - y0
    bw = math.sqrt(w * h) * case["strength"] / 100
    nb = min(int(math.log(bw) / math.log(2.0) - 1.0), int(math.ceil(math.log(max(w, h)) / math.log(2.0))))
    a, gap = 1 << nb, 3 << nb
    wp = -(-w // a) * a
    out = set()
    for (tx, ty), (fw, fh) in zip(case["corners"], sizes):
        px0 = max(x0, tx - gap)
        px1 = min(x0 + wp, tx + fw + gap)
        px0 = x0 + (((px0 - x0) >> nb) << nb)
        pw = -(-(px1 - px0) // a) * a
        for l in range(nb):
            sw = pw >> l
            dw = (sw + 1) // 2
            width0 = min((sw - 3) // 2 + 1, dw)
            out.add((width0 % 4, (sw >> 1) % 4, width0 < 5))
    return out


def run_orders(O, case, Blender, s16):
    """(got, want): the panorama (and the int16 result when the case asks for it) from Blender and the oracle."""
    a, b = Blender("multiband", case["strength"]), O.Blender("multiband", case["strength"])
    sizes = [(im.shape[1], im.shape[0]) for im in case["imgs"]]
    for bl in (a, b):
        bl.prepare(case["corners"], sizes)
        for im, m, c in zip(case["imgs"], case["masks"], case["corners"]):
            bl.feed(im, m, c)
    if s16:
        got = a.blender.blend(want_s16=True)
        want = b.blend_s16()
        return (got[2], got[1]), want
    return a.blend(), b.blend()


def check_orders(O, seed, monkeypatch=None, lanes=False, s16=True):
    import replay
    from stitching_b200 import Blender

    if lanes:
        monkeypatch.setenv("SB_EMU_LANES", "1")
    case = orders_case(seed)
    (g0, g1), (w0, w1) = run_orders(O, case, Blender, s16)
    what = f"orders seed {seed}{' (lanes)' if lanes else ''} {'int16' if s16 else 'uint8'}"
    replay.assert_exact(g0, w0, what)
    replay.assert_exact(g1, w1, what + " mask")


# -- a gain product of exactly 2^31 ---------------------------------------------------------------------------------------
def gain_image(h, w):
    """Columns of 127, 128, 129 and a ramp: products just below, at and above 2^31 with a gain of 2^24."""
    img = np.empty((h, w, 3), np.uint8)
    img[:] = np.array([127, 128, 129], np.uint8)[(np.arange(w) // 3) % 3][None, :, None]
    img[:, :, 1] = np.roll(img[:, :, 1], 1, axis=1)
    img[::4] = np.arange(w, dtype=np.uint8)[None, :, None] + 100
    return img


def check_gain_2p31(O):
    import replay
    from stitching_b200 import Compositor, Warper
    from stitching_b200 import exposure_error_compensator as ec

    img = gain_image(24, 40)
    gains = {"scalar": np.array([[2.0 ** 24]], np.float64), "map1": np.full((3, 4), 2.0 ** 24, np.float32),
             "map3": np.full((2, 3, 3), 2.0 ** 24, np.float32)}
    for name, g in gains.items():
        want = O.gain_apply(img, g)
        assert (want[img == 128] == 0).all() and (want[img == 127] == 255).all(), f"oracle, gain 2^24 {name}"
        replay.assert_exact(np.asarray(ec.apply_gain(img.copy(), g)), want, f"apply, gain 2^24 {name}")
    # the same gains in the warp kernel: a whole-pixel translation, whose warp is an exact copy
    cams = [rigs.Camera(1, 1, 0, 0, np.array([[1, 0, 40.0 * i], [0, 1, 0], [0, 0, 1]], np.float32)) for i in range(3)]
    c = Compositor(cams, [(40, 24)] * 3, "affine", "no", 5)
    try:
        for i, g in enumerate(gains.values()):
            c.set_gain(i, g)
        c.composite([img] * 3)
        for i, (name, g) in enumerate(gains.items()):
            wi, _ = c.download_warped(i)
            rect, oi, _ = O.warp("affine", np.float32(1.0), Warper.get_K(cams[i], 1), cams[i].R, img)
            replay.assert_exact(wi, O.gain_apply(oi, g), f"Compositor.set_gain 2^24 {name}")
    finally:
        c.close()


# -- a ray with z == 0 -----------------------------------------------------------------------------------------------------
# Optical axis along world +x (the third column of R is (1, 0, 0)), so the backward map's z is x_ = rowA * sin(u / s):
# exactly 0 in the column u == 0.  The principal point lies far right of the image, whose rays then come within less than
# a pixel of world +z, so the warped rect starts at u == 0 (roi truncation).
Z0_R = np.array([[0, 0, 1], [0, 1, 0], [-1, 0, 0]], np.float32)


def z0_cameras():
    return [rigs.Camera(8.0, 1.0, 128.0, 30.0, Z0_R), rigs.Camera(8.0, 1.0, 60.0, 30.0, Z0_R)]


def check_z_zero(O, wtype):
    import replay
    from stitching_b200 import Compositor, Warper

    cams = z0_cameras()
    imgs = [rigs.noise_image(60, 120, 70 + i) for i in range(len(cams))]
    w = Warper(wtype)
    w.set_scale(cams)
    scale = np.float32(w.scale)
    c = Compositor(cams, [(120, 60)] * len(cams), wtype, "no", 5)
    try:
        c.composite(imgs)
        hit = False
        for i, (cam, img) in enumerate(zip(cams, imgs)):
            rect, wi, wm = O.warp(wtype, scale, Warper.get_K(cam, 1), cam.R, img)
            hit = hit or rect[0] == 0
            replay.assert_exact(np.asarray(w.warp_image(img, cam)), wi, f"{wtype} Warper.warp_image {i}")
            gi, gm = c.download_warped(i)
            replay.assert_exact(gi, wi, f"{wtype} Compositor.download_warped image {i}")
            replay.assert_exact(gm, wm, f"{wtype} Compositor.download_warped mask {i}")
        assert hit, "a warped rect must start at the column u == 0"
    finally:
        c.close()


# seeds of bin_case whose panorama shows it when level 3 of binary masks takes the single summation order (the first
# three of 15285 searched on an H100 with that fault; its level-4 weights need more than 24 bits)
BIN_SEEDS = [4377, 7789, 10608]


# -- binary masks, four or more bands: level 3 of the shuffle pyrDown needs the reference's orders again -----------------
def bin_case(seed):
    """A compositor rig of sheared affine images without blend masks (the pyrDown's binary-mask shortcut), 4 to 6 bands."""
    import rig_fuzz

    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 5))
    sizes = [(int(rng.integers(40, 140)), int(rng.integers(40, 120))) for _ in range(n)]
    cams = rig_fuzz._affine_cams(rng, sizes)
    c = rig_fuzz.Case(f"bin_{seed}", "affine", cams, sizes, "multiband", 0.0, ["none"] * n, ["none"] * n, ["noise"] * n, seed)
    c.rects = rig_fuzz._rects(c.wtype, c.cams, c.sizes)
    x, y, w, h = c.roi()
    c.strength = 2.0 ** (int(rng.integers(4, 7)) + 1.5) * 100 / math.sqrt(w * h)
    return c


def check_bin(O, seed):
    import rig_fuzz
    from stitching_b200 import Compositor

    c = bin_case(seed)
    imgs, ex = rig_fuzz.images(c), rig_fuzz.extras(c)
    rig_fuzz.check(c, rig_fuzz.compositor_run(Compositor, c, imgs, ex), rig_fuzz.oracle_run(O, c, imgs, ex), seed)


# -- the case lists ------------------------------------------------------------------------------------------------------
def emu_cases():
    """(case id, fn(oracle module, monkeypatch))"""
    out = [(f"orders_{s}_{'s16' if s16 else 'u8'}" + ("_lanes" if lanes else ""),
            lambda O, mp, s=s, lanes=lanes, s16=s16: check_orders(O, s, mp, lanes, s16))
           for s, lanes in ORDER_SEEDS for s16 in (True, False)]
    out += [("gain_2p31", lambda O, mp: check_gain_2p31(O)),
            ("z_zero_spherical", lambda O, mp: check_z_zero(O, "spherical")),
            ("z_zero_cylindrical", lambda O, mp: check_z_zero(O, "cylindrical"))]
    return out


def gpu_cases():
    """(case id, fn(oracle module)): every case above on the device (the lane emulation is the GPU's own)."""
    out = [(f"orders_{s}_{'s16' if s16 else 'u8'}", lambda O, s=s, s16=s16: check_orders(O, s, s16=s16))
           for s in sorted({s for s, _ in ORDER_SEEDS}) for s16 in (True, False)]
    out += [(f"bin_{s}", lambda O, s=s: check_bin(O, s)) for s in BIN_SEEDS]
    out += [("gain_2p31", check_gain_2p31),
            ("z_zero_spherical", lambda O: check_z_zero(O, "spherical")),
            ("z_zero_cylindrical", lambda O: check_z_zero(O, "cylindrical"))]
    return out


# -- the seed search -----------------------------------------------------------------------------------------------------
ORDER_FAULTS = {"tap5h_order": (False, True), "tap5v_order": (False, True), "hs_end_late": (False, True),
                "gather_h_simd_x0": (False,), "gather_v_simd_le": (False,), "walk_h_simd_x0": (True,), "walk_v_simd_le": (True,)}


def search(limit, per_fault, lanes_too):
    """For every order fault of tests/mutants.py and each build it runs in (False: the per-pixel pyrDown, True: the
    shuffle pyrDown under SB_EMU_LANES), the first `per_fault` seeds of orders_case that the faulty library gets wrong
    and the unmutated one right."""
    import tempfile

    import pytest

    import mutants
    from oracle import oracle as O
    from stitching_b200 import _lib

    O.build()
    found = {(f, lanes): [] for f, ls in ORDER_FAULTS.items() for lanes in ls if lanes_too or not lanes}
    with tempfile.TemporaryDirectory() as work:
        b = mutants.EmuBuilder(work, os.cpu_count() or 4)
        libs = {m.id: _lib.bind(b.mutant(m)) for m in mutants.CATALOGUE if m.id in ORDER_FAULTS}
        base = _lib.bind(b.lib)
        for seed in range(limit):
            for lanes in (False, True):
                todo = [f for (f, ln), s in found.items() if ln == lanes and len(s) < per_fault]
                if not todo:
                    continue
                with pytest.MonkeyPatch.context() as mp:
                    mp.setattr(_lib, "_lib", base)
                    check_orders(O, seed, mp, lanes, seed % 2 == 0)  # the unmutated library must agree with the oracle
                    for f in todo:
                        mp.setattr(_lib, "_lib", libs[f])
                        try:
                            check_orders(O, seed, mp, lanes, seed % 2 == 0)
                        except AssertionError:
                            found[(f, lanes)].append(seed)
                            print(f"{f}{' (lanes)' if lanes else ''}: seed {seed}", flush=True)
            if all(len(s) >= per_fault for s in found.values()):
                break
    return found


if __name__ == "__main__":
    import argparse

    ap = argparse.ArgumentParser(description="search the seeds of ORDER_SEEDS")
    ap.add_argument("--search", action="store_true", required=True)
    ap.add_argument("--limit", type=int, default=3000)
    ap.add_argument("--per-fault", type=int, default=1)
    ap.add_argument("--lanes", action="store_true", help="also search under SB_EMU_LANES (slow)")
    a = ap.parse_args()
    res = search(a.limit, a.per_fault, a.lanes)
    seeds = sorted({(s, lanes) for (f, lanes), ss in res.items() for s in ss})
    print("not found:", [k for k, v in res.items() if not v])
    print("ORDER_SEEDS =", seeds)
