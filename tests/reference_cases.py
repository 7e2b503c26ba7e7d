"""Seeded cases whose results the unmodified reference (OpenStitching/stitching 0.7.0 on cv2 4.13.0) returned, pinned
in tests/golden/golden_reference.npz by tests/golden/gen_golden.py.

tests/test_vs_reference_live.py and tests/test_dropin_pipeline.py build the same inputs from the same seeds, run the
oracle or the product's classes on them and compare with the pins: arrays by shape, dtype and SHA-256 of their bytes
(bit for bit, like replay.assert_exact), small values (rois, corners, sizes, gains, cameras, seam masks) as they are.
"""
import hashlib
import os

import numpy as np

from stitching_b200 import rigs

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_reference.npz")
SEED = 20260923
WARP_TYPES = ("spherical", "plane", "affine", "cylindrical", "fisheye", "stereographic", "compressedPlaneA2B1", "compressedPlaneA1.5B1",
              "compressedPlanePortraitA2B1", "compressedPlanePortraitA1.5B1", "paniniA2B1", "paniniA1.5B1", "paniniPortraitA2B1",
              "paniniPortraitA1.5B1", "mercator", "transverseMercator")  # Warper.WARP_TYPE_CHOICES, in its order
COMPENSATORS = ("gain_blocks", "gain", "channel", "channel_blocks", "no")  # ExposureErrorCompensator.COMPENSATOR_CHOICES


def digest(a):
    a = np.ascontiguousarray(np.asarray(a.get() if hasattr(a, "get") else a))
    return f"{a.dtype.str}{list(a.shape)} sha256:{hashlib.sha256(a.tobytes()).hexdigest()}"


class Pins:
    """The reference's results by key: recorded by the generator (record=True), checked by the tests."""

    def __init__(self, record=False):
        self.record = record
        self.data = {} if record else dict(np.load(PATH, allow_pickle=False))

    def array(self, key, a, what=None):
        """Record the digest of `a`, or assert that `a` is bit for bit the array the reference returned for `key`."""
        d = digest(a)
        if self.record:
            self.data[key] = np.array(d)
            return
        assert key in self.data, f"{key}: no pinned reference result"
        assert d == str(self.data[key]), f"{what or key}: got {d}, the reference {self.data[key]}"

    def value(self, key, v=None):
        """Record a small value as it is, or return the recorded one."""
        if self.record:
            self.data[key] = np.asarray(v)
            return v
        return self.data[key]

    def save(self):
        np.savez_compressed(PATH, **self.data)


def rot(rx, ry, rz):
    cz, sz = np.cos(rz), np.sin(rz)
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return (Rz @ rigs.rot_y(ry) @ rigs.rot_x(rx)).astype(np.float32)


def warp_cases():
    """Every projection, three random cameras each, 88x66 noise sources: (key, wtype, camera, scale, aspect, image)."""
    rng = np.random.default_rng(SEED)
    W, H = 88, 66
    for wtype in WARP_TYPES:
        for trial in range(3):
            if wtype == "affine":
                th, s = rng.uniform(-0.2, 0.2), rng.uniform(0.85, 1.2)
                R = np.array([[s * np.cos(th), -s * np.sin(th), rng.uniform(-90, 300)], [s * np.sin(th), s * np.cos(th), rng.uniform(-40, 40)],
                              [0, 0, 1]], np.float32)
                cam, scale = rigs.Camera(1.0, 1.0, 0.0, 0.0, R), 1.0
            else:
                wide = wtype in ("spherical", "cylindrical")
                R = rot(rng.uniform(-0.3, 0.3), rng.uniform(-3.0, 3.0) if wide else rng.uniform(-0.45, 0.45), rng.uniform(-0.15, 0.15))
                cam = rigs.Camera(rng.uniform(70, 120), rng.uniform(0.97, 1.03), W / 2 + rng.uniform(-4, 4), H / 2 + rng.uniform(-3, 3), R)
                scale = float(rng.uniform(60, 120))
            aspect = float(rng.choice([1.0, 0.8, 1.25])) if trial == 2 else 1.0
            img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
            yield f"warp.{wtype}.{trial}", wtype, cam, scale, aspect, img


def blend_cases():
    """The three blenders on 2-4 random images with binary, holed and gray masks: (trial, kind, strength, corners, sizes,
    images, masks)."""
    rng = np.random.default_rng(SEED)
    for trial in range(9):
        kind = ("multiband", "feather", "no")[trial % 3]
        strength = float(rng.choice([1, 5, 20, 60]))
        n = int(rng.integers(2, 5))
        sizes = [(int(rng.integers(40, 120)), int(rng.integers(30, 90))) for _ in range(n)]
        corners = [(int(rng.integers(-20, 20)) + 35 * i, int(rng.integers(-15, 15))) for i in range(n)]
        imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for (w, h) in sizes]
        masks = []
        for (w, h) in sizes:
            m = np.full((h, w), 255, np.uint8)
            if trial % 2:
                m[rng.random((h, w)) < 0.1] = 0
            if trial % 4 == 3:
                m = (m.astype(np.float32) * rng.random((h, w))).astype(np.uint8)  # gray seam-like masks
            masks.append(m)
        yield trial, kind, strength, corners, sizes, imgs, masks


class Scaler:
    def __init__(self, size):
        self.size = size

    def get_scaled_img_size(self, _):
        return self.size


def final_resolution_cases():
    """SeamFinder.resize, Images.resize_img_by_scaler and ExposureErrorCompensator inputs on random shapes, in draw order:
    ("seam", t, seam, mask), ("resize", t, img, size), ("gain", kind, corners, imgs, masks)."""
    rng = np.random.default_rng(SEED)
    for t in range(10):
        sh, sw = int(rng.integers(1, 70)), int(rng.integers(1, 90))
        h, w = int(rng.integers(2, 300)), int(rng.integers(2, 400))
        seam = (rng.integers(0, 256, (sh, sw), dtype=np.uint8) if t % 2 else (rng.random((sh, sw)) < 0.5).astype(np.uint8) * 255)
        mask = (rng.random((h, w)) < 0.85).astype(np.uint8) * 255
        yield "seam", t, seam, mask
    for t in range(10):
        h, w = int(rng.integers(2, 200)), int(rng.integers(2, 260))
        size = (int(rng.integers(1, 300)), int(rng.integers(1, 240)))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        yield "resize", t, img, size
    for kind in COMPENSATORS:
        n = 3
        sizes = [(int(rng.integers(90, 160)), int(rng.integers(70, 120))) for _ in range(n)]
        corners = [(40 * i + int(rng.integers(-5, 5)), int(rng.integers(-5, 5))) for i in range(n)]
        base = rng.integers(30, 220, (200, 400, 3), dtype=np.uint8)
        imgs = []
        for i, ((w, h), (x, y)) in enumerate(zip(sizes, corners)):
            crop = base[20 + y: 20 + y + h, 20 + x: 20 + x + w].astype(np.float32) * (0.8 + 0.2 * i)
            imgs.append(np.clip(crop + rng.normal(0, 2, crop.shape), 0, 255).astype(np.uint8))
        masks = [np.full((h, w), 255, np.uint8) for (w, h) in sizes]
        yield "gain", kind, corners, imgs, masks


def dropin_cases():
    """Three-camera rigs for the drop-in classes: (trial, warper type, blender type, cameras, 120x90 images)."""
    rng = np.random.default_rng(SEED)
    W, H = 120, 90
    for trial, (wtype, btype) in enumerate((("spherical", "multiband"), ("cylindrical", "feather"), ("plane", "no"), ("fisheye", "multiband"),
                                            ("paniniA2B1", "feather"), ("mercator", "multiband"), ("affine", "multiband"))):
        n = 3
        if wtype == "affine":
            cams = [rigs.Camera(1.0, 1.0, 0.0, 0.0, np.array([[1, 0.01 * i, 70.0 * i + rng.uniform(-3, 3)], [-0.01 * i, 1, rng.uniform(-8, 8)], [0, 0, 1]], np.float32))
                    for i in range(n)]
        else:
            f = rng.uniform(90, 130)
            cams = [rigs.Camera(f * rng.uniform(0.98, 1.02), 1.0, W / 2, H / 2, rot(rng.uniform(-0.05, 0.05), 0.45 * (i - 1) + rng.uniform(-0.03, 0.03), rng.uniform(-0.03, 0.03)))
                    for i in range(n)]
        imgs = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(n)]
        yield trial, wtype, btype, cams, imgs


def synthetic_views(cv):
    """Three perspective views of a textured plane at different exposures (the input of the recorded Stitcher run)."""
    rng = np.random.default_rng(5)
    scene = np.zeros((1400, 3000, 3), np.uint8)
    scene[:] = cv.resize(rng.integers(0, 256, (24, 50, 3), dtype=np.uint8), (3000, 1400), interpolation=cv.INTER_CUBIC)
    for _ in range(900):  # random shapes give ORB something to hold on to
        c = tuple(int(v) for v in rng.integers(0, 256, 3))
        p = (int(rng.integers(0, 3000)), int(rng.integers(0, 1400)))
        if rng.random() < 0.5:
            cv.circle(scene, p, int(rng.integers(5, 40)), c, -1)
        else:
            q = (p[0] + int(rng.integers(10, 90)), p[1] + int(rng.integers(10, 90)))
            cv.rectangle(scene, p, q, c, -1)
    views = []
    f, w, h = 900.0, 1000, 750
    K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]])
    Ks = np.array([[f, 0, 1500], [0, f, 700], [0, 0, 1]])
    for yaw in (-0.35, 0.0, 0.35):
        R = np.array([[np.cos(yaw), 0, np.sin(yaw)], [0, 1, 0], [-np.sin(yaw), 0, np.cos(yaw)]])
        H = K @ R @ np.linalg.inv(Ks)
        views.append(cv.warpPerspective(scene, H, (w, h)))
    # different exposures, so that the exposure compensator has something to do
    views[0] = np.clip(views[0].astype(np.float32) * 0.82, 0, 255).astype(np.uint8)
    views[2] = np.clip(views[2].astype(np.float32) * 1.12, 0, 255).astype(np.uint8)
    return views


def synthetic_scans(cv):
    """Three flat scans of one scene, shifted and slightly rotated against each other (the AffineStitcher run)."""
    rng = np.random.default_rng(11)
    scene = cv.resize(rng.integers(0, 256, (30, 40, 3), dtype=np.uint8), (1600, 1200), interpolation=cv.INTER_CUBIC)
    for _ in range(700):
        c = tuple(int(v) for v in rng.integers(0, 256, 3))
        p = (int(rng.integers(0, 1600)), int(rng.integers(0, 1200)))
        cv.circle(scene, p, int(rng.integers(4, 30)), c, -1)
    scans = []
    for dx, ang in ((0, 0.0), (380, 1.5), (760, -1.0)):
        M = cv.getRotationMatrix2D((400, 500), ang, 1.0)
        M[0, 2] -= dx
        scans.append(cv.warpAffine(scene, M, (800, 1000)))
    return scans


def _mix(a, b, salt):
    """A 64-bit hash of integer cell coordinates (uint64 arithmetic wraps the same way on every machine)."""
    with np.errstate(over="ignore"):
        h = a.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + b.astype(np.uint64) * np.uint64(0xC2B2AE3D27D4EB4F) + np.uint64(salt)
        h ^= h >> np.uint64(29)
        h *= np.uint64(0xBF58476D1CE4E5B9)
        h ^= h >> np.uint64(32)
    return h


def _byte(h, shift, lo, hi):
    return (lo + ((h >> np.uint64(shift)) & np.uint64(255)).astype(np.int32) * (hi - lo) // 256).astype(np.int32)


def _discs(u, v, cell, rmin, rmax, salt, out):
    """One disc per `cell` x `cell` square of the scene, centre, radius and colour from the square's hash."""
    cx, cy = np.floor(u / cell), np.floor(v / cell)
    h = _mix(cx.astype(np.int64), cy.astype(np.int64), salt)
    r = rmin + (rmax - rmin) * ((h & np.uint64(255)).astype(np.float64) / 255.0)
    du = u - (cx + 0.5) * cell - (((h >> np.uint64(8)) & np.uint64(255)).astype(np.float64) - 127.5) * (cell / 2 - rmax) / 127.5
    dv = v - (cy + 0.5) * cell - (((h >> np.uint64(16)) & np.uint64(255)).astype(np.float64) - 127.5) * (cell / 2 - rmax) / 127.5
    inside = du * du + dv * dv < r * r
    for ch in range(3):
        out[..., ch] = np.where(inside, _byte(h, 24 + 8 * ch, 0, 256), out[..., ch])


# Camera-resolution views: (tan of half the yaw step, exposure in percent) per view, left to right.  The yaws are
# 2 atan(t); sin and cos are the rationals 2t / (1 + t^2) and (1 - t^2) / (1 + t^2), so no library trigonometry enters.
CAMERA_VIEW_YAWS = {3: (-0.18, 0.0, 0.18), 4: (-0.16, -0.053, 0.053, 0.16)}
CAMERA_VIEW_GAINS = {3: (82, 100, 112), 4: (82, 100, 112, 91)}


def camera_views(w, h, n, seed):
    """`n` views of w x h (camera resolution) of one textured plane, turned by yaw steps of 12 degrees (4 views) or 20
    degrees (3 views), focal 0.9 w, at different exposures: the input of the recorded camera-resolution Stitcher runs.
    Every pair of views overlaps, so that no pair is left to a chance match above the 0.3 confidence threshold.

    Every pixel is rendered at this resolution from the plane point its ray meets -- blocks and two sizes of discs with
    sharp edges (the features ORB finds at MEDIUM resolution) and sensor noise of a few levels on top -- so the FINAL
    images carry detail down to the pixel.  Only integer arithmetic and +, -, *, /, floor in float64 are used (all
    correctly rounded), so the views come out byte-identical on any machine, without cv2."""
    from concurrent.futures import ThreadPoolExecutor

    f = 0.9 * w
    unit = w / 1000.0  # the shapes of synthetic_views, in units of a 1000 px wide view
    xs = (np.arange(w, dtype=np.float64) - w / 2) / f
    band = 256
    views = []

    def render(img, k, gain, u_row, k_row, y0):
        ys = (np.arange(y0, min(h, y0 + band), dtype=np.float64) - h / 2) / f
        u = np.broadcast_to(u_row, (ys.size, w))
        v = ys[:, None] * k_row[None, :]
        hb = _mix(np.floor(u / (60 * unit)).astype(np.int64), np.floor(v / (60 * unit)).astype(np.int64), seed)
        px = np.stack([_byte(hb, 8 * ch, 40, 216) for ch in range(3)], -1)
        hm = _mix(np.floor(u / (9 * unit)).astype(np.int64), np.floor(v / (9 * unit)).astype(np.int64), seed + 3)
        px += _byte(hm, 0, -36, 37)[..., None]  # a cell texture that makes every neighbourhood unlike the others
        _discs(u, v, 120 * unit, 10 * unit, 45 * unit, seed + 1, px)
        _discs(u, v, 36 * unit, 3 * unit, 12 * unit, seed + 2, px)
        px += np.random.default_rng([seed, k, y0]).integers(-6, 7, px.shape, dtype=np.int32)
        img[y0:y0 + ys.size] = np.clip(px * gain // 100, 0, 255).astype(np.uint8)

    with ThreadPoolExecutor(min(8, os.cpu_count() or 1)) as pool:  # bands are independent: any order gives the same bytes
        for k, (t, gain) in enumerate(zip(CAMERA_VIEW_YAWS[n], CAMERA_VIEW_GAINS[n])):
            s, c = 2 * t / (1 + t * t), (1 - t * t) / (1 + t * t)
            den = s * xs + c                                       # ray (x, y, 1) turned by the yaw, divided through by z
            u_row, k_row = f * (c * xs - s) / den, f / den
            img = np.empty((h, w, 3), np.uint8)
            list(pool.map(lambda y0: render(img, k, gain, u_row, k_row, y0), range(0, h, band)))
            views.append(img)
    return views


PIPELINE_SETTINGS = dict(crop=False, detector="orb", confidence_threshold=0.3)


def camera_value(cam):
    """cv.detail.CameraParams -> float64 [focal, aspect, ppx, ppy, R (9), t (3)]."""
    return np.concatenate([[cam.focal, cam.aspect, cam.ppx, cam.ppy], np.asarray(cam.R, np.float64).ravel(),
                           np.asarray(cam.t, np.float64).ravel()])


def camera_from_value(cv, v):
    cam = cv.detail.CameraParams()
    cam.focal, cam.aspect, cam.ppx, cam.ppy = (float(x) for x in v[:4])
    cam.R = v[4:13].reshape(3, 3).astype(np.float32)
    cam.t = v[13:16].reshape(3, 1)
    return cam
