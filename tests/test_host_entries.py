"""The host-buffer entries of the C ABI on their failure paths, in the emulation build (tests/emu).  sb_emu_fail_at(k)
makes the k-th fallible runtime call after it fail: an allocation, a copy, a stream synchronisation or the error check
after a launch.  For every k until the armed call passes, the entry:

* returns an error, and sb_last_error() is a message of its own that names the CUDA call and its error, not the text an
  earlier call left behind;
* frees every temporary: the live device allocations are what they were before the call (kept buffers excepted: those of
  sb_warp_keep on success, those of a blender's feeds until the blender drops them);
* leaves a blender as it was: after a failed feed, blend() gives the panorama of the feeds made before it, bit for bit;
* and a clean call afterwards gives the same bytes as a clean call before."""
import ctypes as C
import re

import numpy as np
import pytest

SENTINEL = b"sb_warp_roi: invalid argument"
CUDA_MSG = re.compile(rb"CUDA error \d+ \([^)]+\) at \S+:\d+ in `(cuda\w+|k_\w+)")
SPHERICAL, FISHEYE = 0, 4
FEATHER, MULTIBAND = 1, 2


def hooked(L):
    """The emulation library with its failure hook bound (the product library has none)."""
    L.sb_emu_fail_at.argtypes = [C.c_int]
    L.sb_emu_fail_at.restype = None
    L.sb_emu_live_allocs.argtypes = []
    L.sb_emu_live_allocs.restype = C.c_long
    return L


@pytest.fixture(scope="module")
def L(emu_lib):
    return hooked(emu_lib)


def cases():
    """(test, its arguments after L) for every test and parameter set here: tests/emu_sweep.py runs them as a corpus."""
    out = []
    for name, fn in globals().items():
        if name.startswith("test_"):
            marks = [m for m in getattr(fn, "pytestmark", []) if m.name == "parametrize"]
            values = marks[0].args[1] if marks else [()]
            out += [(fn, v if isinstance(v, tuple) else (v,)) for v in values]
    return out


def p(a):
    return a.ctypes.data


def f32p(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def set_sentinel(L):
    assert L.sb_warp_roi(-1, 1.0, None, None, 0, 0, None) != 0
    assert L.sb_last_error() == SENTINEL


def drive(L, call, out, setup=lambda: None, after_fail=lambda: None, live_after_setup=True):
    """Fail the k-th fallible call of call() for k = 1, 2, ... until it passes; returns the number of k that failed."""
    L.sb_emu_fail_at(0)
    setup()
    assert call() == 0, L.sb_last_error()
    clean = out()
    k = 0
    while True:
        k += 1
        live = L.sb_emu_live_allocs()
        setup()
        if live_after_setup:
            live = L.sb_emu_live_allocs()
        set_sentinel(L)
        L.sb_emu_fail_at(k)
        rc = call()
        L.sb_emu_fail_at(0)
        if rc == 0:
            assert out() == clean, f"k={k}: the call that met no failure differs from a clean call"
            break
        msg = L.sb_last_error()
        assert msg != SENTINEL, f"k={k}: the failure left the message of an earlier call"
        assert CUDA_MSG.search(msg), f"k={k}: {msg!r}"
        assert L.sb_emu_live_allocs() == live, f"k={k}: {L.sb_emu_live_allocs() - live} device allocations left behind ({msg!r})"
        after_fail()
        setup()
        assert call() == 0, L.sb_last_error()
        assert out() == clean, f"k={k}: a clean call after the failure differs"
    assert k > 1
    return k - 1


def image(rng, h, w, c=3, dtype=np.uint8):
    return rng.integers(0, 256, (h, w, c) if c else (h, w), dtype=np.int64).astype(dtype)


def camera(w, h, f=60.0):
    K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]], np.float32)
    R = np.eye(3, dtype=np.float32)
    return K, R, f


def warp_roi(L, wt, K, R, f, w, h):
    r = (C.c_int * 4)()
    assert L.sb_warp_roi(wt, f, f32p(K), f32p(R), w, h, r) == 0
    return list(r)


def devimg(L, handle, shape):
    """The bytes of a kept device image (the emulation's device memory is host memory)."""
    a = np.zeros(shape, np.uint8)
    assert L.sb_device_copy(p(a), C.cast(handle, C.POINTER(C.c_void_p))[0], a.nbytes) == 0
    return a


def warped(L, rng, wt=SPHERICAL):
    """One warped image and mask kept on the device, with their host copies."""
    src = image(rng, 30, 40)
    K, R, f = camera(40, 30)
    rect = warp_roi(L, wt, K, R, f, 40, 30)
    w, h = rect[2], rect[3]
    img, mask = np.zeros((h, w, 3), np.uint8), np.zeros((h, w), np.uint8)
    ki, km = C.c_void_p(), C.c_void_p()
    assert L.sb_warp_keep(wt, f, f32p(K), f32p(R), p(src), 40, 30, 120, p(img), w * 3, p(mask), w, (C.c_int * 4)(), C.byref(ki), C.byref(km)) == 0
    return ki.value, km.value, img, mask


@pytest.mark.parametrize("wt", [SPHERICAL, FISHEYE])
def test_warp(L, wt):
    rng = np.random.default_rng(1)
    src = image(rng, 30, 40)
    K, R, f = camera(40, 30)
    w, h = warp_roi(L, wt, K, R, f, 40, 30)[2:]
    img, mask = np.zeros((h, w, 3), np.uint8), np.zeros((h, w), np.uint8)
    rect = (C.c_int * 4)()
    call = lambda: L.sb_warp(wt, f, f32p(K), f32p(R), p(src), 40, 30, 120, p(img), w * 3, p(mask), w, rect)
    drive(L, call, lambda: img.tobytes() + mask.tobytes() + bytes(rect))


def test_warp_keep(L):
    rng = np.random.default_rng(2)
    src = image(rng, 30, 40)
    K, R, f = camera(40, 30)
    w, h = warp_roi(L, FISHEYE, K, R, f, 40, 30)[2:]
    img, mask = np.zeros((h, w, 3), np.uint8), np.zeros((h, w), np.uint8)
    kept = []

    def call():
        ki, km = C.c_void_p(), C.c_void_p()
        rc = L.sb_warp_keep(FISHEYE, f, f32p(K), f32p(R), p(src), 40, 30, 120, p(img), w * 3, p(mask), w, (C.c_int * 4)(), C.byref(ki), C.byref(km))
        assert (rc == 0) == bool(ki.value) == bool(km.value), "a handle is given exactly when the call succeeds"
        kept[:] = [ki.value, km.value] if rc == 0 else []
        return rc

    def out():
        ki, km = kept
        b = img.tobytes() + mask.tobytes() + devimg(L, ki, (h, w, 3)).tobytes() + devimg(L, km, (h, w)).tobytes()
        L.sb_devimg_release(ki)
        L.sb_devimg_release(km)
        return b

    drive(L, call, out)


@pytest.mark.parametrize("gain", ["map", "scalar"])
def test_gain_apply(L, gain):
    rng = np.random.default_rng(3)
    orig = image(rng, 21, 34)
    img = orig.copy()
    gmap = rng.uniform(0.5, 1.5, (3, 4, 3)).astype(np.float32)
    gs = (C.c_double * 3)(0.9, 1.1, 1.3)
    args = (p(gmap), 4, 3, 3, None) if gain == "map" else (None, 0, 0, 0, gs)

    def call():
        img[:] = orig
        return L.sb_gain_apply(p(img), 34 * 3, 34, 21, *args)

    assert drive(L, call, lambda: img.tobytes()) >= 4


@pytest.mark.parametrize("gain", ["map", "scalar"])
def test_gain_apply_dev(L, gain):
    rng = np.random.default_rng(4)
    ki, km, img0, _ = warped(L, rng)
    h, w = img0.shape[:2]
    x, y, cw, ch = 3, 2, w - 5, h - 4
    host = np.zeros((ch, cw, 3), np.uint8)
    gmap = rng.uniform(0.5, 1.5, (3, 4, 1)).astype(np.float32)
    gs = (C.c_double * 3)(0.9, 1.1, 1.3)
    args = (p(gmap), 4, 3, 1, None) if gain == "map" else (None, 0, 0, 0, gs)
    dev = C.cast(ki, C.POINTER(C.c_void_p))[0]

    restore = lambda: L.sb_device_copy(dev, p(img0), img0.nbytes)  # the device image as warped
    call = lambda: L.sb_gain_apply_dev(ki, x, y, cw, ch, p(host), cw * 3, *args)
    drive(L, call, lambda: host.tobytes() + devimg(L, ki, (h, w, 3)).tobytes(), setup=restore)
    L.sb_devimg_release(ki)
    L.sb_devimg_release(km)


@pytest.mark.parametrize("source", ["host_u8", "host_s16", "device"])
def test_timelapse_frame(L, source):
    rng = np.random.default_rng(5)
    roi = (C.c_int * 4)(-4, -3, 50, 40)
    dst = np.zeros((40, 50, 3), np.uint8)
    handles = []
    if source == "device":
        ki, km, img, _ = warped(L, rng)
        handles = [ki, km]
        h, w = img.shape[:2]
        args = (None, 0, 0, ki, 1, 2, w - 3, h - 4)
    else:
        s16 = source == "host_s16"
        img = rng.integers(-300, 300, (24, 33, 3)).astype(np.int16) if s16 else image(rng, 24, 33)
        args = (p(img), int(s16), img.strides[0], None, 0, 0, 33, 24)
    call = lambda: L.sb_timelapse_frame(*args, 5, 7, roi, p(dst), 150)
    drive(L, call, lambda: dst.tobytes())
    for d in handles:
        L.sb_devimg_release(d)


@pytest.mark.parametrize("channels", [1, 3])
def test_resize_exact(L, channels):
    rng = np.random.default_rng(6)
    src = image(rng, 23, 31, channels if channels == 3 else 0)
    dst = np.zeros((17, 40, channels), np.uint8)
    call = lambda: L.sb_resize_exact(p(src), 31 * channels, 31, 23, channels, p(dst), 40 * channels, 40, 17)
    drive(L, call, lambda: dst.tobytes())


def test_seam_resize(L):
    rng = np.random.default_rng(7)
    seam = (rng.random((9, 13)) > 0.4).astype(np.uint8) * 255
    mask = (rng.random((27, 38)) > 0.2).astype(np.uint8) * 255
    dst = np.zeros((27, 38), np.uint8)
    call = lambda: L.sb_seam_resize(p(seam), 13, 13, 9, p(mask), 38, 38, 27, p(dst), 38)
    drive(L, call, lambda: dst.tobytes())


def test_selftest_division(L):
    bad = C.c_ulonglong(123)
    call = lambda: L.sb_selftest_division(4096, 7, 0, C.byref(bad))
    drive(L, call, lambda: bad.value)


class Blender:
    """A blender over a 60 x 44 roi and its feeds; A is fed before the entry under test, B by it."""

    def __init__(self, L, kind, s16):
        self.L, self.kind, self.s16 = L, kind, s16
        rng = np.random.default_rng(8 + kind + 2 * s16)
        dt = np.int16 if s16 else np.uint8
        self.a = image(rng, 30, 36, 3, dt)
        self.b = image(rng, 28, 40, 3, dt)
        self.ma = (rng.random((30, 36)) > 0.1).astype(np.uint8) * 255
        self.mb = (rng.random((28, 40)) > 0.1).astype(np.uint8) * 255
        self.h = None

    def prepare(self, feed_a=True):
        L = self.L
        self.h = L.sb_blender_create(self.kind, 2, 0.05)
        assert L.sb_blender_prepare(self.h, 10, 20, 60, 44) == 0
        if feed_a:
            assert self.feed(self.a, self.ma, 12, 21) == 0

    def feed(self, img, mask, x, y):
        return self.L.sb_blender_feed(self.h, p(img), int(self.s16), img.strides[0], p(mask), mask.shape[1], img.shape[1], img.shape[0], x, y)

    def feed_b(self):
        return self.feed(self.b, self.mb, 28, 33)

    def blend(self):
        pano, pmask, s16 = np.zeros((44, 60, 3), np.uint8), np.zeros((44, 60), np.uint8), np.zeros((44, 60, 3), np.int16)
        rc = self.L.sb_blender_blend(self.h, p(pano), 180, p(pmask), 60, p(s16), 360)
        self.L.sb_blender_destroy(self.h)
        self.h = None
        return rc, pano.tobytes() + pmask.tobytes() + s16.tobytes()

    def blend_ok(self):
        rc, b = self.blend()
        assert rc == 0, self.L.sb_last_error()
        return b


@pytest.mark.parametrize("kind,s16", [(MULTIBAND, False), (MULTIBAND, True), (FEATHER, False)])
def test_blender_feed(L, kind, s16):
    B = Blender(L, kind, s16)
    B.prepare()
    only_a = B.blend_ok()
    drive(L, B.feed_b, B.blend_ok, setup=B.prepare, after_fail=lambda: _same(B.blend_ok(), only_a))


def _same(got, want):
    assert got == want, "a failed feed changed what the blender blends"


@pytest.mark.parametrize("kind", [MULTIBAND, FEATHER])
def test_blender_feed_dev(L, kind):
    B = Blender(L, kind, False)
    rng = np.random.default_rng(9)
    ki, km, img, mask = warped(L, rng)
    h, w = img.shape[:2]
    B.prepare()
    only_a = B.blend_ok()
    call = lambda: L.sb_blender_feed_dev(B.h, ki, 1, 2, km, 1, 2, None, 0, min(w - 1, 40), min(h - 2, 30), 25, 30)
    drive(L, call, B.blend_ok, setup=B.prepare, after_fail=lambda: _same(B.blend_ok(), only_a))
    # the mask from the host
    hm = np.ascontiguousarray(mask[2:, 1:])
    call = lambda: L.sb_blender_feed_dev(B.h, ki, 1, 2, None, 0, 0, p(hm), hm.strides[0], min(w - 1, 40), min(h - 2, 30), 25, 30)
    drive(L, call, B.blend_ok, setup=B.prepare, after_fail=lambda: _same(B.blend_ok(), only_a))
    L.sb_devimg_release(ki)
    L.sb_devimg_release(km)


@pytest.mark.parametrize("kind,s16", [(MULTIBAND, False), (MULTIBAND, True), (FEATHER, False)])
def test_blender_blend(L, kind, s16):
    B = Blender(L, kind, s16)
    result = []

    def setup():
        B.prepare()
        assert B.feed_b() == 0

    def call():
        rc, b = B.blend()
        result[:] = [b]
        return rc

    drive(L, call, lambda: result[0], setup=setup, live_after_setup=False)
