"""GPU drop-in for stitching.blender.Blender (reference: stitching/blender.py:5-56).

prepare / feed / blend keep their signatures and return types.  feed() uploads and records the image;
the arithmetic of cv.detail_MultiBandBlender / FeatherBlender / Blender(NO) runs in blend() as one batch
of sm_90a kernels that applies the feeds in call order (bit-identical to eager accumulation).
"""
import ctypes as C

import numpy as np

from . import _lib, device_array, host_pool
from .stitching_error import StitchingError


class _NativeBlender:
    """What `Blender.blender` holds after prepare(): the libstitch_b200 handle (reference: a cv.detail_* object)."""

    def __init__(self, kind, num_bands=0, sharpness=0.0):
        self.kind = kind
        self.sharpness = float(sharpness)
        self._L = _lib.lib()  # the handle is destroyed by the library that created it, whichever is bound later
        self._h = self._L.sb_blender_create(_lib.BLEND_KINDS[kind], int(num_bands), C.c_float(sharpness))
        if not self._h:
            _lib.check(-1, "sb_blender_create")
        self.roi = None

    def prepare(self, dst_roi):
        x, y, w, h = (int(v) for v in dst_roi)
        _lib.check(_lib.lib().sb_blender_prepare(self._h, x, y, w, h), "sb_blender_prepare")
        self.roi = (x, y, w, h)

    @property
    def num_bands(self):
        return _lib.lib().sb_blender_num_bands(self._h)

    def feed(self, img, mask, corner):
        if self._feed_twin(img, mask, corner):
            return
        img = np.asarray(img)
        if img.ndim != 3 or img.shape[2] != 3:
            raise StitchingError("Blender.feed takes an HxWx3 image")
        if img.dtype not in (np.uint8, np.int16):
            img = img.astype(np.int16)  # what blender.py:41 does with every input
        if hasattr(mask, "get") and not isinstance(mask, np.ndarray):
            mask = mask.get()  # cv.UMat (seam_finder.py:38-43 hands those out)
        mask = np.asarray(mask)
        if mask.dtype != np.uint8 or mask.shape != img.shape[:2]:
            raise StitchingError("Blender.feed takes a uint8 mask of the image's size")
        img = np.ascontiguousarray(img)
        mask = np.ascontiguousarray(mask)
        h, w = mask.shape
        _lib.check(
            _lib.lib().sb_blender_feed(
                self._h, img.ctypes.data_as(C.c_void_p), int(img.dtype == np.int16), img.strides[0],
                mask.ctypes.data_as(C.c_void_p), mask.strides[0], w, h, int(corner[0]), int(corner[1]),
            ),
            "sb_blender_feed",
        )

    def _feed_twin(self, img, mask, corner):
        """Blender.feed without the upload when `img` still has its device twin (a warped image, possibly cropped and
        exposure-compensated by the drop-ins); the mask comes from its twin too, or from the host."""
        tw = device_array.twin(img)
        if tw is None or img.ndim != 3:
            return False
        ptr, ix, iy, w, h = tw
        if hasattr(mask, "get") and not isinstance(mask, np.ndarray):
            mask = mask.get()  # cv.UMat (seam_finder.py:38-43 hands those out)
        mtw = device_array.twin(mask) if getattr(mask, "ndim", 0) == 2 else None
        if mtw is not None and (mtw[3], mtw[4]) == (w, h):
            mptr, mx, my, mhost, mpitch = mtw[0], mtw[1], mtw[2], None, 0
        else:
            mask = np.asarray(mask)
            if mask.dtype != np.uint8 or mask.shape != (h, w):
                raise StitchingError("Blender.feed takes a uint8 mask of the image's size")
            mask = np.ascontiguousarray(mask)
            mptr, mx, my, mhost, mpitch = None, 0, 0, mask.ctypes.data_as(C.c_void_p), mask.strides[0]
        _lib.check(
            _lib.lib().sb_blender_feed_dev(self._h, ptr, ix, iy, mptr, mx, my, mhost, mpitch, w, h, int(corner[0]), int(corner[1])),
            "sb_blender_feed_dev",
        )
        return True

    def blend(self, want_s16=False):
        if self.roi is None:
            raise StitchingError("blend() before prepare()")
        _, _, w, h = self.roi
        dst = host_pool.empty((h, w, 3), np.uint8)  # page-locked: the panorama is the largest copy of a stitch
        msk = host_pool.empty((h, w), np.uint8)
        s16 = host_pool.empty((h, w, 3), np.int16) if want_s16 else None
        _lib.check(
            _lib.lib().sb_blender_blend(
                self._h, dst.ctypes.data_as(C.c_void_p), w * 3, msk.ctypes.data_as(C.c_void_p), w,
                s16.ctypes.data_as(C.c_void_p) if want_s16 else None, w * 6,
            ),
            "sb_blender_blend",
        )
        self.roi = None
        return (dst, msk, s16) if want_s16 else (dst, msk)

    def close(self):
        if self._h:
            self._L.sb_blender_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def result_roi(corners, sizes):
    """Bounding rectangle (x, y, w, h) of the rects -- what cv.detail.resultRoi returns (blender.py:24)."""
    x0 = min(int(c[0]) for c in corners)
    y0 = min(int(c[1]) for c in corners)
    x1 = max(int(c[0]) + int(s[0]) for c, s in zip(corners, sizes))
    y1 = max(int(c[1]) + int(s[1]) for c, s in zip(corners, sizes))
    return (x0, y0, x1 - x0, y1 - y0)


class Blender:
    # interface constants of the boundary (blender.py:8-14)
    BLENDER_CHOICES = ("multiband", "feather", "no")
    DEFAULT_BLENDER = "multiband"
    DEFAULT_BLEND_STRENGTH = 5

    def __init__(self, blender_type=DEFAULT_BLENDER, blend_strength=DEFAULT_BLEND_STRENGTH):
        self.blender_type = blender_type
        self.blend_strength = blend_strength
        self.blender = None

    # blender.py:23-38
    def prepare(self, corners, sizes):
        dst_sz = result_roi(corners, sizes)
        # same float64 expression as the reference so that num_bands / sharpness agree to the bit
        blend_width = np.sqrt(dst_sz[2] * dst_sz[3]) * self.blend_strength / 100
        if self.blender is not None:
            self.blender.close()
            self.blender = None  # an unknown blender_type must fail on `None`, not on a closed handle
        if self.blender_type == "no" or blend_width < 1:
            self.blender = _NativeBlender("no")
        elif self.blender_type == "multiband":
            self.blender = _NativeBlender("multiband", num_bands=int(np.log(blend_width) / np.log(2.0) - 1.0))
        elif self.blender_type == "feather":
            self.blender = _NativeBlender("feather", sharpness=1.0 / blend_width)
        # an unknown blender_type leaves self.blender unset and fails below, like the reference
        self.blender.prepare(dst_sz)

    # blender.py:40-41 (the int16 conversion happens on the device)
    def feed(self, img, mask, corner):
        self.blender.feed(img, mask, corner)

    # blender.py:43-48 (convertScaleAbs is fused into the last kernel)
    def blend(self):
        return self.blender.blend()

    # blender.py:50-56
    @classmethod
    def create_panorama(cls, imgs, masks, corners, sizes):
        blender = cls("no")
        blender.prepare(corners, sizes)
        for img, mask, corner in zip(imgs, masks, corners):
            blender.feed(img, mask, corner)
        return blender.blend()
