"""GPU drop-in for stitching.warper.Warper (reference: stitching/warper.py:7-94).

Same class constants, method names, argument meaning and return types; the OpenCV calls behind them
(cv.PyRotationWarper.warp / warpRoi) are replaced by libstitch_b200's fused sm_90a warp kernel.  All sixteen
projections of WARP_TYPE_CHOICES are served bit-identically: spherical, cylindrical, plane, affine and mercator
project on the device from separable trig tables; the other eleven (fisheye, stereographic, compressedPlane*,
panini*, transverseMercator) are not separable and must match glibc's sinf / atan2f / tanf ... bit for bit, so
their float maps are built by the library's host code (libm, all cores) and the device resamples.
"""
import ctypes as C
from statistics import median

import numpy as np

from . import _lib, device_array, host_pool
from .stitching_error import StitchingError


class Warper:
    # interface constants of the boundary (warper.py:10-29)
    WARP_TYPE_CHOICES = (
        "spherical", "plane", "affine", "cylindrical", "fisheye", "stereographic",
        "compressedPlaneA2B1", "compressedPlaneA1.5B1", "compressedPlanePortraitA2B1",
        "compressedPlanePortraitA1.5B1", "paniniA2B1", "paniniA1.5B1", "paniniPortraitA2B1",
        "paniniPortraitA1.5B1", "mercator", "transverseMercator",
    )
    DEFAULT_WARP_TYPE = "spherical"

    def __init__(self, warper_type=DEFAULT_WARP_TYPE):
        self.warper_type = warper_type
        self.scale = None

    # warper.py:35-37
    def set_scale(self, cameras):
        self.scale = median([cam.focal for cam in cameras])

    # warper.py:39-41 -- stays a generator: stitcher.py pulls one image at a time through the pipeline
    def warp_images(self, imgs, cameras, aspect=1):
        for img, camera in zip(imgs, cameras):
            yield self.warp_image(img, camera, aspect)

    # warper.py:43-52
    def warp_image(self, img, camera, aspect=1):
        return self._warp(img, None, camera, aspect, want_image=True, want_mask=False)[0]

    # warper.py:54-56
    def create_and_warp_masks(self, sizes, cameras, aspect=1):
        for size, camera in zip(sizes, cameras):
            yield self.create_and_warp_mask(size, camera, aspect)

    # warper.py:58-68
    def create_and_warp_mask(self, size, camera, aspect=1):
        return self._warp(None, size, camera, aspect, want_image=False, want_mask=True)[1]

    def warp_image_and_mask(self, img, camera, aspect=1):
        """Extension: image and validity mask from the same kernel pass (the reference needs two warps)."""
        return self._warp(img, None, camera, aspect, want_image=True, want_mask=True)

    # warper.py:70-77
    def warp_rois(self, sizes, cameras, aspect=1):
        roi_corners, roi_sizes = [], []
        for size, camera in zip(sizes, cameras):
            roi = self.warp_roi(size, camera, aspect)
            roi_corners.append(roi[0:2])
            roi_sizes.append(roi[2:4])
        return roi_corners, roi_sizes

    # warper.py:79-82
    def warp_roi(self, size, camera, aspect=1):
        wtype, scale, K, R = self._params(camera, aspect)
        rect = (C.c_int * 4)()
        _lib.check(
            _lib.lib().sb_warp_roi(wtype, scale, _fp(K), _fp(R), int(size[0]), int(size[1]), rect), "sb_warp_roi"
        )
        return tuple(rect)

    # warper.py:84-94
    @staticmethod
    def get_K(camera, aspect=1):
        K = camera.K().astype(np.float32)
        # intrinsics were estimated at another resolution than the images being warped
        K[0, 0] *= aspect
        K[0, 2] *= aspect
        K[1, 1] *= aspect
        K[1, 2] *= aspect
        return K

    # ---------------------------------------------------------------------------------------------
    def _params(self, camera, aspect):
        scale = self.scale * aspect  # TypeError when set_scale was never called, like the reference
        if self.warper_type not in _lib.WARP_TYPES:
            raise StitchingError(f"unknown warper type '{self.warper_type}'")
        K = np.ascontiguousarray(Warper.get_K(camera, aspect))
        R = np.asarray(camera.R)
        if R.dtype != np.float32 or R.shape != (3, 3) or K.shape != (3, 3):
            raise _lib_argument_error("K and R must be 3x3 float32 (CV_32F), as cv.PyRotationWarper requires")
        return _lib.WARP_TYPES[self.warper_type], np.float32(scale), K, np.ascontiguousarray(R)

    def _warp(self, img, size, camera, aspect, want_image, want_mask):
        wtype, scale, K, R = self._params(camera, aspect)
        src_p, pitch = None, 0
        if img is not None:
            img = np.asarray(img)
            if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
                raise _lib_argument_error("the GPU warp path takes uint8 HxWx3 images")
            if img.strides[2] != 1 or img.strides[1] != 3 or img.strides[0] < img.shape[1] * 3:
                img = np.ascontiguousarray(img)  # e.g. a column-sliced crop keeps row pitch; anything odder is copied
            size = (img.shape[1], img.shape[0])
            src_p, pitch = img.ctypes.data_as(C.c_void_p), img.strides[0]
        rect = (C.c_int * 4)()
        L = _lib.lib()
        _lib.check(L.sb_warp_roi(wtype, scale, _fp(K), _fp(R), int(size[0]), int(size[1]), rect), "sb_warp_roi")
        w, h = rect[2], rect[3]
        # page-locked result arrays (host_pool): one DMA instead of page faults + a staged copy
        out = host_pool.empty((h, w, 3), np.uint8) if want_image else None
        msk = host_pool.empty((h, w), np.uint8) if want_mask else None
        # the arrays are filled as always; the device copy of the IMAGE stays alive behind it (device_array.DeviceBacked)
        # so that cropping (slicing), ExposureErrorCompensator.apply and Blender.feed can go on without another upload.
        # Masks stay plain writable ndarrays: the reference hands them to cv2 calls that write into them
        # (seam_finder.py:35, the seam finders' find() modifies `masks` in place).
        keep_i = C.c_void_p()
        rc = L.sb_warp_keep(
            wtype, scale, _fp(K), _fp(R), src_p, int(size[0]), int(size[1]), pitch,
            out.ctypes.data_as(C.c_void_p) if want_image else None, w * 3,
            msk.ctypes.data_as(C.c_void_p) if want_mask else None, w, rect,
            C.byref(keep_i) if want_image else None, None,
        )
        if rc == _lib.SB_ERR_INVALID:  # e.g. a side of 32767 px or more, where cv::remap asserts
            raise _lib_argument_error("sb_warp_keep: " + L.sb_last_error().decode(errors="replace"))
        _lib.check(rc, "sb_warp_keep")
        if want_image:
            out = device_array.wrap(out, keep_i.value)
        return out, msk


def _fp(a):
    return a.ctypes.data_as(_lib.c_float_p)


def _lib_argument_error(msg):
    """cv2 raises cv2.error for these; stay catchable as both when cv2 is installed."""
    try:
        import cv2

        class ArgumentError(StitchingError, cv2.error):
            pass

        return ArgumentError(msg)
    except Exception:
        return StitchingError(msg)
