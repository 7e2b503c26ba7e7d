"""GPU drop-in for the FINAL-resolution half of stitching.seam_finder.SeamFinder (reference: stitching/seam_finder.py).

Seam estimation itself (`SeamFinder.find`, OpenCV's graph-cut / dynamic-programming finders at LOW resolution) stays
with the reference.  `resize` -- the step that produces the blend mask of every image at FINAL resolution
(seam_finder.py:38-43, called from stitcher.py:223-225) -- runs on the device: 3x3 dilate, bilinear resize, AND with
the warped mask, bit-identical to the cv2 calls it replaces.  `stitching_b200.install()` patches it into the
reference class; `Compositor.set_seam_mask` is the fused form (no host round trip of the FINAL-resolution mask).
"""
import ctypes as C

import numpy as np

from . import _lib
from .stitching_error import StitchingError


def resize(seam_mask, mask):
    """SeamFinder.resize(seam_mask, mask): uint8 mask of `mask`'s size.  Like the cv2 chain it replaces
    (seam_finder.py:39-43: dilate -> resize -> bitwise_and) the result is a cv.UMat whenever an input was one -- the seam
    finder hands out cv.UMat masks, and SeamFinder.draw_seam_mask (seam_finder.py:47) calls cv.UMat.get on the result --
    and an ndarray when both inputs were ndarrays."""
    was_umat = False
    if hasattr(seam_mask, "get") and not isinstance(seam_mask, np.ndarray):
        seam_mask, was_umat = seam_mask.get(), True  # cv.UMat from the seam finder
    if hasattr(mask, "get") and not isinstance(mask, np.ndarray):
        mask, was_umat = mask.get(), True
    seam_mask = np.ascontiguousarray(seam_mask, np.uint8)
    mask = np.ascontiguousarray(mask, np.uint8)
    if seam_mask.ndim != 2 or mask.ndim != 2:
        raise StitchingError("SeamFinder.resize takes two single-channel uint8 masks")
    h, w = mask.shape
    out = np.empty((h, w), np.uint8)
    _lib.check(
        _lib.lib().sb_seam_resize(
            seam_mask.ctypes.data_as(C.c_void_p), seam_mask.strides[0], seam_mask.shape[1], seam_mask.shape[0],
            mask.ctypes.data_as(C.c_void_p), mask.strides[0], w, h, out.ctypes.data_as(C.c_void_p), out.strides[0],
        ),
        "sb_seam_resize",
    )
    if was_umat:
        import cv2  # a cv.UMat came in, so cv2 is importable

        return cv2.UMat(out)
    return out
