"""GPU drop-in for the resampling step of stitching.images.Images (reference: stitching/images.py:120-123).

`Images.resize_img_by_scaler(scaler, size, img)` produces the MEDIUM / LOW / FINAL resolution inputs of the pipeline
with `cv.resize(img, desired_size, interpolation=cv.INTER_LINEAR_EXACT)`; here the same bit-exact fixed-point bilinear
runs on the device.  The scalers (megapix_scaler.py) stay the reference's: only `get_scaled_img_size` is used.
`stitching_b200.install()` patches the static method into the reference class.
"""
import ctypes as C

import numpy as np

from . import _lib
from .stitching_error import StitchingError


def resize_exact(img, size):
    """cv.resize(img, size, interpolation=cv.INTER_LINEAR_EXACT) for a uint8 image of 1 or 3 channels; size = (w, h)."""
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim not in (2, 3) or (img.ndim == 3 and img.shape[2] not in (1, 3)):
        raise StitchingError("resize takes a uint8 image of 1 or 3 channels")
    cn = 1 if img.ndim == 2 else img.shape[2]
    if img.strides[-1] != 1 or (img.ndim == 3 and img.strides[1] != cn):
        img = np.ascontiguousarray(img)
    w, h = int(size[0]), int(size[1])
    out = np.empty((h, w) if img.ndim == 2 else (h, w, cn), np.uint8)
    _lib.check(
        _lib.lib().sb_resize_exact(img.ctypes.data_as(C.c_void_p), img.strides[0], img.shape[1], img.shape[0], cn,
                                   out.ctypes.data_as(C.c_void_p), out.strides[0], w, h),
        "sb_resize_exact",
    )
    return out


def resize_img_by_scaler(scaler, size, img):
    """Images.resize_img_by_scaler (images.py:120-123)."""
    return resize_exact(img, scaler.get_scaled_img_size(size))
