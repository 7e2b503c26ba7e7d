"""GPU drop-in for the FINAL-resolution half of stitching.exposure_error_compensator.ExposureErrorCompensator
(reference: stitching/exposure_error_compensator.py).

Gain estimation (`feed`, at LOW resolution, stitcher.py:211) stays with OpenCV's compensators.  `apply` -- run on every
warped FINAL-resolution image between warp and blend (exposure_error_compensator.py:43-45, stitcher.py:219-221) -- runs
on the device with the gains the compensator estimated (`getMatGains()`), bit-identical to the cv2 call it replaces.
`stitching_b200.install()` patches it into the reference class; `Compositor.set_gain` is the fused form (the gain is
applied in the warp kernel's epilogue).
"""
import ctypes as C

import numpy as np

from . import _lib, device_array
from .stitching_error import StitchingError


def gain_arguments(gain):
    """(gain_map, gw, gh, gc, gain_scalar) for the C ABI from one entry of getMatGains(): a float32 map of 1 or 3 channels
    (gain_blocks / channel_blocks), a float64 scalar (gain) or float64 vector of >= 3 entries (channel); None: no gain."""
    if gain is None:
        return None, 0, 0, 0, None
    gain = np.asarray(gain)
    if gain.size == 0:
        return None, 0, 0, 0, None
    if gain.dtype == np.float64:
        g = gain.ravel()
        if g.size not in (1, 3, 4):
            raise StitchingError("a scalar gain has 1 value (gain) or 3-4 values (channel)")
        return None, 0, 0, 0, np.ascontiguousarray([g[0]] * 3 if g.size == 1 else g[:3], np.float64)
    if gain.dtype != np.float32 or gain.ndim not in (2, 3) or (gain.ndim == 3 and gain.shape[2] not in (1, 3)):
        raise StitchingError("a gain map is a float32 array of 1 or 3 channels")
    gain = np.ascontiguousarray(gain)
    return gain, gain.shape[1], gain.shape[0], 1 if gain.ndim == 2 else gain.shape[2], None


def apply_gain(img, gain):
    """What cv.detail ...Compensator.apply does to `img` (uint8 HxWx3) given its gain; in place when `img` is a
    C-contiguous-row uint8 array (as the reference modifies its argument), returns the image."""
    gmap, gw, gh, gc, gscalar = gain_arguments(gain)
    tw = device_array.twin(img)
    if tw is not None and img.ndim == 3:
        # the warped image still has its device twin: compensate there, refresh the host copy (the reference modifies
        # its argument in place and returns it -- so do we, for both copies; nobody else can write to this array)
        ptr, x, y, w, h = tw
        img.flags.writeable = True
        try:
            _lib.check(
                _lib.lib().sb_gain_apply_dev(
                    ptr, x, y, w, h, img.ctypes.data_as(C.c_void_p), img.strides[0],
                    gmap.ctypes.data_as(C.c_void_p) if gmap is not None else None, gw, gh, gc,
                    gscalar.ctypes.data_as(C.c_void_p) if gscalar is not None else None,
                ),
                "sb_gain_apply_dev",
            )
        finally:
            img.flags.writeable = False
        return img
    arr = np.asarray(img)
    if arr.dtype != np.uint8 or arr.ndim != 3 or arr.shape[2] != 3:
        raise StitchingError("ExposureErrorCompensator.apply takes a uint8 HxWx3 image")
    if arr.strides[2] != 1 or arr.strides[1] != 3:
        arr = np.ascontiguousarray(arr)
    _lib.check(
        _lib.lib().sb_gain_apply(
            arr.ctypes.data_as(C.c_void_p), arr.strides[0], arr.shape[1], arr.shape[0],
            gmap.ctypes.data_as(C.c_void_p) if gmap is not None else None, gw, gh, gc,
            gscalar.ctypes.data_as(C.c_void_p) if gscalar is not None else None,
        ),
        "sb_gain_apply",
    )
    return arr


def apply(compensator, index, corner, image, mask):
    """ExposureErrorCompensator.apply(index, corner, image, mask) for a cv.detail compensator object that has been fed:
    its gain for image `index` comes from getMatGains(); corner and mask do not enter (as in OpenCV's implementations)."""
    if hasattr(image, "get") and not isinstance(image, np.ndarray):
        image = image.get()
    gains = compensator.getMatGains() if hasattr(compensator, "getMatGains") else []
    gain = gains[index] if index < len(gains) else None  # NoExposureCompensator has none
    return apply_gain(image, gain)
