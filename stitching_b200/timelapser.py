"""GPU drop-in for stitching.timelapser.Timelapser (reference: stitching/timelapser.py:7-56).

The timelapser is the other consumer of the warped FINAL-resolution frames (stitcher.py:242-252): every frame is the
canvas of the prepared roi with ONE warped image pasted at its corner.  Same class constants, constructor, method names
and file naming; cv.detail.Timelapser(AS_IS | CROP).process / getDst and the int16 -> float32 -> convertScaleAbs chain
of get_frame (timelapser.py:40-52) become one kernel pass that writes the uint8 frame, fed from the warped image's
device twin when it still has one (stitching_b200.device_array) -- bit-identical to the reference's frames.  Writing
the file (cv.imwrite, timelapser.py:38) stays with OpenCV.
"""
import ctypes as C
import os

import numpy as np

from . import _lib, device_array, host_pool
from .stitching_error import StitchingError


_EMPTY = object()


class Timelapser:
    # interface constants of the boundary (timelapser.py:10-16)
    TIMELAPSE_CHOICES = ("no", "as_is", "crop")
    DEFAULT_TIMELAPSE = "no"
    DEFAULT_TIMELAPSE_PREFIX = "fixed_"

    def __init__(self, timelapse=DEFAULT_TIMELAPSE, timelapse_prefix=DEFAULT_TIMELAPSE_PREFIX):
        self.do_timelapse = timelapse in ("as_is", "crop")
        self.timelapse_type = timelapse if self.do_timelapse else None
        self.timelapser = self if self.do_timelapse else None  # the reference holds a cv.detail.Timelapser here
        self.timelapse_prefix = timelapse_prefix
        self.roi = None
        self._frame = None

    # timelapser.py:36-37 -> cv.detail.Timelapser.initialize(corners, sizes)
    def initialize(self, corners, sizes):
        if not self.do_timelapse:
            raise AttributeError("'NoneType' object has no attribute 'initialize'")  # what the reference's None raises
        tlx = [int(c[0]) for c in corners]
        tly = [int(c[1]) for c in corners]
        brx = [int(c[0]) + int(s[0]) for c, s in zip(corners, sizes)]
        bry = [int(c[1]) + int(s[1]) for c, s in zip(corners, sizes)]
        if self.timelapse_type == "as_is":  # cv.detail.resultRoi
            x0, y0, x1, y1 = min(tlx), min(tly), max(brx), max(bry)
        else:  # cv.detail.resultRoiIntersection = cv::Rect(Point tl, Point br), which orders its corners
            ax, ay, bx, by = max(tlx), max(tly), min(brx), min(bry)
            x0, y0, x1, y1 = min(ax, bx), min(ay, by), max(ax, bx), max(ay, by)
        self.roi = (x0, y0, x1 - x0, y1 - y0)
        self._frame = None

    # timelapser.py:38-39
    def process_and_save_frame(self, img_name, img, corner):
        import cv2  # file output stays with OpenCV

        self.process_frame(img, corner)
        cv2.imwrite(self.get_fixed_filename(img_name), self.get_frame())

    # timelapser.py:40-43 + :45-49: process and getDst / convertScaleAbs in one pass on the device
    def process_frame(self, img, corner):
        if self.roi is None:
            raise StitchingError("Timelapser.process_frame before initialize")
        _, _, cw, ch = self.roi
        if cw <= 0 or ch <= 0:
            self._frame = _EMPTY  # the reference's get_frame fails on an empty canvas (cv.convertScaleAbs of an empty array)
            return
        roi = (C.c_int * 4)(*self.roi)
        dst = host_pool.empty((ch, cw, 3), np.uint8)
        tw = device_array.twin(img) if getattr(img, "ndim", 0) == 3 else None
        if tw is not None:
            ptr, ix, iy, w, h = tw
            rc = _lib.lib().sb_timelapse_frame(None, 0, 0, ptr, ix, iy, w, h, int(corner[0]), int(corner[1]), roi,
                                               dst.ctypes.data_as(C.c_void_p), cw * 3)
        else:
            img = np.asarray(img)
            if img.ndim != 3 or img.shape[2] != 3:
                raise StitchingError("Timelapser.process_frame takes an HxWx3 image")
            if img.dtype not in (np.uint8, np.int16):
                img = img.astype(np.int16)  # what timelapser.py:42 does with every input
            img = np.ascontiguousarray(img)
            h, w = img.shape[:2]
            rc = _lib.lib().sb_timelapse_frame(img.ctypes.data_as(C.c_void_p), int(img.dtype == np.int16), img.strides[0], None, 0, 0, w, h,
                                               int(corner[0]), int(corner[1]), roi, dst.ctypes.data_as(C.c_void_p), cw * 3)
        _lib.check(rc, "sb_timelapse_frame")
        self._frame = dst

    # timelapser.py:45-49
    def get_frame(self):
        if self._frame is None:
            raise StitchingError("Timelapser.get_frame before process_frame")
        if self._frame is _EMPTY:
            from .warper import _lib_argument_error

            raise _lib_argument_error("Timelapser.get_frame: the prepared roi is empty (the images' rects touch in a line or a point)")
        return self._frame

    # timelapser.py:51-53
    def get_fixed_filename(self, img_name):
        dirname, filename = os.path.split(img_name)
        return os.path.join(dirname, self.timelapse_prefix + filename)
