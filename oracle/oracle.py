"""ctypes front-end of the CPU oracle (oracle/stitch_oracle.c).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  The product (stitching_b200/) never does: it fails loudly without its CUDA library.

Function names mirror the reference call sites they restate:
  warp_roi / warp            stitching/warper.py:43-82
  MultiBand / Simple         stitching/blender.py:23-48 (cv.detail_MultiBandBlender, Feather, NO)
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libstitch_oracle.so")

TYPES = {"spherical": 0, "cylindrical": 1, "plane": 2, "affine": 3, "fisheye": 4, "stereographic": 5,
         "compressedPlaneA2B1": 6, "compressedPlaneA1.5B1": 7, "compressedPlanePortraitA2B1": 8, "compressedPlanePortraitA1.5B1": 9,
         "paniniA2B1": 10, "paniniA1.5B1": 11, "paniniPortraitA2B1": 12, "paniniPortraitA1.5B1": 13, "mercator": 14,
         "transverseMercator": 15}  # warper.py:10-27


def build(force=False):
    src = os.path.join(_HERE, "stitch_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        fp, ip, u8p, s16p = (C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_uint8), C.POINTER(C.c_int16))
        L.so_warp_roi.argtypes = [C.c_int, C.c_float, fp, fp, C.c_int, C.c_int, ip]
        L.so_warp_point.argtypes = [C.c_int, C.c_float, fp, fp, C.c_float, C.c_float, fp]
        L.so_build_maps.argtypes = [C.c_int, C.c_float, fp, fp, C.c_int, C.c_int, ip, fp, fp]
        L.so_remap_linear_u8.argtypes = [u8p, C.c_int, C.c_int, C.c_size_t, C.c_int, fp, fp, C.c_int, C.c_int, u8p, C.c_size_t]
        L.so_warp.argtypes = [C.c_int, C.c_float, fp, fp, u8p, C.c_int, C.c_int, C.c_size_t, u8p, C.c_size_t, u8p, C.c_size_t, ip]
        L.so_pyrdown_s16.argtypes = [s16p, C.c_int, C.c_int, C.c_int, s16p]
        L.so_pyrdown_s16.restype = None
        L.so_pyrdown_f32.argtypes = [fp, C.c_int, C.c_int, fp]
        L.so_pyrdown_f32.restype = None
        L.so_pyrup_s16.argtypes = [s16p, C.c_int, C.c_int, C.c_int, s16p]
        L.so_pyrup_s16.restype = None
        L.so_mb_create.argtypes = [C.c_int] * 5
        L.so_mb_create.restype = C.c_void_p
        L.so_mb_num_bands.argtypes = [C.c_void_p]
        L.so_mb_destroy.argtypes = [C.c_void_p]
        L.so_mb_destroy.restype = None
        L.so_mb_feed_rect.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, ip]
        L.so_mb_feed.argtypes = [C.c_void_p, s16p, C.c_size_t, u8p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int]
        L.so_mb_blend.argtypes = [C.c_void_p, s16p, u8p]
        L.so_dist_l1.argtypes = [u8p, C.c_size_t, C.c_int, C.c_int, fp]
        L.so_dist_l1.restype = None
        L.so_sb_create.argtypes = [C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int]
        L.so_sb_create.restype = C.c_void_p
        L.so_sb_destroy.argtypes = [C.c_void_p]
        L.so_sb_destroy.restype = None
        L.so_sb_feed.argtypes = [C.c_void_p, s16p, C.c_size_t, u8p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int]
        L.so_sb_blend.argtypes = [C.c_void_p, s16p, u8p]
        L.so_mb_fold.argtypes = [C.c_void_p, C.c_void_p]
        L.so_sb_fold.argtypes = [C.c_void_p, C.c_void_p]
        L.so_convert_scale_abs_s16.argtypes = [s16p, C.c_size_t, u8p]
        L.so_resize_linear_f32.argtypes = [fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, fp]
        L.so_resize_linear_exact_u8.argtypes = [u8p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, u8p]
        L.so_gain_apply_blocks.argtypes = [u8p, C.c_size_t, C.c_int, C.c_int, fp, C.c_int, C.c_int, C.c_int]
        L.so_gain_apply_scalar.argtypes = [u8p, C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_double)]
        L.so_dilate3x3_u8.argtypes = [u8p, C.c_size_t, C.c_int, C.c_int, u8p]
        L.so_resize_linear_u8.argtypes = [u8p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, u8p]
        L.so_seam_resize.argtypes = [u8p, C.c_size_t, C.c_int, C.c_int, u8p, C.c_size_t, C.c_int, C.c_int, u8p]
        L.so_convert_scale_abs_s16.restype = None
        _lib = L
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _kr(K, R):
    K = np.ascontiguousarray(K, dtype=np.float32).reshape(9)
    R = np.ascontiguousarray(R, dtype=np.float32).reshape(9)
    return K, R


def warp_roi(wtype, scale, K, R, size):
    """size = (w, h) -> (x, y, w, h) like PyRotationWarper.warpRoi (warper.py:79-82)."""
    K, R = _kr(K, R)
    rect = (C.c_int * 4)()
    lib().so_warp_roi(TYPES[wtype], np.float32(scale), _p(K, C.c_float), _p(R, C.c_float), size[0], size[1], rect)
    return tuple(rect)


def warp_point(wtype, scale, K, R, pt):
    K, R = _kr(K, R)
    uv = (C.c_float * 2)()
    lib().so_warp_point(TYPES[wtype], np.float32(scale), _p(K, C.c_float), _p(R, C.c_float), pt[0], pt[1], uv)
    return np.float32(uv[0]), np.float32(uv[1])


def build_maps(wtype, scale, K, R, size):
    K, R = _kr(K, R)
    rect = warp_roi(wtype, scale, K, R, size)
    xm = np.empty((rect[3], rect[2]), np.float32)
    ym = np.empty_like(xm)
    r = (C.c_int * 4)(*rect)
    lib().so_build_maps(TYPES[wtype], np.float32(scale), _p(K, C.c_float), _p(R, C.c_float), size[0], size[1], r,
                        _p(xm, C.c_float), _p(ym, C.c_float))
    return rect, xm, ym


def remap_linear(src, xmap, ymap):
    src = np.ascontiguousarray(src)
    cn = 1 if src.ndim == 2 else src.shape[2]
    h, w = src.shape[:2]
    xmap = np.ascontiguousarray(xmap, np.float32)
    ymap = np.ascontiguousarray(ymap, np.float32)
    dh, dw = xmap.shape
    dst = np.empty((dh, dw) + ((cn,) if src.ndim == 3 else ()), np.uint8)
    lib().so_remap_linear_u8(_p(src, C.c_uint8), w, h, src.strides[0], cn, _p(xmap, C.c_float), _p(ymap, C.c_float),
                             dw, dh, _p(dst, C.c_uint8), dw * cn)
    return dst


def warp(wtype, scale, K, R, img, want_image=True, want_mask=True):
    """Fused warper.py:43-52 (image) + :58-68 (mask).  Returns (rect, image|None, mask|None)."""
    K, R = _kr(K, R)
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    rect = warp_roi(wtype, scale, K, R, (w, h))
    dst = np.empty((rect[3], rect[2], 3), np.uint8) if want_image else None
    msk = np.empty((rect[3], rect[2]), np.uint8) if want_mask else None
    r = (C.c_int * 4)()
    lib().so_warp(TYPES[wtype], np.float32(scale), _p(K, C.c_float), _p(R, C.c_float), _p(img, C.c_uint8), w, h,
                  img.strides[0], _p(dst, C.c_uint8) if want_image else None, rect[2] * 3,
                  _p(msk, C.c_uint8) if want_mask else None, rect[2], r)
    return tuple(r), dst, msk


def pyrdown_s16(a):
    a = np.ascontiguousarray(a, np.int16)
    h, w = a.shape[:2]
    cn = 1 if a.ndim == 2 else a.shape[2]
    out = np.empty(((h + 1) // 2, (w + 1) // 2) + a.shape[2:], np.int16)
    lib().so_pyrdown_s16(_p(a, C.c_int16), w, h, cn, _p(out, C.c_int16))
    return out


def pyrdown_f32(a):
    a = np.ascontiguousarray(a, np.float32)
    h, w = a.shape
    out = np.empty(((h + 1) // 2, (w + 1) // 2), np.float32)
    lib().so_pyrdown_f32(_p(a, C.c_float), w, h, _p(out, C.c_float))
    return out


def pyrup_s16(a):
    a = np.ascontiguousarray(a, np.int16)
    h, w = a.shape[:2]
    cn = 1 if a.ndim == 2 else a.shape[2]
    out = np.empty((2 * h, 2 * w) + a.shape[2:], np.int16)
    lib().so_pyrup_s16(_p(a, C.c_int16), w, h, cn, _p(out, C.c_int16))
    return out


def dist_l1(mask):
    mask = np.ascontiguousarray(mask, np.uint8)
    h, w = mask.shape
    out = np.empty((h, w), np.float32)
    lib().so_dist_l1(_p(mask, C.c_uint8), mask.strides[0], w, h, _p(out, C.c_float))
    return out


def convert_scale_abs(a):
    a = np.ascontiguousarray(a, np.int16)
    out = np.empty(a.shape, np.uint8)
    lib().so_convert_scale_abs_s16(_p(a, C.c_int16), a.size, _p(out, C.c_uint8))
    return out


def dilate3x3(a):
    """cv.dilate(a, None) for a uint8 image."""
    a = np.ascontiguousarray(a, np.uint8)
    h, w = a.shape
    out = np.empty((h, w), np.uint8)
    lib().so_dilate3x3_u8(_p(a, C.c_uint8), a.strides[0], w, h, _p(out, C.c_uint8))
    return out


def resize_linear(a, size):
    """cv.resize(a, size, interpolation=cv.INTER_LINEAR) for a uint8 image; size = (w, h)."""
    a = np.ascontiguousarray(a, np.uint8)
    h, w = a.shape
    out = np.empty((int(size[1]), int(size[0])), np.uint8)
    lib().so_resize_linear_u8(_p(a, C.c_uint8), a.strides[0], w, h, int(size[0]), int(size[1]), _p(out, C.c_uint8))
    return out


def seam_resize(seam_mask, mask):
    """SeamFinder.resize (seam_finder.py:38-43): dilate, bilinear resize to the mask's size, AND with the mask."""
    seam_mask = np.ascontiguousarray(seam_mask, np.uint8)
    mask = np.ascontiguousarray(mask, np.uint8)
    sh, sw = seam_mask.shape
    h, w = mask.shape
    out = np.empty((h, w), np.uint8)
    lib().so_seam_resize(_p(seam_mask, C.c_uint8), seam_mask.strides[0], sw, sh, _p(mask, C.c_uint8), mask.strides[0], w, h,
                         _p(out, C.c_uint8))
    return out


def resize_linear_exact(a, size):
    """cv.resize(a, size, interpolation=cv.INTER_LINEAR_EXACT) for a uint8 image of 1 or 3 channels (images.py:120-123);
    size = (w, h)."""
    a = np.ascontiguousarray(a, np.uint8)
    h, w = a.shape[:2]
    cn = 1 if a.ndim == 2 else a.shape[2]
    out = np.empty((int(size[1]), int(size[0])) + (() if a.ndim == 2 else (cn,)), np.uint8)
    lib().so_resize_linear_exact_u8(_p(a, C.c_uint8), a.strides[0], w, h, cn, int(size[0]), int(size[1]), _p(out, C.c_uint8))
    return out


def resize_linear_f32(a, size):
    """cv.resize(a, size, interpolation=cv.INTER_LINEAR) for a float32 image of 1 or 3 channels; size = (w, h)."""
    a = np.ascontiguousarray(a, np.float32)
    h, w = a.shape[:2]
    cn = 1 if a.ndim == 2 else a.shape[2]
    out = np.empty((int(size[1]), int(size[0])) + (() if a.ndim == 2 else (cn,)), np.float32)
    lib().so_resize_linear_f32(_p(a, C.c_float), w, h, cn, int(size[0]), int(size[1]), _p(out, C.c_float))
    return out


def gain_apply(img, gain):
    """ExposureErrorCompensator.apply for one image (exposure_error_compensator.py:43-45), given the compensator's gain
    for it (cv.detail ...Compensator.getMatGains()[idx]): a float32 map of 1 or 3 channels (gain_blocks /
    channel_blocks), a float64 scalar (gain) or a float64 vector of >= 3 entries (channel).  Returns a new image."""
    out = np.ascontiguousarray(img, np.uint8).copy()
    h, w = out.shape[:2]
    gain = np.asarray(gain)
    if gain.dtype == np.float64:
        g = gain.ravel()
        g3 = np.array([g[0], g[0], g[0]] if g.size == 1 else g[:3], np.float64)
        lib().so_gain_apply_scalar(_p(out, C.c_uint8), out.strides[0], w, h, g3.ctypes.data_as(C.POINTER(C.c_double)))
    else:
        gain = np.ascontiguousarray(gain, np.float32)
        gc = 1 if gain.ndim == 2 else gain.shape[2]
        lib().so_gain_apply_blocks(_p(out, C.c_uint8), out.strides[0], w, h, _p(gain, C.c_float), gain.shape[1], gain.shape[0], gc)
    return out


def result_roi(corners, sizes):
    """cv.detail.resultRoi (blender.py:24): bounding box of the rects."""
    tlx = min(c[0] for c in corners)
    tly = min(c[1] for c in corners)
    brx = max(c[0] + s[0] for c, s in zip(corners, sizes))
    bry = max(c[1] + s[1] for c, s in zip(corners, sizes))
    return (tlx, tly, brx - tlx, bry - tly)


def result_roi_intersection(corners, sizes):
    """cv.detail.resultRoiIntersection: the rectangle every image covers, built as cv::Rect(Point tl, Point br) -- a
    constructor that orders its two corners, so an EMPTY intersection comes back as the (positive-sized) gap rectangle."""
    tlx = max(c[0] for c in corners)
    tly = max(c[1] for c in corners)
    brx = min(c[0] + s[0] for c, s in zip(corners, sizes))
    bry = min(c[1] + s[1] for c, s in zip(corners, sizes))
    return (min(tlx, brx), min(tly, bry), abs(brx - tlx), abs(bry - tly))


class Timelapser:
    """Restatement of stitching/timelapser.py:7-56 (cv.detail.Timelapser AS_IS / CROP): every frame is a zeroed canvas of
    the prepared roi -- resultRoi for "as_is", resultRoiIntersection for "crop" -- with ONE warped image pasted at its
    corner (pixels outside the canvas dropped), then |.| saturated to uint8 (timelapser.py:44-52: int16 -> float32 ->
    convertScaleAbs)."""

    def __init__(self, timelapse="no"):
        self.timelapse_type = timelapse
        self.do_timelapse = timelapse in ("as_is", "crop")
        self.roi = None
        self._dst = None

    def initialize(self, corners, sizes):
        self.roi = result_roi(corners, sizes) if self.timelapse_type == "as_is" else result_roi_intersection(corners, sizes)
        self._dst = np.zeros((max(self.roi[3], 0), max(self.roi[2], 0), 3), np.int16)

    def process_frame(self, img, corner):
        img = np.asarray(img).astype(np.int16)  # timelapser.py:42
        x, y, w, h = self.roi
        self._dst[...] = 0
        dx, dy = int(corner[0]) - x, int(corner[1]) - y
        x0, y0 = max(dx, 0), max(dy, 0)
        x1, y1 = min(dx + img.shape[1], w), min(dy + img.shape[0], h)
        if x1 > x0 and y1 > y0:
            self._dst[y0:y1, x0:x1] = img[y0 - dy:y1 - dy, x0 - dx:x1 - dx]

    def get_frame(self):
        return convert_scale_abs(self._dst)


class Blender:
    """Restatement of stitching/blender.py:5-56 on top of the C oracle (same method names)."""

    def __init__(self, blender_type="multiband", blend_strength=5):
        self.blender_type = blender_type
        self.blend_strength = blend_strength
        self._h = None
        self._kind = None
        self.num_bands = None
        self.sharpness = None

    def prepare(self, corners, sizes):
        self._free()
        self.roi = result_roi(corners, sizes)
        x, y, w, h = self.roi
        blend_width = np.sqrt(w * h) * self.blend_strength / 100
        if self.blender_type == "no" or blend_width < 1:
            self._kind = "no"
            self._h = lib().so_sb_create(0, 0.0, x, y, w, h)
        elif self.blender_type == "multiband":
            self._kind = "multiband"
            self._h = lib().so_mb_create(int((np.log(blend_width) / np.log(2.0) - 1.0)), x, y, w, h)
            self.num_bands = lib().so_mb_num_bands(self._h)
        elif self.blender_type == "feather":
            self._kind = "feather"
            self.sharpness = np.float32(1.0 / blend_width)
            self._h = lib().so_sb_create(1, self.sharpness, x, y, w, h)
        else:
            raise ValueError(self.blender_type)

    def feed(self, img, mask, corner):
        img = np.ascontiguousarray(np.asarray(img).astype(np.int16))
        mask = np.ascontiguousarray(mask, np.uint8)
        h, w = mask.shape
        f = lib().so_mb_feed if self._kind == "multiband" else lib().so_sb_feed
        rc = f(self._h, _p(img, C.c_int16), w * 3, _p(mask, C.c_uint8), w, w, h, int(corner[0]), int(corner[1]))
        if rc:
            raise ValueError("feed rect outside the prepared roi")

    def fold(self, other):
        """Add `other`'s accumulators into this blender's (int16 sums with wrap-around, float weight sums with a plain
        +=); `other` must be prepared with the same roi and kind and is left as it was.  Restates how the owner of a
        strip in the sharded composite adds another rank's partial sums."""
        if self._kind != other._kind or self.roi != other.roi or self._kind == "no":
            raise ValueError("fold needs two multiband or two feather blenders prepared with the same roi")
        f = lib().so_mb_fold if self._kind == "multiband" else lib().so_sb_fold
        if f(self._h, other._h):
            raise ValueError("fold: blenders of different geometry")

    def blend_s16(self):
        x, y, w, h = self.roi
        dst = np.empty((h, w, 3), np.int16)
        msk = np.empty((h, w), np.uint8)
        (lib().so_mb_blend if self._kind == "multiband" else lib().so_sb_blend)(self._h, _p(dst, C.c_int16), _p(msk, C.c_uint8))
        self._free()
        return dst, msk

    def blend(self):
        dst, msk = self.blend_s16()
        return convert_scale_abs(dst), msk

    def _free(self):
        if self._h is not None:
            (lib().so_mb_destroy if self._kind == "multiband" else lib().so_sb_destroy)(self._h)
            self._h = None

    def __del__(self):
        try:
            self._free()
        except Exception:
            pass
