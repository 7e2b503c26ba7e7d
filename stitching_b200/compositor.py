"""Fused warp + blend on one GPU with every intermediate resident in HBM (sb_compositor_* in the C ABI).

Equivalent to running, for a fixed rig, the FINAL-resolution half of Stitcher.stitch: stitcher.py:178-189
(Warper.warp_images / create_and_warp_masks / warp_rois), the crop of stitcher.py:198-208 when a `Crop` is given,
ExposureErrorCompensator.apply and SeamFinder.resize when gains and seam masks are set, and stitcher.py:241-259
(Blender.prepare / feed / blend) -- with one host->device copy of the sources and one device->host copy of the
panorama.  Without seam masks or masks the warped validity mask is the blend mask (seam finder "no").
"""
import ctypes as C
from statistics import median

import numpy as np

from . import _lib
from .stitching_error import StitchingError
from .warper import Warper


def time_multi(compositors, iters):
    """Device time (ms) of `iters` steps dealt round-robin to several compositors of the same rig (batches in flight)."""
    n = len(compositors)
    arr = (C.c_void_p * n)(*[c._c for c in compositors])
    ms = C.c_float()
    _lib.check(_lib.lib().sb_compositor_time_multi(arr, n, int(iters), C.byref(ms)), "sb_compositor_time_multi")
    return ms.value


def _scaled(rect, aspect):
    """A LOW-resolution (x, y, w, h) in FINAL pixels, each component rounded half to even (Python's round)."""
    return tuple(int(round(v * aspect)) for v in rect)


class Crop:
    """The crop of every image in FINAL pixels, as Stitcher.crop_final_resolution applies it.

    rects[i]: (x, y, w, h), the slice of warped image i that is fed (clipped at the warped image's bottom and right);
    corners[i]: where it is fed (Blender.feed); sizes[i]: its size as Blender.prepare sees it, which sets the pano roi
    and num_bands.  The fed size is the clipped slice, so it may be smaller than sizes[i]."""

    def __init__(self, rects, corners, sizes):
        self.rects = [tuple(int(v) for v in r) for r in rects]
        self.corners = [tuple(int(v) for v in c) for c in corners]
        self.sizes = [tuple(int(v) for v in s) for s in sizes]
        if not (len(self.rects) == len(self.corners) == len(self.sizes)):
            raise StitchingError("Crop needs one rect, corner and size per image")
        if any(len(r) != 4 for r in self.rects) or any(len(c) != 2 for c in self.corners) or any(len(s) != 2 for s in self.sizes):
            raise StitchingError("Crop: rects are (x, y, w, h), corners (x, y), sizes (w, h)")

    @classmethod
    def from_cropper(cls, cropper, aspect=1):
        """The crop a prepared Cropper (cropper.py) applies at `aspect` = LOW -> FINAL ratio; None if it does not crop.

        Image i is sliced by its intersection rectangle and fed at its overlapping rectangle, both scaled separately
        (so their roundings differ); the scaled overlap corners are shifted so that the smallest x and y are 0."""
        if not cropper.do_crop:
            return None
        rects = [_scaled(r, aspect) for r in cropper.intersection_rectangles]
        overlaps = [_scaled(r, aspect) for r in cropper.overlapping_rectangles]
        x0 = min(o[0] for o in overlaps)
        y0 = min(o[1] for o in overlaps)
        return cls(rects, [(o[0] - x0, o[1] - y0) for o in overlaps], [(o[2], o[3]) for o in overlaps])


class Compositor:
    def __init__(self, cameras, sizes, warper_type="spherical", blender_type="multiband", blend_strength=5, scale=None,
                 aspect=1, rank=0, world=1, crop=None, input_sizes=None, timelapse=None):
        """cameras: objects with .focal, .K(), .R (cv.detail.CameraParams or rigs.Camera); sizes: [(w, h)].

        crop: a `Crop` (e.g. Crop.from_cropper(stitcher.cropper, aspect)); every image is then warped only over its
        slice and fed at the crop's corner, and `self.rects` holds the fed rects (corner, fed size): the shapes that
        set_mask and download_warped use, and that set_seam_mask and set_gain resize to.

        world > 1: one panorama over `world` GPUs, one process per GPU.  Every rank passes ALL cameras; rank r owns
        images [r*n/world, (r+1)*n/world) -- `self.first`, `self.count` -- uploads only those and gets the column
        strip `self.strip` = (lo, hi) of the panorama back (stitching_b200.dist.init_comm must have run).

        input_sizes: [(w, h)] of the frames upload / submit / composite then take, e.g. the camera sizes `st.images.sizes`
        of a Stitcher whose final_megapix is set; `sizes` stay the FINAL sizes
        (`st.images.get_scaled_img_sizes(Images.Resolution.FINAL)`).  Frame i is resized from input_sizes[i] to sizes[i] on
        the device, byte for byte as Images.resize_img_by_scaler does (cv.resize INTER_LINEAR_EXACT); a frame whose two
        sizes are equal is taken as it is.  Inputs smaller than their FINAL size on either axis are refused.

        timelapse: "as_is" or "crop" -- a Stitcher with that timelapse setting: every step ends in one frame per image
        (Timelapser.process_frame / get_frame) instead of a panorama.  `self.roi` is then the canvas; submit_timelapse /
        wait / frames, or timelapse(), run the steps; set_gain works, the blend, mask and panorama calls do not.  One GPU
        only; blender_type and blend_strength are unused."""
        n = len(cameras)
        if n == 0 or len(sizes) != n:
            raise StitchingError("Compositor needs one size per camera")
        if timelapse is not None and timelapse not in _lib.TIMELAPSE_KINDS:
            raise StitchingError(f"unknown timelapse kind '{timelapse}' (the compositor writes frames for 'as_is' and 'crop')")
        if timelapse is not None and int(world) != 1:
            raise StitchingError("a timelapse compositor runs on one GPU")
        if crop is not None and len(crop.rects) != n:
            raise StitchingError(f"Crop has {len(crop.rects)} rects for {n} images")
        if warper_type not in _lib.WARP_TYPES:
            raise StitchingError(f"warper type '{warper_type}' is not on the GPU path")
        if blender_type not in _lib.BLEND_KINDS:
            raise StitchingError(f"unknown blender type '{blender_type}'")
        self.n = n
        self.sizes = [(int(w), int(h)) for w, h in sizes]
        if input_sizes is not None and len(input_sizes) != n:
            raise StitchingError(f"Compositor has {len(input_sizes)} input sizes for {n} images")
        self.input_sizes = self.sizes if input_sizes is None else [(int(w), int(h)) for w, h in input_sizes]
        if scale is None:
            scale = median([cam.focal for cam in cameras])  # Warper.set_scale
        # Stitcher's ratios are numpy float64, so Warper.get_K scales the float32 K in double and rounds once; a Python
        # float would make numpy multiply in float32, one rounding off at some ratios.  Take the ratio as the Stitcher does.
        aspect = np.float64(aspect)
        self.scale = scale * aspect
        self._K = np.ascontiguousarray(np.stack([Warper.get_K(c, aspect) for c in cameras]).astype(np.float32))
        self._R = np.ascontiguousarray(np.stack([np.asarray(c.R, np.float32) for c in cameras]))
        self._w = (C.c_int * n)(*[s[0] for s in self.sizes])
        self._h = (C.c_int * n)(*[s[1] for s in self.sizes])
        rig = _lib.Rig(n, _lib.WARP_TYPES[warper_type], np.float32(self.scale), _lib.BLEND_KINDS[blender_type],
                       float(blend_strength), self._w, self._h, self._K.ctypes.data_as(_lib.c_float_p),
                       self._R.ctypes.data_as(_lib.c_float_p))
        L = self._L = _lib.lib()  # close() releases through the library that created the compositor
        self.rank, self.world = int(rank), int(world)
        desc = in_w = in_h = None
        if crop is not None:
            arrs = [(C.c_int * (k * n))(*[v for t in ts for v in t]) for k, ts in ((4, crop.rects), (2, crop.corners), (2, crop.sizes))]
            desc = C.pointer(_lib.CropDesc(*[C.cast(a, _lib.c_int_p) for a in arrs]))
        if input_sizes is not None:
            in_w = (C.c_int * n)(*[s[0] for s in self.input_sizes])
            in_h = (C.c_int * n)(*[s[1] for s in self.input_sizes])
        self.timelapse_kind = timelapse
        opts = _lib.CompositorOpts(desc, in_w, in_h, self.rank, self.world, _lib.TIMELAPSE_KINDS.get(timelapse, 0))
        self._c = L.sb_compositor_create(C.byref(rig), C.byref(opts))
        if not self._c:
            _lib.check(-1, "sb_compositor_create")
        rects = (C.c_int * (4 * n))()
        roi = (C.c_int * 4)()
        nb = C.c_int()
        _lib.check(L.sb_compositor_geometry(self._c, rects, roi, C.byref(nb)), "sb_compositor_geometry")
        self.rects = [tuple(rects[4 * i: 4 * i + 4]) for i in range(n)]
        self.roi = tuple(roi)
        self.num_bands = nb.value
        self._pinned = []
        first, count, strip = C.c_int(), C.c_int(), (C.c_int * 2)()
        _lib.check(L.sb_compositor_shard_info(self._c, C.byref(first), C.byref(count), strip), "sb_compositor_shard_info")
        self.first, self.count, self.strip = first.value, count.value, (strip[0], strip[1])
        self.strip_axis = int(L.sb_compositor_shard_axis(self._c))  # 0: self.strip are columns of the panorama, 1: rows

    # -- data movement ---------------------------------------------------------------------------
    def upload(self, images, pinned=False):
        """images: the frames of THIS rank's block, in order (all n frames when world == 1)."""
        L = _lib.lib()
        if len(images) != self.count:
            raise StitchingError(f"expected {self.count} images (block {self.first}..{self.first + self.count - 1}), got {len(images)}")
        for i, img in enumerate(images, start=self.first):
            img = np.asarray(img)
            w, h = self.input_sizes[i]
            if img.dtype != np.uint8 or img.shape != (h, w, 3):
                raise StitchingError(f"image {i}: expected uint8 {h}x{w}x3")
            if img.strides[2] != 1 or img.strides[1] != 3:
                img = np.ascontiguousarray(img)
            _lib.check(L.sb_compositor_upload(self._c, i, img.ctypes.data_as(C.c_void_p), img.strides[0], int(pinned)),
                       "sb_compositor_upload")

    def set_mask(self, i, mask):
        """Blend mask of image i in warped coordinates (uint8 h' x w', e.g. SeamFinder.resize's output); replaces the
        warped validity mask as blend weight from the next run on."""
        if hasattr(mask, "get") and not isinstance(mask, np.ndarray):
            mask = mask.get()
        mask = np.ascontiguousarray(mask, np.uint8)
        if mask.shape != (self.rects[i][3], self.rects[i][2]):
            raise StitchingError(f"mask {i}: expected {self.rects[i][3]}x{self.rects[i][2]}")
        _lib.check(_lib.lib().sb_compositor_set_mask(self._c, i, mask.ctypes.data_as(C.c_void_p), mask.strides[0]),
                   "sb_compositor_set_mask")

    def set_gain(self, i, gain):
        """Exposure gain of image i (one entry of a fed cv.detail compensator's getMatGains(): float32 map of 1 or 3
        channels, float64 scalar or vector; None removes it): ExposureErrorCompensator.apply (stitcher.py:219-221)
        fused into the warp kernel's epilogue from the next run on."""
        from .exposure_error_compensator import gain_arguments

        gmap, gw, gh, gc, gscalar = gain_arguments(gain)
        _lib.check(_lib.lib().sb_compositor_set_gain(self._c, i, gmap.ctypes.data_as(C.c_void_p) if gmap is not None else None, gw, gh, gc,
                                                     gscalar.ctypes.data_as(C.c_void_p) if gscalar is not None else None),
                   "sb_compositor_set_gain")

    def set_seam_mask(self, i, seam_mask):
        """Blend mask of image i from its LOW-resolution seam mask (what SeamFinder.find returns): SeamFinder.resize
        (seam_finder.py:38-43) runs on the device -- dilate, resize to the warped size, AND with the warped mask."""
        if hasattr(seam_mask, "get") and not isinstance(seam_mask, np.ndarray):
            seam_mask = seam_mask.get()
        seam_mask = np.ascontiguousarray(seam_mask, np.uint8)
        if seam_mask.ndim != 2:
            raise StitchingError(f"seam mask {i}: expected a 2-d uint8 array")
        _lib.check(_lib.lib().sb_compositor_set_seam_mask(self._c, i, seam_mask.ctypes.data_as(C.c_void_p), seam_mask.strides[0],
                                                          seam_mask.shape[1], seam_mask.shape[0]), "sb_compositor_set_seam_mask")

    def run(self):
        _lib.check(_lib.lib().sb_compositor_run(self._c), "sb_compositor_run")

    def sync(self):
        _lib.check(_lib.lib().sb_compositor_sync(self._c), "sb_compositor_sync")

    def download(self, out=None, out_mask=None):
        """(pano, mask); with world > 1 the columns (strip_axis 0) or rows (strip_axis 1) self.strip[0]:self.strip[1]."""
        h, w = self.roi[3], self.roi[2]
        if self.strip_axis == 0:
            w = self.strip[1] - self.strip[0]
        else:
            h = self.strip[1] - self.strip[0]
        pano = np.empty((h, w, 3), np.uint8) if out is None else out
        mask = np.empty((h, w), np.uint8) if out_mask is None else out_mask
        _lib.check(_lib.lib().sb_compositor_download(self._c, pano.ctypes.data_as(C.c_void_p), pano.strides[0],
                                                     mask.ctypes.data_as(C.c_void_p), mask.strides[0]),
                   "sb_compositor_download")
        return pano, mask

    def download_warped(self, i):
        _, _, w, h = self.rects[i]
        img = np.empty((h, w, 3), np.uint8)
        mask = np.empty((h, w), np.uint8)
        _lib.check(_lib.lib().sb_compositor_download_warped(self._c, i, img.ctypes.data_as(C.c_void_p), w * 3,
                                                            mask.ctypes.data_as(C.c_void_p), w),
                   "sb_compositor_download_warped")
        return img, mask

    # -- sharded composite: transport hooks (sb_compositor_run moves the slabs with NCCL itself) ---------
    def shard_phase(self, phase):
        """0: local kernels up to the filled send slabs; 1: finish after the receive slabs were filled."""
        _lib.check(_lib.lib().sb_compositor_shard_phase(self._c, int(phase)), "sb_compositor_shard_phase")

    def shard_slab(self, peer, outgoing):
        """(device pointer, bytes) of the slab sent to (outgoing=True) or received from `peer`; bytes may be 0."""
        p, n = C.c_void_p(), C.c_size_t()
        _lib.check(_lib.lib().sb_compositor_shard_slab(self._c, int(peer), int(bool(outgoing)), C.byref(p), C.byref(n)),
                   "sb_compositor_shard_slab")
        return p.value, n.value

    def _sources(self, images):
        if len(images) != self.n:
            raise StitchingError(f"expected {self.n} images, got {len(images)}")
        ptrs = (C.c_void_p * self.n)()
        pitches = (C.c_size_t * self.n)()
        for i, img in enumerate(images):
            w, h = self.input_sizes[i]
            if img.dtype != np.uint8 or img.shape != (h, w, 3) or img.strides[1:] != (3, 1):
                raise StitchingError(f"image {i}: expected a uint8 {h}x{w}x3 array with packed pixels")
            ptrs[i] = img.ctypes.data
            pitches[i] = img.strides[0]
        return ptrs, pitches

    def submit(self, images, out, out_mask):
        """Pipelined step: enqueue upload of `images`, warp + blend, download into `out` / `out_mask`; returns a
        ticket for wait().  At most three tickets in flight; host arrays should live in pinned memory
        (`pinned_empty`) and must stay untouched until wait(ticket) returns."""
        ptrs, pitches = self._sources(images)
        ticket = C.c_ulonglong()
        _lib.check(_lib.lib().sb_compositor_submit(self._c, ptrs, pitches, out.ctypes.data_as(C.c_void_p), out.strides[0],
                                                   out_mask.ctypes.data_as(C.c_void_p), out_mask.strides[0], C.byref(ticket)),
                   "sb_compositor_submit")
        return ticket.value

    def wait(self, ticket):
        _lib.check(_lib.lib().sb_compositor_wait(self._c, C.c_ulonglong(ticket)), "sb_compositor_wait")

    # -- timelapse (Compositor(..., timelapse="as_is" | "crop")) -------------------------------------------------------
    def submit_timelapse(self, images):
        """Pipelined timelapse step: enqueue upload of `images`, warp, and the copy of every image's part into its frame;
        returns a ticket for wait() and frames().  At most three tickets in flight; host arrays should live in pinned
        memory (`pinned_empty`) and must stay untouched until wait(ticket) returns."""
        ptrs, pitches = self._sources(images)
        ticket = C.c_ulonglong()
        _lib.check(_lib.lib().sb_compositor_submit_timelapse(self._c, ptrs, pitches, C.byref(ticket)), "sb_compositor_submit_timelapse")
        return ticket.value

    def frames(self, ticket):
        """The n frames of `ticket` after wait(ticket): read-only uint8 views (canvas h x w x 3) into the library's
        page-locked frames, valid until ticket + 3 is submitted or close() is called (copy what must live longer).  A
        view keeps the compositor alive, so dropping the compositor does not free the memory under it; an explicit
        close() does."""
        out = []
        for i in range(self.n):
            p, pitch = C.c_void_p(), C.c_size_t()
            _lib.check(_lib.lib().sb_compositor_timelapse_frame(self._c, C.c_ulonglong(ticket), i, C.byref(p), C.byref(pitch)),
                       "sb_compositor_timelapse_frame")
            w, h = self.roi[2], self.roi[3]
            buf = (C.c_uint8 * (pitch.value * h)).from_address(p.value)
            buf.owner = self  # the ndarray's base is `buf`
            a = np.ndarray((h, w, 3), np.uint8, buffer=buf, strides=(pitch.value, 3, 1))
            a.flags.writeable = False
            out.append(a)
        return out

    def timelapse(self, images):
        """One timelapse step: submit_timelapse + wait; returns n owned copies of the frames, as Timelapser.get_frame
        returns them after process_frame of each image."""
        images = [np.ascontiguousarray(img) for img in images]
        t = self.submit_timelapse(images)
        self.wait(t)
        return [f.copy() for f in self.frames(t)]

    def pinned_empty(self, shape):
        """uint8 ndarray in page-locked host memory (freed with the compositor: invalid after close())."""
        nbytes = int(np.prod(shape))
        p = self._L.sb_host_alloc(nbytes)
        if not p:
            _lib.check(-5, "sb_host_alloc")
        self._pinned.append(p)
        return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p)).reshape(shape)

    def composite(self, images):
        """One call: upload, warp + blend, download.  Returns (uint8 pano, uint8 mask) like Blender.blend()."""
        self.upload(images)
        self.run()
        return self.download()

    # -- measurement -------------------------------------------------------------------------------
    def time(self, iters, flush_l2=False):
        """Device time of `iters` runs, CUDA events on the compositor stream.

        Returns (total_ms, [(launch name, ms per run)]) with one entry per kernel launch, in launch order."""
        ms = C.c_float()
        _lib.check(_lib.lib().sb_compositor_time(self._c, int(iters), int(flush_l2), C.byref(ms)), "sb_compositor_time")
        cap = 64
        names = (C.c_char_p * cap)()
        vals = (C.c_float * cap)()
        k = _lib.lib().sb_compositor_stage_times(self._c, names, vals, cap)
        return ms.value, [(names[i].decode(), vals[i]) for i in range(k)]

    def model_bytes(self):
        """Compulsory HBM traffic of one run: (total bytes, [bytes per launch, in launch order])."""
        cap = 64
        tot = C.c_double()
        per = (C.c_double * cap)()
        k = _lib.lib().sb_compositor_model_bytes(self._c, C.byref(tot), per, cap)
        if k < 0:
            _lib.check(k, "sb_compositor_model_bytes")
        return tot.value, [per[i] for i in range(k)]

    def close(self):
        if getattr(self, "_c", None):
            self._L.sb_compositor_destroy(self._c)  # synchronises all its streams first
            self._c = None
            for p in self._pinned:
                self._L.sb_host_free(p)
            self._pinned = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
