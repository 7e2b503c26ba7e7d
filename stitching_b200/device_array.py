"""Device-resident twins of the arrays the drop-in classes hand out (SURVEY.md 8b "device-handle variants").

The reference pipeline moves every FINAL-resolution image through plain ndarrays: Warper.warp_image -> (crop: slicing,
cropper.py:150-151) -> ExposureErrorCompensator.apply -> Blender.feed (stitcher.py:185-189, 219-221, 254).  With host
buffers at every call that is three PCIe round trips per image.  `DeviceBacked` is an ndarray -- a real, filled host
array, so cv2, numpy and every other consumer of the reference keep working on it -- that additionally remembers a
device copy of the same bytes (a `sb_devimg` handle of the C ABI).  Slices stay twins (the view's offset inside the
root buffer selects the same rectangle on the device); anything numpy has to copy (astype, fancy indexing, arithmetic)
is an ordinary ndarray again.  The array is read-only, so host and device copies cannot drift apart behind the
library's back; the drop-ins that legitimately modify an image in place (ExposureErrorCompensator.apply) update both.
"""
import numpy as np

from . import _lib


class _Handle:
    """Owns one sb_devimg."""

    def __init__(self, ptr):
        self.ptr = ptr
        self.L = _lib.lib()  # released by the library that made it, whichever is bound later

    def __del__(self):
        try:
            if self.ptr:
                self.L.sb_devimg_release(self.ptr)
                self.ptr = None
        except Exception:  # interpreter shutdown
            pass


class DeviceBacked(np.ndarray):
    """uint8 ndarray (HxWx3 image or HxW mask) with a device twin; see the module docstring."""

    _sb = None  # (handle, root address, root nbytes, root width, channels)

    def __array_finalize__(self, obj):
        self._sb = None
        info = getattr(obj, "_sb", None)
        if info is None or self.dtype != np.uint8:
            return
        handle, root, nbytes, width, ch = info
        addr = self.__array_interface__["data"][0]
        # a view into the root buffer with the root's row / pixel strides (plain 2-D slicing) keeps the twin
        if not (root <= addr < root + nbytes) or self.ndim != (3 if ch == 3 else 2):
            return
        st = self.strides
        if st[0] != width * ch or st[1] != ch or (ch == 3 and (self.shape[2] != 3 or st[2] != 1)):
            return
        self._sb = info


def wrap(host, handle_ptr):
    """`host`: the freshly filled C-contiguous uint8 array; handle_ptr: sb_devimg* holding the same bytes (or None)."""
    if not handle_ptr:
        return host
    out = host.view(DeviceBacked)
    ch = 3 if host.ndim == 3 else 1
    out._sb = (_Handle(handle_ptr), host.__array_interface__["data"][0], host.nbytes, host.shape[1], ch)
    out.flags.writeable = False
    return out


def twin(arr):
    """(sb_devimg*, x, y, w, h) of the device rectangle that holds `arr`'s bytes, or None when `arr` has no (valid) twin."""
    info = getattr(arr, "_sb", None)
    if info is None or not isinstance(arr, DeviceBacked) or arr.flags.writeable:
        return None  # (a caller that made the array writable may have changed the host copy)
    handle, root, _nbytes, width, ch = info
    off = arr.__array_interface__["data"][0] - root
    y, rem = divmod(off, width * ch)
    if rem % ch:
        return None
    return handle.ptr, rem // ch, y, arr.shape[1], arr.shape[0]


def keep_alive(arr):
    info = getattr(arr, "_sb", None)
    return info[0] if info else None
