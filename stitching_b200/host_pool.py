"""Page-locked host memory for the arrays the drop-in classes hand back (warped images, masks, the panorama).

The reference's calls return fresh ndarrays (warper.py:43-68, blender.py:43-48).  A fresh `np.empty` of tens of
megabytes is untouched virtual memory: the device-to-host copy into it first faults every page in and then goes through
the driver's staging buffer -- where it was measured that was most of a drop-in stitch (bench.py `e2e.dropin.stage_ms`).
Here the arrays live in buffers from `sb_host_alloc` (cudaHostAlloc): the copy is one DMA at PCIe speed, and a buffer
whose last ndarray view died goes back to a free list, so the next stitch of the same rig allocates nothing.

The arrays are ordinary writable ndarrays (views of a ctypes buffer).  The pool is bounded: beyond SB_PINNED_LIMIT_MB
(default 8192) of outstanding + cached page-locked memory `empty()` falls back to `np.empty`.
"""
import ctypes as C
import os
import threading
import weakref

import numpy as np

from . import _lib

_GRAIN = 1 << 20  # buffers come in multiples of 1 MiB so that rigs with slightly different rois share them
_lock = threading.Lock()
_free = {}        # rounded size -> [(address, library that allocated it), ...]
_total = 0        # bytes of page-locked memory alive (handed out + cached)


def _limit():
    try:
        return int(os.environ.get("SB_PINNED_LIMIT_MB", "8192")) << 20
    except ValueError:
        return 8192 << 20


def _release(block, size):
    with _lock:
        _free.setdefault(size, []).append(block)


def empty(shape, dtype=np.uint8):
    """Uninitialised ndarray of `shape` / `dtype` in page-locked memory (pageable when the pool is exhausted or the
    array is small enough not to matter)."""
    global _total
    dtype = np.dtype(dtype)
    nbytes = int(np.prod(shape, dtype=np.int64)) * dtype.itemsize
    if nbytes < (1 << 18):
        return np.empty(shape, dtype)
    size = (nbytes + _GRAIN - 1) // _GRAIN * _GRAIN
    block, drop = None, []
    with _lock:
        lst = _free.get(size)
        if lst:
            block = lst.pop()
        else:
            # make room from the cache of other sizes before giving up on page-locked memory
            for s, cached in list(_free.items()):
                while cached and _total + size > _limit():
                    drop.append(cached.pop())
                    _total -= s
            if _total + size <= _limit():
                _total += size
                block = (0, None)
    for a, L in drop:
        L.sb_host_free(a)
    if block is None:
        return np.empty(shape, dtype)
    if block[0] == 0:
        L = _lib.lib()  # a buffer goes back to the library that allocated it, whichever library is bound later
        block = (L.sb_host_alloc(size), L)
        if not block[0]:
            with _lock:
                _total -= size
            return np.empty(shape, dtype)
    buf = (C.c_uint8 * size).from_address(block[0])
    fin = weakref.finalize(buf, _release, block, size)
    fin.atexit = False  # at interpreter exit the process's memory goes away as a whole
    return np.frombuffer(buf, dtype=dtype, count=nbytes // dtype.itemsize).reshape(shape)


def trim():
    """Gives the cached buffers back to the driver (the handed-out ones follow when their arrays die)."""
    global _total
    with _lock:
        items = [(b, s) for s, lst in _free.items() for b in lst]
        _free.clear()
        _total -= sum(s for _, s in items)
    for (a, L), _ in items:
        L.sb_host_free(a)
