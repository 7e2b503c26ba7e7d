"""The C-ABI shared library loads and exports every symbol include/stitch_b200.h declares (no GPU needed)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT
from stitching_b200 import _lib

HEADER = os.path.join(ROOT, "include", "stitch_b200.h")


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"SB_API\s+[^;(]*?\b(sb_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_entries():
    syms = declared_symbols()
    assert len(syms) >= 25
    for required in ("sb_warp", "sb_warp_roi", "sb_blender_prepare", "sb_blender_feed", "sb_blender_blend", "sb_compositor_run"):
        assert required in syms


def test_library_exports_every_declared_symbol():
    assert os.path.exists(_lib.LIB_PATH), "build the library first: make -C stitching_b200/csrc (or __graft_entry__.build())"
    L = ctypes.CDLL(_lib.LIB_PATH)
    missing = [s for s in declared_symbols() if not hasattr(L, s)]
    assert not missing, f"not exported: {missing}"


def test_binding_covers_the_header():
    bound = {name for name, _, _ in _lib.SIGNATURES}
    assert bound == set(declared_symbols())
    _lib.bind(_lib.LIB_PATH)  # attaches every prototype


def test_library_targets_sm90a_only():
    import shutil
    import subprocess

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "--list-elf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_no_cpu_fallback_without_a_gpu():
    """Geometry is host-only and works; compute entries must fail loudly when no device is usable."""
    import numpy as np

    L = _lib.bind(_lib.LIB_PATH)
    K = np.array([[100, 0, 50], [0, 100, 40], [0, 0, 1]], np.float32)
    R = np.eye(3, dtype=np.float32)
    rect = (ctypes.c_int * 4)()
    fp = lambda a: a.ctypes.data_as(_lib.c_float_p)  # noqa: E731
    assert L.sb_warp_roi(0, 100.0, fp(K), fp(R), 100, 80, rect) == 0
    assert rect[2] > 0 and rect[3] > 0
    if os.path.exists("/dev/nvidia0") or os.path.exists("/dev/nvidiactl"):
        pytest.skip("a GPU is present: the failure path cannot be exercised")
    src = np.zeros((80, 100, 3), np.uint8)
    dst = np.zeros((rect[3], rect[2], 3), np.uint8)
    rc = L.sb_warp(0, 100.0, fp(K), fp(R), src.ctypes.data_as(ctypes.c_void_p), 100, 80, 300,
                   dst.ctypes.data_as(ctypes.c_void_p), rect[2] * 3, None, 0, rect)
    assert rc == -2, rc  # SB_ERR_NO_DEVICE
    assert b"no CPU fallback" in L.sb_last_error()
