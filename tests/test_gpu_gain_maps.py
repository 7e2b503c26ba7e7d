"""Exposure gain maps of every shape against cv2's own results (tests/gain_maps.py) through the real library on the
H100, and at camera scale: maps one block wide or high stretched more than 100 times onto 4000 x 3000-class images
through ExposureErrorCompensator.apply (host buffers and device twins) and Compositor.set_gain."""
import numpy as np
import pytest

import fuzz_chain
import gain_maps as GM
import replay
from stitching_b200 import exposure_error_compensator as ec

pytestmark = pytest.mark.gpu


def _apply(img, gain):
    return ec.apply_gain(img, gain)


def test_goldens(cuda_lib, oracle):
    GM.check_oracle_resize(oracle)
    GM.check_apply_goldens(oracle, _apply)
    GM.check_feed_goldens(oracle, _apply)


def test_device_twin_at_a_crop_offset(cuda_lib, oracle):
    GM.check_device_twin(oracle)
    GM.check_device_twin(oracle, size=(1500, 1100), crop=(13, 31, 7, 2), foil=False)


@pytest.mark.parametrize("seed", range(3, 9))
def test_compositor_set_gain(cuda_lib, oracle, seed):
    """Foil images at the emulation build's sizes, then noise images a few hundred px across."""
    sizes, maps = GM.compositor_draw(seed, 90)
    GM.check_compositor(oracle, sizes, maps, seed)
    sizes, maps = GM.compositor_draw(seed, 700)
    rng = np.random.default_rng(seed)
    arrays = [None if m is None else rng.uniform(0.55, 1.9, m[0] + (m[1],)).astype(np.float32) for m in maps]
    GM.check_compositor(oracle, sizes, arrays, seed, foil=False)


def test_timelapse_with_clipped_parts(cuda_lib, oracle):
    GM.check_timelapse(oracle)


def test_sharded_owner_sets_the_gain(cuda_lib, oracle):
    GM.check_sharded(oracle, fuzz_chain.device_copy, scale_down=4)


def test_live_sweep_against_cv2(cuda_lib, oracle):
    pytest.importorskip("cv2")
    GM.live_sweep(oracle, _apply, 40, 20261018, max_side=700)


# maps one block high or wide stretched onto camera-size images: 1 x 5 (1 x 13) from a LOW image 28 px high at ratios
# 22 and 11, their transposes, and a 1 x 1 map
CAMERA = [((1, 5), 1, (3960, 2990)), ((1, 13), 3, (4000, 300)), ((5, 1), 3, (2990, 3960)), ((9, 1), 1, (220, 3100)),
          ((1, 1), 3, (4000, 3000))]


def _camera_maps():
    rng = np.random.default_rng(2026)
    out = []
    for shape, cn, size in CAMERA:
        m = rng.uniform(0.55, 1.9, shape + (cn,)).astype(np.float32)
        out.append((m[:, :, 0] if cn == 1 else m, size))
    return out


def test_camera_scale_apply(cuda_lib, oracle):
    """sb_gain_apply on host buffers: 1-px maps stretched 100-4000 times."""
    for k, (m, (w, h)) in enumerate(_camera_maps()):
        img = GM.noise(h, w, 70 + k)
        replay.assert_exact(np.asarray(_apply(img.copy(), m)), oracle.gain_apply(img, m), f"camera scale map {m.shape} on {w}x{h}")


def test_camera_scale_compositor(cuda_lib, oracle):
    """Compositor.set_gain with the same maps on camera-size images, one batch."""
    cases = _camera_maps()[:3]
    GM.check_compositor(oracle, [s for _, s in cases], [m for m, _ in cases], foil=False)


def test_camera_scale_device_twin(cuda_lib, oracle):
    GM.check_device_twin(oracle, size=(4000, 3000), crop=(9, 21, 4, 17), foil=False)
