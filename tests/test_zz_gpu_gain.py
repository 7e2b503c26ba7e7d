"""ExposureErrorCompensator.apply on the device (SURVEY 8f, f2): the reference's goldens, fuzz against the oracle and the
fused Compositor.set_gain, through the real library.  Kept in its own file, last in collection order."""
import numpy as np
import pytest

import replay
from stitching_b200 import Blender, Compositor, Warper, rigs
from stitching_b200 import exposure_error_compensator as ec

pytestmark = pytest.mark.gpu


def test_gain_apply_goldens_and_fuzz(cuda_lib, oracle):
    replay.run_gain_goldens(lambda img, gain: ec.apply_gain(img.copy(), gain))
    rng = np.random.default_rng(22)
    for t in range(12):
        h, w = int(rng.integers(20, 900)), int(rng.integers(20, 1200))
        img = rigs.noise_image(h, w, 400 + t)
        if t % 3 == 2:
            gain = np.array([[rng.uniform(0.4, 2.5)]], np.float64)
        else:
            gain = rng.uniform(0.5, 2.5, (int(rng.integers(1, 40)), int(rng.integers(1, 50))) + ((3,) if t % 3 else ())).astype(np.float32)
        replay.assert_exact(ec.apply_gain(img.copy(), gain), oracle.gain_apply(img, gain), f"gain fuzz {t}")



def test_gains_out_of_the_int_range(cuda_lib, oracle):
    """Products beyond the int range and NaN round to INT_MIN (so 0) as on x86, not to the device's saturated 255."""
    replay.run_gain_range_golden(oracle, ec.apply_gain, Warper, Blender, Compositor, rigs, 4)

def test_fused_final_resolution_chain(cuda_lib, oracle):
    """Gains and seam masks together in the fast warp kernel's extras path."""
    got, ref = replay.fused_chain_case(oracle, Warper, Blender, Compositor, rigs, 4)
    replay.assert_exact(got[0], ref[0], "pano of the fused chain")
    replay.assert_exact(got[1], ref[1], "mask of the fused chain")


def test_image_resize_goldens_and_fuzz(cuda_lib, oracle):
    """Images.resize_img_by_scaler (cv.resize INTER_LINEAR_EXACT, SURVEY 8f f3) on the device."""
    from stitching_b200 import images

    replay.run_resize_goldens(images.resize_exact)
    rng = np.random.default_rng(32)
    for t in range(12):
        sh, sw = int(rng.integers(2, 1200)), int(rng.integers(2, 1600))
        sc = rng.uniform(0.05, 1.0) if t % 3 else rng.uniform(1.0, 3.0)
        size = (max(1, int(round(sw * sc))), max(1, int(round(sh * sc))))
        src = rng.integers(0, 256, (sh, sw, 3) if t % 2 else (sh, sw), dtype=np.uint8)
        replay.assert_exact(images.resize_exact(src, size), oracle.resize_linear_exact(src, size), f"resize fuzz {t}")


def test_fused_gain_in_the_compositor(cuda_lib, oracle):
    got, ref, pano0 = replay.fused_gain_case(oracle, Warper, Blender, Compositor, rigs, 4)
    replay.assert_exact(got[0], ref[0], "pano with fused exposure gains")
    replay.assert_exact(got[1], ref[1], "mask with fused exposure gains")
    assert not np.array_equal(got[0], pano0)


def test_device_twins_through_warp_crop_compensate_feed_on_gpu(cuda_lib, oracle):
    """The warped images' device twins (sb_warp_keep / sb_gain_apply_dev / sb_blender_feed_dev) against the host-buffer
    entries on the same arrays: identical panorama and mask."""
    import test_host_logic

    test_host_logic._twin_chain(oracle)


def test_compositor_with_the_other_projections_on_gpu(cuda_lib, oracle):
    import test_host_logic

    test_host_logic._compositor_other_projections(oracle, ["fisheye", "stereographic", "compressedPlaneA1.5B1", "compressedPlanePortraitA2B1", "paniniA2B1",
                                                           "paniniPortraitA1.5B1", "mercator", "transverseMercator"])


def test_timelapser_goldens_and_fuzz(cuda_lib, oracle):
    """Timelapser frames (SURVEY 8f f4) on the device: goldens, fuzz against the oracle, frames from device twins."""
    from stitching_b200 import Timelapser

    replay.run_timelapse_goldens(Timelapser)
    replay.timelapse_fuzz(oracle, Timelapser, Warper, rigs, 4)


def test_parallel_distance_transform_on_gpu(cuda_lib, oracle):
    """Feather weights through the parallel L1 distance transform (ballot words + scans, chunked prefix minima) on mask shapes
    that stress its carries, at sizes the CPU lane emulation cannot afford."""
    import test_host_logic

    test_host_logic._distance_transform_stress(oracle, [(40, 1100), (300, 37), (64, 64), (5, 70), (97, 131), (33, 2100), (700, 4500)])
