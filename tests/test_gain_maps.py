"""Exposure gain maps of every shape against cv2's own results (tests/gain_maps.py), on the emulation build: the
oracle's resize bit for bit against golden_gain_maps.npz, the oracle and ExposureErrorCompensator.apply against the
compensators' apply, sb_gain_apply_dev on a device twin, and Compositor.set_gain plain, in a timelapse and sharded, with
maps one block wide, high or both.  The live sweep against cv2 is skipped where cv2 does not import."""
import pytest

import gain_maps as GM
from stitching_b200 import exposure_error_compensator as ec


def _apply(img, gain):
    return ec.apply_gain(img, gain)


@pytest.mark.parametrize("which", ["1px", "ipp"])
def test_oracle_resize_against_cv2_goldens(oracle, which):
    GM.check_oracle_resize(oracle, which)


@pytest.mark.parametrize("which", ["1px", "ipp"])
def test_apply_against_the_compensators(use_emu, oracle, which):
    GM.check_apply_goldens(oracle, _apply, which)


def test_maps_fed_from_thin_low_images(use_emu, oracle):
    GM.check_feed_goldens(oracle, _apply, ratios=(11,))


def test_device_twin_at_a_crop_offset(use_emu, oracle):
    GM.check_device_twin(oracle)


@pytest.mark.parametrize("seed", [3, 4])
def test_compositor_set_gain(use_emu, oracle, seed):
    sizes, maps = GM.compositor_draw(seed, 90)
    GM.check_compositor(oracle, sizes, maps, seed)


def test_timelapse_with_clipped_parts(use_emu, oracle):
    GM.check_timelapse(oracle)


def test_sharded_owner_sets_the_gain(use_emu, oracle):
    GM.check_sharded(oracle, GM.memmove)


def test_live_sweep_against_cv2(use_emu, oracle):
    pytest.importorskip("cv2")
    GM.live_sweep(oracle, _apply, 24, 20261017, max_side=300)
