"""Camera frames resized to FINAL inside the compositor on the GPU: the resize kernel against the oracle, rig / crop /
shard draws against the compositor fed resized frames, the reference Stitcher's final_megapix records replayed from
the camera views, SB_SRC4=0 in a child process, and one 48 MP camera."""
import numpy as np
import pytest

import crop_fuzz
import final_scale
import fuzz_chain
import reference_cases as RC
import rig_fuzz
import shard_fuzz

pytestmark = pytest.mark.gpu

SEED = final_scale.seed_from_env()
RIG_COUNT = 24
_views = {}


def _record_views(name):
    if name not in _views:
        _views.clear()
        _views[name] = final_scale.views(final_scale.record(name))
    return _views[name]


@pytest.mark.parametrize("k", range(4))
def test_resize_kernel_against_oracle(cuda_lib, oracle, k):
    rng = np.random.default_rng([SEED, 2, k])
    final_scale.kernel_check(oracle, final_scale.kernel_sizes(rng, 10 + 8 * k, 400), SEED + k)


def test_camera_48mp_to_12mp(cuda_lib, oracle):
    """8000 x 6000 frames to 4000 x 3000 (final_megapix 12) and to 4243 x 3182 (non-dyadic)."""
    final_scale.kernel_check(oracle, [((8000, 6000), (4000, 3000)), ((8000, 6000), (4243, 3182))], SEED)


@pytest.mark.parametrize("k", range(RIG_COUNT + 1))
def test_resized_compositor_equals_prefed(cuda_lib, oracle, k):
    cs = list(rig_fuzz.cases(SEED, RIG_COUNT, rig_fuzz.GPU)) + [rig_fuzz.named("many", rig_fuzz.GPU)]
    final_scale.rig_check(oracle, cs[k], SEED)


@pytest.mark.parametrize("k", range(6))
def test_resized_crop_equals_prefed(cuda_lib, oracle, k):
    cc = crop_fuzz.cases(SEED, 6, rig_fuzz.GPU)[k]
    final_scale.rig_check(oracle, cc.case, SEED, crop=cc.crop, ex=rig_fuzz.extras(cc.cropped_case()))


def test_resized_sharded_roles_on_one_gpu(cuda_lib, oracle):
    ran = set()
    for case in shard_fuzz.cases(SEED, 6, rig_fuzz.GPU):
        for world in (2, 3):
            if case.n >= world:
                final_scale.sharded_check(oracle, case, world, fuzz_chain.device_copy, SEED)
                ran.add(world)
    assert ran == {2, 3}


def test_pipelined_steps(cuda_lib, oracle):
    final_scale.pipelined_check(oracle, rig_fuzz.named("odd_origins", rig_fuzz.GPU), 7, SEED)


@pytest.mark.parametrize("name", final_scale.RECORDS)
def test_recorded_stitcher_from_camera_frames(cuda_lib, name):
    """The compositor fed the 4000 x 3000 views, with the record's crop, seam masks and gains: every image after gain and
    its blend weight, the panorama and two pipelined steps equal what the reference Stitcher computed at final_megapix."""
    z = final_scale.record(name)
    final_scale.compositor_replay(z, _record_views(name))


@pytest.mark.parametrize("name", final_scale.RECORDS)
def test_dropin_resize_reproduces_the_record(cuda_lib, name):
    from stitching_b200 import images

    z = final_scale.record(name)
    final_scale.resized_check(images.resize_exact, z, _record_views(name))


def test_packed_sources_are_identical(cuda_lib):
    """SB_SRC4=0 (the resize writes packed FINAL sources, the warp reads them) in a child process: the same panorama,
    mask and warped images as the word layout, on record 5."""
    base = fuzz_chain.ab_run("final_scale:ab_arrays", ["5"], [("SB_SRC4", "0")], "SB_FINAL_SCALE_SEED", timeout=900)
    assert RC.digest(base["pano"]) == str(final_scale.record("5")["pano"])
