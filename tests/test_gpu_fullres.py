"""The default Stitcher at camera resolution on the GPU: the recorded crop=True runs of the reference (12 MP and 48 MP
views, tests/golden/golden_fullres_*.npz) replayed through the fused compositor and through the drop-in classes, stage
by stage; compositor draws at the pipeline's LOW -> FINAL ratios against the oracle; and SeamFinder.resize and
ExposureErrorCompensator.apply through the C ABI on 4000-9000 px images."""
import time

import numpy as np
import pytest

import fullres

pytestmark = pytest.mark.gpu

SEED = fullres.seed_from_env()
GPU_COUNT = 12
_sets, _views = {}, {}


def _record_views(name):
    """One record's views at a time (record B's take 430 MB)."""
    if name not in _views:
        _views.clear()
        _views[name] = fullres.views(fullres.record(name))
    return _views[name]


@pytest.mark.parametrize("name", fullres.RECORDS)
def test_recorded_stitcher_on_the_compositor(cuda_lib, oracle, name):
    """Geometry, every image after its fused gain with its blend weight, the panorama and two pipelined steps equal what
    the reference Stitcher computed; the compositor's panorama also equals the drop-in chain's."""
    z = fullres.record(name)
    imgs = _record_views(name)
    t = time.perf_counter()
    nbytes, pano = fullres.compositor_replay(z, imgs, oracle)
    print(f"\n{fullres.describe(name, z)}, num_bands {int(z['num_bands'])}: compositor replay {time.perf_counter() - t:.1f} s, "
          f"{nbytes / 1e6:.0f} MB compared")


@pytest.mark.parametrize("name", fullres.RECORDS)
def test_recorded_stitcher_on_the_dropins(cuda_lib, oracle, name):
    """Warper, the crop as a numpy slice, ExposureErrorCompensator.apply, SeamFinder.resize and Blender in the
    Stitcher's order: every stage of every image and the panorama equal the record, and the compositor's panorama."""
    z = fullres.record(name)
    imgs = _record_views(name)
    t = time.perf_counter()
    nbytes, pano = fullres.dropin_replay(z, imgs, oracle)
    dt = time.perf_counter() - t
    c = fullres.compositor(z)
    try:
        assert np.array_equal(c.composite(imgs)[0], pano), "the drop-in chain's panorama differs from the compositor's"
    finally:
        c.close()
    print(f"\n{fullres.describe(name, z)}: drop-in replay {dt:.1f} s, {nbytes / 1e6:.0f} MB compared")


def gpu_set():
    if "gpu" not in _sets:
        _sets["gpu"] = fullres.cases(SEED, GPU_COUNT, 1500, 4000, 20_000_000)
    return _sets["gpu"]


@pytest.mark.parametrize("k", range(GPU_COUNT))
def test_ratio_draws_against_oracle(cuda_lib, oracle, k):
    """Rects, pano roi, num_bands, every cropped image after gain and its blend mask, the panorama: bit for bit."""
    cc = gpu_set()[k]
    t = time.perf_counter()
    nbytes = fullres.run_and_check(oracle, cc, SEED)
    print(f"\n{cc.describe()}: {time.perf_counter() - t:.1f} s, {nbytes / 1e6:.0f} MB compared")


def test_ratio_draws_coverage():
    rows = [(c, fullres.coverage(c)) for c in gpu_set()]
    print("\nratio draws coverage, GPU set:\n" + fullres.rig_fuzz.coverage_table(rows))
    reached = set().union(*(t for _, t in rows))
    assert fullres.WANT <= reached, f"not reached: {sorted(fullres.WANT - reached)}"


def test_standalone_entries_at_camera_resolution(cuda_lib, oracle):
    """sb_seam_resize and sb_gain_apply (host buffers) on 4000-9000 px images against the oracle, the LOW sides from
    the pipeline's ratios."""
    from stitching_b200 import exposure_error_compensator, seam_finder

    import replay

    rng = np.random.default_rng([SEED, 9])
    for t in range(6):
        w, h = int(rng.integers(4000, 9001)), int(rng.integers(3000, 6001))
        aspect = fullres.pipeline_aspect(float(rng.uniform(2, 48)))
        sw, sh = max(1, int(round(w / aspect)) - int(rng.integers(0, 2))), max(1, int(round(h / aspect)) - int(rng.integers(0, 2)))
        seam = (rng.random((sh, sw)) < 0.5).astype(np.uint8) * 255 if t % 2 else rng.integers(0, 256, (sh, sw), dtype=np.uint8)
        mask = np.full((h, w), 255, np.uint8)
        mask[:, : int(rng.integers(0, w // 8))] = 0
        replay.assert_exact(seam_finder.resize(seam, mask), oracle.seam_resize(seam, mask), f"seam resize {sw}x{sh} -> {w}x{h}")
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        shape = (-(-sh // fullres.BLOCK), -(-sw // fullres.BLOCK)) + ((3,) if t % 3 == 2 else ())
        gain = rng.uniform(0.6, 1.6, shape).astype(np.float32)
        replay.assert_exact(exposure_error_compensator.apply_gain(img.copy(), gain), oracle.gain_apply(img, gain),
                            f"gain map {shape} on {w}x{h}")
