"""Camera frames resized to FINAL inside the compositor (Compositor(input_sizes=...)), in the emulation build: the resize
kernel against the oracle's cv.resize(INTER_LINEAR_EXACT), the compositor fed camera frames against the compositor fed
resized frames on random rigs, crops and shards, the refusals, and the reference Stitcher's final_megapix records."""
import ctypes

import numpy as np
import pytest

import crop_fuzz
import final_scale
import fuzz_chain
import rig_fuzz
import shard_fuzz
from stitching_b200 import Compositor, StitchingError

SEED = final_scale.seed_from_env()
KERNEL_RIGS = 6
RIG_COUNT = 17


def _kernel_rig(k):
    rng = np.random.default_rng([SEED, 1, k])
    return final_scale.kernel_sizes(rng, 8 + 5 * k, 90)


@pytest.mark.parametrize("k", range(KERNEL_RIGS))
def test_resize_kernel_against_oracle(use_emu, oracle, k):
    """Scales 0.05-1, exact halvings, one axis kept, 1-px sides, FINAL widths of every residue mod 8; rigs of 8 to 33
    images (one launch per 32).  1-px images send their batch through the packed-source warp, so both outputs run."""
    final_scale.kernel_check(oracle, _kernel_rig(k), SEED + k)


def test_resize_kernel_packed_output(use_emu, oracle, monkeypatch):
    """SB_SRC4=0: the kernel writes the packed FINAL source instead of words for every image, not only for those in a
    batch that k_warp_wide warps."""
    monkeypatch.setenv("SB_SRC4", "0")
    final_scale.kernel_check(oracle, _kernel_rig(1), SEED + 100)


def test_kernel_draws_cover_the_cases():
    pairs = [p for k in range(KERNEL_RIGS) for p in _kernel_rig(k)]
    assert {w % 8 for _, (w, _) in pairs} == set(range(8))
    assert any(w == 1 for _, (w, _) in pairs) and any(h == 1 for _, (_, h) in pairs)
    assert any(W == 2 * w and H == 2 * h for (W, H), (w, h) in pairs)
    assert any(W == w and H > h for (W, H), (w, h) in pairs) and any(H == h and W > w for (W, H), (w, h) in pairs)
    assert min(w / W for (W, _), (w, _) in pairs) < 0.1
    assert max(len(_kernel_rig(k)) for k in range(KERNEL_RIGS)) > rig_fuzz.WARP_BATCH


def _rig_cases():
    cs = list(rig_fuzz.cases(SEED, RIG_COUNT, rig_fuzz.EMU))
    return cs + [rig_fuzz.named("many", rig_fuzz.EMU)]


@pytest.mark.parametrize("k", range(RIG_COUNT + 1))
def test_resized_compositor_equals_prefed(use_emu, oracle, k):
    """Panorama, mask and every warped image and mask equal those of a compositor fed the oracle-resized frames, with
    the case's set_mask / set_seam_mask / set_gain."""
    final_scale.rig_check(oracle, _rig_cases()[k], SEED)


def test_rig_draws_coverage():
    cs = _rig_cases()
    tags = set()
    for c in cs:
        tags |= rig_fuzz.coverage(c, pyr_fast=False, tile=False, dt_fast=False) | {c.wtype}
        if any(g != "none" for g in c.gains):
            tags.add("set_gain")
        if "seam" in c.masks:
            tags.add("set_seam_mask")
        ins = final_scale.input_sizes(c, np.random.default_rng([SEED, c.seed]))
        if any(tuple(a) == tuple(b) for a, b in zip(ins, c.sizes)) and any(tuple(a) != tuple(b) for a, b in zip(ins, c.sizes)):
            tags.add("mixed rig")
    want = {"spherical", "affine", "map projection", "multiband", "feather", "no", "nb=0", "nb=1", "nb>=2", "n>32",
            "set_gain", "set_seam_mask", "mixed rig"}
    assert want <= tags, f"not reached: {sorted(want - tags)}"


@pytest.mark.parametrize("k", range(4))
def test_resized_crop_equals_prefed(use_emu, oracle, k):
    cc = crop_fuzz.cases(SEED, 4, rig_fuzz.EMU)[k]
    final_scale.rig_check(oracle, cc.case, SEED, crop=cc.crop, ex=rig_fuzz.extras(cc.cropped_case()))


def _memmove(d, s, n):
    ctypes.memmove(d, s, n)


def test_resized_sharded_equals_grouped_oracle(use_emu, oracle):
    """World 2 and 3: every rank resizes its own block; strips and own warped images equal the grouped oracle fed the
    resized frames."""
    ran = set()
    for case in shard_fuzz.cases(SEED, 6, rig_fuzz.EMU):
        for world in (2, 3):
            if case.n >= world:
                final_scale.sharded_check(oracle, case, world, _memmove, SEED)
                ran.add(world)
    assert ran == {2, 3}


def test_pipelined_steps(use_emu, oracle):
    """Five submit / wait steps over the three buffer sets, new camera frames each step."""
    final_scale.pipelined_check(oracle, rig_fuzz.named("odd_origins", rig_fuzz.EMU), 5, SEED)


def test_equal_input_sizes_change_nothing(use_emu, oracle):
    """input_sizes == sizes: no image is resized -- the same bytes and the same kernel launches as without them."""
    case = rig_fuzz.named("gray_mask_multiband", rig_fuzz.EMU)
    imgs, ex = rig_fuzz.images(case), rig_fuzz.extras(case)
    out, launches = [], []
    for kw in ({}, {"input_sizes": case.sizes}):
        before = use_emu.sb_launch_count()
        out.append(fuzz_chain.compositor_run(case, imgs, ex, **kw))
        launches.append(use_emu.sb_launch_count() - before)
    rig_fuzz.check(case, out[1], out[0], SEED)
    assert launches[0] == launches[1], launches


def test_refusals(use_emu):
    case = rig_fuzz.named("odd_origins", rig_fuzz.EMU)
    (w, h), rest = case.sizes[0], list(case.sizes[1:])

    def make(first):
        return Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength, input_sizes=[first] + rest)

    with pytest.raises(StitchingError, match="image 0 .* smaller than its FINAL size"):
        make((w - 1, 2 * h))
    with pytest.raises(StitchingError, match="image 0 .* smaller than its FINAL size"):
        make((2 * w, h - 1))
    with pytest.raises(StitchingError, match="image 0 has the size"):
        make((0, h))
    with pytest.raises(StitchingError, match="image 0 has the size"):
        make((w, -3))
    with pytest.raises(StitchingError, match="image 0 .* 32767 px or more"):
        make((32767, h))
    with pytest.raises(StitchingError, match="input sizes for"):
        Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength, input_sizes=case.sizes[1:])
    c = make((2 * w, 2 * h))
    try:
        imgs = rig_fuzz.images(case)
        with pytest.raises(StitchingError, match="image 0: expected uint8"):
            c.upload(imgs)  # the FINAL-size frame where the camera frame belongs
        with pytest.raises(StitchingError, match="image 0: expected a uint8"):
            c.submit(imgs, np.empty((1, 1, 3), np.uint8), np.empty((1, 1), np.uint8))
        with pytest.raises(StitchingError, match=f"expected {case.n} images"):
            c.submit(imgs[1:], np.empty((1, 1, 3), np.uint8), np.empty((1, 1), np.uint8))
        with pytest.raises(StitchingError, match="image 0: expected uint8"):
            c.composite(imgs)
    finally:
        c.close()


@pytest.mark.parametrize("name", final_scale.RECORDS)
def test_records_resize_like_the_oracle(oracle, name):
    """The oracle's INTER_LINEAR_EXACT of the rebuilt camera views is what the reference's resize_final_resolution
    handed to the warp, for the exact halving (record 3) and the non-dyadic scale (record 5)."""
    z = final_scale.record(name)
    final_scale.resized_check(oracle.resize_linear_exact, z, final_scale.views(z))
