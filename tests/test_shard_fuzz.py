"""Seeded random rigs (tests/shard_fuzz.py) through the sharded composite of the emulation build, every strip bit for
bit against an oracle that sums in the ranks' groups; the oracle's own self-checks; the multiband block-order check.

All ranks live in this process; the slabs are moved with memmove through the transport hooks, as in
tests/test_sharded.py.  tests/test_gpu_shard_fuzz.py runs a larger set on the GPU and the real exchange."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import replay
import rig_fuzz
import shard_fuzz
from stitching_b200 import Compositor, StitchingError, Warper

SEED = shard_fuzz.seed_from_env()


def _memmove(d, s, n):
    C.memmove(d, s, n)


@pytest.mark.parametrize("k", range(len(shard_fuzz.emu_ids())), ids=shard_fuzz.emu_ids())
def test_shard_fuzz_against_grouped_oracle(use_emu, oracle, monkeypatch, k):
    """One random sharded rig (or a named one): every rank's geometry as restated, slab sizes agreeing on both sides,
    own warped images and masks, and every strip and its mask equal to the grouped oracle's."""
    case = shard_fuzz.emu_set(SEED)[k]
    for key, v in case.env.items():
        monkeypatch.setenv(key, v)
    imgs, ex = rig_fuzz.images(case), rig_fuzz.extras(case)
    ref = shard_fuzz.grouped_oracle(oracle, case, imgs, ex)
    got, sizes = shard_fuzz.hooks_run(case, imgs, ex, _memmove)
    shard_fuzz.check(case, got, sizes, ref, SEED)


def test_grouped_oracle_differs_from_plain_on_the_named_case(oracle):
    """The named case is one where the ranks' grouping changes the result: the exact comparison is stricter than a
    comparison with the single-GPU oracle could be."""
    case = shard_fuzz.named("grouped_differs")
    imgs, ex = rig_fuzz.images(case), rig_fuzz.extras(case)
    ref = shard_fuzz.grouped_oracle(oracle, case, imgs, ex)
    plain = shard_fuzz.plain_oracle(oracle, case, imgs, ex)
    g = shard_fuzz.geometry(case)
    diff = sum(int((shard_fuzz.cut(p, s, g["axis"]) != shard_fuzz.cut(plain["pano"], s, g["axis"])).sum())
               for (p, _), s in zip(ref["panos"], g["strips"]))
    assert diff > 0


def test_shard_fuzz_coverage_under_emulation(oracle):
    """The emulated set reaches what it is there for, by the geometry restated from the rigs."""
    cs = shard_fuzz.emu_set(SEED)
    rows = [(c, shard_fuzz.coverage(c, tile="SB_EMU_BLOCKS" in c.env)) for c in cs]
    print(f"\nshard fuzz coverage, emulation set (seed {SEED}, {len(cs)} cases):\n" + rig_fuzz.coverage_table(rows))
    reached = set().union(*(t for _, t in rows))
    want = {"world=2", "world=3", "world=4", "world=5", "world=8", "multiband", "feather", "empty strip", "column strips",
            "row strips", "row strips reversed", "slab at l>=2", "tile l0 with slab items", "tile l1 with slab items",
            "n == world", "n % world != 0", "nb=1", "3+ ranks in a pixel", "gray blend mask"}
    assert want <= reached, f"not reached: {sorted(want - reached)}"
    assert rig_fuzz.redraw_share(cs) < 1.0, f"{rig_fuzz.redraw_share(cs):.2f} rejected draws per case"


# -- the oracle's self-checks ------------------------------------------------------------------------------------------
def test_grouped_oracle_with_one_rank_is_blend(oracle):
    """World 1: the grouped oracle is Blender.blend(), on the golden blend and end-to-end cases."""
    for c in replay.blend_cases():
        if c["btype"] == "no":
            continue
        _, panos = shard_fuzz.grouped_blend(oracle, c["btype"], c["strength"], c["corners"], c["imgs"], c["masks"], 1)
        replay.assert_exact(panos[0][0], c["pano"], f"blend case {c['i']}")
        replay.assert_exact(panos[0][1], c["pmask"], f"blend case {c['i']} mask")
    for c in replay.e2e_cases():
        cfg = c["cfg"]
        warped = [oracle.warp(cfg["warper"], np.float32(np.median([k.focal for k in c["cams"]])),
                              Warper.get_K(k, 1), k.R, im) for k, im in zip(c["cams"], c["imgs"])]
        _, panos = shard_fuzz.grouped_blend(oracle, cfg["blender"], cfg["strength"], [w[0][:2] for w in warped],
                                            [w[1] for w in warped], [w[2] for w in warped], 1)
        replay.assert_exact(panos[0][0], c["pano"], f"e2e {c['name']}")
        replay.assert_exact(panos[0][1], c["pmask"], f"e2e {c['name']} mask")


@pytest.mark.parametrize("kind", ["multiband", "feather"])
def test_fold_of_an_empty_blender_changes_nothing(oracle, kind):
    c = next(c for c in replay.blend_cases() if c["btype"] == kind)
    sizes = [(m.shape[1], m.shape[0]) for m in c["masks"]]
    b, empty = oracle.Blender(kind, c["strength"]), oracle.Blender(kind, c["strength"])
    b.prepare(c["corners"], sizes)
    empty.prepare(c["corners"], sizes)
    for img, m, corner in zip(c["imgs"], c["masks"], c["corners"]):
        b.feed(img, m, corner)
    b.fold(empty)
    pano, mask = b.blend()
    replay.assert_exact(pano, c["pano"], f"{kind}: fold of an empty blender")
    replay.assert_exact(mask, c["pmask"], f"{kind}: fold of an empty blender, mask")
    # and folding a fed blender into an empty one gives that blender's result
    b2, d = oracle.Blender(kind, c["strength"]), oracle.Blender(kind, c["strength"])
    b2.prepare(c["corners"], sizes)
    d.prepare(c["corners"], sizes)
    for img, m, corner in zip(c["imgs"], c["masks"], c["corners"]):
        b2.feed(img, m, corner)
    d.fold(b2)
    replay.assert_exact(d.blend()[0], c["pano"], f"{kind}: fold into an empty blender")
    with pytest.raises(ValueError):
        oracle.Blender("feather" if kind == "multiband" else "multiband", c["strength"]).fold(b2)


# -- the multiband block order -------------------------------------------------------------------------------------------
def test_multiband_blocks_right_to_left_are_refused(use_emu):
    """Image blocks that run right to left cannot be cut into left-to-right column strips: StitchingError, on every
    rank.  The restated predicate (shard_fuzz.geometry) decides, over raw draws, which rigs must be refused and which
    must build, so both directions of the check run."""
    case = shard_fuzz.named("right_to_left")
    assert not shard_fuzz.geometry(case)["ok"]
    for r in range(case.world):
        with pytest.raises(StitchingError, match="not ordered left to right"):
            Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength, rank=r, world=case.world)
    seen = {True: 0, False: 0}
    for drawn in shard_fuzz.raw_draws(SEED + 1, 80, shard_fuzz.EMU):
        # each draw as it comes and mirrored (images in reverse order: the blocks run the other way), so that both
        # outcomes occur under any seed
        mirrored = dataclasses.replace(drawn, cams=drawn.cams[::-1], sizes=drawn.sizes[::-1], masks=drawn.masks[::-1],
                                       gains=drawn.gains[::-1], gens=drawn.gens[::-1], rects=drawn.rects[::-1])
        for c in (drawn, mirrored):
            g = shard_fuzz.geometry(c)
            if g["kind"] != "multiband" or g["nb"] < 1 or c.n < c.world:
                continue
            seen[g["ok"]] += 1
            if g["ok"]:
                comp = Compositor(c.cams, c.sizes, c.wtype, c.blender, c.strength, rank=c.world - 1, world=c.world)
                assert comp.strip == g["strips"][-1], c.describe()
                comp.close()
            else:
                with pytest.raises(StitchingError, match="not ordered left to right"):
                    Compositor(c.cams, c.sizes, c.wtype, c.blender, c.strength, rank=0, world=c.world)
    assert seen[True] >= 10 and seen[False] >= 10, seen


def test_item_lists_stay_under_sb_max_items(use_emu):
    """SB_MAX_ITEMS (320: own images plus received slabs per level) cannot be exceeded: the compositor takes at most
    SB_MAX_IMAGES = 256 images, and a rank holds at most ceil(n / world) + world - 1 <= 256 items.  The largest list
    there can be -- 256 images on one spot at world 256, where the last rank receives a slab from every other rank at
    every level: 1 + 255 items -- builds; a 257th image is refused."""
    assert max(-(-n // w) + w - 1 for n in range(2, 257) for w in range(2, n + 1)) == 256
    n = 256
    cam = shard_fuzz._affine(0.0, 1.0, 1.0, 0.0, 0.0, 0.0)
    c = Compositor([cam] * n, [(8, 8)] * n, "affine", "multiband", 100.0, rank=n - 1, world=n)
    assert c.num_bands >= 1 and c.count == 1
    assert all(c.shard_slab(p, False)[1] > 0 for p in range(n - 1))
    c.close()
    with pytest.raises(StitchingError):
        Compositor([cam] * (n + 1), [(8, 8)] * (n + 1), "affine", "multiband", 100.0, rank=0, world=2)
