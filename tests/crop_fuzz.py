"""Seeded crops for the compositor against the CPU oracle (helper module: no tests in here).

A crop is what Stitcher.crop_final_resolution does to every warped image: the reference's Cropper intersects each
LOW-resolution warped rect with the largest interior rectangle (LIR), slices image i by the intersection scaled to
FINAL pixels and feeds it at the overlap, scaled separately.  Here the LOW rects are the FINAL warped rects of a
rig_fuzz case scaled down by `aspect`, the LIR is drawn at random, and a duck-typed Cropper carries the rectangles to
Crop.from_cropper -- so the draws reach slices clipped at the warped image's edge, placements that are not the warped
corner plus the slice offset, and pano rois (hence band counts) that differ from the uncropped ones.

SB_CROP_FUZZ_SEED=<int> or =random replaces the fixed default seed (the seed used is printed).
"""
import dataclasses
import functools
import types

import numpy as np

import fuzz_chain
import rig_fuzz
from stitching_b200 import Compositor, Crop

DEFAULT_SEED = 20261016
ASPECTS = (1.0, 1.5, 2.5, 0.5, 1.25, 3.0, 1.7)  # x.5 and x.25 products round half to even


seed_from_env = functools.partial(fuzz_chain.seed_from_env, "SB_CROP_FUZZ_SEED", DEFAULT_SEED)


def _overlap(r, lir):
    x1, y1 = max(r[0], lir[0]), max(r[1], lir[1])
    x2, y2 = min(r[0] + r[2], lir[0] + lir[2]), min(r[1] + r[3], lir[1] + lir[3])
    return (x1, y1, x2 - x1, y2 - y1)


def low_cropper(rects, aspect, lir_frac):
    """A duck-typed prepared Cropper for FINAL warped `rects` seen at LOW = FINAL / aspect; the LIR spans the fractions
    `lir_frac` = (x0, y0, x1, y1) of the LOW pano.  None when some overlap would be empty."""
    low = [(int(round(x / aspect)), int(round(y / aspect)), max(1, int(round(w / aspect))), max(1, int(round(h / aspect))))
           for x, y, w, h in rects]
    x0, y0 = min(r[0] for r in low), min(r[1] for r in low)
    low = [(x - x0, y - y0, w, h) for x, y, w, h in low]  # Cropper.prepare zero-centres the corners
    W, H = max(r[0] + r[2] for r in low), max(r[1] + r[3] for r in low)
    lx, ly = int(lir_frac[0] * W), int(lir_frac[1] * H)
    lir = (lx, ly, max(1, int(lir_frac[2] * W) - lx), max(1, int(lir_frac[3] * H) - ly))
    overlaps = [_overlap(r, lir) for r in low]
    if any(o[2] <= 0 or o[3] <= 0 for o in overlaps):
        return None
    inters = [(abs(o[0] - r[0]), abs(o[1] - r[1]), o[2], o[3]) for r, o in zip(low, overlaps)]
    return types.SimpleNamespace(do_crop=True, overlapping_rectangles=overlaps, intersection_rectangles=inters)


def full_crop(rects, shift=(7, -3)):
    """Every image whole, placed at its warped corner shifted by a constant: must equal no crop."""
    return Crop([(0, 0, w, h) for _, _, w, h in rects], [(x + shift[0], y + shift[1]) for x, y, _, _ in rects],
                [(w, h) for _, _, w, h in rects])


@dataclasses.dataclass
class CropCase:
    case: object      # rig_fuzz.Case (rects: the uncropped warped rects)
    crop: object      # Crop
    aspect: float
    low: object = None  # the LOW Cropper it was drawn as (fuzz_chain.draw_crop)

    @property
    def n(self):
        return self.case.n

    def fed(self):
        """(corner + fed size) per image: the slice clipped like a numpy slice of the warped image."""
        out = []
        for (x, y, w, h), c, r in zip(self.crop.rects, self.crop.corners, self.case.rects):
            out.append((c[0], c[1], max(0, min(w, r[2] - x)), max(0, min(h, r[3] - y))))
        return out

    def cropped_case(self):
        """The rig_fuzz case with the fed rects: extras drawn for it are sized to the cropped images."""
        return dataclasses.replace(self.case, rects=self.fed())

    def describe(self):
        return f"{self.case.describe()} crop@{self.aspect:g}"


def cases(seed, count, budget):
    """`count` seeded crop cases over rig_fuzz rigs drawn with `seed` (a rig none of whose 20 LIR draws crops every
    image to a non-empty slice is passed over)."""
    rng = np.random.default_rng(seed)
    out = []
    for c in rig_fuzz.cases(seed, 4 * count, budget):
        if len(out) == count:
            break
        cc = fuzz_chain.draw_crop(rng, c, ASPECTS, 0.3, 0.7)
        if cc is not None:
            out.append(cc)
    return out


def named(name, budget):
    if name == "full":
        c = rig_fuzz.named("odd_origins", budget)
        return CropCase(c, full_crop(c.rects), 1.0)
    if name == "many":
        c = rig_fuzz.named("many", budget)
        return CropCase(c, Crop.from_cropper(low_cropper(c.rects, 1.5, (0.05, 0.05, 0.95, 0.95)), 1.5), 1.5)
    raise KeyError(name)


# -- the two sides ----------------------------------------------------------------------------------------------------
def compositor(cc, crop=True, **kw):
    case = cc.case
    return Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength, crop=cc.crop if crop else None, **kw)


def run_and_check(O, cc, seed):
    imgs, ex = rig_fuzz.images(cc.case), rig_fuzz.extras(cc.cropped_case())
    ref = rig_fuzz.oracle_run(O, cc.case, imgs, ex, crop=cc.crop)
    got = fuzz_chain.compositor_run(cc.case, imgs, ex, crop=cc.crop)
    rig_fuzz.check(dataclasses.replace(cc.case, name=cc.describe()), got, ref, seed)
    return got


def ab_arrays(seed, count, ks):
    """Cases `ks` of cases(seed, count, GPU) through the compositor: the pano and its mask by name."""
    cs = cases(seed, count, rig_fuzz.GPU)
    out = {}
    for k in ks:
        got = fuzz_chain.compositor_run(cs[k].case, rig_fuzz.images(cs[k].case), rig_fuzz.extras(cs[k].cropped_case()),
                                        crop=cs[k].crop)
        out[f"{k}_pano"], out[f"{k}_pmask"] = got["pano"], got["pmask"]
    return out


# -- sharded ------------------------------------------------------------------------------------------------------------
def sharded_cases(seed, count, budget):
    """Crops of shard_fuzz rigs whose pano roi is the same from the fed and from the prepared sizes (shard_fuzz's
    grouped oracle prepares from the fed images)."""
    import shard_fuzz

    def keep(cc):
        g = fuzz_chain.blend_geometry(cc.crop.corners, cc.crop.sizes, cc.case.blender, cc.case.strength)
        blends = g.nb >= 1 if g.kind == "multiband" else g.kind == "feather"
        return blends and g.roi == fuzz_chain.blend_geometry(cc.crop.corners, [f[2:] for f in cc.fed()]).roi

    rng = np.random.default_rng(seed)
    out = []
    for c in shard_fuzz.cases(seed, 4 * count, budget):
        if len(out) == count:
            break
        cc = fuzz_chain.draw_crop(rng, c, ASPECTS, 0.2, 0.8, keep=keep)
        if cc is not None:
            out.append(cc)
    return out


def sharded_check(O, cc, world, copy, seed):
    """All ranks in this process through the transport hooks (shard_fuzz.hooks_run with the crop): every rank's own
    cropped warped images and its strip equal shard_fuzz.grouped_blend fed with the cropped images.  Returns False
    when the crop's blocks run right to left (the sharded composite refuses those)."""
    import replay
    import shard_fuzz
    from stitching_b200 import StitchingError

    case = dataclasses.replace(cc.case, world=world)
    imgs, ex = rig_fuzz.images(case), rig_fuzz.extras(cc.cropped_case())
    ref = rig_fuzz.oracle_run(O, case, imgs, ex, crop=cc.crop)
    _, panos = shard_fuzz.grouped_blend(O, case.blender, case.strength, cc.crop.corners, ref["warped"], ref["masks"], world)
    try:
        got, slabs = shard_fuzz.hooks_run(case, imgs, ex, copy, crop=cc.crop)
    except StitchingError as e:
        if "right to left" in str(e) or "order" in str(e):
            return False
        raise
    where = f"seed {seed}, {cc.describe()}, world {world}"
    for sn, dn in slabs.values():
        assert sn == dn, where
    for r, rk in enumerate(got):
        assert [tuple(x) for x in rk["rects"]] == ref["rects"] and tuple(rk["roi"]) == tuple(ref["roi"]), where
        assert rk["num_bands"] == ref["num_bands"], where
        for i, (wi, wm) in rk["warped"].items():
            replay.assert_exact(wi, ref["warped"][i], f"{where}: warped image {i}")
            replay.assert_exact(wm, ref["masks"][i], f"{where}: warped mask {i}")
        rp, rm = panos[r]
        replay.assert_exact(rk["pano"], shard_fuzz.cut(rp, rk["strip"], rk["axis"]), f"{where}: rank {r} strip")
        replay.assert_exact(rk["pmask"], shard_fuzz.cut(rm, rk["strip"], rk["axis"]), f"{where}: rank {r} strip mask")
    return True


# -- coverage -----------------------------------------------------------------------------------------------------------
def coverage(cc):
    """What a crop case reaches, from its geometry alone."""
    case = cc.case
    tags = {case.blender, case.wtype}
    if case.wtype in rig_fuzz.MAP_TYPES:
        tags.add("map projection")
    if case.n > rig_fuzz.WARP_BATCH:
        tags.add("n>32")
    g = fuzz_chain.blend_geometry(cc.crop.corners, cc.crop.sizes, case.blender, case.strength)
    _, _, w, h = g.roi
    nb = g.nb if g.kind == "multiband" else -1
    if nb >= 0:
        tags.add("nb=0" if nb == 0 else "nb=1" if nb == 1 else "nb>=2")
        if nb >= 1:
            tags.add("tile l0 yes" if w % 2 == 0 else "tile l0 no")
    whole = case.geometry()
    if nb != (whole.nb if whole.kind == "multiband" else -1):
        tags.add("crop changes num_bands")
    fed = cc.fed()
    if any((f[2], f[3]) != tuple(s) for f, s in zip(fed, cc.crop.sizes)):
        tags.add("fed smaller than prepared")
    # placement vs warped corner + slice offset, both shifted so that image 0 sits at the same place
    off = [(r[0] + s[0] - c[0], r[1] + s[1] - c[1]) for r, s, c in zip(case.rects, cc.crop.rects, cc.crop.corners)]
    if len(set(off)) > 1:
        tags.add("placement off by rounding")
    if any(m != "none" for m in case.masks) or any(g != "none" for g in case.gains):
        tags.add("extras")
    return tags


# -- the recorded reference Stitcher run ----------------------------------------------------------------------------------
def stitch_replay(golden_path):
    """The compositor fed from the recorded crop=True Stitcher run (tests/golden/gen_crop_golden.py): cameras, scale and
    ratios, Crop.from_cropper over the recorded Cropper rectangles, set_seam_mask with the LOW seam masks and set_gain with
    getMatGains().  Returns (digest of the panorama, digest the reference's Stitcher.stitch returned)."""
    import cv2 as cv

    import reference_cases as RC

    z = np.load(golden_path)
    views = RC.synthetic_views(cv)
    assert [RC.digest(v) for v in views] == [str(d) for d in z["stitch_inputs"]], "the FINAL inputs are not the recorded ones"
    cams = [RC.camera_from_value(cv, v) for v in z["stitch_cameras"]]
    cropper = types.SimpleNamespace(do_crop=True, overlapping_rectangles=[tuple(map(int, r)) for r in z["stitch_overlaps"]],
                                    intersection_rectangles=[tuple(map(int, r)) for r in z["stitch_inters"]])
    crop = Crop.from_cropper(cropper, float(z["stitch_low_to_final"]))
    c = Compositor(cams, [(v.shape[1], v.shape[0]) for v in views], "spherical", "multiband", 5, scale=float(z["stitch_scale"]),
                   aspect=float(z["stitch_medium_to_final"]), crop=crop)
    try:
        for i in range(int(z["stitch_n"])):
            c.set_seam_mask(i, z[f"stitch_seam{i}"])
            c.set_gain(i, z[f"stitch_gain{i}"])
        pano, _ = c.composite(views)
        return RC.digest(pano), str(z["stitch_pano"])
    finally:
        c.close()
