"""Seeded crops for the compositor against the CPU oracle (helper module: no tests in here).

A crop is what Stitcher.crop_final_resolution does to every warped image: the reference's Cropper intersects each
LOW-resolution warped rect with the largest interior rectangle (LIR), slices image i by the intersection scaled to
FINAL pixels and feeds it at the overlap, scaled separately.  Here the LOW rects are the FINAL warped rects of a
rig_fuzz case scaled down by `aspect`, the LIR is drawn at random, and a duck-typed Cropper carries the rectangles to
Crop.from_cropper -- so the draws reach slices clipped at the warped image's edge, placements that are not the warped
corner plus the slice offset, and pano rois (hence band counts) that differ from the uncropped ones.

SB_CROP_FUZZ_SEED=<int> replaces the fixed default seed.
"""
import dataclasses
import math
import os
import types

import numpy as np

import rig_fuzz
from stitching_b200 import Compositor, Crop

DEFAULT_SEED = 20261016
ASPECTS = (1.0, 1.5, 2.5, 0.5, 1.25, 3.0, 1.7)  # x.5 and x.25 products round half to even


def seed_from_env():
    s = os.environ.get("SB_CROP_FUZZ_SEED")
    return int(s) if s else DEFAULT_SEED


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
        for _ in range(20):
            aspect = float(rng.choice(ASPECTS))
            frac = (rng.uniform(0, 0.3), rng.uniform(0, 0.3), rng.uniform(0.7, 1.0), rng.uniform(0.7, 1.0))
            cr = low_cropper(c.rects, aspect, frac)
            if cr is None:
                continue
            crop = Crop.from_cropper(cr, aspect)
            cc = CropCase(c, crop, aspect)
            if all(w > 0 and h > 0 for _, _, w, h in cc.fed()):
                out.append(cc)
                break
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
def oracle_run(O, cc, imgs, ex, s16=False):
    """Stitcher order: warp, slice image and mask (a numpy slice), compensator apply on the cropped image, blend mask =
    the caller's mask or SeamFinder.resize(seam, cropped mask) or the cropped mask; Blender.prepare(cropped corners,
    sizes), feed at the cropped corners, blend.  `raw` and "pano16" as in rig_fuzz.oracle_run."""
    case = cc.case
    scale = case.scale()
    warped, masks, raw = [], [], []
    for img, cam, (x, y, w, h), (mask, seam, gain) in zip(imgs, case.cams, cc.crop.rects, ex):
        _, wi, wm = O.warp(case.wtype, scale, rig_fuzz.Warper.get_K(cam, 1), cam.R, img)
        raw.append((wi, wm))
        wi = np.ascontiguousarray(wi[y:y + h, x:x + w])
        wm = np.ascontiguousarray(wm[y:y + h, x:x + w])
        if gain is not None:
            wi = O.gain_apply(wi, gain)
        if mask is not None:
            wm = mask
        elif seam is not None:
            wm = O.seam_resize(seam, wm)
        warped.append(wi)
        masks.append(wm)
    b = O.Blender(case.blender, case.strength)
    b.prepare(cc.crop.corners, cc.crop.sizes)
    for wi, wm, c in zip(warped, masks, cc.crop.corners):
        b.feed(wi, wm, c)
    pano16, pmask = b.blend_s16()
    rects = [tuple(c) + (wi.shape[1], wi.shape[0]) for c, wi in zip(cc.crop.corners, warped)]
    return dict(warped=warped, masks=masks, rects=rects, roi=b.roi, num_bands=b.num_bands if b._kind == "multiband" else -1,
                pano=O.convert_scale_abs(pano16), pmask=pmask, raw=raw, pano16=pano16 if s16 else None)


def compositor(cc, crop=True, **kw):
    case = cc.case
    return Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength, crop=cc.crop if crop else None, **kw)


def compositor_run(cc, imgs, ex):
    c = compositor(cc)
    try:
        for i, (mask, seam, gain) in enumerate(ex):
            if mask is not None:
                c.set_mask(i, mask)
            if seam is not None:
                c.set_seam_mask(i, seam)
            if gain is not None:
                c.set_gain(i, gain)
        pano, pmask = c.composite(imgs)
        warped = [c.download_warped(i) for i in range(cc.n)]
        return dict(rects=list(c.rects), roi=tuple(c.roi), num_bands=c.num_bands, pano=pano, pmask=pmask,
                    warped=[w for w, _ in warped], masks=[m for _, m in warped])
    finally:
        c.close()


def run_and_check(O, cc, seed):
    imgs, ex = rig_fuzz.images(cc.case), rig_fuzz.extras(cc.cropped_case())
    ref = oracle_run(O, cc, imgs, ex)
    got = compositor_run(cc, imgs, ex)
    rig_fuzz.check(dataclasses.replace(cc.case, name=cc.describe()), got, ref, seed)
    return got


# -- sharded ------------------------------------------------------------------------------------------------------------
def sharded_cases(seed, count, budget):
    """Crops of shard_fuzz rigs whose pano roi is the same from the fed and from the prepared sizes (shard_fuzz's
    grouped oracle prepares from the fed images)."""
    import shard_fuzz

    rng = np.random.default_rng(seed)
    out = []
    for c in shard_fuzz.cases(seed, 4 * count, budget):
        if len(out) == count:
            break
        for _ in range(20):
            aspect = float(rng.choice(ASPECTS))
            frac = (rng.uniform(0, 0.2), rng.uniform(0, 0.2), rng.uniform(0.8, 1.0), rng.uniform(0.8, 1.0))
            cr = low_cropper(c.rects, aspect, frac)
            if cr is None:
                continue
            cc = CropCase(c, Crop.from_cropper(cr, aspect), aspect)
            fed = cc.fed()
            _, _, w, h = _roi(cc.crop.corners, cc.crop.sizes)
            blends = _bands(c, w, h) >= 1 if c.blender == "multiband" else math.sqrt(w * h) * c.strength >= 100.0
            if blends and all(f[2] > 0 and f[3] > 0 for f in fed) and \
                    _roi(cc.crop.corners, cc.crop.sizes) == _roi(cc.crop.corners, [f[2:] for f in fed]):
                out.append(cc)
                break
    return out


def sharded_check(O, cc, world, copy, seed):
    """All ranks in this process through the transport hooks: every rank's own cropped warped images and its strip equal
    shard_fuzz.grouped_blend fed with the cropped images.  Returns False when the crop's blocks run right to left (the
    sharded composite refuses those)."""
    import replay
    import shard_fuzz
    from stitching_b200 import StitchingError

    case = cc.case
    imgs, ex = rig_fuzz.images(case), rig_fuzz.extras(cc.cropped_case())
    ref = oracle_run(O, cc, imgs, ex)
    _, panos = shard_fuzz.grouped_blend(O, case.blender, case.strength, cc.crop.corners, ref["warped"], ref["masks"], world)
    ranks = []
    try:
        try:
            for r in range(world):
                ranks.append(compositor(cc, rank=r, world=world))
        except StitchingError as e:
            if "right to left" in str(e) or "order" in str(e):
                return False
            raise
        for c in ranks:
            for i in range(c.first, c.first + c.count):
                mask, seam, gain = ex[i]
                if mask is not None:
                    c.set_mask(i, mask)
                if seam is not None:
                    c.set_seam_mask(i, seam)
                if gain is not None:
                    c.set_gain(i, gain)
            c.upload(imgs[c.first: c.first + c.count])
            c.shard_phase(0)
        for src in ranks:
            for dst in ranks:
                if src is not dst:
                    sp, sn = src.shard_slab(dst.rank, True)
                    dp, dn = dst.shard_slab(src.rank, False)
                    assert sn == dn
                    if sn:
                        copy(dp, sp, sn)
        where = f"seed {seed}, {cc.describe()}, world {world}"
        for c in ranks:
            c.shard_phase(1)
            assert [tuple(x) for x in c.rects] == ref["rects"] and tuple(c.roi) == tuple(ref["roi"]), where
            assert c.num_bands == ref["num_bands"], where
            for i in range(c.first, c.first + c.count):
                wi, wm = c.download_warped(i)
                replay.assert_exact(wi, ref["warped"][i], f"{where}: warped image {i}")
                replay.assert_exact(wm, ref["masks"][i], f"{where}: warped mask {i}")
            pano, pmask = c.download()
            rp, rm = panos[c.rank]
            replay.assert_exact(pano, shard_fuzz.cut(rp, c.strip, c.strip_axis), f"{where}: rank {c.rank} strip")
            replay.assert_exact(pmask, shard_fuzz.cut(rm, c.strip, c.strip_axis), f"{where}: rank {c.rank} strip mask")
        return True
    finally:
        for c in ranks:
            c.close()


# -- coverage -----------------------------------------------------------------------------------------------------------
def _roi(corners, sizes):
    x0, y0 = min(c[0] for c in corners), min(c[1] for c in corners)
    return x0, y0, max(c[0] + s[0] for c, s in zip(corners, sizes)) - x0, max(c[1] + s[1] for c, s in zip(corners, sizes)) - y0


def _bands(case, w, h):
    bw = math.sqrt(w * h) * case.strength / 100.0
    if case.blender != "multiband" or bw < 1.0:
        return -1
    return min(int(math.log(bw) / math.log(2.0) - 1.0), int(math.ceil(math.log(max(w, h)) / math.log(2.0))))


def coverage(cc):
    """What a crop case reaches, from its geometry alone."""
    case = cc.case
    tags = {case.blender, case.wtype}
    if case.wtype in rig_fuzz.MAP_TYPES:
        tags.add("map projection")
    if case.n > rig_fuzz.WARP_BATCH:
        tags.add("n>32")
    _, _, w, h = _roi(cc.crop.corners, cc.crop.sizes)
    nb = _bands(case, w, h)
    if nb >= 0:
        tags.add("nb=0" if nb == 0 else "nb=1" if nb == 1 else "nb>=2")
        if nb >= 1:
            tags.add("tile l0 yes" if w % 2 == 0 else "tile l0 no")
    x, y, W, H = case.roi()
    if nb != _bands(case, W, H):
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
