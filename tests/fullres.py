"""The default Stitcher at camera resolution (helper module: no tests in here).

Two parts:

Records.  tests/golden/gen_fullres_golden.py ran the unmodified reference Stitcher (crop=True, gain_blocks compensator,
seam finder, spherical warper, multiband blender) on reference_cases.camera_views: record "a" is 4 views of
4000 x 3000 (LOW -> FINAL about 11), record "b" 3 views of 8000 x 6000 (about 21.9).  A record holds what the
Stitcher decided at LOW and MEDIUM resolution (cameras, scale, ratios, Cropper rectangles, LOW seam masks,
getMatGains()) and the digest of every FINAL-resolution stage per image, so the FINAL chain can be replayed on the
compositor, the drop-in classes or the oracle and a mismatch names its stage.

Ratio draws.  Crops of rig_fuzz-style rigs at FINAL sizes of 1500-4000 px seen from a LOW resolution at the ratios the
Stitcher's own formula gives for 2-48 MP cameras, sqrt(MP / 0.1), with LOW seam masks and 32 px block gain maps sized
from the LOW cropped images, as the seam finder and the gain_blocks compensator hand them out.  They go through the
compositor against rig_fuzz.oracle_run with the crop; coverage() restates from the geometry what each reaches.

SB_FULLRES_SEED=<int> or =random replaces the fixed default seed of the ratio draws (the seed used is printed).
"""
import dataclasses
import functools
import math
import time
import types

import numpy as np

import crop_fuzz
import fuzz_chain
import reference_cases as RC
import replay
import rig_fuzz
from stitching_b200 import Crop, rigs

RECORDS = ("a", "b")
STAGES = ("warped", "warped_mask", "cropped", "cropped_mask", "compensated", "blend_mask")
DEFAULT_SEED = 20261018
BLOCK = 32   # the gain_blocks compensator's block size at LOW resolution (ExposureErrorCompensator.DEFAULT_BLOCK_SIZE)


seed_from_env = functools.partial(fuzz_chain.seed_from_env, "SB_FULLRES_SEED", DEFAULT_SEED)


# -- the records --------------------------------------------------------------------------------------------------------
_records = {}


def record(name):
    if name not in _records:
        z = replay.load(f"golden_fullres_{name}.npz")
        _records[name] = {k: z[k] for k in (z.files if hasattr(z, "files") else z)}
    return _records[name]


def views(z):
    """The recorded run's FINAL inputs, rebuilt from the seed; fails unless they are the bytes the reference was fed."""
    n, w, h, seed = (int(v) for v in z["views"])
    out = RC.camera_views(w, h, n, seed)
    got = [RC.digest(v) for v in out]
    exp = [str(d) for d in z["inputs"]]
    assert got == exp, f"the rebuilt camera views are not the recorded inputs: {got} != {exp}"
    return out


def cameras(z):
    return [rigs.Camera(v[0], v[1], v[2], v[3], v[4:13].reshape(3, 3)) for v in z["cameras"]]


def cropper(z):
    return types.SimpleNamespace(do_crop=True, overlapping_rectangles=[tuple(map(int, r)) for r in z["overlaps"]],
                                 intersection_rectangles=[tuple(map(int, r)) for r in z["inters"]])


def crop(z):
    return Crop.from_cropper(cropper(z), float(z["low_to_final"]))


def seams(z):
    return [z[f"seam{i}"] for i in range(int(z["n"]))]


def gains(z):
    return [z[f"gain{i}"] for i in range(int(z["n"]))]


def shape_of(d):
    """The shape a digest names: 'u1[h, w, 3] sha256:...' -> (h, w, 3)."""
    return tuple(int(v) for v in d[d.index("[") + 1: d.index("]")].split(",") if v.strip())


def fed_rects(z):
    """(corner, fed size) per image: the prepared corners and the shapes of the cropped images."""
    return [tuple(map(int, c)) + shape_of(str(d))[1::-1] for c, d in zip(z["corners"], z["cropped"])]


def describe(name, z):
    n, w, h, _ = (int(v) for v in z["views"])
    return f"record {name}: {n} x {w}x{h}, LOW -> FINAL {float(z['low_to_final']):.4f}, pano {shape_of(str(z['pano']))}"


# -- replays ------------------------------------------------------------------------------------------------------------
class Mismatch(AssertionError):
    pass


def check_digest(got, z, stage, i=None, explain=None):
    """Assert that `got` is the array the reference handed on at `stage` (for image i); on a mismatch, `explain()` names
    the oracle's array for that stage and the |diff| histogram and first differing coordinates are printed."""
    exp = str(z[stage]) if i is None else str(z[stage][i])
    d = RC.digest(got)
    if d == exp:
        return np.asarray(got).size
    what = stage if i is None else f"{stage} {i}"
    msg = f"{what}: got {d}, the reference {exp}"
    if explain is not None:
        ref = explain()
        msg += "\n" + diff_table(np.asarray(got.get() if hasattr(got, "get") else got), ref, f"{what} against the oracle")
    print(msg)
    raise Mismatch(msg)


def diff_table(got, ref, what):
    if got.shape != ref.shape:
        return f"{what}: shape {got.shape} != {ref.shape}"
    d = np.abs(got.astype(np.int64) - ref.astype(np.int64))
    nz = np.argwhere(d)
    hist = np.bincount(np.minimum(d, 16).ravel(), minlength=17)
    rows = ", ".join(f"{k if k < 16 else '>=16'}: {int(c)}" for k, c in enumerate(hist) if c and k)
    return (f"{what}: {len(nz)} of {d.size} values differ, max |diff| {int(d.max())}; |diff| histogram {rows or 'none'}; "
            f"first at {[tuple(int(v) for v in p) for p in nz[:8]]}")


class OracleChain:
    """The FINAL chain of a record on the CPU oracle (fuzz_chain.oracle_image), image by image, built only when a stage
    has to be explained (or pinned); the blend only for the panorama."""

    def __init__(self, O, z, imgs):
        self.O, self.z, self.imgs = O, z, imgs
        self.cams, self.crop = cameras(z), crop(z)
        self.scale = np.float32(float(z["scale"]) * float(z["medium_to_final"]))
        self._cache = {}

    def stages(self, i):
        if i not in self._cache:
            from stitching_b200.warper import Warper

            cam, (x, y, w, h) = self.cams[i], self.crop.rects[i]
            (_, wi, wm), comp, bm = fuzz_chain.oracle_image(self.O, "spherical", self.scale,
                                                            Warper.get_K(cam, self.z["medium_to_final"]), cam.R, self.imgs[i],
                                                            (x, y, w, h), gains(self.z)[i], seam=seams(self.z)[i])
            # one image at a time: the stages of a 48 MP image take over half a GB
            self._cache = {i: dict(warped=wi, warped_mask=wm, cropped=wi[y:y + h, x:x + w], cropped_mask=wm[y:y + h, x:x + w],
                                   compensated=comp, blend_mask=bm)}
        return self._cache[i]

    def stage(self, stage, i):
        return lambda: self.stages(i)[stage]

    def pano(self):
        def run():
            b = self.O.Blender("multiband", 5)
            b.prepare([tuple(map(int, c)) for c in self.z["corners"]], [tuple(map(int, s)) for s in self.z["sizes"]])
            for i, c in enumerate(self.z["corners"]):
                s = self.stages(i)
                b.feed(s["compensated"], s["blend_mask"], tuple(map(int, c)))
            return b.blend()[0]
        return run


def compositor(z):
    from stitching_b200 import Compositor

    n, w, h, _ = (int(v) for v in z["views"])
    # the ratio goes in as a Python float on purpose: the compositor must scale K like Stitcher's float64 ratio does
    c = Compositor(cameras(z), [(w, h)] * n, "spherical", "multiband", 5, scale=float(z["scale"]), aspect=float(z["medium_to_final"]),
                   crop=crop(z))
    for i in range(int(z["n"])):
        c.set_seam_mask(i, seams(z)[i])
        c.set_gain(i, gains(z)[i])
    return c


def compositor_replay(z, imgs, oracle=None):
    """The fused compositor built from the record: geometry, every image after gain and its blend weight, the panorama,
    and two pipelined steps.  Returns the number of bytes compared."""
    chain = OracleChain(oracle, z, imgs) if oracle is not None else None
    c = compositor(z)
    try:
        n = int(z["n"])
        assert [tuple(r) for r in c.rects] == fed_rects(z), f"rects {c.rects} != {fed_rects(z)}"
        roi = fuzz_chain.blend_geometry([tuple(map(int, v)) for v in z["corners"]], [tuple(map(int, v)) for v in z["sizes"]]).roi
        assert tuple(c.roi) == roi, f"pano roi {c.roi} != {roi}"
        assert c.num_bands == int(z["num_bands"]), f"num_bands {c.num_bands} != {int(z['num_bands'])}"
        pano, pmask = c.composite(imgs)
        nbytes = 0
        # the warp kernel writes the image after gain and, as its fourth byte, the blend weight: the seam mask resized
        # and ANDed with the cropped validity mask (SeamFinder.resize's output), so the blend-mask stage is compared
        for i in range(n):
            wi, wm = c.download_warped(i)
            nbytes += check_digest(wi, z, "compensated", i, chain and chain.stage("compensated", i))
            nbytes += check_digest(wm, z, "blend_mask", i, chain and chain.stage("blend_mask", i))
        nbytes += check_digest(pano, z, "pano", None, chain and chain.pano())
        srcs = []
        for im in imgs:
            p = c.pinned_empty(im.shape)
            p[...] = im
            srcs.append(p)
        outs = [(c.pinned_empty(pano.shape), c.pinned_empty(pmask.shape)) for _ in range(2)]
        tickets = [c.submit(srcs, o, m) for o, m in outs]
        for t in tickets:
            c.wait(t)
        for k, (o, m) in enumerate(outs):
            assert np.array_equal(o, pano) and np.array_equal(m, pmask), f"pipelined step {k} differs from composite()"
            nbytes += o.size + m.size
        return nbytes, pano
    finally:
        c.close()


def dropin_replay(z, imgs, oracle=None):
    """The reference Stitcher's FINAL-resolution calls on the drop-in classes (stitcher.py:117-128): even images keep
    their device twin from the warp to the blender, odd ones travel as host copies.  Returns (bytes compared, pano)."""
    import stitching_b200
    from stitching_b200 import device_array, exposure_error_compensator, seam_finder

    import dropin_fuzz

    chain = OracleChain(oracle, z, imgs) if oracle is not None else None
    n, cams, aspect = int(z["n"]), cameras(z), z["medium_to_final"]  # numpy float64, as Stitcher passes it
    sizes_in = [(im.shape[1], im.shape[0]) for im in imgs]
    warper = stitching_b200.Warper("spherical")
    warper.set_scale(cams)
    assert warper.scale == float(z["scale"]), f"Warper.set_scale: {warper.scale} != {float(z['scale'])}"
    compensator = dropin_fuzz.GainCompensator(gains(z))
    cr = crop(z)
    corners, sizes = [tuple(map(int, v)) for v in z["corners"]], [tuple(map(int, v)) for v in z["sizes"]]
    assert [c for c in cr.corners] == corners and [s for s in cr.sizes] == sizes, "Crop.from_cropper: corners / sizes"
    b = stitching_b200.Blender("multiband", 5)
    b.prepare(corners, sizes)
    assert b.blender.num_bands == int(z["num_bands"]), f"num_bands {b.blender.num_bands} != {int(z['num_bands'])}"
    nbytes = 0
    ex = (lambda s, i: chain.stage(s, i)) if chain else (lambda s, i: None)
    for i, (wi, wm) in enumerate(zip(warper.warp_images(imgs, cams, aspect), warper.create_and_warp_masks(sizes_in, cams, aspect))):
        nbytes += check_digest(wi, z, "warped", i, ex("warped", i))
        nbytes += check_digest(wm, z, "warped_mask", i, ex("warped_mask", i))
        x, y, w, h = cr.rects[i]
        img, m = wi[y:y + h, x:x + w], wm[y:y + h, x:x + w]
        nbytes += check_digest(img, z, "cropped", i, ex("cropped", i))
        nbytes += check_digest(m, z, "cropped_mask", i, ex("cropped_mask", i))
        if i % 2:
            img = np.array(img)
        img = exposure_error_compensator.apply(compensator, i, corners[i], img, m)
        if i % 2 == 0:
            assert device_array.twin(img) is not None, f"image {i} lost its device twin"
        nbytes += check_digest(img, z, "compensated", i, ex("compensated", i))
        bm = seam_finder.resize(seams(z)[i], m)
        nbytes += check_digest(bm, z, "blend_mask", i, ex("blend_mask", i))
        b.feed(img, bm, corners[i])
    pano, _ = b.blend()
    pano = np.array(pano)
    nbytes += check_digest(pano, z, "pano", None, chain and chain.pano())
    return nbytes, pano


def oracle_stages(O, z, imgs, i):
    """The oracle's warp, numpy slice, gain_apply and seam_resize of image i against the recorded stage digests."""
    chain = OracleChain(O, z, imgs)
    s = chain.stages(i)
    return sum(check_digest(s[st], z, st, i) for st in STAGES)


# -- ratio draws --------------------------------------------------------------------------------------------------------
def pipeline_aspect(mp):
    """LOW -> FINAL of the Stitcher for an image of `mp` megapixels: MegapixDownscaler's sqrt(0.1 * 1e6 / area) scale
    for LOW over 1.0 for FINAL (final_megapix -1)."""
    return 1.0 / min(1.0, math.sqrt(0.1 * 1e6 / (mp * 1e6)))


def _draw(rng, index, seed, lo, hi):
    n = int(rng.integers(2, 5))
    sizes = [(int(rng.integers(lo, hi + 1)), int(rng.integers(lo * 3 // 4, hi * 3 // 4 + 1))) for _ in range(n)]
    u = rng.random()
    if u < 0.2:
        wtype, cams = "affine", rig_fuzz._affine_cams(rng, sizes)
    else:
        wtype = str(rng.choice(["spherical", "spherical", "cylindrical", "plane"]))
        cams = rig_fuzz._rot_cams(rng, wtype, sizes, "plane" if wtype == "plane" else "ring")
    blender = str(rng.choice(["multiband"] * 6 + ["feather", "no"]))
    gens = [str(rng.choice(["noise", "synth", "synth"])) for _ in range(n)]
    return rig_fuzz.Case(f"fullres_{index}", wtype, cams, sizes, blender, 5.0, ["seam"] * n, ["map1"] * n, gens, seed * 7919 + 300_000 + index)


def cases(seed, count, lo, hi, max_area):
    """`count` seeded crop cases with sources of lo..hi px (3:4), the Stitcher's LOW -> FINAL aspect of a 2-48 MP camera,
    and a LIR drawn at random; the warped rects stay under `max_area`."""
    rng = np.random.default_rng([seed, 1])
    out = []
    index = 0
    while len(out) < count:
        c = _draw(rng, index, seed, lo, hi)
        index += 1
        c.rects = rig_fuzz._rects(c.wtype, c.cams, c.sizes)
        if not all(0 < r[2] * r[3] <= max_area for r in c.rects):
            continue
        if c.blender == "multiband" and rng.random() < 0.5:
            c.strength = rig_fuzz._strength(rng, c.rects, c.blender)
        mp = float(rng.choice([2, 5, 8, 12, 16, 20, 24, 33, 48])) * float(rng.uniform(0.97, 1.03))
        cc = fuzz_chain.draw_crop(rng, c, pipeline_aspect(mp), 0.3, 0.7)
        if cc is not None:
            out.append(cc)
    return out


def extras(cc):
    """Per image (None, LOW seam mask, gain map): the seam mask at the size of the LOW cropped image (the intersection
    rectangle), a ragged cut through it as the graph-cut finder leaves them; the gain map one value per 32 x 32 block of
    it, as the gain_blocks compensator estimates them."""
    out = []
    for i, (_, _, w, h) in enumerate(cc.low.intersection_rectangles):
        rng = np.random.default_rng(cc.case.seed * 1000 + 700 + i)
        seam = np.zeros((h, w), np.uint8)
        cut = int(rng.integers(0, w + 1))
        for y in range(h):
            cut = int(np.clip(cut + rng.integers(-2, 3), 0, w))
            seam[y, :cut] = 255
        if i % 2:
            seam = 255 - seam
        gain = rng.uniform(0.7, 1.4, (-(-h // BLOCK), -(-w // BLOCK))).astype(np.float32)
        out.append((None, seam, gain))
    return out


def run_and_check(O, cc, seed):
    imgs, ex = rig_fuzz.images(cc.case), extras(cc)
    ref = rig_fuzz.oracle_run(O, cc.case, imgs, ex, crop=cc.crop)
    got = fuzz_chain.compositor_run(cc.case, imgs, ex, crop=cc.crop)
    rig_fuzz.check(dataclasses.replace(cc.case, name=cc.describe()), got, ref, seed)
    return sum(a.size for a in got["warped"] + got["masks"]) + got["pano"].size + got["pmask"].size


def coverage(cc):
    """crop_fuzz.coverage plus what the pipeline's ratios reach, from the geometry: the aspect, the seam-resize and
    gain-map stretch factors of the fed images, and slices the rounding clips at the warped image's bottom or right."""
    tags = crop_fuzz.coverage(cc)
    if cc.aspect > 8:
        tags.add("aspect>8")
    if cc.aspect > 16:
        tags.add("aspect>16")
    for (mask, seam, gain), (_, _, w, h) in zip(extras(cc), cc.fed()):
        if w / seam.shape[1] > 8 and h / seam.shape[0] > 8:
            tags.add("seam resize >8 both axes")
        if max(w / gain.shape[1], h / gain.shape[0]) > 100:
            tags.add("gain stretch >100")
    if any(f[2] < r[2] or f[3] < r[3] for f, r in zip(cc.fed(), cc.crop.rects)):
        tags.add("slice clipped")
    return tags


WANT = {"aspect>8", "aspect>16", "seam resize >8 both axes", "gain stretch >100", "slice clipped", "placement off by rounding",
        "tile l0 yes", "crop changes num_bands"}


def timed(fn, *a):
    t = time.perf_counter()
    r = fn(*a)
    return r, time.perf_counter() - t
