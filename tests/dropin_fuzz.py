"""Seeded random rigs and crops through the drop-in classes against the CPU oracle (helper module: no tests in here).

The drop-ins are what install() puts under every reference Stitcher, so they run here in the reference's order of calls
(stitcher.py:178-259): Warper.set_scale; warp_images / create_and_warp_masks / warp_rois; the crop as a numpy slice
(cropper.py:150-151); ExposureErrorCompensator.apply with a compensator whose getMatGains() hands out the case's gains;
SeamFinder.resize (with cv.UMat seam masks for a share of the cases, as the seam finders hand them out); Blender prepare /
feed / blend, with the int16 result for a share of the multiband cases; and, for some cases, the Timelapser over the same
images.  The oracle side is rig_fuzz.oracle_run on the same draws, with the crop where there is one; everything is
compared bit for bit.

Every case also picks, per image, how the image travels from the warp to the blender (FEEDS):
  twin  the warped image's device twin throughout: sb_gain_apply_dev, sb_blender_feed_dev (k_pack_rgbm from the twin's
        rectangle, at the crop's offset), sb_timelapse_frame from the twin;
  host  a host copy (np.array): sb_gain_apply, sb_blender_feed (k_pack_rgbm from an upload);
  s16   a host copy, compensated, then astype(np.int16): the blender's int16 layout and gather kernels.
A case whose images take different ways blends uint8 and int16 feeds in one pyramid ("mixed").

Three sets: the rig_fuzz and crop_fuzz draws under their own seeds (only the drop-in choices come from this module's
seed), and drop-in-only draws: 1-px source sides, source widths of every residue mod 8 (the byte offsets of k_warp_wide's
paired loads), sources passed as column-sliced views (row pitch > 3 w), strengths that are not float32-exact and
timelapse frames.

SB_DROPIN_FUZZ_SEED=<int> or =random replaces the fixed default seed of the drop-in choices and draws (the seed used
is printed).
"""
import dataclasses
import functools

import numpy as np

import crop_fuzz
import fuzz_chain
import rig_fuzz

DEFAULT_SEED = 20261017
FEEDS = ("twin", "host", "s16")
LANES, BLOCKS = rig_fuzz.LANES, rig_fuzz.BLOCKS


seed_from_env = functools.partial(fuzz_chain.seed_from_env, "SB_DROPIN_FUZZ_SEED", DEFAULT_SEED)


@dataclasses.dataclass
class DropCase:
    name: str
    case: object                # rig_fuzz.Case: cameras, sources, blender, extras (rects: the uncropped warped rects)
    crop: object = None         # crop_fuzz.CropCase, or None
    feeds: list = None          # per image: one of FEEDS
    umat: bool = False          # seam masks handed to SeamFinder.resize as cv.UMat
    s16_out: bool = False       # Blender.blend with the int16 result as well
    views: bool = False         # sources passed as column-sliced views of wider arrays
    timelapse: str = None       # "as_is" | "crop": the Timelapser's frames over the fed images, too
    env: dict = dataclasses.field(default_factory=dict)

    @property
    def n(self):
        return self.case.n

    def corners_sizes(self):
        """What Blender.prepare and Timelapser.initialize receive."""
        if self.crop is not None:
            return self.crop.crop.corners, self.crop.crop.sizes
        return [r[:2] for r in self.case.rects], [r[2:] for r in self.case.rects]

    def slices(self):
        """Per image the (x, y, w, h) slice of its warped image that is fed (the whole image without a crop)."""
        if self.crop is not None:
            return self.crop.crop.rects
        return [(0, 0, r[2], r[3]) for r in self.case.rects]

    def extras(self):
        return rig_fuzz.extras(self.crop.cropped_case() if self.crop is not None else self.case)

    def describe(self):
        base = self.crop.describe() if self.crop is not None else self.case.describe()
        feeds = "/".join(sorted(set(self.feeds)))
        more = [s for s, on in (("umat", self.umat), ("s16 out", self.s16_out), ("views", self.views)) if on]
        if self.timelapse:
            more.append(f"timelapse {self.timelapse}")
        return f"{self.name}: {base} feeds {feeds}" + "".join(f" {m}" for m in more)


# -- drop-in choices for a draw of rig_fuzz / crop_fuzz ------------------------------------------------------------------
def _choose(rng, name, case, crop=None):
    n = case.n
    u = rng.random()
    if u < 0.4:
        feeds = ["twin"] * n
    elif u < 0.55:
        feeds = ["host"] * n
    elif u < 0.7:
        feeds = ["s16"] * n
    else:
        feeds = [str(rng.choice(FEEDS)) for _ in range(n)]
    s16_out = case.blender == "multiband" and rng.random() < 0.3
    return DropCase(name, case, crop, feeds, umat=bool(rng.random() < 0.5), s16_out=bool(s16_out))


def from_rig(seed, k, case):
    dc = _choose(np.random.default_rng([seed, 1, k]), f"rig/{case.name}", case)
    dc.env = dict(case.env)
    return dc


def from_crop(seed, k, cc):
    return _choose(np.random.default_rng([seed, 2, k]), f"crop/{k}", cc.case, cc)


# -- drop-in-only draws ---------------------------------------------------------------------------------------------------
def _own_sizes(rng, n, side, small, k):
    sizes = []
    for i in range(n):
        w, h = rig_fuzz._side(rng, side, small), rig_fuzz._side(rng, side, small)
        w = max(1, w - w % 8 + (3 * k + i) % 8)  # every residue mod 8 over the set
        u = rng.random()
        if u < 0.1:
            w = 1
        elif u < 0.2:
            h = 1
        elif u < 0.3:
            h = int(rng.integers(2, 7))
        sizes.append((w, h))
    return sizes


def _inexact(rng, s):
    """A two-decimal strength near `s` that float32 cannot hold."""
    s = max(0.01, round(s * rng.uniform(0.97, 1.03), 2))
    while float(np.float32(s)) == s:
        s = round(s + 0.01, 2)
    return s


def _own_draw(rng, budget, k, seed):
    side = budget["side"]
    many = k % 12 == 5
    n = int(rng.integers(rig_fuzz.WARP_BATCH + 1, rig_fuzz.WARP_BATCH + 5)) if many else int(rng.choice([1, 2, 3, 3, 4, 5]))
    sizes = _own_sizes(rng, n, side, many, k)
    u = rng.random()
    if u < 0.2:
        wtype = str(rng.choice(rig_fuzz.MAP_TYPES + ("compressedPlaneA2B1", "paniniA1.5B1", "transverseMercator")))
        cams = rig_fuzz._rot_cams(rng, wtype, sizes, "ring")
    elif u < 0.4:
        wtype = "affine"
        cams = rig_fuzz._affine_cams(rng, sizes)
    else:
        wtype = str(rng.choice(["spherical", "cylindrical", "plane", "mercator"]))
        style = "plane" if wtype == "plane" else str(rng.choice(["ring", "ring", "turned"]))
        cams = rig_fuzz._rot_cams(rng, wtype, sizes, style)
    blender = str(rng.choice(["multiband"] * 5 + ["feather", "feather", "no"]))
    masks = [str(rng.choice(rig_fuzz.MASK_KINDS)) for _ in range(n)]
    gains = [str(rng.choice(rig_fuzz.GAIN_KINDS)) for _ in range(n)]
    gens = [str(rng.choice(["noise", "noise", "synth", "const"])) for _ in range(n)]
    return rig_fuzz.Case(f"own_{k}", wtype, cams, sizes, blender, 0.0, masks, gains, gens, seed * 7919 + 100_000 + k)


def own_cases(seed, count, budget, env_every=0):
    """`count` drop-in-only cases; with env_every > 0 every env_every-th case runs under SB_EMU_LANES, the one after it
    under SB_EMU_BLOCKS (emulation build)."""
    rng = np.random.default_rng([seed, 3])
    out = []
    for k in range(count):
        redraws = 0
        while True:
            c = _own_draw(rng, budget, k, seed)
            c.rects = rig_fuzz._rects(c.wtype, c.cams, c.sizes)
            if rig_fuzz._fits(c, budget):
                break
            redraws += 1
        c.redraws = redraws
        s = rig_fuzz._strength(rng, c.rects, c.blender)
        c.strength = _inexact(rng, s) if rng.random() < 0.85 else s
        cc = fuzz_chain.draw_crop(rng, c, crop_fuzz.ASPECTS, 0.3, 0.7, tries=1) if rng.random() < 0.4 else None
        dc = _choose(rng, c.name, c, cc)
        dc.views = bool(rng.random() < 0.5)
        if c.n <= 6 and rng.random() < 0.35:
            dc.timelapse = str(rng.choice(["as_is", "crop"]))
        if env_every and k % env_every == env_every - 2:
            dc.env = dict(LANES)
        elif env_every and k % env_every == env_every - 1:
            dc.env = dict(BLOCKS)
        out.append(dc)
    return out


# -- the seeded sets of the test suite ----------------------------------------------------------------------------------
EMU_RIG = list(range(12)) + list(range(rig_fuzz.EMU_COUNT, rig_fuzz.EMU_COUNT + len(rig_fuzz.EMU_NAMED)))
EMU_CROP = 8
EMU_OWN = 16
GPU_CROP = 40
GPU_OWN = 60

_sets = {}


def emu_set(seed):
    if ("emu", seed) not in _sets:
        rigs = rig_fuzz.emu_set(rig_fuzz.seed_from_env())
        crops = crop_fuzz.cases(crop_fuzz.seed_from_env(), EMU_CROP, rig_fuzz.EMU)
        _sets[("emu", seed)] = ([from_rig(seed, k, rigs[k]) for k in EMU_RIG] + [from_crop(seed, k, c) for k, c in enumerate(crops)] +
                                own_cases(seed, EMU_OWN, rig_fuzz.EMU, env_every=8))
    return _sets[("emu", seed)]


def gpu_set(seed):
    """The GPU rig set of rig_fuzz, the GPU crop set (as tests/test_gpu_crop.py draws it) and GPU_OWN own draws."""
    if ("gpu", seed) not in _sets:
        rigs = rig_fuzz.gpu_set(rig_fuzz.seed_from_env())
        crops = crop_fuzz.cases(crop_fuzz.seed_from_env(), GPU_CROP, rig_fuzz.GPU) + [crop_fuzz.named(n, rig_fuzz.GPU) for n in ("many", "full")]
        _sets[("gpu", seed)] = ([from_rig(seed, k, c) for k, c in enumerate(rigs)] + [from_crop(seed, k, c) for k, c in enumerate(crops)] +
                                own_cases(seed, GPU_OWN, rig_fuzz.GPU))
    return _sets[("gpu", seed)]


def gpu_count():
    return len(rig_fuzz.gpu_ids()) + GPU_CROP + 2 + GPU_OWN


# -- inputs -------------------------------------------------------------------------------------------------------------
def sources(dc):
    """The source images, as the drop-ins see them: column-sliced views of wider arrays when dc.views."""
    imgs = rig_fuzz.images(dc.case)
    if not dc.views:
        return imgs, imgs
    out = []
    for i, img in enumerate(imgs):
        rng = np.random.default_rng(dc.case.seed * 1000 + 900 + i)
        h, w = img.shape[:2]
        left = int(rng.integers(1, 9))
        big = rng.integers(0, 256, (h, w + left + int(rng.integers(0, 9)), 3), dtype=np.uint8)
        big[:, left:left + w] = img
        out.append(big[:, left:left + w])
    return imgs, out


class GainCompensator:
    """What ExposureErrorCompensator.apply reads from a fed cv.detail compensator: getMatGains()."""

    def __init__(self, gains):
        self.gains = gains

    def getMatGains(self):
        return self.gains


# -- the two sides ------------------------------------------------------------------------------------------------------
def oracle_run(O, dc, imgs, ex):
    ref = rig_fuzz.oracle_run(O, dc.case, imgs, ex, s16=dc.s16_out, crop=dc.crop.crop if dc.crop is not None else None)
    if dc.timelapse:
        corners, sizes = dc.corners_sizes()
        t = O.Timelapser(dc.timelapse)
        t.initialize(corners, sizes)
        frames = []
        for wi, c in zip(ref["warped"], corners):
            t.process_frame(wi, c)
            frames.append(t.get_frame() if t.roi[2] > 0 and t.roi[3] > 0 else None)
        ref["frames"] = frames
    return ref


def dropin_run(dc, srcs, ex):
    """The Stitcher's calls on the drop-in classes.  Asserts on the way that every twin-fed image still has its twin."""
    import stitching_b200
    from stitching_b200 import StitchingError, device_array, exposure_error_compensator, seam_finder

    case = dc.case
    warper = stitching_b200.Warper(case.wtype)
    warper.set_scale(case.cams)
    warped = list(warper.warp_images(srcs, case.cams))
    wmasks = list(warper.create_and_warp_masks(case.sizes, case.cams))
    rcorners, rsizes = warper.warp_rois(case.sizes, case.cams)
    raw = [(np.array(wi), wm.copy()) for wi, wm in zip(warped, wmasks)]  # apply() below writes into the warped images
    corners, sizes = dc.corners_sizes()
    compensator = GainCompensator([g for _, _, g in ex])
    umat = None
    if dc.umat:
        try:
            import cv2

            umat = cv2.UMat
        except ImportError:
            pass
    fed, fmasks, comp = [], [], []
    for i, (wi, wm, (x, y, w, h), (mask, seam, _)) in enumerate(zip(warped, wmasks, dc.slices(), ex)):
        img, m = wi[y:y + h, x:x + w], wm[y:y + h, x:x + w]
        if dc.feeds[i] != "twin":
            img = np.array(img)
        img = exposure_error_compensator.apply(compensator, i, corners[i], img, m)
        if dc.feeds[i] == "twin":
            assert device_array.twin(img) is not None, f"{dc.describe()}: image {i} lost its device twin"
        comp.append(np.array(img))
        if mask is not None:
            m = mask
        elif seam is not None:
            m = seam_finder.resize(umat(seam) if umat else seam, m)
        fmasks.append(m)
        fed.append(img.astype(np.int16) if dc.feeds[i] == "s16" else img)
    b = stitching_b200.Blender(case.blender, case.strength)
    b.prepare(corners, sizes)
    num_bands = b.blender.num_bands if b.blender.kind == "multiband" else -1
    for img, m, c in zip(fed, fmasks, corners):
        b.feed(img, m, c)
    if dc.s16_out:
        pano, pmask, pano16 = b.blender.blend(want_s16=True)
    else:
        (pano, pmask), pano16 = b.blend(), None
    got = dict(rects=[tuple(c) + tuple(s) for c, s in zip(rcorners, rsizes)], raw=raw, warped=comp,
               masks=[m.get() if hasattr(m, "get") and not isinstance(m, np.ndarray) else np.asarray(m) for m in fmasks],
               fed_rects=[tuple(c) + (img.shape[1], img.shape[0]) for c, img in zip(corners, fed)], num_bands=num_bands,
               pano=np.array(pano), pmask=np.array(pmask), pano16=pano16)
    if dc.timelapse:
        t = stitching_b200.Timelapser(dc.timelapse)
        t.initialize(corners, sizes)
        frames = []
        for img, c in zip(fed, corners):
            t.process_frame(img, c)
            try:
                frames.append(np.array(t.get_frame()))
            except StitchingError:
                frames.append(None)  # an empty canvas: the reference's get_frame fails as well
        got["frames"] = frames
    return got


def check(dc, got, ref, seed):
    """Bit for bit: the warped rects, every warped image and mask, every compensated (cropped) image and blend mask, the
    fed rects, num_bands, the panorama and its mask, the int16 result and the timelapse frames where asked."""
    import replay

    where = f"seed {seed}, {dc.describe()}"
    assert [tuple(r) for r in got["rects"]] == [tuple(r) for r in dc.case.rects], f"{where}: warp_rois"
    for i in range(dc.n):
        replay.assert_exact(np.asarray(got["raw"][i][0]), ref["raw"][i][0], f"{where}: warped image {i}")
        replay.assert_exact(got["raw"][i][1], ref["raw"][i][1], f"{where}: warped mask {i}")
        replay.assert_exact(got["warped"][i], ref["warped"][i], f"{where}: compensated image {i}")
        replay.assert_exact(got["masks"][i], ref["masks"][i], f"{where}: blend mask {i}")
    assert [tuple(r) for r in got["fed_rects"]] == [tuple(r) for r in ref["rects"]], f"{where}: fed rects"
    assert got["num_bands"] == ref["num_bands"], f"{where}: num_bands {got['num_bands']} != {ref['num_bands']}"
    replay.assert_exact(got["pano"], ref["pano"], f"{where}: pano")
    replay.assert_exact(got["pmask"], ref["pmask"], f"{where}: pano mask")
    if dc.s16_out:
        replay.assert_exact(got["pano16"], ref["pano16"], f"{where}: int16 pano")
    if dc.timelapse:
        for i, (g, r) in enumerate(zip(got["frames"], ref["frames"])):
            assert (g is None) == (r is None), f"{where}: timelapse frame {i} (empty canvas on one side only)"
            if r is not None:
                replay.assert_exact(g, r, f"{where}: timelapse frame {i}")


def run_and_check(O, dc, seed):
    imgs, srcs = sources(dc)
    ex = dc.extras()
    ref = oracle_run(O, dc, imgs, ex)
    got = dropin_run(dc, srcs, ex)
    check(dc, got, ref, seed)
    return imgs, ex, got


# -- coverage -----------------------------------------------------------------------------------------------------------
def plan(dc):
    """(blend kind, band count, pano width) of Blender.prepare on the prepared corners and sizes, in double like the
    reference; band count -1 when not multiband."""
    g = fuzz_chain.blend_geometry(*dc.corners_sizes(), dc.case.blender, dc.case.strength)
    return g.kind, g.nb if g.kind == "multiband" else -1, g.roi[2]


def footprints(O, dc, i):
    """Which paths k_warp_wide takes for image i, from the float maps of its projection: whether a bilinear footprint
    straddles the border (reflected, byte loads) and the byte offsets mod 8 of the paired loads of the inside ones."""
    case = dc.case
    _, xm, ym = O.build_maps(case.wtype, case.scale(), rig_fuzz.Warper.get_K(case.cams[i], 1), case.cams[i].R, case.sizes[i])
    sw, sh = case.sizes[i]
    with np.errstate(invalid="ignore", over="ignore"):
        sx, sy = np.rint(xm * np.float32(32)), np.rint(ym * np.float32(32))
        ok = np.isfinite(sx) & np.isfinite(sy) & (np.abs(sx) < 2 ** 30) & (np.abs(sy) < 2 ** 30)
        ix = np.where(ok, sx, 0).astype(np.int64) >> 5
        iy = np.where(ok, sy, 0).astype(np.int64) >> 5
    inside = ok & (ix >= 0) & (ix < sw - 1) & (iy >= 0) & (iy < sh - 1)
    offsets = set(np.unique((3 * (iy[inside] * sw + ix[inside])) % 8).tolist())
    return bool((~inside).any()), offsets


def coverage(dc, O=None, tile=True):
    """What a drop-in case reaches, from its geometry and choices alone.  `tile`: the tile collapse runs in this build
    (always on the GPU; under SB_EMU_BLOCKS in the emulation build).  With the oracle `O`, the k_warp_wide paths of the
    first two images of the case are restated from the projection's maps as well."""
    case = dc.case
    tags = set()
    kind, nb, pano_w = plan(dc)
    tags.add(kind)
    if kind == "multiband":
        tags.add("nb=0" if nb == 0 else "nb=1" if nb == 1 else "nb>=2")
    feeds = set(dc.feeds)
    for f in feeds:
        tags.add(f"{f} feed")
    if len(feeds) > 1:
        tags.add("mixed feeds")
    if "s16" in feeds and len(feeds) > 1:
        tags.add("uint8 and int16 in one blend")
    slices = dc.slices()
    if any(f == "twin" and s[0] > 0 for f, s in zip(dc.feeds, slices)):
        tags.add("twin at x offset != 0")
    fed_w = [min(s[2], r[2] - s[0]) for s, r in zip(slices, case.rects)]
    byte_only = "s16" not in feeds
    if kind == "multiband" and nb >= 1 and byte_only and not dc.s16_out and pano_w % 2 == 0 and tile and \
            any(w % 4 for w in fed_w):
        tags.add("rgbm pitch != width, tile l0")
    for g, f in zip(case.gains, dc.feeds):
        if g != "none":
            tags.add(f"gain {'map' if g.startswith('map') else g} on {'twin' if f == 'twin' else 'host'}")
    if case.wtype not in rig_fuzz.TABLE_TYPES:  # maps built on the host
        tags.add("map projection")
    if rig_fuzz._z_nonpositive(case):
        tags.add("z<=0")
    if dc.umat and any(m == "seam" for m in case.masks):
        tags.add("UMat seams")
    if case.n > rig_fuzz.WARP_BATCH:
        tags.add("n>32")
    if any(min(s) == 1 for s in case.sizes):
        tags.add("1-px source")
    if float(np.float32(case.strength)) != case.strength:
        tags.add("non-float32 strength")
    if dc.s16_out:
        tags.add("int16 result")
    if dc.views:
        tags.add("column-sliced sources")
    if dc.crop is not None:
        tags.add("crop")
    if dc.timelapse:
        tags.add(f"timelapse {dc.timelapse}")
    for w, _ in case.sizes:
        tags.add(f"src w%8={w % 8}")
    if O is not None:
        for i in range(min(2, case.n)):
            border, offsets = footprints(O, dc, i)
            if border:
                tags.add("border branch")
            tags.update(f"fetch_pair o={o}" for o in offsets)
    return tags


def emu_coverage(dc, O=None):
    return coverage(dc, O, tile="SB_EMU_BLOCKS" in dc.env)


WANT = {"twin feed", "host feed", "s16 feed", "mixed feeds", "uint8 and int16 in one blend", "twin at x offset != 0",
        "rgbm pitch != width, tile l0", "nb=0", "nb=1", "nb>=2", "feather", "no", "map projection", "z<=0", "border branch",
        "gain map on twin", "gain map on host", "gain scalar on twin", "gain scalar on host", "gain vector on twin",
        "gain vector on host", "UMat seams", "n>32", "1-px source", "non-float32 strength", "int16 result",
        "column-sliced sources", "crop", "timelapse as_is", "timelapse crop"} | {f"fetch_pair o={o}" for o in range(8)} | \
       {f"src w%8={r}" for r in range(8)}
