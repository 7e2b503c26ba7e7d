"""Seeded random rigs for the compositor against the CPU oracle (helper module: no tests in here).

cases(seed, count, budget) yields Case records: warper type, cameras and per-image source sizes, blender kind and
strength, per-image extras (set_mask / set_seam_mask / set_gain) and how each source image is generated.  The draws aim
at the launch-time branches of the compositor that the fixed BASELINE rigs never reach: odd and tiny sources, flat
images beside large ones, poles in view, cameras whose warped rect holds directions behind them, steep plane tilts,
sheared affines with rect origins on every alignment, more than SB_WARP_BATCH images, every band count from 0 to the
clipped maximum, and extras mixed within one rig.  `budget` bounds the largest source side and the largest warped-rect
area, so the same generator serves the emulation build (small) and the GPU (large).

coverage(case, ...) restates, from the case's geometry alone, the predicates the launchers use to choose a kernel, so
that a test can prove which branches a seeded set of cases reached.

SB_RIG_FUZZ_SEED=<int> or =random replaces the fixed default seed (the seed used is printed).
"""
import dataclasses
import functools
import math
from statistics import median

import numpy as np

import fuzz_chain
from stitching_b200 import rigs
from stitching_b200.warper import Warper

DEFAULT_SEED = 20261015
EMU = dict(side=120, area=14_000)         # emulation build: serial CPU stand-in for the device
GPU = dict(side=1500, area=1_200_000)     # H100: the oracle (scalar C on the CPU) sets the cost
TABLE_TYPES = ("spherical", "cylindrical", "plane", "affine", "mercator")  # k_warp_rgbm from separable tables
MAP_TYPES = ("fisheye", "stereographic")                                 # host-built maps, k_warp_wide writes RGBM
WARP_BATCH = 32        # SB_WARP_BATCH: the images of one warp launch
MASK_KINDS = ("none", "binary", "ramp", "random", "seam")
GAIN_KINDS = ("none", "map1", "map3", "scalar", "vector")


seed_from_env = functools.partial(fuzz_chain.seed_from_env, "SB_RIG_FUZZ_SEED", DEFAULT_SEED)


@dataclasses.dataclass
class Case:
    name: str
    wtype: str
    cams: list
    sizes: list            # source (w, h) per image
    blender: str
    strength: float
    masks: list            # per image: one of MASK_KINDS
    gains: list            # per image: one of GAIN_KINDS
    gens: list             # per image: "noise" | "synth" | "const"
    seed: int              # of the image / extras content
    rects: list = None     # warped (x, y, w, h) per image, from the oracle
    env: dict = dataclasses.field(default_factory=dict)  # emulation switches this case runs under
    redraws: int = 0       # draws rejected by the budget before this one

    @property
    def n(self):
        return len(self.cams)

    def describe(self):
        ws = [s[0] for s in self.sizes]
        hs = [s[1] for s in self.sizes]
        extras = ",".join(f"{m}/{g}" for m, g in zip(self.masks, self.gains) if (m, g) != ("none", "none")) or "none"
        env = " " + " ".join(f"{k}={v}" for k, v in self.env.items()) if self.env else ""
        return (f"{self.name}: {self.wtype} n={self.n} src w {min(ws)}..{max(ws)} h {min(hs)}..{max(hs)} "
                f"{self.blender}@{self.strength:g} extras {extras}{env}")

    def scale(self):
        return np.float32(median([c.focal for c in self.cams]))  # Warper.set_scale, as float32 like the C ABI

    def geometry(self):
        return fuzz_chain.blend_geometry([r[:2] for r in self.rects], [r[2:] for r in self.rects], self.blender, self.strength)

    def roi(self):
        return self.geometry().roi


# -- inputs -----------------------------------------------------------------------------------------------------------
def images(case):
    out = []
    for i, ((w, h), g) in enumerate(zip(case.sizes, case.gens)):
        s = case.seed * 1000 + i
        if g == "noise":
            out.append(rigs.noise_image(h, w, s))
        elif g == "synth":
            out.append(rigs.synth_image(h, w, s))
        else:
            out.append(np.full((h, w, 3), np.random.default_rng(s).integers(0, 256, 3), np.uint8))
    return out


def extras(case):
    """Per image (mask, seam, gain): a warped-size blend mask for set_mask, a low-resolution seam mask for
    set_seam_mask, a gain in the forms a cv.detail compensator's getMatGains() hands out; None where absent."""
    out = []
    for i, (mk, gk, r) in enumerate(zip(case.masks, case.gains, case.rects)):
        rng = np.random.default_rng(case.seed * 1000 + 500 + i)
        h, w = r[3], r[2]
        mask = seam = gain = None
        if mk == "binary":
            mask = (rng.random((max(1, h // 4 + 1), max(1, w // 4 + 1))) < 0.7).repeat(4, 0).repeat(4, 1)[:h, :w]
            mask = mask.astype(np.uint8) * 255
        elif mk == "ramp":
            mask = np.minimum(np.arange(w)[None, :] * 255 // max(1, w // 3), 255) * np.ones((h, 1), np.int64)
            mask = np.minimum(mask, (np.arange(h)[:, None] * 255 // max(1, h // 2 + 1) + 40)).astype(np.uint8)
        elif mk == "random":
            mask = rng.integers(0, 256, (h, w), dtype=np.uint8)
        elif mk == "seam":
            sh, sw = max(2, int(round(h / rng.uniform(1.5, 4)))), max(2, int(round(w / rng.uniform(1.5, 4))))
            seam = np.zeros((sh, sw), np.uint8)
            seam[:, : int(rng.integers(0, sw + 1))] = 255
            for y in rng.integers(0, sh, 4):
                seam[max(0, y - 1): y + 2, :] = 255 * int(rng.integers(0, 2))
            if i % 2:
                seam = 255 - seam
        if gk == "map1":
            gain = rng.uniform(0.6, 1.6, (int(rng.integers(1, 8)), int(rng.integers(1, 8)))).astype(np.float32)
        elif gk == "map3":
            gain = rng.uniform(0.6, 1.6, (int(rng.integers(1, 8)), int(rng.integers(1, 8)), 3)).astype(np.float32)
        elif gk == "scalar":
            gain = np.array([[rng.uniform(0.6, 1.6)]], np.float64)
        elif gk == "vector":
            gain = np.array([[rng.uniform(0.6, 1.6)], [rng.uniform(0.6, 1.6)], [rng.uniform(0.6, 1.6)], [0.0]], np.float64)
        out.append((mask, seam, gain))
    return out


# -- drawing ----------------------------------------------------------------------------------------------------------
def _side(rng, side, small=False):
    """One source side: mostly log-uniform, with the widths kernels trip over (odd, 1 mod 32, 2) mixed in."""
    hi = max(4, side // 6) if small else side
    u = rng.random()
    if u < 0.08:
        return 2
    if u < 0.2:  # 1 mod 32
        return 32 * int(rng.integers(1, (hi - 1) // 32 + 1)) + 1 if hi > 33 else 3
    v =int(round(math.exp(rng.uniform(math.log(3), math.log(hi)))))
    return v | 1 if u < 0.45 else v


def _sizes(rng, n, side, small=False):
    sizes = []
    for _ in range(n):
        w, h = _side(rng, side, small), _side(rng, side, small)
        u = rng.random()
        if u < 0.12:
            h = int(rng.integers(2, 7))    # very flat
        elif u < 0.2:
            w = int(rng.integers(2, 7))    # very thin
        sizes.append((max(2, w), max(2, h)))
    return sizes


def _quant(x):
    """`x` on a grid of 1/256 (float32-exact).  The compositor takes the strength in double like the oracle, so any
    value would do; the grid stays so that the seeded draws do not move (tests/dropin_fuzz.py draws inexact ones)."""
    return float(np.float32(round(x * 256) / 256))


def _rot_cams(rng, wtype, sizes, style):
    n = len(sizes)
    cams = []
    med = median(max(w, h) for w, h in sizes)
    if style == "pole":
        f = med * rng.uniform(0.5, 1.2)
    elif style == "turned":
        f = med * rng.uniform(0.25, 0.5)  # wide field of view
    else:
        f = med * rng.uniform(0.6, 2.5)
    step = rng.uniform(5, 60)
    for i, (w, h) in enumerate(sizes):
        yaw = np.deg2rad(step * (i - (n - 1) / 2) + rng.uniform(-3, 3))
        pitch = rng.uniform(-0.15, 0.15)
        if style == "pole" and i == 0:
            pitch = float(rng.choice([-1, 1])) * rng.uniform(1.2, 1.6)
        elif style == "turned" and i % 2 == 0:
            pitch = float(rng.choice([-1, 1])) * rng.uniform(0.5, 1.1)
        elif style == "plane":
            pitch = float(rng.choice([-1, 1])) * rng.uniform(0.4, 1.0) if i == 0 else rng.uniform(-0.3, 0.3)
            yaw = np.deg2rad(rng.uniform(-25, 25))
        roll = rng.uniform(-0.1, 0.1)
        R = rigs.rot_y(yaw) @ rigs.rot_x(pitch) @ np.array([[np.cos(roll), -np.sin(roll), 0], [np.sin(roll), np.cos(roll), 0],
                                                             [0, 0, 1]])
        fi = f * rng.uniform(0.97, 1.03)
        cams.append(rigs.Camera(fi, rng.uniform(0.97, 1.03), w / 2 + rng.uniform(-3, 3), h / 2 + rng.uniform(-3, 3),
                                R.astype(np.float32)))
    return cams


def _affine_cams(rng, sizes):
    cams = []
    x = 0.0
    for i, (w, h) in enumerate(sizes):
        th = rng.uniform(-0.5, 0.5)
        sx, sy = rng.uniform(0.6, 1.5), rng.uniform(0.6, 1.5)
        sh = rng.uniform(-0.4, 0.4)
        A = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]) @ np.array([[sx, sh], [0, sy]])
        tx = x + rng.uniform(-0.5, 0.5) * w + rng.integers(0, 64) + rng.random()
        ty = rng.uniform(-0.5, 0.5) * h + rng.integers(0, 64) + rng.random()
        x += 0.6 * w * sx
        H = np.array([[A[0, 0], A[0, 1], tx], [A[1, 0], A[1, 1], ty], [0, 0, 1]], np.float32)
        cams.append(rigs.Camera(1.0, 1.0, 0.0, 0.0, H))
    return cams


def _rects(wtype, cams, sizes):
    from oracle import oracle as O

    scale = np.float32(median([c.focal for c in cams]))
    return [O.warp_roi(wtype, scale, Warper.get_K(c, 1), c.R, s) for c, s in zip(cams, sizes)]


def _strength(rng, rects, blender):
    """Blend strength aimed at a band count: 0, 1, 2, intermediate, the clipped maximum; or a blend width under 1."""
    _, _, w, h = fuzz_chain.blend_geometry([r[:2] for r in rects], [r[2:] for r in rects]).roi
    root = math.sqrt(w * h)
    u = rng.random()
    if u < 0.06:
        return _quant(max(1 / 256, 50.0 / root))                  # blend width about 0.5: the NO blender
    if blender != "multiband" or u < 0.16:
        return float(rng.choice([1, 5, 20, 60, 100]))
    if u < 0.26:
        return 100.0                                                # far past the clip at ceil(log2(max side))
    nb = int(rng.choice([0, 0, 1, 1, 2, 2, 3, 4, 5]))
    bw = 2.0 ** (nb + 1 + rng.uniform(0.1, 0.9))                    # Blender.prepare: int(log2(bw) - 1) == nb
    return _quant(max(1 / 256, bw * 100 / root))


def _draw(rng, budget, index, seed):
    side = budget["side"]
    u = rng.random()
    many = index % 12 == 7                                      # a fixed share crosses SB_WARP_BATCH
    n = int(rng.integers(WARP_BATCH + 1, WARP_BATCH + 9)) if many else int(rng.choice([1, 2, 2, 3, 3, 4, 5, 6]))
    sizes = _sizes(rng, n, side, small=many)
    if u < 0.125:
        wtype = str(rng.choice(MAP_TYPES))
        cams = _rot_cams(rng, wtype, sizes, "ring")
    elif u < 0.35:
        wtype = "affine"
        cams = _affine_cams(rng, sizes)
    else:
        wtype = str(rng.choice(["spherical", "spherical", "cylindrical", "cylindrical", "plane", "mercator"]))
        style = str(rng.choice(["ring", "ring", "pole", "turned"])) if wtype != "plane" else "plane"
        if wtype == "mercator" and style == "pole":
            style = "ring"
        cams = _rot_cams(rng, wtype, sizes, style)
    blender = str(rng.choice(["multiband"] * 6 + ["feather", "feather", "no"]))
    mode = rng.random()
    if mode < 0.4:
        masks, gains = ["none"] * n, ["none"] * n
    elif mode < 0.55:
        mk, gk = str(rng.choice(MASK_KINDS)), str(rng.choice(GAIN_KINDS))
        masks, gains = [mk] * n, [gk] * n
    else:  # mixed within the rig
        masks = [str(rng.choice(MASK_KINDS)) for _ in range(n)]
        gains = [str(rng.choice(GAIN_KINDS)) for _ in range(n)]
    gens = [str(rng.choice(["noise", "noise", "synth", "const"])) for _ in range(n)]
    return Case(f"case_{index}", wtype, cams, sizes, blender, 0.0, masks, gains, gens, seed * 7919 + index)


def _fits(case, budget):
    return all(r[2] > 0 and r[3] > 0 and r[2] * r[3] <= budget["area"] and r[2] <= 12 * budget["side"] for r in case.rects)


def cases(seed, count, budget):
    """`count` seeded cases whose warped rects fit `budget`; each carries the number of rejected draws before it."""
    rng = np.random.default_rng(seed)
    for index in range(count):
        redraws = 0
        while True:
            c = _draw(rng, budget, index, seed)
            c.rects = _rects(c.wtype, c.cams, c.sizes)
            if _fits(c, budget):
                break
            redraws += 1
        c.strength = _strength(rng, c.rects, c.blender)
        c.redraws = redraws
        yield c


def named(name, budget):
    """Cases kept by name: each reaches one branch on purpose."""
    side = budget["side"]
    if name == "flat_top":
        # a flat image whose rect is the top of the pano (no top padding) but whose padded rect reaches further below
        # it than it is high: pyrDown level 0 is not NEAR (launch_pyrdown_fast, the second clause of level 0's test)
        sizes = [(min(side, 90), 3), (min(side, 70), min(side, 40)), (min(side, 60), min(side, 30))]
        cams = [rigs.Camera(1, 1, 0, 0, np.array([[1, 0, 0.3], [0, 1, 36.0], [0, 0, 1]], np.float32)),
                rigs.Camera(1, 1, 0, 0, np.array([[1, 0.1, 40.6], [0, 1, 9.25], [0, 0, 1]], np.float32)),
                rigs.Camera(1, 1, 0, 0, np.array([[0.9, 0, 11.1], [0.2, 1, 20.5], [0, 0, 1]], np.float32))]
        c = Case(name, "affine", cams, sizes, "multiband", 0.0, ["none"] * 3, ["none", "map1", "none"],
                 ["noise", "synth", "noise"], 11)
    elif name == "gray_mask_multiband":
        # gray blend masks switch the compositor's binary-mask shortcut (BIN) off for the whole plan
        sizes = [(min(side, 50), min(side, 36)), (min(side, 47), min(side, 33)), (min(side, 41), min(side, 38))]
        cams = rigs.yaw_ring(3, 50, 36, 60, 30)
        c = Case(name, "spherical", cams, sizes, "multiband", 0.0, ["random", "none", "ramp"], ["none", "scalar", "none"],
                 ["noise"] * 3, 12)
    elif name == "thin_levels":
        # a pano 4 rows high: the padded rects are one lattice cell high, so level 1 has 2 rows and pyrDown past level 0
        # is not NEAR: <false, false, false> runs
        sizes = [(min(side, 60), 3), (min(side, 55), 3)]
        cams = [rigs.Camera(1, 1, 0, 0, np.array([[1, 0, 5.5], [0, 1, 0.0], [0, 0, 1]], np.float32)),
                rigs.Camera(1, 1, 0, 0, np.array([[1, 0, 40.2], [0, 1, 0.5], [0, 0, 1]], np.float32))]
        c = Case(name, "affine", cams, sizes, "multiband", 0.0, ["none"] * 2, ["none"] * 2, ["noise"] * 2, 13)
    elif name == "many":
        n = WARP_BATCH + 5
        sizes = [(9 + i % 7, 7 + (3 * i) % 5) for i in range(n)]
        cams = [rigs.Camera(1, 1, 0, 0, np.array([[1, 0, 7.0 * (i % 9) + 0.4 * i], [0, 1, 6.0 * (i // 9) + 0.1], [0, 0, 1]],
                                                  np.float32)) for i in range(n)]
        masks = ["none"] * n
        masks[WARP_BATCH + 2] = "binary"
        gains = ["none"] * n
        gains[WARP_BATCH + 1] = "map3"
        c = Case(name, "affine", cams, sizes, "multiband", 0.0, masks, gains, ["noise"] * n, 14)
    elif name == "odd_origins":
        # rects at odd origins and an odd pano width: the tile kernel's level 0 declines (launch_collapse_tile: odd
        # output pitches)
        sizes = [(min(side, 61), min(side, 45)), (min(side, 53), min(side, 47)), (min(side, 40), min(side, 31))]
        cams = [rigs.Camera(1, 1, 0, 0, np.array([[1, 0, 3.7], [0, 1, 1.3], [0, 0, 1]], np.float32)),
                rigs.Camera(1, 1, 0, 0, np.array([[0.95, 0.1, 37.2], [-0.1, 1.05, 9.6], [0, 0, 1]], np.float32)),
                rigs.Camera(1, 1, 0, 0, np.array([[1, 0, 19.5], [0, 1, 33.9], [0, 0, 1]], np.float32))]
        c = Case(name, "affine", cams, sizes, "multiband", 0.0, ["none", "seam", "none"], ["none"] * 3, ["synth", "noise", "noise"], 15)
    elif name in ("thin_w", "thin_h"):
        # a pano 4 px wide (thin_w) or high (thin_h) with two bands: every padded rect is one 4-px lattice cell across,
        # so level 2 is 1 px wide (high) and k_collapse_tile's level 1 stages a coarse window of one column (row):
        # fix_borders' reflect-101 of a 1-px level
        sizes = [(4, min(side, 40)), (4, min(side, 37))]
        offs = [(0.0, 0.0), (0.0, 23.0)]
        if name == "thin_h":
            sizes = [(h, w) for w, h in sizes]
            offs = [(y, x) for x, y in offs]
        cams = [rigs.Camera(1, 1, 0, 0, np.array([[1, 0, ox], [0, 1, oy], [0, 0, 1]], np.float32)) for ox, oy in offs]
        c = Case(name, "affine", cams, sizes, "multiband", 0.0, ["none", "ramp"], ["none"] * 2, ["noise", "synth"], 17)
    elif name == "wide_feather":
        # a feather image wider than 8192 px: the two-sweep distance-transform row kernel (launch_feather_weights_fast)
        sizes = [(8300, 9), (700, 60)]
        cams = [rigs.Camera(1, 1, 0, 0, np.array([[1, 0, 0.5], [0, 1, 0.0], [0, 0, 1]], np.float32)),
                rigs.Camera(1, 1, 0, 0, np.array([[1, 0, 4000.25], [0.02, 1, 4.5], [0, 0, 1]], np.float32))]
        c = Case(name, "affine", cams, sizes, "feather", 5.0, ["none", "binary"], ["none", "vector"], ["noise", "synth"], 16)
    else:
        raise KeyError(name)
    c.rects = _rects(c.wtype, c.cams, c.sizes)
    if c.blender == "multiband" and c.strength == 0.0:
        x0, y0, w, h = c.roi()
        c.strength = _quant(2.0 ** 3.5 * 100 / math.sqrt(w * h))  # two bands
    return c


# -- the seeded sets of the test suite ----------------------------------------------------------------------------------
LANES, BLOCKS = {"SB_EMU_LANES": "1"}, {"SB_EMU_BLOCKS": "1"}
EMU_COUNT = 36
# emulation: the shuffle pyrDown runs only under SB_EMU_LANES and the tile collapse only under SB_EMU_BLOCKS (slow)
EMU_NAMED = [("flat_top", LANES), ("gray_mask_multiband", LANES), ("thin_levels", LANES),
             ("odd_origins", BLOCKS), ("many", BLOCKS), ("gray_mask_multiband", BLOCKS), ("thin_w", BLOCKS), ("thin_h", BLOCKS)]
GPU_COUNT = 200
GPU_NAMED = ["many", "wide_feather", "flat_top", "thin_levels", "odd_origins", "gray_mask_multiband", "thin_w", "thin_h"]


def emu_ids():
    return [f"case_{k}" for k in range(EMU_COUNT)] + [f"{n}-{'lanes' if e is LANES else 'blocks'}" for n, e in EMU_NAMED]


def gpu_ids():
    return [f"case_{k}" for k in range(GPU_COUNT)] + GPU_NAMED


_sets = {}


def emu_set(seed):
    if ("emu", seed) not in _sets:
        out = list(cases(seed, EMU_COUNT, EMU))
        for name, env in EMU_NAMED:
            c = named(name, EMU)
            c.env = dict(env)
            c.name = f"{name}-{'lanes' if env is LANES else 'blocks'}"
            out.append(c)
        _sets[("emu", seed)] = out
    return _sets[("emu", seed)]


def gpu_set(seed):
    if ("gpu", seed) not in _sets:
        _sets[("gpu", seed)] = list(cases(seed, GPU_COUNT, GPU)) + [named(n, GPU) for n in GPU_NAMED]
    return _sets[("gpu", seed)]


def ab_arrays(seed, ks):
    """Cases `ks` of the GPU set through the compositor: the pano, its mask, every warped image and mask by name."""
    cs = gpu_set(seed)
    out = {}
    for k in ks:
        c = cs[k]
        got = fuzz_chain.compositor_run(c, images(c), extras(c))
        out[f"{k}_pano"], out[f"{k}_pmask"] = got["pano"], got["pmask"]
        for i in range(c.n):
            out[f"{k}_w{i}"], out[f"{k}_m{i}"] = got["warped"][i], got["masks"][i]
    return out


def emu_coverage(case):
    lanes, blocks = "SB_EMU_LANES" in case.env, "SB_EMU_BLOCKS" in case.env
    return coverage(case, pyr_fast=lanes, tile=blocks, dt_fast=lanes)


def redraw_share(cs):
    """Rejected draws per accepted case: kept small, or the budget has silently reshaped the distribution."""
    return sum(c.redraws for c in cs) / max(1, len(cs))


# -- the oracle side ----------------------------------------------------------------------------------------------------
def oracle_run(O, case, imgs, ex, s16=False, crop=None):
    """fuzz_chain.oracle_image per image, sliced by `crop`'s rects when given, then oracle_blend at the warped corners
    and sizes or at the crop's corners and prepared sizes.  `rects` are the fed ones (corner, fed size), `raw` holds the
    warped images and masks before slice and compensation; s16: also the blend's int16 result ("pano16")."""
    scale = case.scale()
    slices = crop.rects if crop is not None else [None] * case.n
    raw, warped, masks, rects = [], [], [], []
    for img, cam, sl, (mask, seam, gain) in zip(imgs, case.cams, slices, ex):
        (rect, ri, rm), wi, wm = fuzz_chain.oracle_image(O, case.wtype, scale, Warper.get_K(cam, 1), cam.R, img, sl, gain,
                                                         mask, seam)
        raw.append((ri, rm))
        warped.append(wi)
        masks.append(wm)
        rects.append(rect)
    corners, sizes = (crop.corners, crop.sizes) if crop is not None else ([r[:2] for r in rects], [r[2:] for r in rects])
    b, pano16, pmask = fuzz_chain.oracle_blend(O, case.blender, case.strength, corners, sizes, warped, masks)
    return dict(warped=warped, masks=masks, rects=[tuple(c) + (wi.shape[1], wi.shape[0]) for c, wi in zip(corners, warped)],
                roi=b.roi, num_bands=b.num_bands if b._kind == "multiband" else -1, pano=O.convert_scale_abs(pano16),
                pmask=pmask, raw=raw, pano16=pano16 if s16 else None)


def check(case, got, ref, seed):
    """Bit for bit: rects, pano roi, num_bands (-1: not multiband), every warped image and mask, pano and its mask."""
    import replay

    where = f"seed {seed}, {case.describe()}"
    assert [tuple(r) for r in got["rects"]] == [tuple(r) for r in ref["rects"]], f"{where}: rects"
    assert tuple(got["roi"]) == tuple(ref["roi"]), f"{where}: pano roi {got['roi']} != {ref['roi']}"
    assert got["num_bands"] == ref["num_bands"], f"{where}: num_bands {got['num_bands']} != {ref['num_bands']}"
    for i in range(case.n):
        replay.assert_exact(got["warped"][i], ref["warped"][i], f"{where}: warped image {i}")
        replay.assert_exact(got["masks"][i], ref["masks"][i], f"{where}: warped mask {i}")
    replay.assert_exact(got["pano"], ref["pano"], f"{where}: pano")
    replay.assert_exact(got["pmask"], ref["pmask"], f"{where}: pano mask")


# -- coverage accounting ------------------------------------------------------------------------------------------------
def plan(case):
    """Blend kind, band count and the padded feed rects of a case's rects (fuzz_chain.blend_geometry)."""
    g = fuzz_chain.blend_geometry([r[:2] for r in case.rects], [r[2:] for r in case.rects], case.blender, case.strength)
    return g.kind, g.nb, g.feeds


def _z_nonpositive(case):
    """Whether some pixel of a warped rect maps back to a ray with z <= 0 (the table projections of k_warp_rgbm)."""
    if case.wtype not in ("spherical", "cylindrical", "plane"):
        return False
    s = float(case.scale())
    for cam, (rx, ry, rw, rh) in zip(case.cams, case.rects):
        kr = Warper.get_K(cam, 1).astype(np.float64) @ np.linalg.inv(cam.R.astype(np.float64))
        u = (rx + np.arange(rw)) / s
        v = (ry + np.arange(rh)) / s
        if case.wtype == "spherical":
            a = np.sin(np.pi - v)[:, None]
            X, Y, Z = a * np.sin(u)[None, :], np.cos(np.pi - v)[:, None] + 0 * u[None, :], a * np.cos(u)[None, :]
        elif case.wtype == "cylindrical":
            X, Y, Z = np.sin(u)[None, :] + 0 * v[:, None], v[:, None] + 0 * u[None, :], np.cos(u)[None, :] + 0 * v[:, None]
        else:
            X, Y, Z = u[None, :] + 0 * v[:, None], v[:, None] + 0 * u[None, :], np.ones((rh, rw))
        if ((kr[2, 0] * X + kr[2, 1] * Y + kr[2, 2] * Z) <= 0).any():
            return True
    return False


def coverage(case, pyr_fast=True, tile=True, dt_fast=True, pd_bin=True):
    """The kernels and branches a case reaches, from its geometry: `pyr_fast` / `tile` / `dt_fast` say whether the
    shuffle pyrDown, the tile collapse and the fast distance transform run in this build (always on the GPU; in the
    emulation build the first and the last only under SB_EMU_LANES, the tile collapse only under SB_EMU_BLOCKS)."""
    tags = set()
    kind, nb, padded = plan(case)
    tags.add(kind)
    if case.blender != "no" and kind == "no":
        tags.add("blend width < 1")
    if kind == "multiband":
        tags.add("nb=0" if nb == 0 else "nb=1" if nb == 1 else "nb>=2")
    x, y, w, h = case.roi()
    if w % 2:
        tags.add("odd pano width")
    if case.n > WARP_BATCH:
        tags.add("n>32")
    if _z_nonpositive(case):
        tags.add("z<=0")
    # launch_warp: maps or a 1-px source take k_warp_wide; else k_warp_rgbm<HAS_BM, ...>
    has_bm = any(m != "none" or g != "none" for m, g in zip(case.masks, case.gains))
    tags.add("k_warp_wide" if case.wtype in MAP_TYPES else f"k_warp_rgbm<HAS_BM={int(has_bm)}>")
    if case.wtype in MAP_TYPES:
        tags.add("map projection")
    kinds = {(m, g) for m, g in zip(case.masks, case.gains)}
    if len(kinds) >= 3 and ("none", "none") in kinds:
        tags.add("mixed extras")
    if any(m in ("ramp", "random", "seam") for m in case.masks):
        tags.add("gray blend mask")
    if any(s[0] == 2 for s in case.sizes):
        tags.add("2-px source")
    binary = pd_bin and all(m == "none" for m in case.masks)  # use_blend_mask: set_mask / set_seam_mask turn it off
    if kind == "multiband" and pyr_fast:
        for l in range(nb):  # launch_pyrdown_fast
            near = all((p["ph"] >> l) >= 4 for p in padded)
            if l == 0:
                near = near and all(p["top"] <= p["h"] and p["ph"] - p["top"] - p["h"] <= p["h"] for p in padded)
            if l == 0:
                inst = (1, int(near), int(binary))
            elif l <= 2 and binary and near:
                inst = (0, 1, 1)
            else:
                inst = (0, int(near), 0)
            tags.add("k_pyrdown_walk<%d,%d,%d>" % inst)
    if kind == "multiband" and tile and nb >= 1:
        # tile_images_ok (BlendPlan) holds for every compositor; launch_collapse_tile at level 0 wants even output
        # pitches: 3 * pano width and the mask pitch
        tags.add("tile l0 yes" if w % 2 == 0 else "tile l0 no")
        if nb >= 2:
            tags.add("tile l1 yes")
        # the coarse windows a tile level stages (level l + 1 of each image and of the pano) one element across:
        # fix_borders' reflect-101 of a 1-px level
        for up in [l + 1 for l in (0, 1) if l < nb and (l == 1 or w % 2 == 0)]:
            if any(p["pw"] >> up == 1 for p in padded) or -(-w // (1 << nb)) * (1 << nb) >> up == 1:
                tags.add("tile coarse 1 px wide")
            if any(p["ph"] >> up == 1 for p in padded) or -(-h // (1 << nb)) * (1 << nb) >> up == 1:
                tags.add("tile coarse 1 px high")
    if kind == "feather" and max(r[2] for r in case.rects) > 8192:
        tags.add("feather w>8192")
        if dt_fast:
            tags.add("k_dt_rows_warp")
    # gain_upload: a map with a side of 1 takes OpenCV's own resize taps (gain_mode 3), as cv::resize does
    for _, _, g in extras(case):
        if g is not None and g.dtype == np.float32 and 1 in g.shape[:2]:
            gh, gw = g.shape[:2]
            tags.add("gain map 1x1" if gh == gw else "gain map 1 px wide" if gw == 1 else "gain map 1 px high")
    return tags


PYRDOWN_INSTANCES = ["k_pyrdown_walk<%d,%d,%d>" % t for t in ((1, 1, 1), (1, 0, 1), (1, 1, 0), (1, 0, 0), (0, 1, 1), (0, 1, 0), (0, 0, 0))]


def coverage_table(rows):
    """rows: [(case, tags)] -> printable table of how many cases reached each tag."""
    counts = {}
    for _, tags in rows:
        for t in tags:
            counts[t] = counts.get(t, 0) + 1
    width = max(len(t) for t in counts) if counts else 10
    return "\n".join(f"  {t:<{width}}  {counts[t]:4d}" for t in sorted(counts))
