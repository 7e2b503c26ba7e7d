"""Seeded random rigs for the sharded composite against an oracle that sums in the ranks' groups (helper module: no
tests in here).

The sharded composite (sb_shard.cpp, DESIGN §7) deals the images to `world` ranks in contiguous blocks and cuts the
panorama into strips, one per rank.  The owner of a strip adds, per level and pixel: the partial sums (slabs) of the
lower ranks, its own images one at a time, then the slabs of the higher ranks; each slab is a sum that starts at 0.  The
int16 sums are exact under any grouping, the float weight sums are not, so the single-GPU oracle is not the right
yardstick.  grouped_oracle() restates the owner's grouping with oracle.Blender.fold, which makes the comparison exact.

cases(seed, count, budget) yields ShardCase records (rig_fuzz.Case plus `world`): yaw rings on four projections,
left-to-right affine strips with three or more images per pixel, one huge image spanning other ranks' strips, clustered
blocks whose strip bounds snap to the same lattice column, feather rings and stacked feather grids in both directions,
and per-image extras mixed within a rig.  geometry(case) restates the strip bounds and slab extents from the rig alone;
coverage(case) turns them into tags a test can count.

SB_SHARD_FUZZ_SEED=<int> or =random replaces the fixed default seed (the seed used is printed).
"""
import dataclasses
import functools
import math
from statistics import median

import numpy as np

import fuzz_chain
import rig_fuzz
from stitching_b200 import rigs
from stitching_b200.warper import Warper

DEFAULT_SEED = 20261016
EMU = dict(side=48, area=2_600)           # emulation build: serial CPU stand-in for the device
GPU = dict(side=400, area=160_000)        # H100: the oracle (scalar C on the CPU, world + 1 blenders) sets the cost
WORLDS = (2, 3, 4, 5, 8)


seed_from_env = functools.partial(fuzz_chain.seed_from_env, "SB_SHARD_FUZZ_SEED", DEFAULT_SEED)


@dataclasses.dataclass
class ShardCase(rig_fuzz.Case):
    world: int = 2
    layout: str = ""

    def describe(self):
        return f"{rig_fuzz.Case.describe(self)} world={self.world} layout={self.layout}"


def block_of(n, world, r):
    """ShardPlan::block_of: rank r owns images [first, first + count)."""
    first = r * n // world
    return first, (r + 1) * n // world - first


def rank_of(n, world, i):
    return next(r for r in range(world) if block_of(n, world, r)[0] <= i < sum(block_of(n, world, r)))


# -- drawing ----------------------------------------------------------------------------------------------------------
def _ring_cams(rng, sizes, sign=1):
    """A yaw ring with overlap between neighbours, random step and jitter, never closing on itself."""
    n = len(sizes)
    f = median(max(w, h) for w, h in sizes) * rng.uniform(0.7, 2.0)
    fov = math.degrees(2 * math.atan(median(w for w, _ in sizes) / (2 * f)))
    step = min(fov * rng.uniform(0.3, 0.9), 280.0 / n)
    cams = []
    for i, (w, h) in enumerate(sizes):
        yaw = np.deg2rad(sign * step * (i - (n - 1) / 2) + rng.uniform(-0.15, 0.15) * step)
        R = rigs.rot_y(yaw) @ rigs.rot_x(rng.uniform(-0.1, 0.1))
        cams.append(rigs.Camera(f * rng.uniform(0.97, 1.03), 1.0, w / 2 + rng.uniform(-2, 2), h / 2 + rng.uniform(-2, 2),
                                R.astype(np.float32)))
    return cams


def _affine(th, sx, sy, sh, tx, ty):
    """An affine camera whose warped image lies near (tx, ty) (the affine warper applies the camera's inverse)."""
    A = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]) @ np.array([[sx, sh], [0, sy]])
    t = -A @ np.array([tx, ty])
    return rigs.Camera(1.0, 1.0, 0.0, 0.0, np.array([[A[0, 0], A[0, 1], t[0]], [A[1, 0], A[1, 1], t[1]], [0, 0, 1]], np.float32))


def _at(cam):
    """(tx, ty) of an _affine camera."""
    A = cam.R[:2, :2].astype(np.float64)
    return -np.linalg.solve(A, cam.R[:2, 2].astype(np.float64))


def _strip_cams(rng, sizes, advance, sign=1):
    """Affine images along x; each starts `advance` (share of the previous width) further on: 0.3 -> 3+ per pixel."""
    cams, x = [], 0.0
    for w, h in sizes:
        sx, sy = rng.uniform(0.8, 1.25), rng.uniform(0.8, 1.25)
        tx = sign * x + (-w * sx if sign < 0 else 0) + rng.uniform(0, 3) + rng.random()
        cams.append(_affine(rng.uniform(-0.15, 0.15), sx, sy, rng.uniform(-0.2, 0.2), tx, rng.uniform(0, 12) + rng.random()))
        x += advance * w * sx
    return cams


def _grid_cams(rng, n, world, sizes, sign=1):
    """Feather grid: rank r's block is one row; rows run down (sign 1) or up (sign -1) the panorama."""
    cams = []
    rh = max(h for _, h in sizes) * 0.7
    for i, (w, h) in enumerate(sizes):
        r = rank_of(n, world, i)
        k = i - block_of(n, world, r)[0]
        row = r if sign > 0 else world - 1 - r
        cams.append(_affine(rng.uniform(-0.05, 0.05), 1.0, 1.0, 0.0, k * 0.7 * w + rng.uniform(0, 3) + rng.random(),
                            row * rh + rng.uniform(0, 3) + rng.random()))
    return cams


def _sizes(rng, n, side):
    """Mostly ordinary sources (odd sizes mixed in), a few flat or thin ones."""
    out = []
    for _ in range(n):
        w, h = int(rng.integers(side // 3, side + 1)), int(rng.integers(side // 3, side + 1))
        u = rng.random()
        if u < 0.06:
            h = int(rng.integers(2, 6))
        elif u < 0.1:
            w = int(rng.integers(2, 6))
        out.append((max(2, w), max(2, h)))
    return out


def _extras(rng, n):
    mode = rng.random()
    if mode < 0.35:
        return ["none"] * n, ["none"] * n
    if mode < 0.5:
        return [str(rng.choice(rig_fuzz.MASK_KINDS))] * n, [str(rng.choice(rig_fuzz.GAIN_KINDS))] * n
    return ([str(rng.choice(rig_fuzz.MASK_KINDS)) for _ in range(n)], [str(rng.choice(rig_fuzz.GAIN_KINDS)) for _ in range(n)])


def _mb_strength(rng, rects):
    """A multiband strength aimed at nb = 1, 2, an intermediate count or the clipped maximum (never 0: the sharded
    composite needs a band)."""
    _, _, w, h = fuzz_chain.blend_geometry([r[:2] for r in rects], [r[2:] for r in rects]).roi
    if rng.random() < 0.15:
        return 400.0                                                # past the clip at ceil(log2(max side))
    nb = int(rng.choice([1, 1, 2, 2, 3, 4, 5]))
    return rig_fuzz._quant(max(1 / 256, 2.0 ** (nb + 1 + rng.uniform(0.1, 0.9)) * 100 / math.sqrt(w * h)))


LAYOUTS_MB = ("ring", "ring", "strip", "strip", "huge", "cluster")
LAYOUTS_FEATHER = ("ring", "ring_rtl", "grid_down", "grid_up")


def _draw(rng, budget, index, seed):
    side = budget["side"]
    world = int(rng.choice(WORLDS))
    u = rng.random()
    n = world if u < 0.15 else int(rng.integers(world, 5 * world + 1))
    if u > 0.85 and n % world == 0:
        n += 1
    multiband = rng.random() < 0.7
    layout = str(rng.choice(LAYOUTS_MB if multiband else LAYOUTS_FEATHER))
    sizes = _sizes(rng, n, side)
    wtype = "affine"
    if layout == "ring":
        wtype = str(rng.choice(["spherical", "cylindrical", "mercator", str(rng.choice(rig_fuzz.MAP_TYPES))]))
        cams = _ring_cams(rng, sizes)
    elif layout == "ring_rtl":
        wtype = str(rng.choice(["spherical", "cylindrical"]))
        cams = _ring_cams(rng, sizes, -1)
    elif layout == "strip":
        cams = _strip_cams(rng, sizes, rng.uniform(0.15, 0.35))
    elif layout == "huge":
        cams = _strip_cams(rng, sizes, rng.uniform(0.3, 0.6))
        k = int(rng.integers(0, n))
        sizes[k] = (max(4, side // 3), max(4, side // 3))
        s = rng.uniform(2.5, 4.0) * side / sizes[k][0]
        tx, ty = _at(cams[k])
        cams[k] = _affine(0.0, s, s * rng.uniform(0.5, 1.0), 0.0, tx - side * rng.uniform(0, 1.5), ty)
    elif layout == "cluster":
        # one middle block piled onto a single spot between its neighbours: its two strip bounds snap to one column
        cams = _strip_cams(rng, sizes, rng.uniform(0.3, 0.6))
        if world >= 3:
            r = int(rng.integers(1, world - 1))
            f0, fc = block_of(n, world, r)
            x = _at(cams[f0])[0]
            nxt = _at(cams[f0 + fc])[0] if f0 + fc < n else 0.0
            for i in range(f0, f0 + fc):
                sizes[i] = (int(rng.integers(3, 7)), sizes[i][1])
                cams[i] = _affine(0.0, 1.0, 1.0, 0.0, x + rng.uniform(0, 2), _at(cams[i])[1])
            for i in range(f0 + fc, n):  # the rest follows right after the pile
                tx, ty = _at(cams[i])
                cams[i] = _affine(0.0, 1.0, 1.0, 0.0, tx - nxt + x + 4, ty)
    else:
        cams = _grid_cams(rng, n, world, sizes, 1 if layout == "grid_down" else -1)
    masks, gains = _extras(rng, n)
    gens = [str(rng.choice(["noise", "noise", "synth", "const"])) for _ in range(n)]
    return ShardCase(f"case_{index}", wtype, cams, sizes, "multiband" if multiband else "feather", 0.0, masks, gains, gens,
                     seed * 7919 + index, world=world, layout=layout)


def _fits(case, budget):
    area = sum(r[2] * r[3] for r in case.rects)
    return (all(r[2] > 0 and r[3] > 0 and r[2] * r[3] <= budget["area"] for r in case.rects)
            and area <= 12 * budget["area"] and case.roi()[2] <= 40 * budget["side"])


def _finish(case, rng):
    if case.blender == "multiband":
        case.strength = _mb_strength(rng, case.rects)
    else:
        case.strength = float(rng.choice([5, 20, 60, 100]))
    return case


def cases(seed, count, budget):
    """`count` seeded cases that fit `budget` and that the sharded composite accepts (blocks in order, a band or the
    feather blender with a blend width of at least 1); each carries the number of rejected draws before it."""
    rng = np.random.default_rng(seed)
    for index in range(count):
        redraws = 0
        while True:
            c = _draw(rng, budget, index, seed)
            c.rects = rig_fuzz._rects(c.wtype, c.cams, c.sizes)
            if _fits(c, budget):
                _finish(c, rng)
                if geometry(c)["ok"]:
                    break
            redraws += 1
        c.redraws = redraws
        yield c


def raw_draws(seed, count, budget):
    """Draws as they come (also those the sharded composite must reject), for the order predicate's test."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        c = _draw(rng, budget, len(out), seed)
        c.rects = rig_fuzz._rects(c.wtype, c.cams, c.sizes)
        if _fits(c, budget):
            out.append(_finish(c, rng))
    return out


def named(name, budget=None):
    """Cases kept by name (the same rig for every budget)."""
    if name == "grouped_differs":
        # found by searching seeded rigs with the oracle alone (gray masks, about seven images on each pixel, four
        # ranks): the grouped float weight sums round three values of the panorama differently from the single-GPU order
        n, world, side = 23, 4, 116
        sizes = [(side, side)] * n
        cams = _strip_cams(np.random.default_rng(15), sizes, 0.13854914882478564)
        c = ShardCase(name, "affine", cams, sizes, "multiband", 1.18359375, ["random"] * n, ["none"] * n, ["noise"] * n, 15,
                      world=world, layout="strip")
    elif name == "lower_slabs_first":
        # found the same way: the owner's grouping (lower ranks' slabs, own images, higher ranks' slabs) and the owner's
        # own images first, then all slabs, give five different values in the strips of ranks 1 and 2
        n, world, side = 24, 3, 80
        sizes = [(side, side)] * n
        cams = _strip_cams(np.random.default_rng(52), sizes, 0.16832240846228785)
        c = ShardCase(name, "affine", cams, sizes, "multiband", 1.48046875, ["random"] * n, ["none"] * n, ["noise"] * n, 52,
                      world=world, layout="strip")
    elif name == "right_to_left":
        # multiband image blocks that run right to left: ShardPlan::build must refuse them
        n, world = 9, 3
        sizes = [(40, 36)] * n
        cams = _strip_cams(np.random.default_rng(5), sizes, 0.5, -1)
        c = ShardCase(name, "affine", cams, sizes, "multiband", 0.0, ["none"] * n, ["none"] * n, ["noise"] * n, 22,
                      world=world, layout="strip_rtl")
    else:
        raise KeyError(name)
    c.rects = rig_fuzz._rects(c.wtype, c.cams, c.sizes)
    if c.strength == 0.0:
        x0, y0, w, h = c.roi()
        c.strength = rig_fuzz._quant(2.0 ** 3.5 * 100 / math.sqrt(w * h))  # two bands
    return c


# -- the geometry, restated from the library's ShardPlan --------------------------------------------------------------
def geometry(case):
    """Strip geometry of every rank, restated from the rig: dict(ok, kind, nb, axis, reversed, bounds, strips, empty,
    slab_levels (levels at which some slab is non-empty), has_slabs[r][l] (rank r receives a slab at level l))."""
    bg = case.geometry()
    kind, nb = bg.kind, bg.nb
    n, world = case.n, case.world
    x, y, w, h = bg.roi
    g = dict(kind=kind, nb=nb, axis=0, reversed=False, ok=n >= world and (kind == "feather" or (kind == "multiband" and nb >= 1)))
    if not g["ok"]:
        return g
    blocks = [block_of(n, world, r) for r in range(world)]
    if kind == "multiband":
        imgs, (wp, hp) = bg.feeds, bg.padded
        a = 1 << nb
        snapped = []
        for r in range(1, world):
            L, R = imgs[sum(blocks[r - 1]) - 1], imgs[blocks[r][0]]
            mid = (L["dx"] + L["w"] // 2 + R["dx"] + R["w"] // 2) // 2
            snapped.append(min((mid + a // 2) // a * a, wp))
        g["ok"] = all(b >= a_ for a_, b in zip(snapped, snapped[1:]))  # blocks left to right (equal: an empty strip)
        bounds = [0] + snapped + [wp]
        g["bounds"] = bounds
        g["strips"] = [(min(bounds[r], w), min(bounds[r + 1], w)) for r in range(world)]

        def region(r, l):
            if l == 0:
                lo, hi = bounds[r], min(bounds[r + 1], (w + 1) // 2 * 2)
            else:
                lo, hi = max(0, (bounds[r] >> l) - 2), min(wp >> l, (bounds[r + 1] >> l) + 2)
            return lo, max(lo, hi)

        def slab(src, dst, l):
            f0, fc = blocks[src]
            even = ~1 if l < nb else ~0
            fx0 = fy0 = 1 << 30
            fx1 = fy1 = -1
            for im in imgs[f0: f0 + fc]:
                X0, Y0 = im["px"] + im["left"], im["py"] + im["top"]
                X1, Y1 = X0 + im["w"], Y0 + im["h"]
                fx0 = min(fx0, max(im["px"] >> l, ((X0 >> l) - 3) & even))
                fy0 = min(fy0, max(im["py"] >> l, ((Y0 >> l) - 3) & even))
                fx1 = max(fx1, min((im["px"] + im["pw"]) >> l, ((((X1 - 1) >> l) + 4) + 1) & even))
                fy1 = max(fy1, min((im["py"] + im["ph"]) >> l, ((((Y1 - 1) >> l) + 4) + 1) & even))
            lo, hi = region(dst, l)
            return fc > 0 and min(hi, fx1) > max(lo, fx0) and fy1 > fy0

        g["has_slabs"] = [[any(slab(p, r, l) for p in range(world) if p != r) for l in range(nb + 1)] for r in range(world)]
        g["region"] = region
    else:
        lo_x, hi_x, lo_y, hi_y = [], [], [], []
        for f0, fc in blocks:
            rs = case.rects[f0: f0 + fc]
            lo_x.append(min(r[0] - x for r in rs))
            hi_x.append(max(r[0] - x + r[2] for r in rs))
            lo_y.append(min(r[1] - y for r in rs))
            hi_y.append(max(r[1] - y + r[3] for r in rs))
        cx = [0.5 * (a + b) for a, b in zip(lo_x, hi_x)]
        cy = [0.5 * (a + b) for a, b in zip(lo_y, hi_y)]
        inc_x = all(cx[r] > cx[r - 1] for r in range(1, world))
        dec_x = all(cx[r] < cx[r - 1] for r in range(1, world))
        inc_y = all(cy[r] > cy[r - 1] for r in range(1, world))
        dec_y = all(cy[r] < cy[r - 1] for r in range(1, world))
        mono_x, mono_y = inc_x or dec_x, inc_y or dec_y
        g["ok"] = mono_x or mono_y
        if not g["ok"]:
            return g
        axis = 1 if mono_y and (not mono_x or abs(cy[-1] - cy[0]) > abs(cx[-1] - cx[0])) else 0
        rev = not inc_x if axis == 0 else not inc_y
        extent = w if axis == 0 else h
        lo, hi = (lo_x, hi_x) if axis == 0 else (lo_y, hi_y)
        bounds = [0] * (world + 1)
        bounds[world] = extent
        for q in range(1, world):
            ra, rb = (world - q, world - 1 - q) if rev else (q - 1, q)
            bounds[q] = min(max((hi[ra] + lo[rb]) // 2, bounds[q - 1]), extent)
        place = [world - 1 - r if rev else r for r in range(world)]
        g.update(axis=axis, reversed=rev, bounds=bounds,
                 strips=[(min(bounds[place[r]], extent), min(bounds[place[r] + 1], extent)) for r in range(world)])

        def fslab(src, dst):
            q = place[dst]
            a0, a1 = max(lo[src], bounds[q]), min(hi[src], bounds[q + 1])
            o = (lo_y, hi_y) if axis == 0 else (lo_x, hi_x)
            return blocks[src][1] > 0 and a1 > a0 and o[1][src] > o[0][src]

        g["has_slabs"] = [[any(fslab(p, r) for p in range(world) if p != r)] for r in range(world)]
    g["empty"] = [a == b for a, b in g["strips"]]
    return g


def _ranks_per_pixel(case):
    x, y, w, h = case.roi()
    cnt = np.zeros((h, w), np.int16)
    for r in range(case.world):
        f0, fc = block_of(case.n, case.world, r)
        m = np.zeros((h, w), bool)
        for rx, ry, rw, rh in case.rects[f0: f0 + fc]:
            m[ry - y: ry - y + rh, rx - x: rx - x + rw] = True
        cnt += m
    return int(cnt.max())


def coverage(case, tile=True):
    """Tags of what a case reaches, from its geometry alone; `tile`: whether the tile collapse runs in this build (always
    on the GPU, under SB_EMU_BLOCKS in the emulation build)."""
    g = geometry(case)
    tags = {f"world={case.world}", case.blender, f"layout {case.layout}"}
    if not g["ok"]:
        tags.add("rejected")
        return tags
    n, world = case.n, case.world
    if n == world:
        tags.add("n == world")
    if n % world:
        tags.add("n % world != 0")
    x, y, w, h = case.roi()
    if w % 2:
        tags.add("odd pano width")
    if any(g["empty"]):
        tags.add("empty strip")
    tags.add(("row" if g["axis"] else "column") + " strips" + (" reversed" if g["reversed"] else ""))
    if _ranks_per_pixel(case) >= 3:
        tags.add("3+ ranks in a pixel")
    if any(m in ("ramp", "random", "seam") for m in case.masks):
        tags.add("gray blend mask")
    kinds = {(m, gk) for m, gk in zip(case.masks, case.gains)}
    if len(kinds) >= 3 and ("none", "none") in kinds:
        tags.add("mixed extras")
    if case.wtype in rig_fuzz.MAP_TYPES:
        tags.add("map projection")
    if g["kind"] == "multiband":
        nb = g["nb"]
        clipped = int(math.ceil(math.log(max(w, h)) / math.log(2.0)))
        tags.add("nb=1" if nb == 1 else "nb=max" if nb == clipped else "nb=2.." if nb >= 2 else "")
        if w % (1 << nb):
            tags.add("roi.w % 2^nb != 0")
        levels = {l for r in range(world) for l in range(nb + 1) if g["has_slabs"][r][l]}
        for l in levels:
            tags.add("slab at l0" if l == 0 else "slab at l1" if l == 1 else "slab at l>=2")
        if tile:
            for r in range(world):
                lo, hi = g["strips"][r]
                a, b = g["region"](r, 0)
                if g["has_slabs"][r][0] and (hi - lo) % 2 == 0 and b > a:
                    tags.add("tile l0 with slab items")
                if nb >= 2 and g["has_slabs"][r][1]:
                    tags.add("tile l1 with slab items")
    tags.discard("")
    return tags


# -- the oracle side ----------------------------------------------------------------------------------------------------
def grouped_oracle(O, case, imgs, ex, world=None):
    """What every rank computes: per rank r, a blender that folds in the blocks of the lower ranks (each fed on its
    own, from 0), is fed r's images one at a time, folds in the blocks of the higher ranks, and blends.  Returns the
    warped images and masks, rects, roi, num_bands, and per rank the WHOLE blended panorama and mask (the rank keeps
    its strip of it, the test slices)."""
    world = case.world if world is None else world
    scale = case.scale()
    rects, warped, masks = [], [], []
    for img, cam, (mask, seam, gain) in zip(imgs, case.cams, ex):
        (rect, _, _), wi, wm = fuzz_chain.oracle_image(O, case.wtype, scale, Warper.get_K(cam, 1), cam.R, img, None, gain,
                                                       mask, seam)
        rects.append(tuple(rect))
        warped.append(wi)
        masks.append(wm)
    b0, panos = grouped_blend(O, case.blender, case.strength, [r[:2] for r in rects], warped, masks, world)
    return dict(warped=warped, masks=masks, rects=rects, roi=b0.roi, num_bands=b0.num_bands if b0._kind == "multiband" else -1,
                panos=panos)


def grouped_blend(O, kind, strength, corners, imgs, masks, world):
    """Blender.prepare / feed / blend in the ranks' groups -> (a prepared blender, [(pano, mask) per rank])."""
    n = len(imgs)
    sizes = [(m.shape[1], m.shape[0]) for m in masks]

    def blender():
        b = O.Blender(kind, strength)
        b.prepare(corners, sizes)
        return b

    blocks = [block_of(n, world, r) for r in range(world)]
    part = []
    for f0, fc in blocks:
        b = blender()
        for i in range(f0, f0 + fc):
            b.feed(imgs[i], masks[i], corners[i])
        part.append(b)
    panos = []
    for r, (f0, fc) in enumerate(blocks):
        d = blender()
        for p in range(r):
            d.fold(part[p])
        for i in range(f0, f0 + fc):
            d.feed(imgs[i], masks[i], corners[i])
        for p in range(r + 1, world):
            d.fold(part[p])
        panos.append(d.blend())
    return part[0], panos


def config_case(cfg, world, cams=None):
    """A ShardCase for one of the fixed rigs of stitching_b200.rigs.config (no extras)."""
    cams = cfg["cameras"] if cams is None else cams
    n = len(cams)
    c = ShardCase("config", cfg["warper"], cams, [(cfg["w"], cfg["h"])] * n, cfg["blender"], float(cfg["strength"]),
                  ["none"] * n, ["none"] * n, ["noise"] * n, 0, world=world, layout="config")
    c.rects = rig_fuzz._rects(c.wtype, c.cams, c.sizes)
    return c


def grouped_panorama(O, case, imgs):
    """The grouped oracle's strips put together in spatial order: (panorama, mask, num_bands) of what the ranks compute
    together (num_bands -1: not multiband)."""
    ref = grouped_oracle(O, case, imgs, [(None, None, None)] * case.n)
    g = geometry(case)
    order = sorted(range(case.world), key=lambda r: g["strips"][r])
    ax = 1 if g["axis"] == 0 else 0
    return (np.concatenate([cut(ref["panos"][r][0], g["strips"][r], g["axis"]) for r in order], axis=ax),
            np.concatenate([cut(ref["panos"][r][1], g["strips"][r], g["axis"]) for r in order], axis=ax), ref["num_bands"])


def plain_oracle(O, case, imgs, ex):
    return rig_fuzz.oracle_run(O, case, imgs, ex)


def cut(a, strip, axis):
    return a[:, strip[0]: strip[1]] if axis == 0 else a[strip[0]: strip[1]]


# -- the product side ---------------------------------------------------------------------------------------------------
def hooks_run(case, imgs, ex, copy, **compositor_kwargs):
    """All ranks in this process (Compositor keywords `compositor_kwargs`: crop, input_sizes): each sets the extras of
    its own images, uploads its block and runs phase 0; the slabs are moved with `copy(dst, src, bytes)`; phase 1;
    strips and own warped images are downloaded."""
    from stitching_b200 import Compositor

    ranks = []
    try:
        for r in range(case.world):
            ranks.append(Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength, rank=r, world=case.world,
                                    **compositor_kwargs))
        for c in ranks:
            fuzz_chain.set_extras(c, ex, range(c.first, c.first + c.count))
            c.upload(imgs[c.first: c.first + c.count])
            c.shard_phase(0)
        sizes = {}
        for src in ranks:
            for dst in ranks:
                if src is dst:
                    continue
                sp, sn = src.shard_slab(dst.rank, True)
                dp, dn = dst.shard_slab(src.rank, False)
                sizes[(src.rank, dst.rank)] = (sn, dn)
                if sn and sn == dn:
                    copy(dp, sp, sn)
        out = []
        for c in ranks:
            c.shard_phase(1)
            pano, mask = c.download()
            warped = {i: c.download_warped(i) for i in range(c.first, c.first + c.count)}
            out.append(dict(rects=list(c.rects), roi=tuple(c.roi), num_bands=c.num_bands, first=c.first, count=c.count,
                            strip=tuple(c.strip), axis=c.strip_axis, pano=pano, pmask=mask, warped=warped))
        return out, sizes
    finally:
        for c in ranks:
            c.close()


def check(case, got, slab_sizes, ref, seed):
    """Every rank: rects, roi, num_bands, block, strip and strip axis as restated; slab sizes agree on both sides; own
    warped images and masks, the strip and its mask equal the grouped oracle's bit for bit."""
    import replay

    where = f"seed {seed}, {case.describe()}"
    g = geometry(case)
    for (s, d), (sn, dn) in slab_sizes.items():
        assert sn == dn, f"{where}: slab {s}->{d}: {sn} bytes sent, {dn} expected by the receiver"
    for r, rk in enumerate(got):
        at = f"{where}, rank {r}"
        assert [tuple(x) for x in rk["rects"]] == ref["rects"], f"{at}: rects"
        assert tuple(rk["roi"]) == tuple(ref["roi"]), f"{at}: roi {rk['roi']} != {ref['roi']}"
        assert rk["num_bands"] == ref["num_bands"], f"{at}: num_bands {rk['num_bands']} != {ref['num_bands']}"
        assert (rk["first"], rk["count"]) == block_of(case.n, case.world, r), f"{at}: image block"
        assert rk["axis"] == g["axis"], f"{at}: strip axis {rk['axis']} != {g['axis']}"
        assert rk["strip"] == g["strips"][r], f"{at}: strip {rk['strip']} != restated {g['strips'][r]}"
        for i, (wi, wm) in rk["warped"].items():
            replay.assert_exact(wi, ref["warped"][i], f"{at}: warped image {i}")
            replay.assert_exact(wm, ref["masks"][i], f"{at}: warped mask {i}")
        pano, pmask = ref["panos"][r]
        replay.assert_exact(rk["pano"], cut(pano, rk["strip"], rk["axis"]), f"{at}: strip {rk['strip']}")
        replay.assert_exact(rk["pmask"], cut(pmask, rk["strip"], rk["axis"]), f"{at}: strip mask")


def ab_arrays(seed, ks):
    """Cases `ks` of the GPU set, all ranks on this device: every rank's strip and its mask by name."""
    cs = gpu_set(seed)
    out = {}
    for k in ks:
        got, _ = hooks_run(cs[k], rig_fuzz.images(cs[k]), rig_fuzz.extras(cs[k]), fuzz_chain.device_copy)
        for r, g in enumerate(got):
            out[f"{k}_{r}_pano"], out[f"{k}_{r}_pmask"] = g["pano"], g["pmask"]
    return out


def assemble(got):
    """The strips of all ranks in spatial order -> the whole panorama and mask."""
    order = sorted(range(len(got)), key=lambda r: got[r]["strip"])
    ax = 1 if got[0]["axis"] == 0 else 0
    return (np.concatenate([got[r]["pano"] for r in order], axis=ax), np.concatenate([got[r]["pmask"] for r in order], axis=ax))


# -- the seeded sets of the test suite ----------------------------------------------------------------------------------
LANES, BLOCKS = rig_fuzz.LANES, rig_fuzz.BLOCKS
EMU_COUNT = 26
EMU_ENV = {3: LANES, 8: LANES, 13: LANES, 5: BLOCKS, 10: BLOCKS, 17: BLOCKS}   # case index -> emulation switch
EMU_NAMED = [("grouped_differs", {}), ("grouped_differs", BLOCKS), ("lower_slabs_first", {})]
GPU_COUNT = 60
GPU_NAMED = ["grouped_differs", "lower_slabs_first"]


def _env_name(env):
    return "" if not env else "-lanes" if env is LANES else "-blocks"


def emu_ids():
    return ([f"case_{k}{_env_name(EMU_ENV.get(k))}" for k in range(EMU_COUNT)] + [f"{n}{_env_name(e)}" for n, e in EMU_NAMED])


def gpu_ids():
    return [f"case_{k}" for k in range(GPU_COUNT)] + GPU_NAMED


_sets = {}


def emu_set(seed):
    if ("emu", seed) not in _sets:
        out = list(cases(seed, EMU_COUNT, EMU))
        for k, env in EMU_ENV.items():
            out[k].env = dict(env)
            out[k].name += _env_name(env)
        for name, env in EMU_NAMED:
            c = named(name, EMU)
            c.env = dict(env)
            c.name += _env_name(env)
            out.append(c)
        _sets[("emu", seed)] = out
    return _sets[("emu", seed)]


def gpu_set(seed):
    if ("gpu", seed) not in _sets:
        _sets[("gpu", seed)] = list(cases(seed, GPU_COUNT, GPU)) + [named(n, GPU) for n in GPU_NAMED]
    return _sets[("gpu", seed)]
