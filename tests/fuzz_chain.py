"""What every seeded fuzz set shares (helper module: no tests in here).

seed_from_env    the seed of a set: its fixed default, an integer or a fresh random draw.
oracle_image     one image through the Stitcher's FINAL chain on the CPU oracle; oracle_blend: the Blender after it.
set_extras       a case's per-image extras on a Compositor; compositor_run: one Compositor over a rig_fuzz case.
device_copy      the slab mover of the transport hooks with every rank on one GPU.
blend_geometry   the pano roi, blend kind, band count and padded feed rects the library derives from a rig.
draw_crop        the search for a random largest interior rectangle that leaves every image a non-empty slice.
ab_run           a function in child processes, with the library's defaults and under each A/B switch.
"""
import collections
import json
import math
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def seed_from_env(var, default):
    """$var=<int> or =random replaces the fixed default seed of a set (the seed used is printed)."""
    s = os.environ.get(var)
    if not s:
        return default
    seed = int(np.random.SeedSequence().entropy % (1 << 31)) if s == "random" else int(s)
    print(f"{var}={seed}")
    return seed


# -- the oracle side ----------------------------------------------------------------------------------------------------
def oracle_image(O, wtype, scale, K, R, img, slice=None, gain=None, mask=None, seam=None, want_mask=True):
    """One image in the Stitcher's order (warp_final_resolution, crop_final_resolution, compensate_exposure_errors,
    resize_seam_masks): warp; the crop's (x, y, w, h) as a numpy slice of the warped image and mask; the compensator's
    gain on the sliced image; blend mask = the caller's mask, or SeamFinder.resize(seam, sliced mask), or the sliced mask.
    Returns ((rect, warped image, warped mask) before the slice, fed image, blend mask)."""
    rect, wi, wm = O.warp(wtype, scale, K, R, img, want_mask=want_mask)
    raw = (rect, wi, wm)
    if slice is not None:
        x, y, w, h = slice
        wi = np.ascontiguousarray(wi[y:y + h, x:x + w])
        wm = np.ascontiguousarray(wm[y:y + h, x:x + w]) if want_mask else None
    if gain is not None:
        wi = O.gain_apply(wi, gain)
    if mask is not None:
        wm = mask
    elif seam is not None:
        wm = O.seam_resize(seam, wm)
    return raw, wi, wm


def oracle_blend(O, kind, strength, corners, sizes, imgs, masks):
    """Blender.prepare(corners, sizes), feed every image at its corner in order, blend -> (blender, int16 pano, mask)."""
    b = O.Blender(kind, strength)
    b.prepare(corners, sizes)
    for wi, wm, c in zip(imgs, masks, corners):
        b.feed(wi, wm, c)
    pano16, pmask = b.blend_s16()
    return b, pano16, pmask


# -- the product side ---------------------------------------------------------------------------------------------------
def set_extras(c, ex, images):
    """set_mask / set_seam_mask / set_gain of `ex` (per image (mask, seam, gain), None where absent) for `images`."""
    for i in images:
        mask, seam, gain = ex[i]
        if mask is not None:
            c.set_mask(i, mask)
        if seam is not None:
            c.set_seam_mask(i, seam)
        if gain is not None:
            c.set_gain(i, gain)


def compositor_run(case, imgs, ex, **compositor_kwargs):
    """A Compositor over a rig_fuzz case (with `compositor_kwargs`: crop, input_sizes), the extras set, one composite:
    rects, roi, num_bands, the pano and its mask, every warped image and mask."""
    from stitching_b200 import Compositor

    c = Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength, **compositor_kwargs)
    try:
        set_extras(c, ex, range(case.n))
        pano, pmask = c.composite(imgs)
        warped = [c.download_warped(i) for i in range(case.n)]
        return dict(rects=list(c.rects), roi=tuple(c.roi), num_bands=c.num_bands, pano=pano, pmask=pmask,
                    warped=[w for w, _ in warped], masks=[m for _, m in warped])
    finally:
        c.close()


def device_copy(dst, src, nbytes):
    """copy(dst, src, bytes) for shard_fuzz.hooks_run with all ranks on one GPU: sb_device_copy of a slab."""
    from stitching_b200 import _lib

    _lib.check(_lib.lib().sb_device_copy(dst, src, nbytes), "sb_device_copy")


# -- the blend geometry, restated from the library's plan ---------------------------------------------------------------
BlendGeometry = collections.namedtuple("BlendGeometry", "kind nb roi padded feeds")


def blend_geometry(corners, sizes, blender="no", strength=0.0):
    """What the library derives from the prepared corners and sizes: the pano roi (resultRoi); the blend kind and band
    count (derive_blend_params: a blend width under 1 px is the "no" blender; the count clipped at ceil(log2(max side))
    by BlendPlan::set_geometry; 0 when not multiband); and for multiband the pano size padded to 2^nb and per feed the
    padded rect of BlendPlan::add_feed: origin px, py and size pw, ph in the padded pano, the image's offset left, top
    inside it, its size w, h and its corner dx, dy in the pano."""
    x, y = min(c[0] for c in corners), min(c[1] for c in corners)
    w = max(c[0] + s[0] for c, s in zip(corners, sizes)) - x
    h = max(c[1] + s[1] for c, s in zip(corners, sizes)) - y
    roi = (x, y, w, h)
    bw = math.sqrt(w * h) * strength / 100.0
    if blender == "no" or bw < 1.0:
        return BlendGeometry("no", 0, roi, None, [])
    if blender == "feather":
        return BlendGeometry("feather", 0, roi, None, [])
    nb = min(int(math.log(bw) / math.log(2.0) - 1.0), int(math.ceil(math.log(max(w, h)) / math.log(2.0))))
    a, gap = 1 << nb, 3 << nb
    wp, hp = -(-w // a) * a, -(-h // a) * a
    feeds = []
    for (tx, ty), (fw, fh) in zip(corners, sizes):
        px0, py0 = max(x, tx - gap), max(y, ty - gap)
        px1, py1 = min(x + wp, tx + fw + gap), min(y + hp, ty + fh + gap)
        px0 = x + (((px0 - x) >> nb) << nb)
        py0 = y + (((py0 - y) >> nb) << nb)
        feeds.append(dict(px=px0 - x, py=py0 - y, pw=-(-(px1 - px0) // a) * a, ph=-(-(py1 - py0) // a) * a, left=tx - px0,
                          top=ty - py0, w=fw, h=fh, dx=tx - x, dy=ty - y))
    return BlendGeometry("multiband", nb, roi, (wp, hp), feeds)


# -- the crop search ----------------------------------------------------------------------------------------------------
def draw_crop(rng, case, aspect, frac_lo, frac_hi, tries=20, keep=None):
    """Up to `tries` draws of a LOW -> FINAL aspect (a float, or a tuple to choose one from per draw) and of a LIR
    spanning (< frac_lo, < frac_lo) to (> frac_hi, > frac_hi) of the LOW pano of `case`'s warped rects: the first crop
    whose every slice is non-empty and that `keep(crop case)` accepts, as a crop_fuzz.CropCase; None if none is."""
    import crop_fuzz
    from stitching_b200 import Crop

    for _ in range(tries):
        a = float(rng.choice(aspect)) if isinstance(aspect, tuple) else aspect
        frac = (rng.uniform(0, frac_lo), rng.uniform(0, frac_lo), rng.uniform(frac_hi, 1.0), rng.uniform(frac_hi, 1.0))
        cr = crop_fuzz.low_cropper(case.rects, a, frac)
        if cr is None:
            continue
        cc = crop_fuzz.CropCase(case, Crop.from_cropper(cr, a), a, cr)
        if all(w > 0 and h > 0 for _, _, w, h in cc.fed()) and (keep is None or keep(cc)):
            return cc
    return None


# -- A/B switches -------------------------------------------------------------------------------------------------------
_CHILD = """
import importlib, json, pickle, sys
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
from stitching_b200 import _lib
_lib.check(_lib.lib().sb_init(0), "sb_init")
mod, fn = sys.argv[2].split(":")
res = getattr(importlib.import_module(mod), fn)(*json.loads(sys.argv[3]))
with open(sys.argv[4], "wb") as f:
    pickle.dump(res, f)
"""


def _same(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return a == b


def ab_run(target, args, switches, seed_var=None, timeout=1800):
    """`module:function(*args)` (args: JSON) in a child process with the library's defaults, and once more per
    (name, value) of `switches`: the library reads each switch once per process.  Every child's environment holds no
    SB_* variable of this process but `seed_var`, plus its one switch.  The function returns a dict of arrays or of
    digests; every entry under a switch must equal the defaults' byte for byte.  Returns the defaults' result."""
    res = {}
    with tempfile.TemporaryDirectory() as d:
        for sw in [None] + list(switches):
            env = {k: v for k, v in os.environ.items() if not k.startswith("SB_") or k == seed_var}
            if sw:
                env[sw[0]] = sw[1]
            out = os.path.join(d, "result.pkl")
            subprocess.run([sys.executable, "-c", _CHILD, ROOT, target, json.dumps(args), out], env=env, check=True,
                           timeout=timeout)
            with open(out, "rb") as f:
                res[sw] = pickle.load(f)
    base = res.pop(None)
    for (key, val), got in res.items():
        assert got.keys() == base.keys(), f"{key}={val}: {sorted(got)} != {sorted(base)}"
        for name, a in got.items():
            assert _same(a, base[name]), f"{key}={val}: {name} differs"
    return base
