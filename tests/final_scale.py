"""Camera-resolution frames resized to FINAL on the compositor (helper module: no tests in here).

A Stitcher with final_megapix set resizes every camera frame to its FINAL size before the warp
(Images.resize_img_by_scaler: cv.resize INTER_LINEAR_EXACT).  Compositor(..., input_sizes=...) takes the camera frames
and does that resize on the device (k_resize_src).  Two kinds of draws check it:

Kernel draws.  Rigs of integer-translated identity homographies ("affine" warper, "no" blender): the warp of such an
image is an exact copy of its FINAL source, so download_warped(i) shows what the resize kernel wrote, against
oracle.resize_linear_exact.  The sizes cover scales 0.05-1, exact halvings, one axis kept, 1-px sides and every width
mod 8 (the kernel stores groups of four pixels in row-major order).

Rig draws.  rig_fuzz / crop_fuzz / shard_fuzz cases with camera sizes drawn per image above the case's FINAL sizes (some
kept equal: a mixed rig); the compositor fed camera frames must equal the one fed the oracle's resized frames.

Records.  tests/golden/gen_final_scale_golden.py ran the unmodified reference Stitcher with final_megapix 3 (scale 0.5
exactly) and 5 on the 4 views of 4000 x 3000 of golden_fullres_a; the records hold the fullres fields plus "resized",
the digest of every frame resize_final_resolution handed to the warp.

SB_FINAL_SCALE_SEED=<int> or =random replaces the fixed default seed (the seed used is printed).
"""
import dataclasses
import functools

import numpy as np

import fullres
import fuzz_chain
import reference_cases as RC
import replay
import rig_fuzz
from stitching_b200 import Compositor, rigs

DEFAULT_SEED = 20261019
RECORDS = ("3", "5")


seed_from_env = functools.partial(fuzz_chain.seed_from_env, "SB_FINAL_SCALE_SEED", DEFAULT_SEED)


# -- kernel draws -------------------------------------------------------------------------------------------------------
def _input_side(rng, final, kind):
    if kind == "keep":
        return final
    if kind == "half":
        return 2 * final
    return max(final, int(round(final / rng.uniform(0.05, 1.0))))


def kernel_sizes(rng, count, side):
    """`count` pairs ((W, H) camera, (w, h) FINAL): FINAL widths of every residue mod 8, 1-px sides, exact halvings,
    one axis kept, and scales down to 0.05."""
    out = []
    for k in range(count):
        w = int(rng.integers(1, side // 8 + 1)) * 8 + k % 8
        h = int(rng.integers(2, side + 1))
        if k % 11 == 3:
            h = 1
        if k % 13 == 5:
            w = 1
        kinds = [("half", "half"), ("keep", "any"), ("any", "keep"), ("any", "any"), ("any", "any")][k % 5]
        out.append(((_input_side(rng, w, kinds[0]), _input_side(rng, h, kinds[1])), (w, h)))
    return out


def identity_rig(final_sizes):
    """Cameras of the "affine" warper that translate each image by whole pixels, side by side: every warped image is
    its source, byte for byte."""
    cams, x = [], 0
    for k, (w, h) in enumerate(final_sizes):
        cams.append(rigs.Camera(1.0, 1.0, 0.0, 0.0, np.array([[1, 0, x], [0, 1, 7 * (k % 3)], [0, 0, 1]], np.float32)))
        x += w + 5
    return cams


def frames(sizes, seed):
    return [rigs.noise_image(h, w, seed * 1000 + i) if i % 3 else rigs.synth_image(h, w, seed * 1000 + i)
            for i, (w, h) in enumerate(sizes)]


def kernel_check(O, pairs, seed, **kw):
    """Every image of one identity rig: download_warped equals the oracle's resize of its frame."""
    finals = [f for _, f in pairs]
    ins = [c for c, _ in pairs]
    imgs = frames(ins, seed)
    c = Compositor(identity_rig(finals), finals, "affine", "no", 5, input_sizes=ins, **kw)
    try:
        c.upload(imgs)
        c.run()
        for i, (img, (w, h)) in enumerate(zip(imgs, finals)):
            assert tuple(c.rects[i][2:]) == (w, h), f"image {i}: warped size {c.rects[i][2:]} != {(w, h)}"
            got, mask = c.download_warped(i)
            replay.assert_exact(got, O.resize_linear_exact(img, (w, h)), f"seed {seed}: image {i} {img.shape[1]}x{img.shape[0]} -> {w}x{h}")
            assert (mask == 255).all()
    finally:
        c.close()


# -- rig draws ----------------------------------------------------------------------------------------------------------
def input_sizes(case, rng, keep=0.2, max_factor=4.0):
    """Camera sizes for a case's FINAL sizes: about `keep` of the images unchanged, a share halved exactly, the rest
    scaled by 1/s for s in [1/max_factor, 1], per axis rounded like MegapixDownscaler (the FINAL size is what the
    reference gets back from round(camera * s))."""
    out = []
    for w, h in case.sizes:
        u = rng.random()
        if u < keep:
            out.append((w, h))
        elif u < keep + 0.2:
            out.append((2 * w, 2 * h))
        else:
            f = rng.uniform(1.0, max_factor)
            out.append((max(w, int(round(w * f))), max(h, int(round(h * f)))))
    return out


def oracle_resized(O, imgs, sizes):
    return [img if (img.shape[1], img.shape[0]) == tuple(s) else O.resize_linear_exact(img, s) for img, s in zip(imgs, sizes)]


def rig_check(O, case, seed, crop=None, ex=None):
    """The compositor fed camera frames equals the compositor fed the oracle's resize of them, byte for byte."""
    rng = np.random.default_rng([seed, case.seed])
    ins = input_sizes(case, rng)
    cams = frames(ins, case.seed)
    ex = rig_fuzz.extras(case) if ex is None else ex
    want = fuzz_chain.compositor_run(case, oracle_resized(O, cams, case.sizes), ex, crop=crop)
    got = fuzz_chain.compositor_run(case, cams, ex, crop=crop, input_sizes=ins)
    rig_fuzz.check(dataclasses.replace(case, name=f"{case.describe()} inputs {ins}"), got, want, seed)
    return ins


def sharded_check(O, case, world, copy, seed):
    """All ranks through the transport hooks, fed camera frames: equal to shard_fuzz's grouped oracle fed the
    oracle's resized frames."""
    import shard_fuzz

    case = dataclasses.replace(case, world=world)
    rng = np.random.default_rng([seed, case.seed, world])
    ins = input_sizes(case, rng)
    cams = frames(ins, case.seed)
    ex = [(None, None, None)] * case.n
    ref = shard_fuzz.grouped_oracle(O, case, oracle_resized(O, cams, case.sizes), ex, world)
    got, slabs = shard_fuzz.hooks_run(case, cams, ex, copy, input_sizes=ins)
    shard_fuzz.check(case, got, slabs, ref, seed)


def pipelined_check(O, case, steps, seed):
    """submit / wait over `steps` steps (more than the three buffer sets) with new frames per step: every output equals
    composite() of the oracle-resized frames of that step."""
    rng = np.random.default_rng([seed, case.seed, 7])
    ins = input_sizes(case, rng, keep=0.3)
    c = Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength, input_sizes=ins)
    ref = Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength)
    try:
        w, h = ref.roi[2], ref.roi[3]
        batches = [frames(ins, case.seed + 101 * k) for k in range(steps)]
        pinned = []
        for b in batches:
            ps = []
            for img in b:
                p = c.pinned_empty(img.shape)
                p[...] = img
                ps.append(p)
            pinned.append(ps)
        outs = [(c.pinned_empty((h, w, 3)), c.pinned_empty((h, w))) for _ in range(steps)]
        tickets = []
        for k in range(steps):
            if len(tickets) == 3:
                c.wait(tickets[-3])
            tickets.append(c.submit(pinned[k], *outs[k]))
        for t in tickets[-3:]:
            c.wait(t)
        for k in range(steps):
            pano, pmask = ref.composite(oracle_resized(O, batches[k], case.sizes))
            replay.assert_exact(outs[k][0], pano, f"seed {seed}, {case.describe()}: step {k} pano")
            replay.assert_exact(outs[k][1], pmask, f"seed {seed}, {case.describe()}: step {k} mask")
    finally:
        c.close()
        ref.close()


# -- the records --------------------------------------------------------------------------------------------------------
_records = {}


def record(name):
    if name not in _records:
        z = replay.load(f"golden_final_scale_{name}.npz")
        _records[name] = {k: z[k] for k in (z.files if hasattr(z, "files") else z)}
    return _records[name]


def final_sizes(z):
    return [tuple(int(v) for v in s) for s in z["final_sizes"]]


def resized_check(resize, z, views):
    """`resize(view, size)` of every rebuilt camera view against the recorded resize_final_resolution digests."""
    for i, (v, s) in enumerate(zip(views, final_sizes(z))):
        fullres.check_digest(resize(v, s), z, "resized", i)


def compositor(z, crop=True, **kw):
    n, w, h, _ = (int(v) for v in z["views"])
    c = Compositor(fullres.cameras(z), final_sizes(z), "spherical", "multiband", 5, scale=float(z["scale"]),
                   aspect=float(z["medium_to_final"]), crop=fullres.crop(z) if crop else None, input_sizes=[(w, h)] * n, **kw)
    for i in range(int(z["n"])):
        c.set_seam_mask(i, fullres.seams(z)[i])
        c.set_gain(i, fullres.gains(z)[i])
    return c


def ab_arrays(name):
    """Record `name` through the compositor from its camera views: the pano, its mask and every warped image and mask."""
    z = record(name)
    c = compositor(z)
    try:
        pano, mask = c.composite(views(z))
        return dict(pano=pano, mask=mask, warped=np.concatenate([np.concatenate([a.ravel(), b.ravel()])
                                                                 for a, b in (c.download_warped(i) for i in range(c.n))]))
    finally:
        c.close()


def compositor_replay(z, views):
    """The compositor built from a record and fed the camera views: rects, every image after gain with its blend
    weight, the panorama and two pipelined steps equal the record.  Returns the panorama."""
    c = compositor(z)
    try:
        n = int(z["n"])
        assert [tuple(r) for r in c.rects] == fullres.fed_rects(z), f"rects {c.rects} != {fullres.fed_rects(z)}"
        assert c.num_bands == int(z["num_bands"]), f"num_bands {c.num_bands} != {int(z['num_bands'])}"
        pano, pmask = c.composite(views)
        for i in range(n):
            wi, wm = c.download_warped(i)
            fullres.check_digest(wi, z, "compensated", i)
            fullres.check_digest(wm, z, "blend_mask", i)
        fullres.check_digest(pano, z, "pano")
        srcs = []
        for v in views:
            p = c.pinned_empty(v.shape)
            p[...] = v
            srcs.append(p)
        outs = [(c.pinned_empty(pano.shape), c.pinned_empty(pmask.shape)) for _ in range(2)]
        for t in [c.submit(srcs, o, m) for o, m in outs]:
            c.wait(t)
        for k, (o, m) in enumerate(outs):
            assert np.array_equal(o, pano) and np.array_equal(m, pmask), f"pipelined step {k} differs from composite()"
        return pano
    finally:
        c.close()


def views(z):
    n, w, h, seed = (int(v) for v in z["views"])
    out = RC.camera_views(w, h, n, seed)
    assert [RC.digest(v) for v in out] == [str(d) for d in z["inputs"]], "the rebuilt camera views are not the recorded inputs"
    return out
