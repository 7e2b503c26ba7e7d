"""Seeded timelapse compositors against the CPU oracle (helper module: no tests in here).

A Stitcher with timelapse="as_is" or "crop" ends every FINAL-resolution image in a frame instead of a blend: the warped
image is sliced by the crop, compensated, and pasted at its corner on a zeroed canvas -- resultRoi ("as_is") or
resultRoiIntersection ("crop") of what Blender.prepare would have received.  Compositor(..., timelapse=kind) does that
on the device, warping only the part P_i of each image that lands on the canvas.  The draws cross both kinds with
rig_fuzz rigs (no crop) and crop_fuzz crops, camera frames resized on the device (final_scale.input_sizes) and every
form of gain; the oracle is the warp, the numpy slice, oracle.gain_apply and oracle.Timelapser.  Rects, canvas and every
frame are compared bit for bit.

SB_TIMELAPSE_FUZZ_SEED=<int> or =random replaces the fixed default seed (the seed used is printed).
"""
import dataclasses
import functools

import numpy as np

import crop_fuzz
import final_scale
import fuzz_chain
import replay
import rig_fuzz
from stitching_b200 import Compositor

DEFAULT_SEED = 20261020
KINDS = ("as_is", "crop")


seed_from_env = functools.partial(fuzz_chain.seed_from_env, "SB_TIMELAPSE_FUZZ_SEED", DEFAULT_SEED)


@dataclasses.dataclass
class TLCase:
    case: object          # rig_fuzz.Case; rects: the uncropped warped rects, gains: per image one of GAIN_KINDS
    kind: str             # "as_is" | "crop"
    crop: object = None   # Crop or None
    input_sizes: list = None  # camera sizes resized on the device, or None

    @property
    def n(self):
        return self.case.n

    def fed(self):
        """The fed rects (corner, fed size): the warped rects, or the crop's clipped slices at the crop corners."""
        if self.crop is None:
            return [tuple(r) for r in self.case.rects]
        return crop_fuzz.CropCase(self.case, self.crop, 1.0).fed()

    def prepared(self):
        """(corners, sizes) as Timelapser.initialize receives them."""
        if self.crop is None:
            return [r[:2] for r in self.case.rects], [r[2:] for r in self.case.rects]
        return list(self.crop.corners), list(self.crop.sizes)

    def describe(self):
        crop = " crop" if self.crop is not None else ""
        ins = " resized" if self.input_sizes is not None else ""
        return f"{self.case.describe()} timelapse={self.kind}{crop}{ins} gains {','.join(self.case.gains)}"


def cases(seed, count, budget):
    """`count` seeded cases: kinds alternate, every other pair is cropped, a third take camera frames, gains drawn per
    image; then the two "many" rigs (more than SB_WARP_BATCH images), uncropped and cropped."""
    rng = np.random.default_rng([seed, 1])
    plain = list(rig_fuzz.cases(seed, count, budget))
    crops = crop_fuzz.cases(seed + 1, count, budget)
    bases = []
    for k in range(count):
        if (k // 2) % 2 and crops:
            cc = crops[k % len(crops)]
            bases.append((cc.case, cc.crop))
        else:
            bases.append((plain[k], None))
    bases.append((rig_fuzz.named("many", budget), None))
    mc = crop_fuzz.named("many", budget)
    bases.append((mc.case, mc.crop))
    out = []
    for k, (case, crop) in enumerate(bases):
        gains = [str(rng.choice(rig_fuzz.GAIN_KINDS)) for _ in range(case.n)]
        case = dataclasses.replace(case, name=f"tl_{k}", gains=gains, masks=["none"] * case.n)
        ins = final_scale.input_sizes(case, rng) if k % 3 == 1 else None
        out.append(TLCase(case, KINDS[k % 2], crop, ins))
    return out


def gains(tc):
    """Per image the gain (or None), drawn for the fed size as rig_fuzz.extras draws it."""
    fed_case = dataclasses.replace(tc.case, rects=tc.fed())
    return [g for _, _, g in rig_fuzz.extras(fed_case)]


def frames_in(tc):
    """The frames a caller feeds: camera size when the case resizes on the device."""
    if tc.input_sizes is None:
        return rig_fuzz.images(tc.case)
    return final_scale.frames(tc.input_sizes, tc.case.seed)


# -- the two sides ----------------------------------------------------------------------------------------------------
def oracle_run(O, tc, imgs, gs):
    """Stitcher order: (resize), warp, slice, compensator apply, Timelapser.initialize(prepared corners, sizes),
    process_frame + get_frame per image."""
    case = tc.case
    if tc.input_sizes is not None:
        imgs = final_scale.oracle_resized(O, imgs, case.sizes)
    scale = case.scale()
    fed = tc.fed()
    t = O.Timelapser(tc.kind)
    t.initialize(*tc.prepared())
    frames = []
    for i, (img, cam, gain) in enumerate(zip(imgs, case.cams, gs)):
        _, wi, _ = fuzz_chain.oracle_image(O, case.wtype, scale, rig_fuzz.Warper.get_K(cam, 1), cam.R, img,
                                           tc.crop.rects[i] if tc.crop is not None else None, gain, want_mask=False)
        t.process_frame(wi, fed[i][:2])
        frames.append(t.get_frame())
    return dict(rects=fed, roi=tuple(t.roi), frames=frames)


def compositor(tc, **kw):
    case = tc.case
    return Compositor(case.cams, case.sizes, case.wtype, timelapse=tc.kind, crop=tc.crop, input_sizes=tc.input_sizes, **kw)


def compositor_run(tc, imgs, gs):
    c = compositor(tc)
    try:
        for i, g in enumerate(gs):
            if g is not None:
                c.set_gain(i, g)
        return dict(rects=list(c.rects), roi=tuple(c.roi), num_bands=c.num_bands, frames=c.timelapse(imgs))
    finally:
        c.close()


def check(tc, got, ref, seed, what=""):
    where = f"seed {seed}, {tc.describe()}{what}"
    assert [tuple(r) for r in got["rects"]] == [tuple(r) for r in ref["rects"]], f"{where}: rects {got['rects']} != {ref['rects']}"
    assert tuple(got["roi"]) == tuple(ref["roi"]), f"{where}: canvas {got['roi']} != {ref['roi']}"
    assert len(got["frames"]) == tc.n
    for i in range(tc.n):
        replay.assert_exact(got["frames"][i], ref["frames"][i], f"{where}: frame {i}")


def run_and_check(O, tc, seed):
    if 0 in canvas(tc)[2:]:
        # the reference's get_frame fails on such a canvas; the compositor refuses it at creation
        import pytest

        from stitching_b200 import StitchingError

        with pytest.raises(StitchingError, match="has a zero side"):
            compositor(tc)
        return
    imgs, gs = frames_in(tc), gains(tc)
    ref = oracle_run(O, tc, imgs, gs)
    got = compositor_run(tc, imgs, gs)
    assert got["num_bands"] == -1
    check(tc, got, ref, seed)


def frame_digests(seed, count, ks, budget):
    """Case index -> the digests of every frame, for cases `ks` of cases(seed, count, budget) with a canvas."""
    import reference_cases as RC

    out = {}
    cs = cases(seed, count, budget)
    for k in ks:
        tc = cs[k]
        if 0 in canvas(tc)[2:]:
            continue
        got = compositor_run(tc, frames_in(tc), gains(tc))
        out[k] = [RC.digest(f) for f in got["frames"]]
    return out


# -- the recorded reference Stitcher runs -------------------------------------------------------------------------------
# tests/golden/gen_timelapse_stitcher_golden.py ran the unmodified reference Stitcher with timelapse="as_is" and "crop",
# crop=True and final_megapix=3 on record "a"'s four 4000 x 3000 views; each record holds the final_scale fields minus the
# blend plus "frames", the digest of every frame the Timelapser produced, and "canvas_gap".
RECORDS = ("as_is", "crop")


def record(name):
    z = replay.load(f"golden_timelapse_stitcher_{name}.npz")
    return {k: z[k] for k in (z.files if hasattr(z, "files") else z)}


def record_replay(z):
    """The compositor built from a record and fed the camera views: rects, canvas, every frame of timelapse() and of two
    pipelined steps equal the reference's.  Returns the canvas."""
    import fullres
    import reference_cases as RC

    kind = str(z["timelapse"])
    n, w, h, _ = (int(v) for v in z["views"])
    views = final_scale.views(z)
    c = Compositor(fullres.cameras(z), final_scale.final_sizes(z), "spherical", scale=float(z["scale"]),
                   aspect=float(z["medium_to_final"]), crop=fullres.crop(z), input_sizes=[(w, h)] * n, timelapse=kind)
    try:
        assert [tuple(r) for r in c.rects] == fullres.fed_rects(z), f"{kind}: rects {c.rects} != {fullres.fed_rects(z)}"
        corners, sizes = [tuple(map(int, v)) for v in z["corners"]], [tuple(map(int, v)) for v in z["sizes"]]
        assert tuple(c.roi) == canvas_of(kind, corners, sizes), f"{kind}: canvas {c.roi} != {canvas_of(kind, corners, sizes)}"
        assert int(z["canvas_gap"]) == int("gap canvas" in _gap_tags(kind, corners, sizes))
        for i, g in enumerate(fullres.gains(z)):
            c.set_gain(i, g)
        frames = c.timelapse(views)
        for i, f in enumerate(frames):
            assert RC.digest(f) == str(z["frames"][i]), f"{kind}: frame {i}: {RC.digest(f)}, the reference {z['frames'][i]}"
        srcs = []
        for v in views:
            p = c.pinned_empty(v.shape)
            p[...] = v
            srcs.append(p)
        tickets = [c.submit_timelapse(srcs) for _ in range(2)]
        for t in tickets:
            c.wait(t)
            assert all(np.array_equal(a, b) for a, b in zip(c.frames(t), frames)), f"{kind}: pipelined step {t} differs"
        return tuple(c.roi)
    finally:
        c.close()


def _gap_tags(kind, corners, sizes):
    if kind == "crop" and (max(c[0] for c in corners) > min(c[0] + s[0] for c, s in zip(corners, sizes)) or
                           max(c[1] for c in corners) > min(c[1] + s[1] for c, s in zip(corners, sizes))):
        return {"gap canvas"}
    return set()


# -- coverage -----------------------------------------------------------------------------------------------------------
def canvas(tc):
    return canvas_of(tc.kind, *tc.prepared())


def canvas_of(kind, corners, sizes):
    """Timelapser.initialize's roi: resultRoi, or resultRoiIntersection built as cv::Rect(tl, br)."""
    if kind == "as_is":
        return fuzz_chain.blend_geometry(corners, sizes).roi
    tlx, tly = max(c[0] for c in corners), max(c[1] for c in corners)
    brx, bry = min(c[0] + s[0] for c, s in zip(corners, sizes)), min(c[1] + s[1] for c, s in zip(corners, sizes))
    return (min(tlx, brx), min(tly, bry), abs(brx - tlx), abs(bry - tly))


def parts(tc):
    """P_i per image: its fed rect on the canvas, or None."""
    cx, cy, cw, ch = canvas(tc)
    out = []
    for x, y, w, h in tc.fed():
        x0, y0, x1, y1 = max(x, cx), max(y, cy), min(x + w, cx + cw), min(y + h, cy + ch)
        out.append((x0, y0, x1 - x0, y1 - y0) if x1 > x0 and y1 > y0 else None)
    return out


def coverage(tc):
    """What a case reaches, restated from its geometry."""
    tags = set()
    if 0 in canvas(tc)[2:]:
        return {"zero-side canvas"}
    tags |= _gap_tags(tc.kind, *tc.prepared())
    if tc.case.wtype in rig_fuzz.MAP_TYPES:
        tags.add("map projection")  # host-built maps: the batch runs k_warp_wide
    if tc.n > rig_fuzz.WARP_BATCH:
        tags.add("n>32")
    for f, p, g in zip(tc.fed(), parts(tc), tc.case.gains):
        if p is None:
            tags.add("empty P")
            continue
        clipped = set()
        if p[0] > f[0]:
            clipped.add("clip left")
        if p[1] > f[1]:
            clipped.add("clip top")
        if p[0] + p[2] < f[0] + f[2]:
            clipped.add("clip right")
        if p[1] + p[3] < f[1] + f[3]:
            clipped.add("clip bottom")
        tags |= clipped
        if clipped and g != "none":
            tags.add("gain on clipped P")
            if g.startswith("map"):
                tags.add("gain map on clipped P")
    if tc.input_sizes is not None:
        same = [tuple(a) == tuple(b) for a, b in zip(tc.input_sizes, tc.case.sizes)]
        if any(same) and not all(same):
            tags.add("mixed rig")
    return tags


WANT = {"empty P", "clip left", "clip right", "clip top", "clip bottom", "gap canvas", "map projection", "n>32",
        "gain on clipped P", "gain map on clipped P", "mixed rig"}
