"""Exposure gain maps of every shape, against cv2's own results (helper module: no tests in here).

Blocks*Compensator::apply resizes the float32 gain map to the image with cv::resize(INTER_LINEAR), and cv2 runs two
different kernels for it: IPP's on a map whose sides are both >= 2, OpenCV's own on a map with a side of 1 (1 x k,
k x 1, 1 x 1: the maps the compensators hand out for LOW images of 32 px or less on a side).  The product follows the
same dispatch (gain_upload: gain_mode 1 or 3).  tests/golden/golden_gain_maps.npz, written by gen_gain_map_golden.py
with cv2 and the reference's compensators, pins:
  - cv.resize of a grid of map shapes over destinations from 1 px to camera scale (raw float32 or digests);
  - apply on foil images (foil_image): each value is a byte whose product with the gain rounds differently under the
    rule cv2 does not pick for the map, where such a byte exists;
  - the maps feed() hands out for LOW images 20-31 px on a side, applied at FINAL sizes 11 and 22 times larger.
The checks here run those against the oracle and the product's entries (ExposureErrorCompensator.apply on host
buffers and on device twins, Compositor.set_gain plain, timelapse and sharded); `live_sweep` draws shapes on both
sides of the dispatch against cv2 itself when it imports.
"""
import ctypes as C

import numpy as np

import final_scale
import reference_cases as RC
import replay
import rig_fuzz
import shard_fuzz
import timelapse_fuzz as TF
from stitching_b200 import Compositor, Warper, device_array, rigs
from stitching_b200 import exposure_error_compensator as ec


def golden():
    return replay.load("golden_gain_maps.npz")


def one_px(shape):
    return shape[0] == 1 or shape[1] == 1


def resize_cases(z, which=None):
    """(index, map, (W, H), stored result or digest string); which: "1px", "ipp" or None for all."""
    for n in range(int(z["n_resize"])):
        m = z[f"map_{n}"]
        if which is not None and one_px(m.shape) != (which == "1px"):
            continue
        want = z[f"resized_{n}"] if f"resized_{n}" in z else str(z[f"digest_{n}"])
        yield n, m, tuple(int(v) for v in z[f"size_{n}"]), want


def check_oracle_resize(O, which=None):
    """oracle.resize_linear_f32 against cv.resize of every golden map, bit for bit (digests for the large ones)."""
    z = golden()
    bad, count = [], 0
    for n, m, size, want in resize_cases(z, which):
        got = O.resize_linear_f32(m, size).reshape((size[1], size[0]) + m.shape[2:])
        count += 1
        if isinstance(want, str):
            if RC.digest(got) != want:
                bad.append(f"{m.shape} -> {size}: digest differs")
        elif not np.array_equal(got.view(np.uint32), want.reshape(got.shape).view(np.uint32)):
            d = got.view(np.uint32) != want.reshape(got.shape).view(np.uint32)
            bad.append(f"{m.shape} -> {size}: {int(d.sum())} of {d.size} values differ")
    assert count and not bad, f"oracle resize_linear_f32 vs cv.resize, {len(bad)} of {count} maps:\n  " + "\n  ".join(bad[:20])


def check_apply_goldens(O, apply_fn, which=None):
    """The oracle and apply_fn(img, gain) -> image against the compensators' apply on the foil images (each case
    shows that the other rule would change bytes), and on noise images with non-finite maps (which="1px" or None)."""
    z = golden()
    count = 0
    for k in range(int(z["n_apply"])):
        m, img, want = z[f"apply_map_{k}"], z[f"apply_img_{k}"], z[f"apply_out_{k}"]
        if which is not None and one_px(m.shape) != (which == "1px"):
            continue
        assert_tells_apart(img, *gains_and_foil(O, m, (img.shape[1], img.shape[0])), want, f"apply case {k}, map {m.shape}")
        replay.assert_exact(O.gain_apply(img, m), want, f"oracle, apply case {k}, map {m.shape} on {img.shape[1]}x{img.shape[0]}")
        replay.assert_exact(np.asarray(apply_fn(img.copy(), m)), want, f"apply case {k}, map {m.shape} on {img.shape[1]}x{img.shape[0]}")
        count += 1
    for k in range(int(z["n_nonfinite"]) if which in (None, "1px") else 0):
        m = z[f"nonfinite_map_{k}"]
        for j in range(3):
            want = z[f"nonfinite_resized_{k}_{j}"]
            H, W = want.shape[:2]
            got = O.resize_linear_f32(m, (W, H))
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"oracle resize, non-finite map {k} -> {W}x{H}"
            img, out = noise(H, W, 900 + 10 * k + j), z[f"nonfinite_out_{k}_{j}"]
            replay.assert_exact(O.gain_apply(img, m), out, f"oracle, non-finite map {k} on {W}x{H}")
            replay.assert_exact(np.asarray(apply_fn(img.copy(), m)), out, f"apply, non-finite map {k} on {W}x{H}")
            count += 1
    assert count


def fed_maps(z):
    """(index, kind, LOW (w, h), map) of the maps feed() handed out."""
    for k in range(int(z["n_feed"])):
        yield k, str(z[f"feed_kind_{k}"]), tuple(int(v) for v in z[f"feed_low_{k}"]), z[f"feed_map_{k}"]


def check_feed_goldens(O, apply_fn, ratios=(11, 22)):
    """The maps feed() hands out for LOW images of 32 px or less on a side are one block on that side (what the Stitcher
    really produces); their apply at FINAL sizes 11 and 22 times larger, by the oracle and apply_fn, against digests."""
    z = golden()
    shapes = set()
    for k, kind, (lw, lh), m in fed_maps(z):
        assert m.shape[:2] == (-(-lh // 32), -(-lw // 32)), f"fed map {k}: {m.shape} for LOW {lw}x{lh}"
        assert m.dtype == np.float32 and (m.ndim == 3) == (kind == "channel_blocks")
        shapes.add("1xk" if m.shape[:2][0] == 1 and m.shape[1] > 1 else "kx1" if m.shape[1] == 1 and m.shape[0] > 1 else "1x1")
        for r in ratios:
            img = noise(lh * r, lw * r, 100 * k + r)
            want = str(z[f"feed_out_{k}_{r}"])
            assert RC.digest(O.gain_apply(img, m)) == want, f"oracle, fed map {k} {m.shape} at {r}x LOW {lw}x{lh}"
            assert RC.digest(np.asarray(apply_fn(img.copy(), m))) == want, f"apply, fed map {k} {m.shape} at {r}x LOW {lw}x{lh}"
    assert shapes == {"1xk", "kx1", "1x1"}, shapes


def noise(h, w, seed):
    """The FINAL images of the feed cases (gen_gain_map_golden.noise)."""
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def foil_image(g, *foils):
    """uint8 H x W x 3 for a resized gain g (H x W x cn) and foils, gains of the same shape that a wrong resize would
    give (first the map resized by the rule cv2 does not pick for it): per value, of the bytes whose rounded product
    with g differs from their rounded product with some foil, the one whose product sits nearest a half-integer; where
    no byte tells them apart, the one nearest a half-integer.  Products stay below 254.5, so saturation hides nothing."""
    b3 = lambda a: np.broadcast_to(a if a.ndim == 3 else a[:, :, None], g.shape[:2] + (3,)).astype(np.float32)
    cols = np.stack([b3(a).view(np.uint32).ravel() for a in (g,) + foils], axis=1)
    u, inv = np.unique(cols, axis=0, return_inverse=True)
    us = u.view(np.float32)
    v = np.arange(256, dtype=np.float32)
    best = np.empty(len(u), np.uint8)
    for a in range(0, len(u), 2048):
        p = us[a:a + 2048, 0, None] * v  # float32 products
        dist = np.abs(p - np.floor(p) - np.float32(0.5))
        dist[p >= 254.5] = np.inf
        flips = np.zeros(p.shape, bool)
        for k in range(1, us.shape[1]):
            flips |= np.rint(p) != np.rint(us[a:a + 2048, k, None] * v)
        best[a:a + 2048] = np.argmin(np.where(flips, dist, dist + 2), axis=-1)  # bytes that tell g from a foil first
    return best[inv.ravel()].reshape(g.shape[:2] + (3,))


def fused_rows(m, size):
    """The map resized by OpenCV's own rule with the vertical pass fused (h1 t + round(h0 (1 - t)) rounded once): a
    foil for the rounding of that pass.  numpy, with the fused product and sum taken in double."""
    w, h = size
    cn = 1 if m.ndim == 2 else m.shape[2]
    a = m.reshape(m.shape[0], m.shape[1], cn).astype(np.float32)

    def taps(n_src, n_dst, cols):
        d = np.arange(n_dst, dtype=np.float64)
        f = ((d + 0.5) * (1.0 / (n_dst / n_src)) - 0.5).astype(np.float32)
        s = np.floor(f).astype(np.int64)
        t = (f - s.astype(np.float32)).astype(np.float32)
        if cols:
            t[(s < 0) | (s >= n_src - 1)] = 0
            s = np.maximum(s, 0)
        return np.clip(s, 0, n_src - 1), np.clip(s + 1, 0, n_src - 1), t

    x0, x1, tx = taps(a.shape[1], w, True)
    y0, y1, ty = taps(a.shape[0], h, False)
    ux, uy = (np.float32(1) - tx)[None, :, None], (np.float32(1) - ty)[:, None, None]
    hp = (a[:, x0] * ux).astype(np.float32) + (a[:, x1] * tx[None, :, None]).astype(np.float32)
    r = (hp[y0] * uy).astype(np.float32)
    return (hp[y1].astype(np.float64) * ty[:, None, None].astype(np.float64) + r).astype(np.float32)


def apply_resized(img, g):
    """Blocks*Compensator::apply's product with an already resized finite gain: saturate(cvRound(float(v) * g))."""
    g3 = np.broadcast_to(g if g.ndim == 3 else g[:, :, None], img.shape).astype(np.float32)
    return np.clip(np.rint(img.astype(np.float32) * g3), 0, 255).astype(np.uint8)


def gains_and_foil(O, m, size):
    """(g, gf): the map resized to size = (w, h) by cv2's rule and by the other one, each H x W x cn."""
    w, h = size
    cn = 1 if m.ndim == 2 else m.shape[2]
    g = O.resize_linear_f32(m, size).reshape(h, w, cn)
    gf = O.resize_linear_f32(m, size, rule="ipp" if one_px(m.shape) else "generic").reshape(h, w, cn)
    return g, gf


def foils_of(O, m, size):
    """The foils of a map at size = (w, h): the other rule's resize, and for a map with a side of 1 also fused_rows."""
    g, gf = gains_and_foil(O, m, size)
    return (g, gf, fused_rows(m, size)) if one_px(m.shape) else (g, gf)


def searched_map(O, shape, cn, size, rng, part=None, tries=2000):
    """A map of `shape` drawn from rng (0.55-1.9) until its foil image at `size` tells cv2's rule from the other rule in
    `part` (a pair of slices; the whole image by default); the other foils are told apart where the image can.  With a
    few hundred distinct gains a byte that flips under a one-ulp error exists only for some maps, and a 1 x 1 map that
    the two rules resize alike (a (1 - t) + a t == a at every t) is drawn again.  Returns (map, foil image, g, gf)."""
    part = part or (slice(None), slice(None))
    for _ in range(tries):
        m = rng.uniform(0.55, 1.9, shape + (cn,)).astype(np.float32)
        m = m[:, :, 0] if cn == 1 else m
        fs = foils_of(O, m, size)
        img = foil_image(*fs)
        want = apply_resized(img[part], fs[0][part])
        if (want != apply_resized(img[part], fs[1][part])).any():
            return m, img, fs[0], fs[1]
    raise AssertionError(f"no {shape} x {cn} map in {tries} draws tells the rules apart at {size}")


def assert_tells_apart(img, g, gf, want, what):
    """The image shows the rule in its bytes: `want` is its product with g and not its product with the foil gf (the
    test could not pass if the entry under test took the other rule)."""
    assert np.array_equal(apply_resized(img, g), want), f"{what}: want is not the image times the resized gain"
    d = int((apply_resized(img, gf) != want).sum())
    assert d > 0, f"{what}: the foil rule gives the same bytes"
    return d


# (shape, channels) of the maps with a side of 1 that the twin, timelapse and sharded checks set
PROBES = [((1, 7), 1), ((9, 1), 3), ((1, 1), 1), ((1, 2), 3), ((3, 1), 1)]


def probe_maps(seed):
    rng = np.random.default_rng(seed)
    out = []
    for (h, w), c in PROBES:
        m = rng.uniform(0.55, 1.9, (h, w, c)).astype(np.float32)
        out.append(m[:, :, 0] if c == 1 else m)
    return out


def check_device_twin(O, size=(150, 110), crop=(5, 7, 11, 3), foil=True):
    """sb_gain_apply_dev on warped images' device twins sliced at a crop offset (the Stitcher's crop is a slice):
    the twin and the host copy both equal the oracle's apply of the same bytes.  With foil the cropped parts are foil
    images of searched maps (the other rule would change bytes); without, noise (camera scale)."""
    w, h = size
    top, left, bottom, right = crop
    cw, ch = w - left - right, h - top - bottom
    rng = np.random.default_rng(7)
    maps, imgs, foils = [], [], []
    for i, (shape, cn) in enumerate(PROBES):  # the warp copies each image: its cropped part is a foil image
        img = rigs.noise_image(h, w, 40 + i)
        if foil:
            m, part, g, gf = searched_map(O, shape, cn, (cw, ch), rng)
            img[top:h - bottom, left:w - right] = part
        else:  # camera scale: noise, the maps as drawn
            m = probe_maps(7)[i]
            g = gf = None
        maps.append(m)
        imgs.append(img)
        foils.append((g, gf))
    cams = final_scale.identity_rig([(w, h)] * len(maps))
    warper = Warper("affine")
    warper.set_scale(cams)
    warped = list(warper.warp_images(imgs, cams))
    for i, (wi, m, (g, gf)) in enumerate(zip(warped, maps, foils)):
        v = wi[top:-bottom, left:-right]
        tw = device_array.twin(v)
        assert tw is not None and tw[1:3] == (left, top)
        plain = np.array(v)
        out = ec.apply_gain(v, m)
        assert out is v and device_array.twin(out) is not None
        want = O.gain_apply(plain, m)
        if foil:
            assert_tells_apart(plain, g, gf, want, f"device twin, map {m.shape}")
        replay.assert_exact(np.asarray(out), want, f"device twin at ({left}, {top}), map {m.shape}")


def check_compositor(O, sizes, maps, seed=3, foil=True):
    """Compositor.set_gain on a rig of whole-pixel translations (the "affine" warper copies every image exactly, see
    final_scale.identity_rig): download_warped(i) is the image after the gain, against the oracle's apply.  maps: per
    image None (no gain), a map, or with foil a (shape, channels) to draw by searched_map, whose foil image tells the
    rules apart (checked again here); without foil the images are noise."""
    rng = np.random.default_rng(seed)
    imgs, ms = [], []
    for i, ((w, h), m) in enumerate(zip(sizes, maps)):
        if m is None or not foil:
            imgs.append(rigs.noise_image(h, w, seed * 100 + i))
        elif isinstance(m, tuple):
            m, img, _, _ = searched_map(O, m[0], m[1], (w, h), rng)
            imgs.append(img)
        else:
            imgs.append(foil_image(*foils_of(O, m, (w, h))))
        ms.append(m)
    c = Compositor(final_scale.identity_rig(sizes), sizes, "affine", "no", 5)
    try:
        for i, m in enumerate(ms):
            c.set_gain(i, m)
        c.upload(imgs)
        c.run()
        for i, (img, m) in enumerate(zip(imgs, ms)):
            got, mask = c.download_warped(i)
            want = img if m is None else O.gain_apply(img, m)
            if m is not None and foil:
                assert_tells_apart(img, *gains_and_foil(O, m, (img.shape[1], img.shape[0])), want, f"compositor image {i}")
            replay.assert_exact(got, want, f"compositor image {i} {img.shape[1]}x{img.shape[0]}, map {None if m is None else m.shape}")
            assert (mask == 255).all()
    finally:
        c.close()


def timelapse_case():
    """A "crop" timelapse of whole-pixel translations (the warp copies each image): the canvas is the rects'
    intersection, so every part P_i is clipped on one or two sides and the gain taps are sliced at P_i's place."""
    sizes = [(61, 43), (70, 47), (52, 40), (66, 39), (58, 45)]
    offs = [(0, 0), (9, 4), (4, -6), (-7, 3), (12, -2)]
    cams = [rigs.Camera(1.0, 1.0, 0.0, 0.0, np.array([[1, 0, x], [0, 1, y], [0, 0, 1]], np.float32)) for x, y in offs]
    case = rig_fuzz.Case("gain_timelapse", "affine", cams, sizes, "no", 0.0, ["none"] * 5, ["map1"] * 5, ["noise"] * 5, 31)
    case.rects = rig_fuzz._rects(case.wtype, case.cams, case.sizes)
    return TF.TLCase(case, "crop")


def check_timelapse(O):
    """The timelapse case, every image with a map with a side of 1: frames against the oracle's warp, apply,
    Timelapser.  Each image is a foil image for its whole fed size, and its part on the canvas alone tells the rules
    apart."""
    tc = timelapse_case()
    fed, parts = tc.fed(), TF.parts(tc)
    assert all(p is not None and (p[2], p[3]) != (f[2], f[3]) for p, f in zip(parts, fed)), "every P_i clipped"
    rng = np.random.default_rng(11)
    gs, imgs = [], []
    for i, ((x, y, w, h), (px, py, pw, ph), (shape, cn)) in enumerate(zip(fed, parts, PROBES)):
        assert (w, h) == tc.case.sizes[i], "the warp copies the image"
        s = (slice(py - y, py - y + ph), slice(px - x, px - x + pw))
        m, img, g, gf = searched_map(O, shape, cn, (w, h), rng, part=s)
        assert_tells_apart(img[s], g[s], gf[s], apply_resized(img[s], g[s]), f"timelapse image {i}, P_i")
        gs.append(m)
        imgs.append(img)
    ref = TF.oracle_run(O, tc, imgs, gs)
    TF.check(tc, TF.compositor_run(tc, imgs, gs), ref, 0, " 1-px gain maps")


def check_sharded(O, copy, scale_down=16):
    """A world-2 sharded rig: each owning rank sets maps with a side of 1 (and one IPP map) on its images; every
    rank's warped images and strip against the grouped oracle."""
    cfg = rigs.config("cfg2", scale_down)
    case = shard_fuzz.config_case(cfg, 2)
    imgs = [rigs.noise_image(cfg["h"], cfg["w"], 90 + i) for i in range(case.n)]
    maps = probe_maps(13) + [np.random.default_rng(5).uniform(0.6, 1.5, (3, 4)).astype(np.float32)]
    ex = [(None, None, maps[i % len(maps)]) for i in range(case.n)]
    ref = shard_fuzz.grouped_oracle(O, case, imgs, ex)
    got, sizes = shard_fuzz.hooks_run(case, imgs, ex, copy)
    shard_fuzz.check(case, got, sizes, ref, 0)


def memmove(d, s, n):
    C.memmove(d, s, n)


def live_sweep(O, apply_fn, count, seed, max_side=700):
    """Seeded random maps on both sides of the dispatch against cv2 itself: the oracle's resize bit for bit against
    cv.resize, apply_fn against BlocksGainCompensator / BlocksChannelsCompensator.apply."""
    import cv2

    rng = np.random.default_rng(seed)
    for t in range(count):
        kind = t % 4
        a, b = int(rng.integers(1, 45)), int(rng.integers(2, 45))
        shape = [(1, b), (b, 1), (1, 1), (b, max(2, a))][kind]
        cn = int(rng.choice([1, 3]))
        m = rng.uniform(0.5, 2.0, shape + (cn,)).astype(np.float32)
        m = m[:, :, 0] if cn == 1 else m
        W, H = int(rng.integers(1, max_side)), int(rng.integers(1, max_side))
        want = cv2.resize(m, (W, H), interpolation=cv2.INTER_LINEAR).reshape((H, W) + m.shape[2:])
        got = O.resize_linear_f32(m, (W, H)).reshape(want.shape)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"draw {t}: oracle vs cv.resize, map {m.shape} -> {W}x{H}"
        img = foil_image(*foils_of(O, m, (W, H))) if one_px(m.shape) else noise(H, W, t)
        comp = cv2.detail.BlocksGainCompensator() if cn == 1 else cv2.detail.BlocksChannelsCompensator()
        comp.setMatGains([m])
        ref = np.asarray(comp.apply(0, (0, 0), img.copy(), np.full((H, W), 255, np.uint8)))
        replay.assert_exact(np.asarray(apply_fn(img.copy(), m)), ref, f"draw {t}: apply vs cv2, map {m.shape} on {W}x{H}")


# the compositor draws: sizes and (shape, channels) of 1 x k, k x 1 and 1 x 1 maps (one and three channels), an IPP map
# and an image without a gain in one batch, on images 1 px to a few hundred px across
def compositor_draw(seed, side):
    rng = np.random.default_rng(seed)
    shapes = [(1, 6), (8, 1), (1, 1), (1, 2), (2, 1), (1, 12), (4, 3), None, (1, 1)]
    cns = [1, 3, 1, 3, 1, 3, 3, None, 3]
    sizes, maps = [], []
    for k, (s, c) in enumerate(zip(shapes, cns)):
        w, h = int(rng.integers(2, side)), int(rng.integers(2, side))
        if k == 3:
            h = 1
        if k == 4:
            w = 1
        sizes.append((w, h))
        maps.append(None if s is None else (s, c))
    return sizes, maps
