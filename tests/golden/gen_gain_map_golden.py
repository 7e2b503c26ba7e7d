"""Writes tests/golden/golden_gain_maps.npz: how the reference's wheel resizes the exposure compensators' float32 gain maps
(cv.resize INTER_LINEAR, Blocks*Compensator::apply) over a grid of map shapes and destination sizes, what
BlocksGainCompensator / BlocksChannelsCompensator.apply make of images chosen to show a one-ulp error of that resize in
their bytes, and the maps the compensators' own feed() hands out for LOW images of 32 px or less on a side.  Only this
file is written; no other golden moves, and two runs write identical bytes.

    python tests/golden/gen_gain_map_golden.py

cv2 runs IPP's kernel on a map whose sides are both >= 2 and OpenCV's own on a map with a side of 1 (1 x k, k x 1,
1 x 1), so the grid holds both kinds: 1 x 1, 1 x k and k x 1 for k in K, 2 x 2, 2 x k, k x 2, 3 x 5 and 30 x 40, each
with 1 and 3 channels.  The destinations of each map: its own size, a 1-px side each way, a size below the map's, ratios
of 2-3, exactly 32 px per sample (the block size) and a camera-scale size of 100-4000 px a side (FINAL is 11-22 x LOW,
and a block is 32 LOW px).  Results of up to SMALL values are stored as float32, larger ones as a digest of their bytes.

apply cases: maps drawn by tests/gain_maps.py searched_map with their foil images: each value is a byte whose product
with the resized gain rounds differently from its product with the map resized by the other rule (the oracle's, forced),
where such a byte exists, and the map is drawn again until some byte does, so that apply under the wrong rule changes
bytes.  nonfinite: 1 x 3 and 3 x 1 maps holding inf and NaN, resized
and applied to noise images.  feed cases: LOW images 20-31 px on one side
fed to each compensator (block size 32, as ExposureErrorCompensator's default), the maps getMatGains() hands out, and
apply of each map at FINAL sizes 11 and 22 times the LOW one, on noise images seeded by the case (digests).
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "golden_gain_maps.npz")
K = (2, 3, 5, 12, 40)
SMALL = 4096  # values stored as float32; more than this: a digest


def map_shapes():
    """(rows, columns) of every map of the grid."""
    return ([(1, 1)] + [(1, k) for k in K] + [(k, 1) for k in K] + [(2, 2)] + [(2, k) for k in K if k > 2] +
            [(k, 2) for k in K if k > 2] + [(3, 5), (30, 40)])


def gain_map(h, w, cn, seed):
    """Gains like a compensator's, 0.55-1.9, distinct per block and channel."""
    g = np.random.default_rng(seed).uniform(0.55, 1.9, (h, w, cn)).astype(np.float32)
    return g[:, :, 0] if cn == 1 else g


def destinations(h, w):
    """(W, H) sizes for a map of h x w, without repeats."""
    big = (min(4000, max(100, 352 * w)), min(4000, max(100, 352 * h)))
    if big[0] * big[1] > 4_000_000:  # camera scale, but a few million values at most
        big = (big[0], 4_000_000 // big[0]) if big[0] >= big[1] else (4_000_000 // big[1], big[1])
    out = [(w, h), (3 * w + 2, 1), (1, 3 * h + 1), (max(1, w // 2), max(1, (2 * h) // 3)), (2 * w + 1, 3 * h),
           (3 * w, 2 * h + 1), (32 * w, 32 * h), big]
    seen = []
    for d in out:
        if d not in seen:
            seen.append(d)
    return seen


def digest(a):
    a = np.ascontiguousarray(a)
    return f"{a.dtype.str}{list(a.shape)} sha256:{hashlib.sha256(a.tobytes()).hexdigest()}"


# (map shape, channels, image W x H): IPP maps and maps with a side of 1 (the maps drawn by searched_map)
APPLY = [((1, 12), 1, (250, 160)), ((1, 40), 1, (700, 60)), ((12, 1), 3, (130, 300)), ((1, 1), 1, (97, 61)),
         ((1, 1), 3, (64, 90)), ((5, 1), 1, (70, 260)), ((1, 3), 3, (200, 40)), ((2, 5), 1, (170, 90)),
         ((3, 5), 3, (150, 110)), ((30, 40), 1, (260, 200)), ((12, 2), 3, (60, 330))]

# LOW images (w, h) fed together, side by side, to each blocks compensator: sides of 32 px or less give maps one block
# across on that side
FEED = [[(150, 28), (140, 28), (160, 28)], [(24, 130), (24, 120)], [(20, 20), (31, 31), (25, 90)]]


def noise(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def feed_low(sizes, seed):
    """LOW images of one feed case whose exposures differ per image, with their corners (left to right, overlapping by
    a third)."""
    rng = np.random.default_rng(seed)
    imgs, corners, x = [], [], 0
    for k, (w, h) in enumerate(sizes):
        base = rng.integers(60, 190, (h, w, 3)).astype(np.float32)
        scale = np.array([0.8 + 0.2 * k, 1.0, 1.2 - 0.1 * k], np.float32)
        imgs.append(np.clip(base * scale, 0, 255).astype(np.uint8))
        corners.append((x, 0))
        x += 2 * w // 3
    return imgs, corners


# non-finite gains (set_gain takes any float32 map): a left-clamped column reads its neighbour with weight 0 as cv2 does
NONFINITE = [np.array([[1.5, np.inf, 1.25]], np.float32), np.array([[np.nan], [1.2], [0.9]], np.float32)]
NONFINITE_SIZES = [(12, 1), (12, 5), (7, 9)]


def main():
    import cv2

    for p in (ROOT, os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import gain_maps
    from oracle import oracle as O

    O.build()
    out = {"cv2_version": np.array(cv2.__version__)}
    n = 0
    maps = {}
    for (h, w) in map_shapes():
        for cn in (1, 3):
            m = gain_map(h, w, cn, 1000 * h + 10 * w + cn)
            maps[(h, w, cn)] = m
            for (W, H) in destinations(h, w):
                r = cv2.resize(m, (W, H), interpolation=cv2.INTER_LINEAR)
                out[f"map_{n}"] = m
                out[f"size_{n}"] = np.array([W, H], np.int64)
                if r.size <= SMALL:
                    out[f"resized_{n}"] = r
                else:
                    out[f"digest_{n}"] = np.array(digest(r))
                n += 1
    out["n_resize"] = n
    for k, ((h, w), cn, (W, H)) in enumerate(APPLY):
        m, img, _, _ = gain_maps.searched_map(O, (h, w), cn, (W, H), np.random.default_rng(7000 + k))
        comp = cv2.detail.BlocksGainCompensator() if cn == 1 else cv2.detail.BlocksChannelsCompensator()
        comp.setMatGains([m])
        got = comp.apply(0, (0, 0), img.copy(), np.full((H, W), 255, np.uint8))
        out[f"apply_map_{k}"], out[f"apply_img_{k}"], out[f"apply_out_{k}"] = m, img, np.asarray(got)
    out["n_apply"] = len(APPLY)
    for k, m in enumerate(NONFINITE):
        out[f"nonfinite_map_{k}"] = m
        for j, (W, H) in enumerate(NONFINITE_SIZES):
            out[f"nonfinite_resized_{k}_{j}"] = cv2.resize(m, (W, H), interpolation=cv2.INTER_LINEAR)
            img = noise(H, W, 900 + 10 * k + j)
            comp = cv2.detail.BlocksGainCompensator()
            comp.setMatGains([m])
            out[f"nonfinite_out_{k}_{j}"] = np.asarray(comp.apply(0, (0, 0), img, np.full((H, W), 255, np.uint8)))
    out["n_nonfinite"] = len(NONFINITE)
    k = 0
    for f, sizes in enumerate(FEED):
        imgs, corners = feed_low(sizes, 500 + f)
        masks = [np.full((h, w), 255, np.uint8) for w, h in sizes]
        for kind, comp in (("gain_blocks", cv2.detail.BlocksGainCompensator(32, 32, 1)),
                           ("channel_blocks", cv2.detail.BlocksChannelsCompensator(32, 32, 1))):
            comp.feed(corners, imgs, masks)
            for i, g in enumerate(comp.getMatGains()):
                g = np.asarray(g)
                out[f"feed_kind_{k}"], out[f"feed_low_{k}"], out[f"feed_map_{k}"] = np.array(kind), np.array(sizes[i], np.int64), g
                for ratio in (11, 22):
                    W, H = sizes[i][0] * ratio, sizes[i][1] * ratio
                    img = noise(H, W, 100 * k + ratio)
                    got = comp.apply(i, corners[i], img, np.full((H, W), 255, np.uint8))
                    out[f"feed_out_{k}_{ratio}"] = np.array(digest(np.asarray(got)))
                k += 1
    out["n_feed"] = k
    np.savez_compressed(OUT, **out)
    # npz members carry their time stamps: rewrite them at a fixed date so that two runs write identical bytes
    _fix_zip_dates(OUT)
    print(f"wrote {OUT}: {n} resizes, {len(APPLY)} apply cases, {k} fed maps, cv2 {cv2.__version__}, "
          f"{os.path.getsize(OUT) / 1e3:.0f} kB")


def _fix_zip_dates(path):
    import zipfile

    src = zipfile.ZipFile(path)
    items = [(i, src.read(i.filename)) for i in src.infolist()]
    src.close()
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for info, data in items:
            zi = zipfile.ZipInfo(info.filename, date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(zi, data)


if __name__ == "__main__":
    main()
