"""Writes tests/golden/golden_gain_range.npz: what the reference's compensators (cv.detail, through cv2) do to an image
whose products value * gain leave the int range.  Only this file is written; no other golden moves.

    python tests/golden/gen_gain_range_golden.py

ExposureErrorCompensator.apply hands the image to cv.detail ...Compensator.apply, which rounds value * gain with
cvRound, i.e. cvtss2si / cvtsd2si on x86: a product outside the int range, infinite or NaN rounds to INT_MIN, and
saturate_cast<uchar> makes that 0 -- not 255.  Gains like these do not come out of the compensators' own feed(), but
set_gain / apply take any float32 map or float64 scalar.  The cases: the 256 byte values of every channel against
BlocksGainCompensator (1-channel map) and BlocksChannelsCompensator (3-channel map) with maps of large, infinite, NaN
and negative gains mixed with ordinary ones, and GainCompensator with scalars around the limit.
"""
import os

import cv2
import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_gain_range.npz")


def image(h, w):
    """Every byte value in every channel, twice, in a different order per channel."""
    v = np.arange(h * w, dtype=np.int64)
    return np.stack([(v * 7) % 256, (v * 11 + 3) % 256, (v * 13 + 5) % 256], axis=-1).reshape(h, w, 3).astype(np.uint8)


def maps():
    big = [1.0e7, 8.5e6, 1.0e9, 3.0e38, np.inf, -np.inf, np.nan, -1.0e9, 1.5, 0.7]
    m1 = np.array(big[:8], np.float32).reshape(2, 4)
    m3 = np.array([big[(k * 3 + c) % len(big)] for k in range(6) for c in range(3)], np.float32).reshape(2, 3, 3)
    return {"map1": m1, "map3": m3}


SCALARS = [2.0, 8.4e6, 8.5e6, 1.0e7, 1.0e9, 1.0e300, np.inf, np.nan, -1.0e9]


def main():
    img = image(24, 32)
    mask = np.full(img.shape[:2], 255, np.uint8)
    out = {"img": img, "scalars": np.array(SCALARS, np.float64)}
    for name, m in maps().items():
        comp = cv2.detail.BlocksGainCompensator() if m.ndim == 2 else cv2.detail.BlocksChannelsCompensator()
        comp.setMatGains([m])
        got = img.copy()
        comp.apply(0, (0, 0), got, mask)
        out[name], out[name + "_out"] = m, got
    for k, g in enumerate(SCALARS):
        comp = cv2.detail.GainCompensator()
        comp.setMatGains([np.array([[g]], np.float64)])
        got = img.copy()
        comp.apply(0, (0, 0), got, mask)
        out[f"scalar{k}_out"] = got
    out["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: maps {list(maps())}, {len(SCALARS)} scalars, cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
