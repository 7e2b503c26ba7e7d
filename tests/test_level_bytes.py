"""The byte model of the multiband launches (BlendPlan::launch_bytes, bench.py's roofline) counts the pyramid levels of
byte-fed images as they are stored: one colour word + one float weight per pixel (4 + 4 B), and 4 B per pixel of the
coarser level's colours read by the pyrUp.  Restated here from the padded rects (rig_fuzz.plan) and checked launch by
launch on the emulation build."""
import types

import pytest

import rig_fuzz
from stitching_b200 import Compositor, rigs


def test_byte_model_counts_levels_as_stored(use_emu):
    cfg = rigs.config("cfg2", 25)
    cams = cfg["cameras"]
    c = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), cfg["warper"], cfg["blender"], cfg["strength"])
    try:
        case = types.SimpleNamespace(roi=lambda: c.roi, rects=c.rects, strength=cfg["strength"], blender=cfg["blender"])
        kind, nb, padded = rig_fuzz.plan(case)
        assert kind == "multiband" and nb == c.num_bands and nb >= 2
        _, _, w, h = c.roi
        a = 1 << nb
        wp, hp = -(-w // a) * a, -(-h // a) * a
        _, per_launch = c.model_bytes()
        assert len(per_launch) == 1 + nb + (nb + 1)  # warp, pyrDown l0 .. nb-1, collapse nb .. 0

        def px(p, l):
            return (p["pw"] >> l) * (p["ph"] >> l)

        for l in range(nb):  # read level l (RGBM at level 0), write level l+1
            want = sum((4.0 if l == 0 else 8.0) * px(p, l) + 8.0 * px(p, l) / 4 for p in padded)
            assert per_launch[1 + l] == pytest.approx(want, rel=1e-12), f"pyrdown_l{l}"
        for l in range(nb, -1, -1):  # own level, the coarser level's colours, C_{l+1}, C_l or the final roi
            P = (wp >> l) * (hp >> l)
            want = sum((4.0 if l == 0 else 8.0) * px(p, l) + (4.0 * px(p, l) / 4 if l < nb else 0.0) for p in padded)
            want += (6.0 * P / 4 if l < nb else 0.0) + (6.0 * P if l > 0 else 4.0 * w * h)
            assert per_launch[1 + nb + (nb - l)] == pytest.approx(want, rel=1e-12), f"collapse_l{l}"
    finally:
        c.close()
