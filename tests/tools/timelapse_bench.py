"""What a timelapse step costs on the fused compositor (run on a GPU box:
python tests/tools/timelapse_bench.py [--steps K] [--warmup W]).

Two rigs, each a Stitcher with a timelapse setting:
- "as_is": the cfg2 rig (8 x 4000 x 3000, spherical, yaw ring of 30 degrees), canvas = the whole panorama;
- "crop": 8 x 4000 x 3000 views of one direction, each turned by 1-2 degrees (the reference's timelapse use: a fixed
  camera that wobbles), canvas = what all of them cover.
One JSON line with the card name and power limit (nvidia-smi) and per rig:
- e2e_ms_final / e2e_ms_camera: ms per pipelined submit_timelapse / wait step fed FINAL frames, and fed the 4000 x 3000
  camera frames at final_megapix 3 (resized on the device);
- warp_ms / paste_ms: the kernels per step from torch.profiler in a run of their own, with their model bytes and the
  share of the 3.35 TB/s HBM peak of the H100 SXM data sheet;
- h2d_bytes / d2h_bytes: PCIe bytes per step (sources in, the parts P_i out) against n whole canvases;
- dropin_ms: the drop-in chain in the Stitcher's call order (Warper.warp_image, Timelapser.process_frame / get_frame per
  image) on the same FINAL frames, and parity: its frames equal the compositor's byte for byte.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from final_scale_bench import HBM_BYTES_PER_S, card, final_size  # noqa: E402
from stitching_b200 import Compositor, Timelapser, Warper, _lib, rigs  # noqa: E402


def wobble(n, w, h, focal, seed=5):
    """n cameras looking the same way, each turned by 1-2 degrees about a random axis."""
    rng = np.random.default_rng(seed)
    cams = []
    for _ in range(n):
        a = np.deg2rad(rng.uniform(1.0, 2.0)) * rng.choice([-1, 1], 2)
        R = rigs.rot_y(a[0] * rng.uniform(0.3, 1)) @ rigs.rot_x(a[1] * rng.uniform(0.3, 1))
        cams.append(rigs.Camera(focal, 1.0, w / 2.0, h / 2.0, R.astype(np.float32)))
    return cams


def pinned(c, frames):
    out = []
    for f in frames:
        p = c.pinned_empty(f.shape)
        p[...] = f
        out.append(p)
    return out


def pipelined_ms(c, frames, steps, warmup):
    srcs = pinned(c, frames)
    tickets = []

    def step():
        if len(tickets) >= 3:
            c.wait(tickets[-3])
        tickets.append(c.submit_timelapse(srcs))

    for _ in range(warmup):
        step()
    for t in tickets[-3:]:
        c.wait(t)
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    for t in tickets[-3:]:
        c.wait(t)
    return 1e3 * (time.perf_counter() - t0) / steps, [f.copy() for f in c.frames(tickets[-1])]


def kernel_ms(c, frames, steps):
    """k_warp_* and k_timelapse_paste per step from torch.profiler (a run of its own)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    srcs = pinned(c, frames)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            c.wait(c.submit_timelapse(srcs))
    warp = [e.time_range.elapsed_us() for e in prof.events() if "k_warp" in e.name]
    paste = [e.time_range.elapsed_us() for e in prof.events() if "k_timelapse_paste" in e.name]
    return sum(warp) / 1e3 / steps, sum(paste) / 1e3 / steps, len(paste)


def dropin(cams, frames, wtype, kind, scale):
    """Warper.warp_image + Timelapser per image, the Stitcher's order (no crop, no compensator)."""
    t0 = time.perf_counter()
    w = Warper(wtype)
    w.scale = scale
    warped = [np.asarray(w.warp_image(f, cam, 1)) for f, cam in zip(frames, cams)]
    rois = [w.warp_roi((f.shape[1], f.shape[0]), cam, 1) for f, cam in zip(frames, cams)]
    t = Timelapser(kind)
    t.initialize([r[:2] for r in rois], [r[2:] for r in rois])
    out = []
    for img, r in zip(warped, rois):
        t.process_frame(img, r[:2])
        out.append(np.array(t.get_frame()))
    return 1e3 * (time.perf_counter() - t0), out


def measure(name, kind, cams, W, H, wtype, steps, warmup):
    n = len(cams)
    scale = float(np.median([c.focal for c in cams]))
    cam_frames = [rigs.synth_image(H, W, i) for i in range(n)]
    s, (w, h) = final_size(W, H, 3)
    fin = Compositor(cams, [(W, H)] * n, wtype, timelapse=kind)
    res = Compositor(cams, [(w, h)] * n, wtype, aspect=s, timelapse=kind, input_sizes=[(W, H)] * n)
    try:
        e2e_fin, frames_fin = pipelined_ms(fin, cam_frames, steps, warmup)
        e2e_cam, _ = pipelined_ms(res, cam_frames, steps, warmup)
        warp_ms, paste_ms, launches = kernel_ms(fin, cam_frames, 5)
        _, per = fin.model_bytes()
        cw, ch = fin.roi[2], fin.roi[3]
        parts = []
        for x, y, rw, rh in fin.rects:
            x0, y0 = max(x, fin.roi[0]), max(y, fin.roi[1])
            x1, y1 = min(x + rw, fin.roi[0] + cw), min(y + rh, fin.roi[1] + ch)
            parts.append(max(0, x1 - x0) * max(0, y1 - y0))
        d_ms, d_frames = dropin(cams, cam_frames, wtype, kind, scale)
        parity = all(np.array_equal(a, b) for a, b in zip(frames_fin, d_frames))
        return dict(rig=name, kind=kind, canvas=[cw, ch], e2e_ms_final=round(e2e_fin, 3), e2e_ms_camera_fm3=round(e2e_cam, 3),
                    final_size_fm3=[w, h], warp_ms=round(warp_ms, 4), paste_ms=round(paste_ms, 4), paste_launches=launches,
                    warp_model_bytes=per[0], paste_model_bytes=per[1],
                    warp_share_of_hbm_peak=round(per[0] / (warp_ms * 1e-3) / HBM_BYTES_PER_S, 3),
                    paste_share_of_hbm_peak=round(per[1] / (paste_ms * 1e-3) / HBM_BYTES_PER_S, 3),
                    h2d_bytes=3 * n * W * H, d2h_bytes=3 * sum(parts), whole_canvases_bytes=3 * n * cw * ch,
                    dropin_ms=round(d_ms, 1), parity=bool(parity))
    finally:
        fin.close()
        res.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    _lib.check(_lib.lib().sb_init(0), "sb_init")
    name, limit = card()
    cfg = rigs.config("cfg2", 1)
    runs = [measure("cfg2", "as_is", cfg["cameras"], cfg["w"], cfg["h"], cfg["warper"], a.steps, a.warmup),
            measure("wobble 8 x 4000x3000", "crop", wobble(8, 4000, 3000, 4000.0), 4000, 3000, "spherical", a.steps, a.warmup)]
    print(json.dumps(dict(card=name, power_limit=limit, steps=a.steps, warmup=a.warmup, runs=runs,
                          parity=all(r["parity"] for r in runs))))


if __name__ == "__main__":
    main()
