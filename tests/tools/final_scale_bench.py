"""What final_megapix costs with camera frames resized inside the compositor (run on a GPU box:
python tests/tools/final_scale_bench.py [--steps K] [--warmup W]).

The cfg2 rig (8 x 4000 x 3000, spherical, multiband) at final_megapix 3 (scale 0.5 exactly) and 6 (scale 0.7071), the
FINAL sizes and the camera scaling the reference Stitcher derives (MegapixDownscaler, Warper.get_K).  One JSON line:

- card name and power limit (nvidia-smi);
- e2e_ms_camera: ms per pipelined submit / wait step fed the 4000 x 3000 frames (copy, resize, warp, blend, download);
- e2e_ms_final: the same rig on a compositor fed frames already at FINAL size;
- cpu_resize_ms: cv.resize(INTER_LINEAR_EXACT) of the 8 frames on all host cores (what a caller pays without the
  feature); null when cv2 is missing;
- resize_kernel_ms: k_resize_src per step (8 images, one launch) from torch.profiler in a run of its own, its bytes
  (camera frames read once, FINAL words written) over that time against the 3.35 TB/s of the H100 SXM data sheet;
- parity: the panorama from camera frames equals the one from cv.resize'd frames (or the oracle's resize when cv2 is
  missing) byte for byte.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from stitching_b200 import Compositor, _lib, rigs  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()[0]
        name, limit = (v.strip() for v in out.split(","))
        return name, limit
    except Exception:
        return None, None


def final_size(w, h, megapix):
    """MegapixDownscaler: scale min(1, sqrt(megapix * 1e6 / (w h))) of the first image, sizes rounded."""
    s = min(1.0, math.sqrt(megapix * 1e6 / (w * h)))
    return s, (int(round(w * s)), int(round(h * s)))


def pipelined_ms(c, frames, steps, warmup):
    srcs = []
    for f in frames:
        p = c.pinned_empty(f.shape)
        p[...] = f
        srcs.append(p)
    outs = [(c.pinned_empty((c.roi[3], c.roi[2], 3)), c.pinned_empty((c.roi[3], c.roi[2]))) for _ in range(3)]
    tickets = []

    def step(k):
        if len(tickets) >= 3:
            c.wait(tickets[-3])
        tickets.append(c.submit(srcs, *outs[k % 3]))

    for k in range(warmup):
        step(k)
    for t in tickets[-3:]:
        c.wait(t)
    t0 = time.perf_counter()
    for k in range(steps):
        step(k)
    for t in tickets[-3:]:
        c.wait(t)
    return 1e3 * (time.perf_counter() - t0) / steps, outs[(steps - 1) % 3][0].copy()


def cpu_resize_ms(frames, size, reps=5):
    try:
        import cv2 as cv
    except ImportError:
        return None, None
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        def run():
            return list(ex.map(lambda f: cv.resize(f, size, interpolation=cv.INTER_LINEAR_EXACT), frames))
        out = run()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            run()
            ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts)), out


def kernel_ms(c, frames, steps):
    """k_resize_src per step from torch.profiler (a run of its own); None when the trace has no such kernel."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    srcs = []
    for f in frames:
        p = c.pinned_empty(f.shape)
        p[...] = f
        srcs.append(p)
    out = (c.pinned_empty((c.roi[3], c.roi[2], 3)), c.pinned_empty((c.roi[3], c.roi[2])))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            c.wait(c.submit(srcs, *out))
    ds = [e.time_range.elapsed_us() for e in prof.events() if "k_resize_src" in e.name]
    return (sum(ds) / 1e3 / len(ds), len(ds)) if ds else (None, 0)


def measure(cfg, megapix, steps, warmup):
    n, W, H = cfg["n"], cfg["w"], cfg["h"]
    s, (w, h) = final_size(W, H, megapix)
    frames = [rigs.synth_image(H, W, i) for i in range(n)]
    args = (cfg["cameras"], [(w, h)] * n, cfg["warper"], cfg["blender"], cfg["strength"])
    cam = Compositor(*args, aspect=s, input_sizes=[(W, H)] * n)
    fin = Compositor(*args, aspect=s)
    try:
        cpu_ms, resized = cpu_resize_ms(frames, (w, h))
        if resized is None:
            from oracle import oracle as O

            resized = [O.resize_linear_exact(f, (w, h)) for f in frames]
        e2e_cam, pano_cam = pipelined_ms(cam, frames, steps, warmup)
        e2e_fin, pano_fin = pipelined_ms(fin, resized, steps, warmup)
        k_ms, k_n = kernel_ms(cam, frames, 5)
        nbytes = n * (3.0 * W * H + 4.0 * w * h)
        return dict(final_megapix=megapix, scale=s, final_size=[w, h], e2e_ms_camera=round(e2e_cam, 3), e2e_ms_final=round(e2e_fin, 3),
                    cpu_resize_ms=None if cpu_ms is None else round(cpu_ms, 2),
                    resize_kernel_ms=None if k_ms is None else round(k_ms, 4), resize_kernel_launches=k_n, resize_bytes=nbytes,
                    resize_gb_per_s=None if k_ms is None else round(nbytes / (k_ms * 1e-3) / 1e9, 1),
                    resize_share_of_hbm_peak=None if k_ms is None else round(nbytes / (k_ms * 1e-3) / HBM_BYTES_PER_S, 3),
                    parity=bool(np.array_equal(pano_cam, pano_fin)))
    finally:
        cam.close()
        fin.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    _lib.check(_lib.lib().sb_init(0), "sb_init")
    name, limit = card()
    cfg = rigs.config("cfg2", 1)
    runs = [measure(cfg, mp, a.steps, a.warmup) for mp in (3, 6)]
    print(json.dumps(dict(card=name, power_limit=limit, rig="cfg2 8 x 4000x3000 spherical multiband", steps=a.steps, runs=runs,
                          parity=all(r["parity"] for r in runs))))


if __name__ == "__main__":
    main()
