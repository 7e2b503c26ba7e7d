#!/usr/bin/env python
"""ab_collapse.py -- two builds of libstitch_b200.so through bench.py, alternated in one session on one GPU.

    python tools/ab_collapse.py --parent build/ab/parent.so [--new stitching_b200/libstitch_b200.so] [--out build/ab/out]

Builds nothing.  `--parent` is the library of the commit to compare against, built beforehand from that commit's sources;
`--new` is this tree's.  stitching_b200/_lib.py loads the one path next to itself, so an arm is selected by copying its
file over that path before the bench.py subprocess starts; this tree's file is put back when the script ends, however it
ends.  The arms run one after the other, never two at once: cfg 2 alternated `--reps` times (bench.py --gpus 1 --steps 50
--warmup 5 --no-cpu-baseline --no-dropin --dump-outputs DIR), then cfg 4 and cfg 3 once per arm (--steps 10 --warmup 3).

Prints the card and its power limit (read here, in the same session as the timings), per run `value`, `ms_per_step` and
the collapse l1 / l0 launch times of `roofline.launches_ms`, and whether the two builds gave the same `result_checksum`
and byte-identical --dump-outputs files.  The JSON line of every run and the summary land in --out.  There is no
fallback: without a GPU the script fails.  `--scale-down N` (bench.py's debug switch) is for rehearsing the plumbing;
its numbers are not measurements.  The whole sequence takes about eleven minutes on an H100 (the synthetic frames of
the ten bench.py runs are generated on the host).
"""
import argparse
import filecmp
import json
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "stitching_b200", "libstitch_b200.so")
DUMPED = ["pano.npy", "mask.npy", "pixel_index.npy", "pano_shape.npy"]


def card():
    """Name, power limit and max SM clock of GPU 0; exits when there is none."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        sys.exit(f"ab_collapse: no GPU to measure on ({e})")
    if not out:
        sys.exit("ab_collapse: no GPU to measure on (nvidia-smi lists none)")
    return out


def bench(workload, steps, warmup, dump_dir, scale_down):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--workload", workload, "--steps", str(steps), "--warmup", str(warmup),
           "--no-cpu-baseline", "--no-dropin", "--dump-outputs", dump_dir]
    if scale_down != 1:
        cmd += ["--scale-down", str(scale_down)]
    p = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    lines = [ln for ln in p.stdout.split("\n") if ln.startswith("{")]
    if p.returncode != 0 or not lines:
        sys.exit(f"ab_collapse: {' '.join(cmd)} failed ({p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
    return json.loads(lines[-1])


def row(arm, workload, rep, r):
    ms = r["roofline"]["launches_ms"]
    return {"arm": arm, "workload": workload, "rep": rep, "value": r["value"], "ms_per_step": r["ms_per_step"],
            "collapse_l1_ms": ms.get("collapse_l1"), "collapse_l0_ms": ms.get("collapse_l0"), "result_checksum": r["result_checksum"],
            "sm_mhz": r["clocks"].get("sm_mhz"), "clock_reasons": r["clocks"].get("reasons")}


def same_dump(a, b):
    return all(os.path.exists(os.path.join(a, f)) and filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False) for f in DUMPED)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--parent", required=True, help="libstitch_b200.so built from the commit to compare against")
    ap.add_argument("--new", default=LIB, help="this tree's library (default: the one in place)")
    ap.add_argument("--out", default=os.path.join(ROOT, "build", "ab", "out"))
    ap.add_argument("--reps", type=int, default=3, help="alternations of the two builds on cfg 2")
    ap.add_argument("--scale-down", type=int, default=1, help="rehearsal only: shrink the workloads (not a measurement)")
    args = ap.parse_args()
    for p in (args.parent, args.new):
        if not os.path.isfile(p):
            sys.exit(f"ab_collapse: {p} does not exist")
    gpu = card()
    print(f"card: {gpu} (name, power limit, max SM clock)", flush=True)
    os.makedirs(args.out, exist_ok=True)
    libs = {"parent": os.path.join(args.out, "parent.so"), "new": os.path.join(args.out, "new.so")}
    shutil.copyfile(args.parent, libs["parent"])
    shutil.copyfile(args.new, libs["new"])

    plan = [("cfg2", rep, 50, 5) for rep in range(args.reps)] + [("cfg4", 0, 10, 3), ("cfg3", 0, 10, 3)]
    rows, identical = [], {}
    try:
        for workload, rep, steps, warmup in plan:
            dumps = {}
            for arm in ("parent", "new"):
                shutil.copyfile(libs[arm], LIB)
                dumps[arm] = os.path.join(args.out, f"dump_{workload}_{rep}_{arm}")
                r = bench(workload, steps, warmup, dumps[arm], args.scale_down)
                with open(os.path.join(args.out, f"bench_{workload}_{rep}_{arm}.json"), "w") as f:
                    json.dump(r, f)
                rows.append(row(arm, workload, rep, r))
                print("  ".join(f"{k}={v:.4f}" if isinstance(v, float) else f"{k}={v}" for k, v in rows[-1].items()), flush=True)
            same = same_dump(dumps["parent"], dumps["new"]) and rows[-1]["result_checksum"] == rows[-2]["result_checksum"]
            identical[workload] = identical.get(workload, True) and same
            for d in dumps.values():  # compared: the samples themselves need not travel back
                shutil.rmtree(d, ignore_errors=True)
    finally:
        shutil.copyfile(libs["new"], LIB)
        for p in libs.values():
            os.remove(p)

    print(f"\ncard: {gpu}" + (f"   SCALED DOWN x{args.scale_down}: not a measurement" if args.scale_down != 1 else ""))
    print(f"{'workload':8} {'rep':>3} {'arm':6} {'value MPix/s':>13} {'ms/step':>9} {'collapse l1 ms':>15} {'collapse l0 ms':>15}")
    for r in rows:
        print(f"{r['workload']:8} {r['rep']:>3} {r['arm']:6} {r['value']:>13.0f} {r['ms_per_step']:>9.4f} "
              f"{r['collapse_l1_ms'] or float('nan'):>15.4f} {r['collapse_l0_ms'] or float('nan'):>15.4f}")
    c2 = {arm: [r for r in rows if r["workload"] == "cfg2" and r["arm"] == arm] for arm in ("parent", "new")}
    best_parent, worst_new = max(r["value"] for r in c2["parent"]), min(r["value"] for r in c2["new"])
    print(f"cfg2 value: worst new {worst_new:.0f} vs best parent {best_parent:.0f}: {100 * (worst_new / best_parent - 1):+.1f} %")
    for w, same in identical.items():
        print(f"{w}: result_checksum and --dump-outputs files {'byte-identical' if same else 'DIFFER'} between the two builds")
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump({"card": gpu, "scale_down": args.scale_down, "runs": rows, "identical": identical}, f, indent=1)
    sys.exit(0 if all(identical.values()) else 1)


if __name__ == "__main__":
    main()
