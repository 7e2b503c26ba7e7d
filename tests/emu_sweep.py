"""The emulation corpora of the CPU suite, by name, run through their own tests' runners and checks against the oracle,
in one process on one library: tests/test_emu_memory.py runs it in child processes, on the emulation build whose
allocations start filled with a byte (SB_EMU_FILL) and on the same sources under AddressSanitizer + UBSan.

    python tests/emu_sweep.py --lib tests/emu/libstitch_b200_emu.so [--corpora rig_fuzz,crop_fuzz]
    python tests/emu_sweep.py --lib <mutant>.so --cases rig_fuzz:case_3,kernel_edges:gain_2p31

Each case is one call of an existing test function with its parameters (its env set as the test sets it, through a
MonkeyPatch undone after the case); a case passes when the call returns.  Prints one line per corpus with its number of
cases and failures, the failures' messages, and exits 1 when any case failed."""
import argparse
import os
import sys
import time
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def corpora(L, O):
    """name -> [(case id, fn(monkeypatch))].  L is the bound library (what the tests' use_emu fixture yields), O the
    oracle module."""
    import crop_fuzz
    import dropin_fuzz
    import kernel_edges
    import rig_fuzz
    import shard_fuzz
    import test_crop
    import test_dropin_fuzz
    import test_final_scale
    import test_fullres
    import test_gain_maps as GT
    import test_host_entries as HE
    import test_host_logic as H
    import test_shard_fuzz
    import test_timelapse_compositor as TL
    import timelapse_fuzz

    n_dropin = len(dropin_fuzz.EMU_RIG) + dropin_fuzz.EMU_CROP + dropin_fuzz.EMU_OWN
    return {
        "rig_fuzz": [(i, lambda mp, k=k: H.test_rig_fuzz_against_oracle(L, O, mp, k)) for k, i in enumerate(rig_fuzz.emu_ids())],
        "crop_fuzz": [(f"case_{k}", lambda mp, k=k: test_crop.test_crop_fuzz_against_oracle(L, O, k)) for k in range(test_crop.EMU_COUNT + 1)]
        + [("full_crop", lambda mp: test_crop.test_full_crop_equals_no_crop(L, O))],
        "shard_fuzz": [(i, lambda mp, k=k: test_shard_fuzz.test_shard_fuzz_against_grouped_oracle(L, O, mp, k)) for k, i in enumerate(shard_fuzz.emu_ids())]
        + [("item_lists_256_ranks", lambda mp: test_shard_fuzz.test_item_lists_stay_under_sb_max_items(L))],
        "dropin_fuzz": [(f"case_{k}", lambda mp, k=k: test_dropin_fuzz.test_dropin_fuzz_against_oracle(L, O, mp, k)) for k in range(n_dropin)],
        "final_scale": [(f"kernel_{k}", lambda mp, k=k: test_final_scale.test_resize_kernel_against_oracle(L, O, k)) for k in range(test_final_scale.KERNEL_RIGS)]
        + [("kernel_packed", lambda mp: test_final_scale.test_resize_kernel_packed_output(L, O, mp))]
        + [(f"rig_{k}", lambda mp, k=k: test_final_scale.test_resized_compositor_equals_prefed(L, O, k)) for k in range(test_final_scale.RIG_COUNT + 1)]
        + [(f"crop_{k}", lambda mp, k=k: test_final_scale.test_resized_crop_equals_prefed(L, O, k)) for k in range(4)]
        + [("sharded", lambda mp: test_final_scale.test_resized_sharded_equals_grouped_oracle(L, O)),
           ("pipelined", lambda mp: test_final_scale.test_pipelined_steps(L, O))],
        "timelapse_fuzz": [(f"case_{k}", lambda mp, k=k: TL.test_fuzz_against_oracle(L, O, k)) for k in range(TL.COUNT + 2)]
        + [(f"pipelined_{kind}", lambda mp, kind=kind: TL.test_pipelined_steps(L, O, kind)) for kind in timelapse_fuzz.KINDS]
        + [("set_gain_between_submits", lambda mp: TL.test_set_gain_between_submits(L, O)),
           ("zero_side_canvas", lambda mp: TL.test_zero_side_canvas(L, O))],
        "fullres": [(f"draw_{k}", lambda mp, k=k: test_fullres.test_ratio_draws_against_oracle(L, O, k)) for k in range(test_fullres.EMU_COUNT)],
        "goldens": [("warper", lambda mp: H.test_warper_goldens_through_emulated_library(L)),
                    ("blender", lambda mp: H.test_blender_goldens_through_emulated_library(L)),
                    ("e2e", lambda mp: H.test_e2e_goldens_through_emulated_library(L)),
                    ("seam_resize", lambda mp: H.test_seam_resize_drop_in_and_fused(L, O)),
                    ("image_resize", lambda mp: H.test_image_resize_drop_in(L, O)),
                    ("gain", lambda mp: H.test_exposure_gain_drop_in_and_fused(L, O)),
                    ("gain_out_of_int_range", lambda mp: H.test_gains_out_of_the_int_range(L, O)),
                    ("timelapser", lambda mp: H.test_timelapser_drop_in(L, O)),
                    ("compositor", lambda mp: H.test_compositor_matches_oracle(L, O))],
        "setters": [("between_submits", lambda mp: H.check_setters_between_submits(25))],
        "lanes_blocks": [("lanes_shuffle_pyrdown", lambda mp: H.test_warp_collective_kernels_under_lane_emulation(L, O, mp)),
                         ("blocks_tile_collapse", lambda mp: H.test_shared_memory_tile_kernels_under_block_emulation(L, O, mp)),
                         ("lanes_distance_transform", lambda mp: H.test_parallel_distance_transform_under_lane_emulation(L, O, mp))],
        "kernel_edges": [(cid, lambda mp, fn=fn: fn(O, mp)) for cid, fn in kernel_edges.emu_cases()],
        "gain_maps": [(f"apply_{w}", lambda mp, w=w: GT.test_apply_against_the_compensators(L, O, w)) for w in ("1px", "ipp")]
        + [("feed", lambda mp: GT.test_maps_fed_from_thin_low_images(L, O)),
           ("device_twin", lambda mp: GT.test_device_twin_at_a_crop_offset(L, O)),
           ("timelapse", lambda mp: GT.test_timelapse_with_clipped_parts(L, O)),
           ("sharded", lambda mp: GT.test_sharded_owner_sets_the_gain(L, O))]
        + [(f"compositor_{k}", lambda mp, k=k: GT.test_compositor_set_gain(L, O, k)) for k in (3, 4)],
        "host_entries": [(f"{fn.__name__}[{a}]", lambda mp, fn=fn, a=a: fn(HE.hooked(L), *a)) for fn, a in HE.cases()],
    }


NAMES = ["rig_fuzz", "crop_fuzz", "shard_fuzz", "dropin_fuzz", "final_scale", "timelapse_fuzz", "fullres", "goldens",
         "setters", "lanes_blocks", "kernel_edges", "gain_maps", "host_entries"]


def run(lib_path, names, out=sys.stdout, only=None):
    """Run the named corpora on the library at lib_path; returns {corpus: (cases, [(case id, message)])}.  `only`: a set
    of "corpus:case id" to run instead of whole corpora."""
    import pytest

    from oracle import oracle as O
    from stitching_b200 import _lib

    O.build()
    L = _lib.bind(lib_path)
    _lib._lib = L  # what the use_emu fixture does, for the whole process
    table = corpora(L, O)
    res = {}
    for name in names:
        cases, failed, t0 = table[name], [], time.time()
        if only is not None:
            cases = [(cid, fn) for cid, fn in cases if f"{name}:{cid}" in only]
        for cid, fn in cases:
            with pytest.MonkeyPatch.context() as mp:
                try:
                    fn(mp)
                except Exception as e:  # noqa: BLE001 (every failure is reported with its case)
                    failed.append((cid, f"{type(e).__name__}: {e}"[:2000]))
                    traceback.print_exc(file=out)
        res[name] = (len(cases), failed)
        print(f"sweep {name}: {len(cases)} cases, {len(failed)} failed, {time.time() - t0:.0f} s", file=out, flush=True)
        for cid, msg in failed:
            print(f"  FAILED {name}[{cid}]: {msg}", file=out, flush=True)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--lib", default=os.path.join(ROOT, "tests", "emu", "libstitch_b200_emu.so"))
    ap.add_argument("--corpora", default=",".join(NAMES))
    ap.add_argument("--cases", default="", help="comma-separated corpus:case ids (replaces --corpora)")
    a = ap.parse_args()
    names = [n for n in a.corpora.split(",") if n]
    only = None
    if a.cases:
        only = {c for c in a.cases.split(",") if c}
        names = [n for n in NAMES if any(c.split(":", 1)[0] == n for c in only)]
    unknown = sorted(set(names) - set(NAMES))
    if unknown:
        ap.error(f"unknown corpora {unknown}; known: {NAMES}")
    print(f"sweep on {a.lib}, SB_EMU_FILL={os.environ.get('SB_EMU_FILL', '(unset)')}", flush=True)
    res = run(a.lib, names, only=only)
    total = sum(n for n, _ in res.values())
    bad = sum(len(f) for _, f in res.values())
    if only is not None and total != len(only):
        print(f"unknown cases: {total} of {len(only)} found", flush=True)
        bad += 1
    print(f"all corpora: {total} cases, {bad} failed", flush=True)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
