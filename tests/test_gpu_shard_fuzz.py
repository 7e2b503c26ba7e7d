"""Seeded random sharded rigs (tests/shard_fuzz.py) on the GPU, every strip bit for bit against the oracle summed in the
ranks' groups: all ranks on one device with the slabs moved by device copies through the transport hooks; the same
strips under the A/B switches SB_TILE=0 and SB_PD_BIN=0; and, with two or more GPUs, the real exchange (IPC pushes, direct
stores and the NCCL fallback) through sb_compositor_run."""
import os

import pytest

import fuzz_chain
import rig_fuzz
import shard_fuzz
import torchrun_job
from conftest import ROOT

pytestmark = pytest.mark.gpu

SEED = shard_fuzz.seed_from_env()


@pytest.mark.parametrize("k", range(len(shard_fuzz.gpu_ids())), ids=shard_fuzz.gpu_ids())
def test_shard_fuzz_on_one_gpu(cuda_lib, oracle, k):
    case = shard_fuzz.gpu_set(SEED)[k]
    imgs, ex = rig_fuzz.images(case), rig_fuzz.extras(case)
    ref = shard_fuzz.grouped_oracle(oracle, case, imgs, ex)
    got, sizes = shard_fuzz.hooks_run(case, imgs, ex, fuzz_chain.device_copy)
    shard_fuzz.check(case, got, sizes, ref, SEED)


def test_shard_fuzz_coverage_on_the_gpu(oracle):
    cs = shard_fuzz.gpu_set(SEED)
    rows = [(c, shard_fuzz.coverage(c)) for c in cs]
    print(f"\nshard fuzz coverage, GPU set (seed {SEED}, {len(cs)} cases):\n" + rig_fuzz.coverage_table(rows))
    reached = set().union(*(t for _, t in rows))
    want = {"world=2", "world=3", "world=4", "world=5", "world=8", "multiband", "feather", "empty strip", "column strips",
            "column strips reversed", "row strips", "row strips reversed", "slab at l>=2", "tile l0 with slab items",
            "tile l1 with slab items", "n == world", "n % world != 0", "nb=1", "nb=2..", "nb=max", "3+ ranks in a pixel",
            "gray blend mask", "odd pano width"}
    assert want <= reached, f"not reached: {sorted(want - reached)}"
    assert rig_fuzz.redraw_share(cs) < 1.0, f"{rig_fuzz.redraw_share(cs):.2f} rejected draws per case"


# -- A/B switches: read once per process, so each setting runs in a child process --------------------------------------
def _ab_cases(cs):
    """Multiband with slabs at the tile levels, with and without gray masks, and a feather rig."""
    tile = [k for k, c in enumerate(cs) if c.blender == "multiband" and "tile l0 with slab items" in shard_fuzz.coverage(c)]
    gray = [k for k in tile if any(m in ("ramp", "random") for m in cs[k].masks)]
    plain = [k for k in tile if all(m == "none" for m in cs[k].masks)]
    feather = [k for k, c in enumerate(cs) if c.blender == "feather"]
    return sorted({*gray[:1], *plain[:2], *feather[:1], len(cs) - 1})


def test_shard_ab_switches_give_identical_strips(cuda_lib):
    cs = shard_fuzz.gpu_set(SEED)
    picked = _ab_cases(cs)
    print("A/B cases: " + "; ".join(f"{k}: {cs[k].describe()}" for k in picked))
    fuzz_chain.ab_run("shard_fuzz:ab_arrays", [SEED, picked], [("SB_TILE", "0"), ("SB_PD_BIN", "0")], "SB_SHARD_FUZZ_SEED",
                      timeout=900)


# -- two or more GPUs: the real exchange ----------------------------------------------------------------------------------
WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import numpy as np
import torch.distributed as dist
import fuzz_chain, rig_fuzz, shard_fuzz
from stitching_b200 import Compositor
from stitching_b200 import dist as sbdist

rank, world = sbdist.init_comm_torchrun()
seed = int(sys.argv[2])
ks = [int(k) for k in sys.argv[3].split(",")]
cs = shard_fuzz.gpu_set(seed)
for k in ks:
    case = cs[k]
    imgs, ex = rig_fuzz.images(case), rig_fuzz.extras(case)
    c = Compositor(case.cams, case.sizes, case.wtype, case.blender, case.strength, rank=rank, world=world)
    fuzz_chain.set_extras(c, ex, range(c.first, c.first + c.count))
    c.upload(imgs[c.first: c.first + c.count])
    for _ in range(3):           # repeated steps reuse the slab buffers and the step-counted flags
        c.run()
    pano, mask = c.download()
    parts = [None] * world
    dist.all_gather_object(parts, (c.strip, c.strip_axis, pano, mask))
    c.close()
    if rank == 0:
        from oracle import oracle as O
        ref = shard_fuzz.grouped_oracle(O, case, imgs, ex)
        g = shard_fuzz.geometry(case)
        for r, (strip, axis, p, m) in enumerate(parts):
            assert strip == g["strips"][r] and axis == g["axis"], (k, r, strip, g["strips"][r])
            assert np.array_equal(p, shard_fuzz.cut(ref["panos"][r][0], strip, axis)), f"case {k} rank {r}: strip differs"
            assert np.array_equal(m, shard_fuzz.cut(ref["panos"][r][1], strip, axis)), f"case {k} rank {r}: mask differs"
        print("SHARD_FUZZ_OK", k, case.describe(), flush=True)
    dist.barrier()
sbdist.shutdown()
dist.destroy_process_group()
"""


def gpu_count():
    import test_gpu_sharded

    return test_gpu_sharded.gpu_count()


@pytest.mark.parametrize("peer", ["default", "0", "direct"])
def test_shard_fuzz_real_exchange(tmp_path, peer):
    n = gpu_count()
    if n < 2:
        pytest.skip(f"needs >= 2 GPUs, found {n}")
    world = 2 if n < 4 else 4
    cs = shard_fuzz.gpu_set(SEED)
    ks = [k for k, c in enumerate(cs) if c.world == world][:4]
    if not ks:
        pytest.skip(f"no case of world {world} in this seed")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    if peer != "default":
        env["SB_PEER"] = peer
    out = torchrun_job.run(world, 29627, script, [ROOT, SEED, ",".join(map(str, ks))], env, timeout=900)
    print(out["stdout"][-3000:])
    assert not out["timed_out"] and not out["leftover"], out["stdout"][-3000:] + out["stderr"][-3000:]
    assert out["returncode"] == 0 and out["stdout"].count("SHARD_FUZZ_OK") == len(ks), out["stdout"][-3000:] + out["stderr"][-3000:]
