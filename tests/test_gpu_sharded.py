"""The sharded composite over real GPUs: torchrun, one rank per GPU, slabs exchanged with NCCL send/recv.

Needs >= 2 GPUs on the box (gpurun --gpus 2); on a 1-GPU box the test is skipped -- the kernel roles are then still
covered by tests/test_gpu_parity.py::test_sharded_roles_on_one_gpu and the host logic by tests/test_sharded.py.
"""
import os

import pytest

import torchrun_job
from conftest import ROOT

pytestmark = pytest.mark.gpu

WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1])
import numpy as np
import torch.distributed as dist
from stitching_b200 import Compositor, rigs
from stitching_b200 import dist as sbdist

rank, world = sbdist.init_comm_torchrun()
name, sd = sys.argv[2], int(sys.argv[3])
cfg = rigs.config(name, sd)
cams = cfg["cameras"][: int(sys.argv[4])]
sizes = [(cfg["w"], cfg["h"])] * len(cams)
imgs = [rigs.noise_image(cfg["h"], cfg["w"], 70 + i) if i % 2 else rigs.synth_image(cfg["h"], cfg["w"], 70 + i) for i in range(len(cams))]
c = Compositor(cams, sizes, cfg["warper"], cfg["blender"], cfg["strength"], rank=rank, world=world)
c.upload(imgs[c.first: c.first + c.count])
for _ in range(3):           # repeated steps reuse the slab buffers
    c.run()
pano, mask = c.download()
ms, launches = c.time(5)
parts = [None] * world
dist.all_gather_object(parts, (c.strip, pano, mask))
if rank == 0:
    parts.sort(key=lambda p: p[0])   # spatial order of the strips (a feather grid may run against the rank order)
    ax = 0 if c.strip_axis else 1
    full = np.concatenate([p[1] for p in parts], axis=ax)
    fmask = np.concatenate([p[2] for p in parts], axis=ax)
    # the oracle summed in the ranks' groups (tests/shard_fuzz.py), bit for bit
    sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
    import shard_fuzz
    from oracle import oracle as O
    ref, rmask, _ = shard_fuzz.grouped_panorama(O, shard_fuzz.config_case(cfg, world, cams), imgs)
    assert full.shape == ref.shape and np.array_equal(fmask, rmask), (full.shape, ref.shape)
    assert np.array_equal(full, ref), int((full != ref).sum())
    print("SHARDED_OK", name, world, "ranks; step ms", ms / 5, dict((k, round(v, 3)) for k, v in launches))
c.close()
sbdist.shutdown()
dist.destroy_process_group()
"""


def gpu_count():
    try:
        import pynvml

        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetCount()
    except Exception:  # noqa: BLE001
        return len([d for d in os.listdir("/dev") if d.startswith("nvidia") and d[6:].isdigit()])


@pytest.mark.parametrize("name,scale_down,n_images", [("cfg2", 2, 8), ("cfg3", 4, 16), ("cfg5", 1, 16)])
def test_nccl_sharded_composite(tmp_path, name, scale_down, n_images):
    n = gpu_count()
    if n < 2:
        pytest.skip(f"needs >= 2 GPUs, found {n}")
    world = 2 if n < 4 else 4
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    out = torchrun_job.run(world, 29621, script, [ROOT, name, scale_down, n_images], dict(os.environ, MASTER_ADDR="127.0.0.1"),
                           timeout=900)
    print(out["stdout"][-1500:])
    assert not out["timed_out"] and not out["leftover"], out["stdout"][-3000:] + out["stderr"][-3000:]
    assert out["returncode"] == 0 and "SHARDED_OK" in out["stdout"], out["stdout"][-3000:] + out["stderr"][-3000:]
