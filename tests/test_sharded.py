"""Multi-GPU sharded composite (SURVEY 8e): host logic and kernel roles without GPUs, and the rendezvous plumbing.

The product sources run through tests/emu (serial CUDA stand-in); the slabs that NCCL would move are copied by the
test through the transport hooks (sb_compositor_shard_phase / _shard_slab).  The NCCL path itself is covered on
real GPUs by tests/test_gpu_sharded.py.
"""
import ctypes as C
import os

import numpy as np
import pytest

import replay
import shard_fuzz
import torchrun_job
from conftest import ROOT
from stitching_b200 import Compositor, rigs


def run_sharded(cfg, cams, imgs, world, copy):
    """All ranks of a fixed rig through the transport hooks (shard_fuzz.hooks_run), the slabs moved with `copy`:
    (panorama, mask, slab bytes moved) of the strips put together."""
    case = shard_fuzz.config_case(cfg, world, cams)
    got, sizes = shard_fuzz.hooks_run(case, imgs, [(None, None, None)] * case.n, copy)
    assert sum(g["count"] for g in got) == len(cams) and [g["first"] for g in got] == sorted(g["first"] for g in got)
    assert all(sn == dn for sn, dn in sizes.values()), "both sides must agree on the slab size"
    axis = got[0]["axis"]
    assert all(g["axis"] == axis for g in got)
    los = sorted(g["strip"] for g in got)  # spatial order of the strips (feather may run against the rank order)
    assert los[0][0] == 0 and all(a[1] == b[0] for a, b in zip(los, los[1:])) and los[-1][1] == got[0]["roi"][3 if axis else 2]
    pano, mask = shard_fuzz.assemble(got)
    return pano, mask, sum(sn for sn, _ in sizes.values())


def assert_grouped(oracle, cfg, cams, imgs, world, pano, mask):
    """The strips put together equal the oracle summed in the ranks' groups (tests/shard_fuzz.py) bit for bit: the
    int16 sums are exact under any grouping and the float weight sums are grouped as the ranks group them.  Returns
    the oracle's num_bands."""
    ref_pano, ref_mask, nb = shard_fuzz.grouped_panorama(oracle, shard_fuzz.config_case(cfg, world, cams), imgs)
    replay.assert_exact(mask, ref_mask, f"sharded x{world} mask")
    replay.assert_exact(pano, ref_pano, f"sharded x{world} pano")
    return nb


@pytest.mark.parametrize("world", [2, 3, 4])
def test_sharded_equals_grouped_oracle(use_emu, oracle, world):
    cfg = rigs.config("cfg2", 16)
    cams = cfg["cameras"]
    imgs = [rigs.noise_image(cfg["h"], cfg["w"], 70 + i) if i % 2 else rigs.synth_image(cfg["h"], cfg["w"], 70 + i) for i in range(len(cams))]
    pano, mask, moved = run_sharded(cfg, cams, imgs, world, lambda d, s, n: C.memmove(d, s, n))
    assert moved > 0
    assert assert_grouped(oracle, cfg, cams, imgs, world, pano, mask) >= 2


def test_sharded_cylindrical_many_images(use_emu, oracle):
    cfg = rigs.config("cfg3", 20)  # 32 images, cylindrical (BASELINE configs[2] layout: 4 images per rank at world 8)
    cams = cfg["cameras"]
    imgs = [rigs.synth_image(cfg["h"], cfg["w"], 5 + i) for i in range(len(cams))]
    pano, mask, _ = run_sharded(cfg, cams, imgs, 8, lambda d, s, n: C.memmove(d, s, n))
    assert_grouped(oracle, cfg, cams, imgs, 8, pano, mask)


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_feather_grid(use_emu, oracle, world):
    """BASELINE configs[4]: 4x4 plane grid, feather blender; image blocks are grid rows, so the ranks own ROW strips."""
    cfg = rigs.config("cfg5", 12)
    cams = cfg["cameras"]
    imgs = [rigs.noise_image(cfg["h"], cfg["w"], 30 + i) if i % 3 == 0 else rigs.synth_image(cfg["h"], cfg["w"], 30 + i) for i in range(len(cams))]
    pano, mask, moved = run_sharded(cfg, cams, imgs, world, lambda d, s, n: C.memmove(d, s, n))
    assert moved > 0
    assert_grouped(oracle, cfg, cams, imgs, world, pano, mask)


def test_sharded_feather_side_by_side(use_emu, oracle):
    """Feather on a single-row rig: the blocks lie side by side and the strips are columns, as for multiband."""
    cfg = dict(rigs.config("cfg2", 16), blender="feather")
    cams = cfg["cameras"]
    imgs = [rigs.synth_image(cfg["h"], cfg["w"], 11 + i) for i in range(len(cams))]
    pano, mask, _ = run_sharded(cfg, cams, imgs, 2, lambda d, s, n: C.memmove(d, s, n))
    assert_grouped(oracle, cfg, cams, imgs, 2, pano, mask)


def test_sharded_rejects_what_it_cannot_do(use_emu):
    from stitching_b200 import StitchingError

    cfg = rigs.config("cfg5", 12)  # "no" blender: nothing to exchange, not sharded
    with pytest.raises(StitchingError):
        Compositor(cfg["cameras"], [(cfg["w"], cfg["h"])] * cfg["n"], cfg["warper"], "no", cfg["strength"], rank=0, world=2)
    cfg = rigs.config("cfg2", 16)
    c = Compositor(cfg["cameras"], [(cfg["w"], cfg["h"])] * cfg["n"], cfg["warper"], cfg["blender"], cfg["strength"], rank=1, world=2)
    with pytest.raises(StitchingError):
        c.upload([rigs.noise_image(cfg["h"], cfg["w"], 0)] * cfg["n"])  # only the own block may be uploaded
    c.close()


def test_sharded_create_rejects_an_unknown_blend_kind(use_emu):
    """A sharded create checks the rig like a single-GPU one: a blend kind outside sb_blend_kind is refused, not built as
    a feather blend."""
    from stitching_b200 import Warper, _lib

    cams = rigs.yaw_ring(4, 64, 48, 70, 25)  # blocks run left to right: a feather blend of this rig can be sharded
    K = np.ascontiguousarray(np.stack([Warper.get_K(cam, 1) for cam in cams]).astype(np.float32))
    R = np.ascontiguousarray(np.stack([cam.R for cam in cams]).astype(np.float32))
    w, h = (C.c_int * 4)(*[64] * 4), (C.c_int * 4)(*[48] * 4)

    def create(kind):
        rig = _lib.Rig(4, _lib.WARP_TYPES["spherical"], 70.0, kind, 5.0, w, h, K.ctypes.data_as(_lib.c_float_p),
                       R.ctypes.data_as(_lib.c_float_p))
        return use_emu.sb_compositor_create(C.byref(rig), C.byref(_lib.CompositorOpts(rank=0, world=2)))

    c = create(_lib.BLEND_KINDS["feather"])
    assert c
    use_emu.sb_compositor_destroy(c)
    assert not create(7)
    assert b"invalid" in use_emu.sb_last_error()


GLOO_WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1])
import torch.distributed as dist
dist.init_process_group(backend="gloo")
rank, world = dist.get_rank(), dist.get_world_size()
# the rendezvous used by stitching_b200.dist.init_comm_torchrun: rank 0's 128-byte id reaches every rank
payload = bytes(range(128)) if rank == 0 else None
box = [payload]
dist.broadcast_object_list(box, src=0)
assert box[0] == bytes(range(128))
# every rank derives the same partition and strip geometry from the same rig (host logic, emulation build)
from stitching_b200 import _lib, Compositor, rigs
_lib._lib = _lib.bind(os.path.join(sys.argv[1], "tests", "emu", "libstitch_b200_emu.so"))
cfg = rigs.config("cfg2", 16)
c = Compositor(cfg["cameras"], [(cfg["w"], cfg["h"])] * cfg["n"], cfg["warper"], cfg["blender"], cfg["strength"], rank=rank, world=world)
info = [None] * world
dist.all_gather_object(info, (c.first, c.count, c.strip, [c.shard_slab(p, True)[1] for p in range(world) if p != rank],
                              [c.shard_slab(p, False)[1] for p in range(world) if p != rank]))
if rank == 0:
    assert [i[0] for i in info] == [0, 4] and [i[1] for i in info] == [4, 4]
    assert info[0][2][1] == info[1][2][0]          # strips meet
    assert info[0][3] == info[1][4] and info[1][3] == info[0][4]   # send size on one side == receive size on the other
    print("GLOO_OK")
dist.destroy_process_group()
"""


def test_world_size_2_gloo_rendezvous_and_partition(emu_lib, tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(GLOO_WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    out = torchrun_job.run(2, 29613, script, [ROOT], env, timeout=300)
    assert not out["timed_out"] and not out["leftover"], out["stdout"][-2000:] + out["stderr"][-2000:]
    assert out["returncode"] == 0 and "GLOO_OK" in out["stdout"], out["stdout"][-2000:] + out["stderr"][-2000:]


STUCK_WORKER = r"""
import signal, sys, time
signal.signal(signal.SIGTERM, signal.SIG_IGN)   # a rank that does not stop when asked
print("STARTED", flush=True)
time.sleep(3600)
"""


def test_torchrun_job_timeout_leaves_no_process(tmp_path):
    """The torchrun helper of the multi-GPU tests: a job that overruns its timeout is torn down -- the launcher and every
    worker, also workers that ignore SIGTERM -- and reported as timed out (CPU only: the workers just sleep)."""
    script = tmp_path / "stuck.py"
    script.write_text(STUCK_WORKER)
    out = torchrun_job.run(2, 29617, script, [], dict(os.environ, MASTER_ADDR="127.0.0.1"), timeout=15, grace=3)
    assert out["timed_out"], out["stdout"][-2000:] + out["stderr"][-2000:]
    assert out["stdout"].count("STARTED") == 2, out["stdout"][-2000:] + out["stderr"][-2000:]
    assert out["leftover"] == []
