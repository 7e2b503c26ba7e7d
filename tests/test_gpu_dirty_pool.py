"""The compositor paths on a dirty memory pool, on the GPU: every result equals the oracle when the pool's pages hold a
fill byte instead of the fresh zeros a test process mostly starts with.

sb_init sets the device's default pool to keep what is freed (release threshold: all of it), so a long-running process
hands its kernels pages an earlier caller wrote.  Each child process here, one per fill (0x00, 0xff, 0x7f), poisons that
pool through the driver API before every case -- cuMemAllocAsync of POOL_BYTES, cuMemsetD8Async(fill), cuMemFreeAsync,
synchronize -- and checks with probe allocations from the same pool that the fill is what they read back (or the test
would pass on clean pages).  The cases, each created on freshly poisoned pages: slices of the GPU rig, crop, drop-in,
final-scale, timelapse and shard fuzz sets as their own test files check them, the sharded roles on one GPU with slabs
moved by sb_device_copy into receive buffers nobody clears, a scaled cfg2 rig pipelined over more submits than it has
buffer sets, and the Warper / Blender one-shot calls that run on pooled temporaries."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
import traceback

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILLS = ["0x00", "0xff", "0x7f"]
POOL_BYTES = 1 << 30                       # poisoned per case: far above what any case here allocates
PROBES = (4 << 10, 1 << 20, 64 << 20)
CU_MEMPOOL_ATTR_RELEASE_THRESHOLD, CU_MEMPOOL_ATTR_RESERVED_MEM_CURRENT = 4, 5
CU_STREAM_NON_BLOCKING = 1
TIMEOUT = 1200


# -- the child: poison, probe, run ----------------------------------------------------------------------------------------
class DirtyPool:
    """The default memory pool of the current device, filled with one byte through the driver API."""

    def __init__(self, fill):
        self.fill = fill
        cu = self.cu = C.CDLL("libcuda.so.1")
        cu.cuMemAllocAsync.argtypes = [C.POINTER(C.c_uint64), C.c_size_t, C.c_void_p]
        cu.cuMemsetD8Async.argtypes = [C.c_uint64, C.c_ubyte, C.c_size_t, C.c_void_p]
        cu.cuMemFreeAsync.argtypes = [C.c_uint64, C.c_void_p]
        cu.cuMemcpyDtoH_v2.argtypes = [C.c_void_p, C.c_uint64, C.c_size_t]
        cu.cuDeviceGetDefaultMemPool.argtypes = [C.POINTER(C.c_void_p), C.c_int]
        cu.cuMemPoolGetAttribute.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        cu.cuStreamCreate.argtypes = [C.POINTER(C.c_void_p), C.c_uint]
        dev = C.c_int()
        self._ok(cu.cuCtxGetDevice(C.byref(dev)), "cuCtxGetDevice (sb_init made the device's context current)")
        self.pool = C.c_void_p()
        self._ok(cu.cuDeviceGetDefaultMemPool(C.byref(self.pool), dev.value), "cuDeviceGetDefaultMemPool")
        # the probes allocate on a stream of their own, non-blocking like the library's (sb_context.cpp): what they read
        # back is what the pool hands to another stream after the poison, not only to the stream that freed it
        self.stream = C.c_void_p()
        self._ok(cu.cuStreamCreate(C.byref(self.stream), CU_STREAM_NON_BLOCKING), "cuStreamCreate")

    def _ok(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed: CUresult {rc}")

    def attr(self, a):
        v = C.c_uint64()
        self._ok(self.cu.cuMemPoolGetAttribute(self.pool, a, C.byref(v)), "cuMemPoolGetAttribute")
        return v.value

    def poison(self):
        p = C.c_uint64()
        self._ok(self.cu.cuMemAllocAsync(C.byref(p), POOL_BYTES, None), "cuMemAllocAsync")
        self._ok(self.cu.cuMemsetD8Async(p, self.fill, POOL_BYTES, None), "cuMemsetD8Async")
        self._ok(self.cu.cuMemFreeAsync(p, None), "cuMemFreeAsync")
        self._ok(self.cu.cuCtxSynchronize(), "cuCtxSynchronize")

    def probe(self, nbytes):
        """An allocation from the pool, read back before anything writes it: {byte value: count}."""
        p = C.c_uint64()
        host = np.empty(nbytes, np.uint8)
        self._ok(self.cu.cuMemAllocAsync(C.byref(p), nbytes, self.stream), "cuMemAllocAsync (probe)")
        self._ok(self.cu.cuCtxSynchronize(), "cuCtxSynchronize")
        self._ok(self.cu.cuMemcpyDtoH_v2(host.ctypes.data, p, nbytes), "cuMemcpyDtoH")
        self._ok(self.cu.cuMemFreeAsync(p, self.stream), "cuMemFreeAsync (probe)")
        self._ok(self.cu.cuCtxSynchronize(), "cuCtxSynchronize")
        vals, counts = np.unique(host, return_counts=True)
        return {int(v): int(c) for v, c in zip(vals, counts)}


def _pipelined_cfg2(L, O):
    """A scaled cfg2 rig, six submits with two in flight over the compositor's buffer sets, every result against the
    oracle of its own batch."""
    import replay
    from stitching_b200 import Compositor, rigs
    from test_gpu_parity import assert_parity

    cfg = rigs.config("cfg2", 5)
    cams = cfg["cameras"]
    c = Compositor(cams, [(cfg["w"], cfg["h"])] * len(cams), cfg["warper"], cfg["blender"], cfg["strength"])
    try:
        _, _, pw, ph = c.roi
        raw = [[rigs.noise_image(cfg["h"], cfg["w"], 300 + 10 * b + i) for i in range(len(cams))] for b in range(6)]
        batches = []
        for b in raw:
            pinned = [c.pinned_empty(img.shape) for img in b]
            for p, img in zip(pinned, b):
                p[...] = img
            batches.append(pinned)
        outs = [(c.pinned_empty((ph, pw, 3)), c.pinned_empty((ph, pw))) for _ in batches]
        tickets = []
        for k, b in enumerate(batches):
            if k >= 2:
                c.wait(tickets[k - 2])
            tickets.append(c.submit(b, *outs[k]))
        for t in tickets[-2:]:
            c.wait(t)
        for k, b in enumerate(raw):
            ref = replay.oracle_composite(O, cfg, cams, b)
            assert_parity(outs[k][0], ref["pano"], f"pipelined cfg2 step {k} pano")
            assert np.array_equal(outs[k][1], ref["pmask"]), f"pipelined cfg2 step {k} mask"
    finally:
        c.close()


def cases(L, O):
    """[(case id, fn())]: each a call of an existing GPU test function (or the pipelined cfg2 run above)."""
    import dropin_fuzz
    import rig_fuzz
    import test_gpu_crop as GC
    import test_gpu_dropin_fuzz as GD
    import test_gpu_final_scale as GF
    import test_gpu_parity as GP
    import test_gpu_rig_fuzz as GR
    import test_gpu_shard_fuzz as GS
    import test_gpu_timelapse_compositor as GT
    import test_zz_gpu_gain as GG

    n_rig = len(rig_fuzz.gpu_ids())
    out = [(f"rig_fuzz[{k}]", lambda k=k: GR.test_rig_fuzz_against_oracle(L, O, k)) for k in [0, 1, 2, 3] + list(range(rig_fuzz.GPU_COUNT, n_rig))]
    out += [(f"crop_fuzz[{k}]", lambda k=k: GC.test_crop_fuzz_against_oracle(L, O, k)) for k in (0, 1, 2, GC.GPU_COUNT, GC.GPU_COUNT + 1)]
    out += [(f"dropin_fuzz[{k}]", lambda k=k: GD.test_dropin_fuzz_against_oracle_and_compositor(L, O, k))
            for k in (0, n_rig - 1, n_rig, n_rig + 1, dropin_fuzz.gpu_count() - 3, dropin_fuzz.gpu_count() - 2, dropin_fuzz.gpu_count() - 1)]
    out += [("final_scale kernel[0]", lambda: GF.test_resize_kernel_against_oracle(L, O, 0))]
    out += [(f"final_scale rig[{k}]", lambda k=k: GF.test_resized_compositor_equals_prefed(L, O, k)) for k in (0, 1, GF.RIG_COUNT)]
    out += [("final_scale crop[0]", lambda: GF.test_resized_crop_equals_prefed(L, O, 0)),
            ("final_scale sharded", lambda: GF.test_resized_sharded_roles_on_one_gpu(L, O)),
            ("final_scale pipelined", lambda: GF.test_pipelined_steps(L, O))]
    out += [(f"timelapse_fuzz[{k}]", lambda k=k: GT.test_fuzz_against_oracle(L, O, k)) for k in (0, 1, 2, 3, GT.COUNT, GT.COUNT + 1)]
    out += [(f"shard_fuzz[{k}]", lambda k=k: GS.test_shard_fuzz_on_one_gpu(L, O, k)) for k in (0, 1, 2, 3, GS.shard_fuzz.GPU_COUNT, GS.shard_fuzz.GPU_COUNT + 1)]
    out += [("sharded roles cfg2 x2", lambda: GP.test_sharded_roles_on_one_gpu(L, O, "cfg2", 4, 2)),
            ("sharded roles cfg3 x8", lambda: GP.test_sharded_roles_on_one_gpu(L, O, "cfg3", 8, 8)),
            ("pipelined cfg2", lambda: _pipelined_cfg2(L, O)),
            ("setters between submits", lambda: GP.test_setters_between_pipelined_submits(L)),
            ("warper goldens", lambda: GP.test_warper_goldens(L)),
            ("blender goldens", lambda: GP.test_blender_goldens(L)),
            ("e2e goldens", lambda: GP.test_e2e_goldens(L)),
            ("warp fuzz", lambda: GP.test_warp_fuzz_against_oracle(L, O)),
            ("blend fuzz", lambda: GP.test_blend_fuzz_against_oracle(L, O)),
            ("gain goldens and fuzz", lambda: GG.test_gain_apply_goldens_and_fuzz(L, O)),
            ("gains out of the int range", lambda: GG.test_gains_out_of_the_int_range(L, O)),
            ("timelapser goldens and fuzz", lambda: GG.test_timelapser_goldens_and_fuzz(L, O))]
    return out


def child(fill):
    for p in (ROOT, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    from oracle import oracle as O
    from stitching_b200 import _lib

    O.build()
    L = _lib.lib()
    _lib.check(L.sb_init(0), "sb_init")
    pool = DirtyPool(fill)
    threshold = pool.attr(CU_MEMPOOL_ATTR_RELEASE_THRESHOLD)
    failed, probes, t0 = [], [], time.time()

    def poison_and_probe(sizes):
        pool.poison()
        for n in sizes:
            h = pool.probe(n)
            probes.append(n)
            if h != {fill: n}:
                raise AssertionError(f"probe of {n} bytes after poisoning with {fill:#04x} reads {h}")

    poison_and_probe(PROBES)
    reserved0 = pool.attr(CU_MEMPOOL_ATTR_RESERVED_MEM_CURRENT)
    todo = cases(L, O)
    for cid, fn in todo:
        try:
            poison_and_probe(PROBES[:1])
            fn()
            # a pool that grew gave the case fresh pages beyond the poisoned ones
            grown = pool.attr(CU_MEMPOOL_ATTR_RESERVED_MEM_CURRENT)
            if grown != reserved0:
                raise AssertionError(f"the pool grew from {reserved0} to {grown} bytes: the case ran partly on unpoisoned pages")
        except Exception as e:  # noqa: BLE001 (every failure is reported with its case)
            traceback.print_exc()
            failed.append(f"{cid}: {type(e).__name__}: {e}"[:2000])
    poison_and_probe(PROBES)
    print(json.dumps(dict(fill=fill, cases=len(todo), failed=failed, probes=len(probes), release_threshold=threshold,
                          reserved_mb=[reserved0 >> 20, pool.attr(CU_MEMPOOL_ATTR_RESERVED_MEM_CURRENT) >> 20],
                          seconds=round(time.time() - t0, 1))), flush=True)
    return 1 if failed else 0


# -- the test: one child per fill, in parallel ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def children(cuda_lib, oracle, tmp_path_factory):
    d = tmp_path_factory.mktemp("dirty_pool")
    procs = {}
    for f in FILLS:
        log = open(os.path.join(d, f"fill_{f}.log"), "w+")
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--fill", f]
        procs[f] = (subprocess.Popen(cmd, cwd=ROOT, stdout=log, stderr=subprocess.STDOUT), log)
    yield procs
    for p, log in procs.values():
        if p.poll() is None:
            p.kill()
            p.wait()
        log.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fill", FILLS)
def test_compositor_paths_on_a_dirty_pool(children, fill):
    p, log = children[fill]
    try:
        rc = p.wait(timeout=TIMEOUT)
    except subprocess.TimeoutExpired:
        p.kill()
        p.wait()
        rc = "timeout"
    log.seek(0)
    out = log.read()
    last = [ln for ln in out.splitlines() if ln.startswith("{")]
    assert last, f"fill {fill}: exit {rc}, no summary\n{out[-6000:]}"
    res = json.loads(last[-1])
    print(f"\nfill {fill}: {res}")
    assert res["release_threshold"] == 2 ** 64 - 1, "sb_init keeps every freed block in the pool"
    assert res["probes"] >= res["cases"] + 2 * len(PROBES), res
    assert res["reserved_mb"][0] == res["reserved_mb"][1] == POOL_BYTES >> 20, res
    assert rc == 0 and not res["failed"], f"fill {fill}:\n" + "\n".join(res["failed"]) + f"\n{out[-6000:]}"


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description="one dirty-pool run (a child of test_compositor_paths_on_a_dirty_pool)")
    ap.add_argument("--fill", required=True)
    sys.exit(child(int(ap.parse_args().fill, 0)))
