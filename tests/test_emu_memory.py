"""The emulation corpora (tests/emu_sweep.py) on dirty and fenced memory, in child processes that run in parallel:

* once per fill byte, on the emulation build whose device and page-locked allocations start filled with that byte
  (SB_EMU_FILL).  Large mallocs are fresh zero pages, and zero times a weight of zero is zero, so a kernel that reads
  memory no step wrote passes every other test; 0xff (NaN floats, int16 -1), 0x7f (3.4e38, int16 32639) do not
  hide it.  SB_EMU_FILLS=0xa5,... selects other fills (0x00 is what the rest of the suite runs);
* once on libstitch_b200_emu_san.so, the same sources under AddressSanitizer and UBSan (float-cast-overflow
  included), with libasan preloaded into the child only: the run must exit 0 with no sanitizer report.  It sees
  overruns of every buffer the library allocates on its own -- sources, word sources, resized frames, RGBM, tables,
  maps, gains, outputs, paste and slab buffers, pooled temporaries -- but not overruns between the buffers carved out
  of the one plan arena (sb_plan.cpp), which is a single allocation to it;
* a self-check that the sanitizer child really is instrumented: a probe built with the same flags and preloaded the
  same way must be stopped on a one-past-the-end read and reported on an out-of-range float -> int conversion.

Every case of every run must equal the oracle bit for bit, exactly as its own test file checks it."""
import os
import re
import subprocess
import sys

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")
SWEEP = os.path.join(ROOT, "tests", "emu_sweep.py")
FILLS = [f.strip() for f in os.environ.get("SB_EMU_FILLS", "0xff,0x7f").split(",") if f.strip()]
ASAN_OPTIONS = "detect_leaks=0:halt_on_error=1:abort_on_error=0"
REPORT = re.compile(r"ERROR: AddressSanitizer|runtime error:|SUMMARY: \w+Sanitizer")
TIMEOUT = 1800


def _python():
    return [sys.executable] + (["-s"] if sys.flags.no_user_site else [])


def _san_env():
    """The environment of an instrumented child: the runtime of the compiler that built the library preloaded (the
    parent's python is not instrumented), leaks not checked (the interpreter keeps its objects at exit)."""
    cxx = os.environ.get("SAN_CXX", "g++")
    rt = subprocess.check_output([cxx, "-print-file-name=libasan.so"], text=True).strip()
    assert os.path.isabs(rt) and os.path.exists(rt), f"{cxx} names no AddressSanitizer runtime ({rt!r})"
    env = dict(os.environ, LD_PRELOAD=os.path.realpath(rt), ASAN_OPTIONS=ASAN_OPTIONS, UBSAN_OPTIONS="print_stacktrace=1")
    env.pop("SB_EMU_FILL", None)
    return env


def _start(log_dir, name, lib, env):
    log = open(os.path.join(log_dir, f"{name}.log"), "w+")
    p = subprocess.Popen(_python() + [SWEEP, "--lib", lib], cwd=ROOT, env=env, stdout=log, stderr=subprocess.STDOUT)
    return p, log


def _finish(child):
    p, log = child
    try:
        rc = p.wait(timeout=TIMEOUT)
    except subprocess.TimeoutExpired:
        p.kill()
        p.wait()
        rc = "timeout"
    log.seek(0)
    return rc, log.read()


@pytest.fixture(scope="module")
def children(oracle, tmp_path_factory):
    """Every sweep at once: the fills start while the sanitizer build compiles."""
    d = tmp_path_factory.mktemp("emu_memory")
    subprocess.check_call(["make", "-C", EMU, "-s", "libstitch_b200_emu.so"])
    procs = {}
    try:
        for f in FILLS:
            procs[f"fill {f}"] = _start(d, f"fill_{f}", os.path.join(EMU, "libstitch_b200_emu.so"), dict(os.environ, SB_EMU_FILL=f))
        subprocess.check_call(["make", "-C", EMU, "-s", "libstitch_b200_emu_san.so", "san_probe.so"])
        procs["sanitizer"] = _start(d, "sanitizer", os.path.join(EMU, "libstitch_b200_emu_san.so"), _san_env())
        yield procs
    finally:  # also when the sanitizer build fails: no sweep outlives the fixture
        for p, log in procs.values():
            if p.poll() is None:
                p.kill()
                p.wait()
            log.close()


def _check_sweep(name, rc, out):
    import emu_sweep

    lines = [ln for ln in out.splitlines() if ln.startswith("sweep ")]
    print(f"\n{name}:\n" + "\n".join(lines))
    counts = {m.group(1): (int(m.group(2)), int(m.group(3))) for m in (re.match(r"sweep (\w+): (\d+) cases, (\d+) failed", ln) for ln in lines) if m}
    assert sorted(counts) == sorted(emu_sweep.NAMES), f"{name}: corpora run {sorted(counts)}\n{out[-4000:]}"
    failed = [ln for ln in out.splitlines() if ln.lstrip().startswith("FAILED ")]
    assert rc == 0 and not failed, f"{name}: exit {rc}\n" + "\n".join(failed) + f"\n{out[-4000:]}"
    assert all(n > 0 and f == 0 for n, f in counts.values()), counts


@pytest.mark.parametrize("fill", FILLS)
def test_sweep_on_filled_allocations(children, fill):
    """Every case equals the oracle when every allocation starts as `fill`."""
    rc, out = _finish(children[f"fill {fill}"])
    assert out.startswith("sweep on ") and f"SB_EMU_FILL={fill}" in out.splitlines()[0], f"fill {fill}: exit {rc}\n{out[-4000:]}"
    _check_sweep(f"fill {fill}", rc, out)


def test_sweep_under_address_and_undefined_behaviour_sanitizers(children):
    """Every case equals the oracle on the instrumented build, which exits 0 and reports nothing."""
    rc, out = _finish(children["sanitizer"])
    reports = [ln for ln in out.splitlines() if REPORT.search(ln)]
    assert not reports, "sanitizer report:\n" + out[-8000:]
    _check_sweep("sanitizer", rc, out)


def test_sanitizer_child_is_instrumented(children):
    """A child started like the sanitizer sweep reports an out-of-range float -> int conversion and is stopped by a
    one-past-the-end heap read, each named with its function and file."""
    probe = os.path.join(EMU, "san_probe.so")
    code = ("import ctypes, sys\nL = ctypes.CDLL(sys.argv[1])\nL.sb_probe_cast.argtypes = [ctypes.c_float]\n"
            "L.sb_probe_cast(3e9)\nL.sb_probe_overread(24)\nprint('probe survived')\n")
    r = subprocess.run(_python() + ["-c", code, probe], env=_san_env(), capture_output=True, text=True, timeout=120)
    out = r.stdout + r.stderr
    assert "probe survived" not in out and r.returncode != 0, out
    assert re.search(r"san_probe\.cpp:\d+:\d+: runtime error: .*outside the range of representable values", out), out
    assert "ERROR: AddressSanitizer: heap-buffer-overflow" in out and "READ of size 1" in out, out
    assert re.search(r"in sb_probe_overread .*san_probe\.cpp:\d+", out), out
