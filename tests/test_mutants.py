"""The fault catalogue of tests/mutants.py against the emulation build: every snippet is present exactly once, the
unmutated library passes every entry's killers, and every mutant fails at least one of them (a crash or a timeout counts).
The mutants are built and judged in parallel child processes (one per core) at the first test that needs them; about
70 s on an 8-core machine."""
import concurrent.futures as cf
import os
import tempfile

import pytest

import mutants

CPU = [m for m in mutants.CATALOGUE if m.killers]
TIMEOUT = 600


@pytest.mark.parametrize("m", mutants.CATALOGUE, ids=[m.id for m in mutants.CATALOGUE])
def test_snippet_present_once(m):
    assert mutants.check_snippet(m) == 1, f"{m.id}: the snippet must occur exactly once in {m.file}"
    assert m.old != m.new and m.breaks
    assert m.killers or m.gpu, f"{m.id}: no killer"
    assert m.kind in mutants.KINDS
    assert not m.gpu or m.value_only, f"{m.id}: only value-only mutations may run on a GPU"
    assert not (m.san and m.gpu), f"{m.id}: a memory fault may not run on a GPU"


@pytest.fixture(scope="module")
def verdicts():
    """{id or None (the unmutated library): (passed, failed case ids, output)}"""
    jobs = os.cpu_count() or 4
    with tempfile.TemporaryDirectory(prefix="sb_mutants_") as work:
        b = mutants.EmuBuilder(work, jobs)
        bs = mutants.EmuBuilder(os.path.join(work, "san"), jobs, san=True)
        every = sorted({k for m in CPU for k in m.killers})
        every_san = sorted({k for m in CPU if m.san for k in m.killers})

        def one(m):
            if m is None:
                return None, mutants.run_cases(b.lib, every, TIMEOUT)
            if m == "san":  # the sanitizer build of the unmutated sources passes the killers of the memory faults
                return "san", mutants.run_cases(bs.lib, every_san, TIMEOUT, True)
            return m.id, mutants.run_cases((bs if m.san else b).mutant(m), m.killers, TIMEOUT, m.san)

        with cf.ThreadPoolExecutor(jobs) as ex:
            return dict(ex.map(one, [None, "san"] + CPU))


@pytest.mark.parametrize("build", [None, "san"], ids=["plain", "sanitizer"])
def test_unmutated_library_passes_every_killer(verdicts, build):
    ok, failed, out = verdicts[build]
    assert ok, f"killers failing on the unmutated library: {failed}\n{out[-3000:]}"


@pytest.mark.parametrize("m", CPU, ids=[m.id for m in CPU])
def test_mutant_is_killed(verdicts, m):
    ok, failed, out = verdicts[m.id]
    assert not ok, f"{m.id} ({m.breaks}) survived {m.killers}"
