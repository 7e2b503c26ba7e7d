"""Run a torchrun job from a test with a fixed timeout, and leave no process behind (helper module: no tests in here).

torchrun starts its workers in sessions of their own, so killing the launcher alone would orphan them: a worker stuck in
the job (a rank waiting for a peer that never answers) would keep running and keep its GPU.  On timeout the launcher gets
SIGTERM first, which makes its agent stop the workers; after a grace period everything still alive is killed.  Every
process of the job carries a unique token on its command line (appended to the worker's arguments, after the ones it
reads), which is how the workers are found once the launcher is gone.
"""
import os
import signal
import subprocess
import sys
import time
import uuid


def _pids_with(token):
    tok = token.encode()
    pids = []
    for d in os.listdir("/proc"):
        if not d.isdigit() or int(d) == os.getpid():
            continue
        try:
            with open(f"/proc/{d}/cmdline", "rb") as f:
                if tok in f.read():
                    pids.append(int(d))
        except OSError:
            pass
    return pids


def _kill_all(token, wait=10.0):
    """SIGKILL every process of the job; returns the pids still there after `wait` seconds."""
    deadline = time.monotonic() + wait
    while True:
        pids = _pids_with(token)
        for pid in pids:
            try:
                os.kill(pid, signal.SIGKILL)
            except OSError:
                pass
        if not pids or time.monotonic() > deadline:
            return pids
        time.sleep(0.2)


def run(nproc, port, script, args, env, timeout, grace=30.0):
    """torchrun --nproc-per-node=nproc script *args -> dict(returncode, stdout, stderr, timed_out, leftover).

    `leftover` lists the pids of the job that could not be killed (always checked, also after a normal exit)."""
    token = f"sb-torchrun-job-{uuid.uuid4().hex}"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), str(script), *map(str, args), token]
    p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env)
    timed_out = False
    try:
        out, err = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        timed_out = True
        p.send_signal(signal.SIGTERM)  # the elastic agent stops its workers
        try:
            out, err = p.communicate(timeout=grace)
        except subprocess.TimeoutExpired:
            p.kill()
            _kill_all(token)  # before reading on: an orphaned worker would hold the pipes open
            out, err = p.communicate()
    finally:
        if p.poll() is None:
            p.kill()
        leftover = _kill_all(token)
    return dict(returncode=p.wait(), stdout=out or "", stderr=err or "", timed_out=timed_out, leftover=leftover)
