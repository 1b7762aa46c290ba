"""GPU: every value mutant of tests/kernel_mutants.py is killed by its kill selection.

All mutants are built first, in parallel on the CPU, each into a temporary directory of its own.  Then, one GPU process at a time
(the Burgers kernel's in-kernel tail wants its whole grid resident):
  1. the union of the kill selections runs against the product library, as the control: it must pass, or "killed" means nothing;
  2. each mutant's selection runs as `python -m pytest -x -q <selection>` with PINN_LIB naming the mutant's library (every
     worker subprocess inherits it) and PINN_CSRC its sources (for the tests that compile a harness from them), under a timeout.
A mutant is killed when its run fails.  The table (mutant, outcome, first failing test, wall time) is printed; run with -s to
read it.  PINN_MUTANTS=name,name,... restricts the run to those mutants.  Every mutant without an equivalence reason must die.
"""
import os
import re
import signal
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import pytest

import kernel_mutants as km
from conftest import ROOT

pytestmark = pytest.mark.gpu

TIMEOUT = 1800


def selected():
    names = [n for n in os.environ.get("PINN_MUTANTS", "").split(",") if n]
    return [km.by_name(n) for n in names] if names else list(km.MUTANTS)


def run_selection(ids, env):
    """pytest -x on the node ids in a fresh process group (its workers go with it on a timeout).  Returns (exit code or None on
    a timeout, first failing test, wall seconds)."""
    t0 = time.time()
    p = subprocess.Popen([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider"] + list(ids), cwd=ROOT,
                         env=dict(os.environ, **env), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         start_new_session=True)
    try:
        out, _ = p.communicate(timeout=TIMEOUT)
        rc = p.returncode
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        out, _ = p.communicate()
        rc = None
    failed = re.findall(r"^(?:FAILED|ERROR) (\S+)", out, re.M)
    return rc, (failed[0] if failed else ""), time.time() - t0, out


def test_every_mutant_is_killed(tmp_path_factory):
    mutants = selected()
    root = tmp_path_factory.mktemp("mutants")
    workers = max(1, len(os.sched_getaffinity(0)))
    t0 = time.time()
    with ThreadPoolExecutor(workers) as ex:
        libs = list(ex.map(lambda m: km.build(ROOT, m, str(root / m.name)), mutants))
    t_build = time.time() - t0
    print("\n[mutants] built %d mutants on %d CPUs in %.0f s" % (len(mutants), workers, t_build), flush=True)

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    t_gpu = time.time()
    union = sorted({k for m in mutants for k in m.kill})
    rc, first, wall, out = run_selection(union, {})
    print("[mutants] control: %d selections against the product library, exit %s in %.0f s" % (len(union), rc, wall), flush=True)
    assert rc == 0, "the control run fails on the product library:\n" + out[-4000:]

    rows = []
    for m, lib in zip(mutants, libs):
        rc, first, wall, _ = run_selection(m.kill, {"PINN_LIB": lib, "PINN_CSRC": os.path.join(os.path.dirname(lib), km.CSRC_REL)})
        outcome = "survived" if rc == 0 else ("killed (timeout)" if rc is None else "killed")
        rows.append((m, outcome, first, wall))
        print("[mutants] %-36s %-12s %7.1f s" % (m.name, outcome, wall), flush=True)
    t_gpu = time.time() - t_gpu

    print("[mutants] %-36s %-10s %-12s %7s  %s" % ("mutant", "equivalent", "outcome", "wall s", "first failing test"))
    for m, outcome, first, wall in rows:
        print("[mutants] %-36s %-10s %-12s %7.1f  %s" % (m.name, "yes" if m.equivalent else "", outcome, wall, first))
    print("[mutants] %d killed, %d survived; GPU runs %.0f s (control included), builds %.0f s; card: %s"
          % (sum(r[1] != "survived" for r in rows), sum(r[1] == "survived" for r in rows), t_gpu, t_build, card))
    survivors = [m.name for m, outcome, _, _ in rows if outcome == "survived" and m.equivalent is None]
    assert not survivors, "mutants no test kills: %s" % survivors
