"""The mutant catalogue (tests/kernel_mutants.py) without a GPU: every mutant still applies to the current source, is a value
change the deny-list accepts, names kill selections that collect, and a few of them build with the library's own flags."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest

import kernel_mutants as km
from conftest import ROOT


def test_names_are_unique():
    names = [m.name for m in km.MUTANTS]
    assert len(names) == len(set(names))
    assert len(names) >= 40


@pytest.mark.parametrize("m", km.MUTANTS, ids=[m.name for m in km.MUTANTS])
def test_mutant_applies_once_and_is_a_value_change(m):
    assert m.before in km.source(m), "the code moved: update the catalogue"
    assert km.source(m).count(m.before) == 1
    assert m.after != m.before
    assert km.check_safe(m)
    assert m.kill and m.models
    assert m.equivalent is None or len(m.equivalent) > 40


@pytest.mark.parametrize("before,after", [
    ("mbar_wait(bar, parity);", "mbar_wait(bar, parity ^ 1);"),
    ("for (int k = 0; k < K; k++) acc += a[k];", "for (int k = 1; k < K; k++) acc += a[k];"),
    ("x = a[i];", "x = a[i + 1];"),
    ("n++;", "n--;"),
    ("if (seq == want) ok = 1.0;", "if (seq != want) ok = 1.0;"),
    ("const int s = 4;", "const int s = 3;"),
    ("v = pt < npts ? a : b;", "v = pt <= npts ? a : b;"),
    ("atomicAdd(ctr, 1);", "atomicAdd(ctr, 2);"),
    ("while (!ok) spin();", "if (!ok) spin();"),
    ("const double c = x < y ? a : b;", "const double c = x <= y ? a : b;"),
])
def test_deny_list_rejects_control_and_addressing_changes(before, after):
    with pytest.raises(ValueError):
        km.check_safe(km.Mutant("probe", "generic_fused.cuh", before, after, "", ["x"], None))


def test_every_kill_selection_collects():
    ids = sorted({k for m in km.MUTANTS for k in m.kill})
    r = subprocess.run([sys.executable, "-m", "pytest", "--collect-only", "-q", "-p", "no:cacheprovider"] + ids, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    collected = [ln for ln in r.stdout.splitlines() if "::" in ln]
    for k in ids:
        assert any(ln == k or ln.startswith(k + "[") for ln in collected), k


def test_apply_copies_the_tree_and_changes_one_file(tmp_path):
    m = km.by_name("probe_q1_t_zero")
    csrc = km.apply(ROOT, m, str(tmp_path))
    assert os.path.exists(os.path.join(csrc, "..", "..", "include", "pinn_b200.h"))
    for name in os.listdir(os.path.join(ROOT, km.CSRC_REL)):
        with open(os.path.join(ROOT, km.CSRC_REL, name)) as f:
            orig = f.read()
        with open(os.path.join(csrc, name)) as f:
            new = f.read()
        assert (new != orig) == (name == m.file), name
        if name == m.file:
            assert new == orig.replace(m.before, m.after)


# one mutant per kernel family that compiles differently: the fused-kernel header path, the tail/optimiser header and the tanh
BUILT = ["tanh_coef_5fact_is_4fact", "gen_wide_head_drops_uxx", "lbfgs_solve_curvature_1e9"]


def test_a_few_mutants_build_with_the_library_flags(tmp_path):
    def one(name):
        return km.build(ROOT, km.by_name(name), str(tmp_path / name))
    with ThreadPoolExecutor(len(BUILT)) as ex:
        libs = list(ex.map(one, BUILT))
    for lib in libs:
        assert os.path.getsize(lib) > 100000
