"""CPU: every kernel of libpinn_b200.so keeps the SASS recorded in tests/golden/kernel_sass.json (tests/golden/make_sass_golden.py
explains when that file is regenerated).  The fused, optimiser, probe, LHS and RAD kernels of the parent are all listed, so adding
the source-table kernels left their machine code exactly as it was."""
import importlib.util
import json
import os

import pytest

from conftest import GOLDEN


def _maker():
    spec = importlib.util.spec_from_file_location("make_sass_golden", os.path.join(GOLDEN, "make_sass_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_every_kernel_keeps_its_recorded_sass(lib_built):
    m = _maker()
    with open(m.GOLDEN) as f:
        want = json.load(f)
    if m.nvcc_build() != want["nvcc"]:
        pytest.skip("the digests were recorded with %s, this toolkit is %s" % (want["nvcc"], m.nvcc_build()))
    got = m.sass_digests(lib_built)
    missing = sorted(set(want["functions"]) - set(got))
    changed = sorted(k for k in want["functions"] if k in got and got[k] != want["functions"][k])
    assert not missing and not changed, {"missing": missing, "changed": changed}
    assert sorted(set(got) - set(want["functions"])) == [], "a new kernel: record it with tests/golden/make_sass_golden.py"
    for name in ("fused_loss_grad", "reduce_tail", "lbfgs_iterate", "mlp_forward_generic", "draw_kernel", "head_kernel",
                 "pick_kernel", "eval_kernel"):
        assert any(name in k for k in want["functions"]), name
