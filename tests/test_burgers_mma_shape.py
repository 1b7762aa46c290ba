"""The default Burgers kernel (v2) runs its GEMMs on Hopper's 16x8 FP64 MMA shapes, which issue twice the FMAs per cycle of
m8n8k4 on the H100 (profiles/microbench/fp64_peak_h100.jsonl), and still computes what v1 (still m8n8k4) computes.

The SASS check runs on the CPU.  The GPU check compares v2 with v1 per parameter block at the benchmark's sizes (N_f = 100 000,
and 250 000), where the other tests only compare one relative norm over the whole gradient.
"""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from oracle import taylor as ty

TESTS = os.path.dirname(os.path.abspath(__file__))
REL = 1e-12                      # per kernel: ||g_B - g*_B|| <= REL ||S_B|| (tests/test_gpu_precision.py); two kernels: 2 REL
SIZES = [100_000, 250_000]


def _sass_functions(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    return {m.group(1): m.group(2) for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", out, re.S)}


def test_burgers_v2_uses_only_16x8_dmma(lib_built):
    funcs = _sass_functions(lib_built)
    v2 = [k for k in funcs if "burgers2" in k and "fused_loss_grad" in k]
    assert len(v2) == 1, v2
    shapes = set(re.findall(r"DMMA\.(\d+x\d+x\d+)", funcs[v2[0]]))
    assert shapes == {"16x8x4", "16x8x8"}, shapes          # chain GEMMs k4 (K = 20 unpadded), weight gradient k8
    v1 = [k for k in funcs if "burgers" in k and "burgers2" not in k and "fused_loss_grad" in k]
    assert len(v1) == 1 and "DMMA.8x8x4" in funcs[v1[0]], v1  # the cross-check kernel keeps the other shape


def bench_problem(n_f):
    import bench
    X_f, X_u, u = bench.synthetic_problem(1234, n_f)
    return bench, X_f, X_u, u, bench.init_weights()


def worker():
    """one JSON line: loss, gradient and loss parts of the kernel PINN_BURGERS_KERNEL selects, at each of SIZES"""
    import bench                 # puts the package's utils/ on sys.path
    import pinn_cabi
    out = {}
    for n_f in SIZES:
        bench, X_f, X_u, u, w = bench_problem(n_f)
        p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, bench.LAYERS, bench.LB, bench.UB)
        p.set_pde_params([bench.NU])
        p.set_data(X_u, u)
        p.set_collocation(X_f[:, 0], X_f[:, 1])
        loss, grad, parts = p.loss_grad(w=w)
        out[str(n_f)] = [loss, grad.tolist(), parts.tolist()]
        out["kernel"] = p.kernel_info()
        p.close()
    print(json.dumps(out))


@pytest.fixture(scope="module")
def runs():
    code = "import sys; sys.path[:0] = [%r, %r]; import test_burgers_mma_shape as m; m.worker()" % (ROOT, TESTS)
    res = {}
    for k in ("v2", "v1"):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PINN_BURGERS_KERNEL=k), capture_output=True,
                           text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        res[k] = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["v2"]["kernel"] != res["v1"]["kernel"]        # two different kernels actually ran
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("n_f", SIZES)
def test_v2_matches_v1_per_block_at_benchmark_sizes(runs, n_f):
    bench, X_f, X_u, u, w = bench_problem(n_f)
    _, _, _, mag = ty.burgers_loss_grad(w, bench.LAYERS, bench.LB, bench.UB, X_f, X_u, u, nu=bench.NU, magnitudes=True)
    l2, g2, p2 = runs["v2"][str(n_f)]
    l1, g1, p1 = runs["v1"][str(n_f)]
    g2, g1 = np.array(g2), np.array(g1)
    bad = []
    for name, sl in ty.param_blocks(bench.LAYERS, 0):
        err, bound = np.linalg.norm(g2[sl] - g1[sl]), 2 * REL * np.linalg.norm(mag[sl])
        if not err <= bound:
            bad.append((name, err, bound))
    for name, a, b in [("loss", l2, l1), ("part0", p2[0], p1[0]), ("part2", p2[2], p1[2])]:
        if not abs(a - b) <= 2 * REL * abs(b):
            bad.append((name, a, b))
    assert not bad, bad
