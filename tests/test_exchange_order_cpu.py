"""CPU: the host restatement of the evaluation tail's summation order (tests/exchange_order.py) that
tests/test_gpu_exchange_sim.py holds the simulated ranks to bit for bit, the harness build, and the models pinn_create refuses
to shard."""
import re
import subprocess

import numpy as np
import pytest

import exchange_order as xo

LD = np.longdouble
EPS = np.finfo(np.float64).eps


def _rank_partials(seed, n_ctas, stride):
    return xo.cancelling_ranks(np.random.default_rng(seed), n_ctas, stride)


@pytest.mark.parametrize("n_ctas", [[1, 5], [8, 9, 132], [264, 1, 5, 8, 9], [1, 5, 8, 9, 132, 264, 7, 16]],
                         ids=lambda v: "W%d" % len(v))
def test_restatement_is_a_sum_of_the_partials(n_ctas):
    parts = _rank_partials(len(n_ctas), n_ctas, 40)
    cols = xo.columns(37, [39, 37, 38])
    got = xo.tail_sum(parts, cols)
    allp = np.concatenate(parts)[:, cols]
    exact = np.sum(allp.astype(LD), axis=0)
    bound = (max(n_ctas) + 2 * xo.P2P_MAX) * EPS * np.sum(np.abs(allp), axis=0)
    assert np.all(np.abs(got.astype(LD) - exact) <= bound)
    # and the data cancels enough that the rounding shows: the fp64 result is not the correctly rounded sum everywhere
    assert np.any(got != exact.astype(np.float64))


def test_restatement_tells_apart_a_swapped_rank_order_and_a_shifted_warp_slice():
    """The bitwise checks of the GPU test can fail: on the cancelling data, the sums in a wrong order are just as accurate
    but differ in their bits."""
    n_ctas = [9, 132, 5]
    parts = _rank_partials(7, n_ctas, 48)
    cols = xo.columns(45, [45, 46, 47])
    good = xo.tail_sum(parts, cols)
    swapped = xo.tail_sum([parts[2], parts[1], parts[0]], cols)      # (0+1) = (1+0): only a swap across pairs shows

    def shifted_local_sum(p):                        # warp w takes the CTAs b = w + 1 (mod 8)
        p = p[:, cols]
        acc = np.zeros((8, p.shape[1]))
        for b in range(p.shape[0]):
            acc[(b - 1) % 8] = acc[(b - 1) % 8] + p[b]
        return xo.combine8(acc)

    shifted = xo.exchanged([shifted_local_sum(p) for p in parts])
    allp = np.concatenate(parts)[:, cols]
    exact = np.sum(allp.astype(LD), axis=0)
    bound = 160 * EPS * np.sum(np.abs(allp), axis=0)
    for wrong in (swapped, shifted):
        assert np.all(np.abs(wrong.astype(LD) - exact) <= bound)
        assert np.count_nonzero(wrong != good) > len(cols) // 4


def test_restatement_pads_the_missing_ranks_with_zero():
    v = np.array([[-0.0, 1.0, np.inf]])
    out = xo.exchanged(v)
    assert np.signbit(out[0]) == np.signbit(-0.0 + 0.0) and out[1] == 1.0 and out[2] == np.inf
    with pytest.raises(ValueError):
        xo.exchanged(np.zeros((9, 2)))


def test_harness_builds_for_sm90a_without_stack(tmp_path):
    so = xo.compile_harness(str(tmp_path))
    import build as pinn_build                        # on sys.path through exchange_order.compile_harness
    r = subprocess.run([pinn_build._nvcc().replace("nvcc", "cuobjdump"), "-res-usage", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "arch = sm_90a" in r.stdout
    funcs = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:\d+ STACK:\d+ SHARED:\d+ LOCAL:\d+)", r.stdout))
    for name in ("reduce_tail", "adam_update", "fused_tail_kernel"):
        hits = [v for k, v in funcs.items() if name in k]
        assert len(hits) == 1, (name, sorted(funcs))
        assert "STACK:0 " in hits[0] and "LOCAL:0" in hits[0], (name, hits[0])


# pde id -> a net pinn_create accepts for it
UNSHARDABLE = {1: ("Burgers identification", [2, 20, 1], "no data weight"), 3: ("Burgers discrete", [1, 20, 3], "collocation set"),
               4: ("Burgers discrete identification", [1, 20, 2], "collocation set"), 5: ("KdV", [1, 20, 2], "collocation set"),
               6: ("Allen-Cahn", [1, 20, 3], "collocation set")}


@pytest.mark.parametrize("pde", sorted(UNSHARDABLE), ids=[UNSHARDABLE[k][0] for k in sorted(UNSHARDABLE)])
def test_models_that_cannot_be_sharded_are_refused(lib_built, pde):
    """Refused before any device query or NCCL set-up, so no GPU is needed to see it."""
    import pinn_cabi
    name, layers, why = UNSHARDABLE[pde]
    with pytest.raises(pinn_cabi.PinnError, match="world must be 1.*" + why):
        pinn_cabi.Pinn(pde, layers, [-1.0, 0.0], [1.0, 1.0], rank=1, world=2)
