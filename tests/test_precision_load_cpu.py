"""CPU: the method of tests/test_gpu_precision_load.py, on the fp64 oracles.

* Shuffled replication is invariant: the Burgers, Schrodinger and Navier-Stokes oracles on R shuffled copies of a base set equal
  the base set's oracle (x R for the Navier-Stokes sums) within check()'s rule.
* The shuffle has teeth: the faults that file exists for -- one CTA's block of points read twice and its neighbour skipped, the
  last ragged round of a CTA dropped, a probe chunk read one row off -- are each rejected against the base reference.  The
  duplicated block on an unshuffled replication, where copy boundaries line up with the CTAs, passes: that is why the copies
  are shuffled.
* The load helpers give the per-CTA counts, rounds and chunks of pinn_api.cu's formulas at 132 SMs (an H100 SXM)."""
import numpy as np
import pytest

from oracle import taylor as ty, taylor_ns as tn
from test_gpu_precision import LD, _rand_w, check, points
from test_gpu_precision_load import (burgers_load, generic_load, nls_load, ns_load, ns_probe_chunks, probe_check, replicate,
                                     scaled)

NET = [2, 20, 20, 20, 1]


def _kernel_parts(parts, part_idx):
    out = np.zeros(3)
    out[list(part_idx)] = parts
    return out


def burgers_problem(B, seed=0, lb=(0.0, 0.0), ub=(1e-2, 1e-3)):
    """Burgers inference with nu = 1 on the small domain: a base collocation set of B points, 40 data points, and a function
    of the collocation array (the kernel's 1 / n_f weight fixed by n_f_global)."""
    rng = np.random.default_rng(seed)
    lb, ub = np.array(lb), np.array(ub)
    Xb = points(rng, lb, ub, B)
    X_u, u = points(rng, lb, ub, 40), rng.uniform(-1, 1, (40, 1))
    w = _rand_w(NET, seed)
    run = lambda X_f, n_f_global=None, **kw: ty.burgers_loss_grad(w, NET, lb, ub, X_f, X_u, u, nu=1.0, n_f_global=n_f_global,
                                                                 **kw)
    return Xb, run


def _as_kernel(r, part_idx):
    return r[0], r[1], _kernel_parts(r[2], part_idx)


# -------------------------------------------------------------------------------------------------- replication is invariant
def test_burgers_oracle_is_invariant_under_shuffled_replication():
    Xb, run = burgers_problem(300)
    ref, ref64 = run(Xb, dtype=LD, magnitudes=True), run(Xb)
    got = run(Xb[replicate(300, 7, 1)])
    check("replication/burgers", _as_kernel(got, (0, 2)), ref, ref64, ty.param_blocks(NET), (0, 2))


def test_schrodinger_oracle_is_invariant_under_shuffled_replication():
    layers = [2, 30, 30, 2]
    lb, ub = np.array([-0.7, 0.25]), np.array([1.3, 0.5])
    rng = np.random.default_rng(2)
    Xb = points(rng, lb, ub, 200)
    tb = rng.uniform(lb[1], ub[1], (7, 1))
    X0 = np.concatenate([rng.uniform(lb[0], ub[0], (9, 1)), np.full((9, 1), lb[1])], 1)
    uv0 = rng.standard_normal((9, 2))
    w = _rand_w(layers, 2)
    run = lambda X, **kw: ty.schrodinger_loss_grad(w, layers, lb, ub, X, tb, X0, uv0, **kw)
    got = run(Xb[replicate(200, 5, 2)])
    check("replication/nls", got, run(Xb, dtype=LD, magnitudes=True), run(Xb), ty.param_blocks(layers), (0, 1, 2))


def test_navier_stokes_oracle_is_replication_times_R():
    layers = [3, 20, 20, 2]
    rng = np.random.default_rng(3)
    lb, ub = np.zeros(3), np.array([1e-2, 2e-2, 1e-3])
    X = lb + (ub - lb) * rng.random((100, 3))
    uv = rng.standard_normal((100, 2))
    w = np.concatenate([_rand_w(layers, 3), [0.6, 0.05]])
    run = lambda idx, **kw: tn.ns_ide_loss_grad(w, layers, lb, ub, X[idx], uv[idx], **kw)
    base = np.arange(100)
    got = run(replicate(100, 9, 3))
    check("replication/ns", _as_kernel(got, (0, 2)), scaled(run(base, dtype=LD, magnitudes=True), 9), scaled(run(base), 9),
          ty.param_blocks(layers, 2), (0, 2))


# -------------------------------------------------------------------------------------------------------- the shuffle has teeth
B, R = 250, 7


@pytest.fixture(scope="module")
def teeth():
    Xb, run = burgers_problem(B, seed=5)
    return Xb, run, run(Xb, dtype=LD, magnitudes=True), run(Xb)


def _duplicate_block(X, pts, j):
    """CTA j's block of pts points read twice: CTA j + 1 computes on CTA j's points and its own are skipped."""
    X = X.copy()
    X[(j + 1) * pts:(j + 2) * pts] = X[j * pts:(j + 1) * pts]
    return X


@pytest.mark.parametrize("shuffled", [True, False], ids=["shuffled", "unshuffled"])
def test_a_block_read_twice(teeth, shuffled):
    """A CTA holds one copy's worth of points (pts = B): on unshuffled copies the duplicated block is the next copy, and the
    fault is invisible; shuffled, check() rejects it."""
    Xb, run, ref, ref64 = teeth
    X = Xb[replicate(B, R, 5) if shuffled else np.tile(np.arange(B), R)]
    got = _as_kernel(run(_duplicate_block(X, B, 2)), (0, 2))
    if shuffled:
        with pytest.raises(AssertionError):
            check("teeth/duplicate_block_shuffled", got, ref, ref64, ty.param_blocks(NET), (0, 2))
    else:
        check("teeth/duplicate_block_unshuffled", got, ref, ref64, ty.param_blocks(NET), (0, 2))


def test_the_last_ragged_round_of_a_cta_dropped(teeth):
    """Rounds of 16 points over 12 CTAs (nls_load): the last CTA that owns points ends in a partial round; without it the sum
    misses those points while the mean still divides by all of them."""
    Xb, run, ref, ref64 = teeth
    X = Xb[replicate(B, R, 5)]
    load = nls_load(len(X), 12)
    ragged = load["last CTA points"] % 16
    assert ragged > 0
    got = _as_kernel(run(X[:len(X) - ragged], n_f_global=len(X)), (0, 2))
    with pytest.raises(AssertionError):
        check("teeth/ragged_round_dropped", got, ref, ref64, ty.param_blocks(NET), (0, 2))


def test_a_probe_chunk_one_row_off():
    """The Navier-Stokes probe of a width-256 net over 16 000 points: chunk 1 reads its points one row late.  The clean streams
    pass probe_check against the base oracle row by row; the shifted chunk fails it."""
    layers = [3, 256, 2]
    rng = np.random.default_rng(6)
    lb, ub = np.zeros(3), np.array([1e-2, 2e-2, 1e-3])
    Xb = lb + (ub - lb) * rng.random((500, 3))
    w = _rand_w(layers, 6)
    idx = replicate(500, 32, 6)
    X = Xb[idx]
    chunk = ns_probe_chunks(len(X), 256)["chunk"]
    ref = [v[idx] for v in tn.forward_ns(w, layers, lb, ub, Xb, dtype=LD)[0]]
    ref64 = [v[idx] for v in tn.forward_ns(w, layers, lb, ub, Xb)[0]]
    streams = lambda O: [("stream %d" % k, O[k], ref[k], ref64[k], 1e-13 if sum(m) <= 1 else 1e-12)
                         for k, m in enumerate(tn.STREAMS)]
    probe_check("teeth/probe_clean", streams(tn.forward_ns(w, layers, lb, ub, X)[0]))
    Xs = X.copy()
    Xs[chunk:2 * chunk] = X[chunk + 1:2 * chunk + 1]
    with pytest.raises(AssertionError):
        probe_check("teeth/probe_chunk_one_row_off", streams(tn.forward_ns(w, layers, lb, ub, Xs)[0]))


# ------------------------------------------------------------------------------------------------------------------ the loads
SMS = 132


def test_burgers_loads():
    # pinn_api.cu: burgers_launch_eval; burgers_fused_v2.cuh:361-365, burgers_fused.cuh:315
    assert burgers_load(100100, SMS, "v2") == {"grid": 132, "tiles per CTA": 95, "rounds per chain warp": 24}
    assert burgers_load(100100, SMS, "v1") == {"grid": 132, "rounds per CTA": 24}
    assert burgers_load(2000100, SMS, "v2") == {"grid": 132, "tiles per CTA": 1895, "rounds per chain warp": 474}
    assert burgers_load(250100, SMS, "v2")["tiles per CTA"] == 237
    assert burgers_load(7, SMS, "v2") == {"grid": 1, "tiles per CTA": 1, "rounds per chain warp": 1}


def test_schrodinger_loads():
    # pinn_api.cu: nls_launch_eval: the upstream 20 000 + 50 + 2 x 50 points take 10 rounds per CTA
    assert nls_load(20150, SMS) == {"points per CTA": 160, "rounds per CTA": 10, "last CTA points": 150}
    assert nls_load(106150, SMS)["rounds per CTA"] == 51
    assert nls_load(1950, SMS)["rounds per CTA"] == 1


def test_generic_loads():
    # pinn_api.cu: generic_launch_eval, C = 264 CTAs
    assert generic_load(16 * 264 - 1, SMS) == {"points per CTA": 16, "8-point groups per CTA": 2, "grid": 264,
                                               "last CTA points": 15}
    assert generic_load(16 * 264 + 1, SMS) == {"points per CTA": 32, "8-point groups per CTA": 4, "grid": 133,
                                               "last CTA points": 1}
    assert generic_load(100101, SMS) == {"points per CTA": 384, "8-point groups per CTA": 48, "grid": 261,
                                         "last CTA points": 261}
    assert generic_load(263, SMS)["points per CTA"] == 2


def test_navier_stokes_loads():
    # pinn_api.cu: ns_launch_eval and, for the probe, ns_probe
    assert ns_load(5000, SMS) == {"points per CTA": 38, "M tiles per CTA": 3, "grid": 132, "last CTA points": 22}
    assert ns_load(50000, SMS) == {"points per CTA": 379, "M tiles per CTA": 24, "grid": 132, "last CTA points": 351}
    assert ns_probe_chunks(16000, 256) == {"chunk": 5041, "chunks": 4, "last chunk": 877}
    assert ns_probe_chunks(200000, 20) == {"chunk": 64527, "chunks": 4, "last chunk": 6419}
    assert ns_probe_chunks(700, 256)["chunks"] == 1                # 700 points on a width-256 net fit in one chunk
