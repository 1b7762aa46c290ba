"""GPU: residual-based adaptive resampling on the device (pinn_draw_collocation_rad, DESIGN §4.7).

The drawn set equals, bit for bit, what the numpy restatement (oracle/rad_draw.py) picks from pinn_residual on the same pool and
weights, on the Burgers v2, v1 and wide generic nets and on both Schrodinger kernels.  A handle after RAD equals, bit for bit, a
fresh handle fed those points through pinn_set_collocation, also over five asynchronous Adam steps.  RAD enqueued behind
asynchronous Adam steps reads the stepped weights.  Refused calls change nothing, and the mirror with hp["rad_every"] equals the
same calls made by hand."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from oracle import lhs_draw as ld
from oracle import rad_draw as rd
from test_gpu_lhs_draw import BURGERS, NLS, STD, NLS_BOX, BIG_SEED, BIG_DRAW, create, setup, same, assert_same, fresh_with

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
FAMILIES = {
    "burgers_v2": dict(pde="BURGERS_INF", layers=BURGERS, box=STD),
    "burgers_v1": dict(pde="BURGERS_INF", layers=BURGERS, box=STD, env={"PINN_BURGERS_KERNEL": "v1"}),
    "burgers_wide": dict(pde="BURGERS_INF", layers=[2, 160, 160, 1], box=([0.3, -0.5], [3.7, 2.0])),   # the MAXW_WIDE probe
    "nls": dict(pde="NLS_INF", layers=NLS, box=NLS_BOX),
    "nls_generic": dict(pde="NLS_INF", layers=NLS, box=NLS_BOX, env={"PINN_FORCE_GENERIC": "1"}),
}
RAD_LAUNCHES = 5            # pool draw, probe forward, head, quantise, pick


def expected(fam, seed, draw, n, n_pool, k, c, weights=None):
    """The oracle's points: handle A draws the pool with pinn_draw_collocation and returns pinn_residual on it."""
    a = setup(create(fam), fam)
    if weights is not None:
        a.set_weights(weights)
    a.draw_collocation(seed, draw, n_pool)
    f = a.residual()
    px, pt = a.get_collocation()
    a.close()
    wx, wt = ld.lhs_draw(seed, draw, n_pool, 0, n_pool, *fam["box"])
    assert same(px, wx) and same(pt, wt)
    i = rd.rad_indices(f, seed, draw, n, k, c)
    return px[i], pt[i]


def check_points(name, cases):
    fam = FAMILIES[name]
    b = setup(create(fam), fam)
    for n_pool, n, k, c, seed, draw in cases:
        launches = b.launch_count()
        b.draw_collocation_rad(seed, draw, n, n_pool, k, c)
        assert b.launch_count() == launches + RAD_LAUNCHES * (n > 0)
        assert int(b.lib.pinn_num_residual_points(b.h)) == n
        x, t = b.get_collocation()
        wx, wt = expected(fam, seed, draw, n, n_pool, k, c)
        assert same(x, wx) and same(t, wt), (name, n_pool, n, k, c)
    b.close()


def run_worker(call, env):
    """`call` of this module in a fresh interpreter with env set."""
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_rad as m; m.%s" % (ROOT, TESTS, call)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-1500:] + r.stderr[-3000:])


# ---------------------------------------------------------------------------------------------------- the points themselves
SMALL = [(1, 5, 1, 1.0, 3, 0), (7, 3, 2, 0.0, BIG_SEED, BIG_DRAW), (7, 40, 4, 1024.0, 5, 1), (1000, 300, 1, 1.0, BIG_SEED, 2),
         (1000, 4000, 3, 0.5, 6, BIG_DRAW), (1000, 0, 1, 1.0, 6, 7), (1000, 900, 0, 0.0, 6, 8)]
LARGE = [(1000000, 100000, 1, 1.0, BIG_SEED, BIG_DRAW), (1000000, 2000000, 2, 0.0, 17, 3)]


@pytest.mark.parametrize("name", ["burgers_v2", "nls"])
def test_rad_points_equal_the_oracle_on_pinn_residual(name):
    check_points(name, SMALL + LARGE)


@pytest.mark.parametrize("name", ["burgers_wide", "nls_generic"])
def test_rad_points_equal_the_oracle_on_other_nets(name):
    check_points(name, SMALL)


def check_points_v1():
    check_points("burgers_v1", SMALL)


def test_rad_points_equal_the_oracle_on_the_v1_kernel():
    run_worker("check_points_v1()", FAMILIES["burgers_v1"]["env"])


# ------------------------------------------------------------------------------------------ a RAD set is an uploaded set
@pytest.mark.parametrize("name", ["burgers_v2", "nls"])
def test_rad_handle_equals_a_fresh_handle_fed_the_points(name):
    fam, n_pool, n = FAMILIES[name], 50000, 20011
    p = setup(create(fam), fam)
    p.set_collocation(*ld.lhs_draw(1, 1, 3000, 0, 3000, *fam["box"]))
    p.loss_grad()
    p.draw_collocation_rad(BIG_SEED, BIG_DRAW, n, n_pool, 2, 1.0)
    x, t = expected(fam, BIG_SEED, BIG_DRAW, n, n_pool, 2, 1.0)
    q = fresh_with(fam, x, t, n)
    assert_same(p, q, name)
    for _ in range(5):
        p.adam_step(1e-3, sync=False)
        q.adam_step(1e-3, sync=False)
    assert same(p.get_weights(), q.get_weights()) and same(p.last_loss(), q.last_loss())
    p.close(); q.close()


def test_rad_replaces_a_mapped_batch():
    import ctypes as C
    import pinn_cabi
    fam = FAMILIES["burgers_v2"]
    p = setup(create(fam), fam)
    bufs = [pinn_cabi.host_alloc(20000) for _ in range(2)]
    for (arr, _), v in zip(bufs, (np.linspace(-1, 1, 20000), np.linspace(0, 0.99, 20000))):
        arr[:] = v
    dp = C.POINTER(C.c_double)
    p.set_collocation_mapped(C.cast(bufs[0][1], dp), C.cast(bufs[1][1], dp), 20000)
    p.loss_grad()
    p.draw_collocation_rad(9, 4, 5000, 30000, 1, 1.0)
    assert_same(p, fresh_with(fam, *expected(fam, 9, 4, 5000, 30000, 1, 1.0), 5000), "after a mapped batch")
    p.close()
    for _, ptr in bufs:
        pinn_cabi.load().pinn_host_free(ptr)


def test_rad_after_asynchronous_adam_steps_reads_the_stepped_weights():
    fam = FAMILIES["burgers_v2"]
    p, q = setup(create(fam), fam), setup(create(fam), fam)
    for h in (p, q):
        h.set_collocation(*ld.lhs_draw(2, 0, 20000, 0, 20000, *fam["box"]))
    for _ in range(5):
        p.adam_step(3e-3, sync=False)                       # no host synchronisation between these steps and the draw
    p.draw_collocation_rad(31, 5, 40000, 200000, 1, 1.0)
    x, t = p.get_collocation()
    for _ in range(5):
        q.adam_step(3e-3, sync=True)
    w = q.get_weights()
    assert same(p.get_weights(), w)
    wx, wt = expected(fam, 31, 5, 40000, 200000, 1, 1.0, weights=w)
    assert same(x, wx) and same(t, wt)
    # and not the weights the handle started from
    x0, _ = expected(fam, 31, 5, 40000, 200000, 1, 1.0)
    assert not same(x, x0)
    p.close(); q.close()


def test_refused_calls_change_nothing():
    import pinn_cabi
    fam = FAMILIES["burgers_v2"]
    x, t = ld.lhs_draw(1, 2, 3000, 0, 3000, *fam["box"])
    q = fresh_with(fam, x, t, 3000)
    p = fresh_with(fam, x, t, 3000)
    p.loss_grad()
    launches = p.launch_count()
    for n_pool, n, k, c in ((100, 10, -1, 1.0), (100, 10, 5, 1.0), (100, 10, 1, -0.5), (100, 10, 1, 1024.5),
                            (100, 10, 1, float("nan")), (100, 10, 1, float("inf")), (0, 10, 1, 1.0), ((1 << 29) + 1, 10, 1, 1.0),
                            (100, -1, 1, 1.0)):
        assert p.lib.pinn_draw_collocation_rad(p.h, 1, 1, n_pool, n, k, c) != 0, (n_pool, n, k, c)
        assert "pinn_draw_collocation_rad" in p.lib.pinn_last_error().decode()
    assert p.launch_count() == launches
    assert_same(p, q, "after refused RAD calls")
    p.close(); q.close()
    for pde, layers, box, why in (("BURGERS_IDE", BURGERS, STD, "identification"), ("POLY_IDE", [2, 20, 20, 1], STD, "identification"),
                                  ("NS_IDE", [3, 20, 20, 2], ([0.0, 0.0, 0.0], [1.0, 1.0, 1.0]), "identification"),
                                  ("BURGERS_DISC", [1, 30, 30, 9], ([-1.0], [1.0]), "discrete-time"),
                                  ("POLY_INF", [2, 20, 20, 1], STD, "POLY_INF")):
        p = pinn_cabi.Pinn(getattr(pinn_cabi, pde), layers, *box)
        with pytest.raises(pinn_cabi.PinnError, match="pinn_draw_collocation_rad: .*" + why):
            p.draw_collocation_rad(1, 1, 100, 1000)
        assert p.launch_count() == 0
        p.close()


# ------------------------------------------------------------------------------------------------------------------- mirror
def test_mirror_rad_every_equals_the_c_abi_loop():
    import pinn_cabi
    from neuralnetwork import NeuralNetwork
    N_f = 4000
    hp = {"layers": BURGERS, "tf_epochs": 7, "tf_lr": 3e-3, "tf_b1": 0.9, "tf_eps": None, "nt_epochs": 0, "nt_lr": 0.8,
          "nt_ncorr": 50, "rad_every": 3, "resample_seed": 21, "rad_pool": 12345, "rad_k": 2, "rad_c": 0.5}

    class Quiet(object):
        def log_train_opt(self, name):
            pass

        def log_train_epoch(self, epoch, loss, custom="", is_iter=False):
            float(loss)

    class BurgersInformedNN(NeuralNetwork):
        def __init__(self, X_f):
            super().__init__(hp, Quiet(), np.array(STD[1]), np.array(STD[0]))
            self.nu = 0.01 / np.pi
            self.x_f, self.t_f = X_f[:, 0:1], X_f[:, 1:2]

    rng = np.random.default_rng(3)
    X_u = np.stack([rng.uniform(-1, 1, 80), rng.uniform(0, 0.99, 80)], 1)
    u = np.sin(np.pi * X_u[:, :1])
    X_f = np.stack(ld.lhs_draw(1, 0, N_f, 0, N_f, *STD), 1)
    net = BurgersInformedNN(X_f)
    net.tf_optimization(X_u, u)
    p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, BURGERS, STD[0], STD[1])
    p.set_pde_params([0.01 / np.pi])
    p.set_collocation(X_f[:, 0], X_f[:, 1])
    p.set_weights(net._w0)
    p.set_data(X_u, u)
    for e in range(7):
        if e > 0 and e % 3 == 0:
            assert p.lib.pinn_draw_collocation_rad(p.h, 21, e // 3, 12345, N_f, 2, 0.5) == 0
        p.adam_step(3e-3, 0.9, 0.999, 1e-7, sync=False)
    assert same(net.get_weights(), p.get_weights())
    assert same(net._native().get_collocation()[0], p.get_collocation()[0])
    p.close()
