"""GPU: the device Latin-hypercube draw (pinn_draw_collocation, DESIGN §4.6).

The drawn points equal the numpy restatement (oracle/lhs_draw.py) bit for bit, and a handle that drew its collocation set equals,
bit for bit, a fresh handle fed the restated points through pinn_set_collocation: loss, parts, gradient and residual on every
kernel that has a collocation set, Adam trajectories with no host synchronisation between draw and step, after a mapped batch,
after larger and smaller sets, and through the reference-style mirror with hp["resample_every"].  Refused calls leave the handle
as a fresh one."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, load_golden
from oracle import lhs_draw as ld

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
BURGERS = [2] + [20] * 8 + [1]
NLS = [2, 100, 100, 100, 100, 2]
STD = ([-1.0, 0.0], [1.0, 0.99])
NLS_BOX = ([-5.0, 0.0], [5.0, np.pi / 2])
SHIFTED = ([0.3, -0.5], [3.7, 2.0])
BIG_SEED, BIG_DRAW = 0xFEDCBA9876543210, 0x100000003
HEAT = [(1.0, 0, (0, 0, 1, 0)), (-0.5, 0, (0, 0, 0, 1)), (0.3, 0, (1, 1, 0, 0))]
FAMILIES = {
    "burgers_v2": dict(pde="BURGERS_INF", layers=BURGERS, box=STD),
    "burgers_v1": dict(pde="BURGERS_INF", layers=BURGERS, box=STD, env={"PINN_BURGERS_KERNEL": "v1"}),
    "burgers_generic": dict(pde="BURGERS_INF", layers=[2] + [40] * 8 + [1], box=SHIFTED),
    "nls": dict(pde="NLS_INF", layers=NLS, box=NLS_BOX),
    "nls_generic": dict(pde="NLS_INF", layers=NLS, box=NLS_BOX, env={"PINN_FORCE_GENERIC": "1"}),
    "poly_inf": dict(pde="POLY_INF", layers=[2, 20, 20, 20, 1], box=STD),
}


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def same(a, b):
    a, b = bits(a), bits(b)
    return a.shape == b.shape and bool(np.all(a == b))


def create(fam):
    import pinn_cabi
    env = fam.get("env", {})
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return pinn_cabi.Pinn(getattr(pinn_cabi, fam["pde"]), fam["layers"], fam["box"][0], fam["box"][1])
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k)
            else:
                os.environ[k] = v


def setup(p, fam, seed=5):
    """Constants, data (and boundary) points and weights: every input but the collocation set."""
    from neuralnetwork import _glorot_normal
    rng = np.random.default_rng(seed)
    lb, ub = (np.asarray(v, float) for v in fam["box"])
    if fam["pde"] == "BURGERS_INF":
        p.set_pde_params([0.01 / np.pi])
    if fam["pde"] == "POLY_INF":
        p.set_residual(HEAT)
    X = lb + (ub - lb) * rng.random((60, 2))
    p.set_data(X, rng.standard_normal((60, fam["layers"][-1])))
    if fam["pde"] == "NLS_INF":
        p.set_boundary(lb[1] + (ub[1] - lb[1]) * rng.random(37))
    p.set_weights(_glorot_normal(fam["layers"], np.random.default_rng(seed + 1)))
    return p


def restated(fam, seed, draw, n_global, rank=0, world=1):
    from sharding import shard_rows
    lo, hi = shard_rows(n_global, rank, world)
    return ld.lhs_draw(seed, draw, n_global, lo, hi - lo, *fam["box"])


def raw_draw(p, seed, draw, first, n, n_global):
    """pinn_draw_collocation with explicit rows (the binding takes them from sharding.shard_rows)."""
    if p.lib.pinn_draw_collocation(p.h, seed, draw, first, n, n_global) != 0:
        pytest.fail(p.lib.pinn_last_error().decode())


def observe(p, with_residual=True):
    loss, grad, parts = p.loss_grad()
    out = {"loss": loss, "grad": grad, "parts": parts, "weights": p.get_weights()}
    if with_residual:
        out["residual"] = p.residual()
    return out


def assert_same(p, q, tag):
    a, b = observe(p), observe(q)
    bad = [k for k in a if not same(a[k], b[k])]
    assert not bad, "%s: %s differ (loss %r vs %r)" % (tag, bad, a["loss"], b["loss"])


def fresh_with(fam, x, t, n_global, source=None):
    q = setup(create(fam), fam)
    q.set_collocation(x, t, n_global)
    if source is not None:
        q.set_source(source)
    return q


def run_worker(call, env):
    """`call` of this module in a fresh interpreter with env set."""
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_lhs_draw as m; m.%s" % (ROOT, TESTS, call)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-1500:] + r.stderr[-3000:])


# ---------------------------------------------------------------------------------------------------- the points themselves
@pytest.mark.parametrize("box", [STD, NLS_BOX, SHIFTED], ids=["burgers", "nls", "shifted"])
def test_device_draw_equals_the_restatement(box):
    fam = dict(FAMILIES["burgers_v2"], box=box)
    p = create(fam)
    sizes = (1, 7, 4097, 100000) + ((2000000,) if box is STD else ())
    for N in sizes:
        for seed, draw, first, n in ((BIG_SEED, BIG_DRAW, 0, N), (3, 11, N // 3, N - N // 3 - (N > 2)), (0, 0, N - 1, 1)):
            launches = p.launch_count()
            raw_draw(p, seed, draw, first, n, N)
            assert p.launch_count() == launches + (n > 0)
            x, t = p.get_collocation()
            wx, wt = ld.lhs_draw(seed, draw, N, first, n, *box)
            assert same(x, wx) and same(t, wt), (box, N, seed, draw, first, n)
            assert int(p.lib.pinn_num_residual_points(p.h)) == n
    p.close()


def test_device_draw_reproduces_the_golden_file():
    g = load_golden("lhs_draw")
    k = 0
    while "case%d_params" % k in g:
        seed, draw, N = (int(v) for v in g["case%d_params" % k])
        box = g["case%d_box" % k]
        p = create(dict(FAMILIES["burgers_v2"], box=(box[:2], box[2:])))
        p.draw_collocation(seed, draw, N)
        x, t = p.get_collocation()
        assert same(x, g["case%d_x" % k]) and same(t, g["case%d_t" % k]), k
        p.close()
        k += 1


# ------------------------------------------------------------------------------------------ a drawn set is an uploaded set
def check_draw_equals_upload(name, n_global=20011):
    fam = FAMILIES[name]
    for rank, world in ((0, 1), (1, 3)):
        p = setup(create(fam), fam)
        p.draw_collocation(BIG_SEED, BIG_DRAW, n_global, rank=rank, world=world)
        x, t = restated(fam, BIG_SEED, BIG_DRAW, n_global, rank, world)
        q = fresh_with(fam, x, t, n_global)
        assert_same(p, q, "%s, rows of rank %d of %d" % (name, rank, world))
        p.close(); q.close()


@pytest.mark.parametrize("name", [n for n in FAMILIES if n != "burgers_v1"])
def test_draw_equals_a_fresh_handle_fed_the_restated_points(name):
    check_draw_equals_upload(name)


def test_draw_equals_a_fresh_handle_fed_the_restated_points_v1():
    run_worker("check_draw_equals_upload('burgers_v1')", FAMILIES["burgers_v1"]["env"])


@pytest.mark.parametrize("name", ["burgers_v2", "nls"])
def test_adam_steps_on_drawn_sets_equal_the_upload_loop(name):
    """Five (draw k, asynchronous Adam step) pairs, no host synchronisation in between, against the same loop fed the restated
    points through pinn_set_collocation."""
    fam, N = FAMILIES[name], 30000
    p, q = setup(create(fam), fam), setup(create(fam), fam)
    for k in range(5):
        p.draw_collocation(77, k, N)
        p.adam_step(1e-3, sync=False)
    for k in range(5):
        q.set_collocation(*restated(fam, 77, k, N))
        q.adam_step(1e-3, sync=False)
    assert same(p.get_weights(), q.get_weights()) and same(p.last_loss(), q.last_loss())
    p.close(); q.close()


def test_draw_replaces_a_mapped_batch_and_any_earlier_set():
    import pinn_cabi
    fam = FAMILIES["burgers_v2"]
    x, t = restated(fam, 9, 4, 5000)
    # a mapped batch first
    p = setup(create(fam), fam)
    bufs = [pinn_cabi.host_alloc(20000) for _ in range(2)]
    for (arr, _), v in zip(bufs, (np.linspace(-1, 1, 20000), np.linspace(0, 0.99, 20000))):
        arr[:] = v
    dp = C.POINTER(C.c_double)
    p.set_collocation_mapped(C.cast(bufs[0][1], dp), C.cast(bufs[1][1], dp), 20000)
    p.loss_grad()
    p.draw_collocation(9, 4, 5000)
    q = fresh_with(fam, x, t, 5000)
    assert_same(p, q, "after a mapped batch")
    p.close()
    for _, ptr in bufs:
        q.lib.pinn_host_free(ptr)
    # after a larger set (no growth) and after a smaller one (the region grows)
    for n_before in (150000, 10):
        p = setup(create(fam), fam)
        p.set_collocation(*restated(fam, 1, 1, n_before))
        p.loss_grad()
        p.draw_collocation(9, 4, 5000)
        assert_same(p, q, "after a set of %d points" % n_before)
        p.close()
    p = setup(create(fam), fam)
    p.set_collocation(*restated(fam, 1, 1, 10))
    p.draw_collocation(9, 4, 200000)
    q2 = fresh_with(fam, *restated(fam, 9, 4, 200000), 200000)
    assert_same(p, q2, "grown by the draw")
    p.close(); q.close(); q2.close()


def test_draws_leave_the_schrodinger_data_terms_alone():
    fam = FAMILIES["nls"]
    p = setup(create(fam), fam)
    p.set_collocation(*restated(fam, 2, 2, 3000))
    _, _, parts0 = p.loss_grad()
    for k, n in enumerate((100, 40000, 7, 3000)):
        p.draw_collocation(4, k, n)
        _, _, parts = p.loss_grad()
        assert same(parts[:2], parts0[:2]), (k, n)          # mse_0 and mse_b: initial-condition points and boundary pairs
    p.close()


def test_poly_draw_resets_the_source_and_takes_one_read_back():
    fam, N = FAMILIES["poly_inf"], 8000
    x, t = restated(fam, 6, 1, N)
    src = np.sin(3 * x) * np.exp(-t)
    p = setup(create(fam), fam)
    p.set_collocation(x, t)
    p.set_source(src)
    p.draw_collocation(6, 1, N)                         # the same points again: the source still goes
    assert_same(p, fresh_with(fam, x, t, N), "draw resets the source")
    gx, gt = p.get_collocation()
    p.set_source(np.sin(3 * gx) * np.exp(-gt))
    assert_same(p, fresh_with(fam, x, t, N, source=src), "draw -> get_collocation -> set_source")
    p.close()


def test_refused_calls_leave_the_handle_as_a_fresh_one():
    import pinn_cabi
    fam = FAMILIES["burgers_v2"]
    x, t = restated(fam, 1, 2, 3000)
    q = fresh_with(fam, x, t, 3000)
    p = fresh_with(fam, x, t, 3000)
    p.loss_grad()
    for first, n, n_global in ((0, -1, 10), (-1, 5, 10), (6, 5, 10), (0, 11, 10), (0, 0, 0), (0, 1, (1 << 53) + 1)):
        assert p.lib.pinn_draw_collocation(p.h, 1, 1, first, n, n_global) != 0, (first, n, n_global)
        assert "pinn_draw_collocation" in p.lib.pinn_last_error().decode()
    w = np.empty(3001)
    assert p.lib.pinn_get_collocation(p.h, w.ctypes.data_as(C.POINTER(C.c_double)), w.ctypes.data_as(C.POINTER(C.c_double)), 3001) != 0
    assert "3001" in p.lib.pinn_last_error().decode()
    assert_same(p, q, "after refused draws")
    p.close(); q.close()
    # models without a collocation set
    for pde, layers, box in (("BURGERS_IDE", BURGERS, STD), ("POLY_IDE", [2, 20, 20, 1], STD), ("BURGERS_DISC", [1, 30, 30, 9],
                                                                                                      ([-1.0], [1.0]))):
        p = pinn_cabi.Pinn(getattr(pinn_cabi, pde), layers, *box)
        with pytest.raises(pinn_cabi.PinnError, match="pinn_draw_collocation: (identification|the discrete-time)"):
            p.draw_collocation(1, 1, 100)
        with pytest.raises(pinn_cabi.PinnError, match="no collocation set"):
            p.get_collocation()
        assert int(p.lib.pinn_launch_count(p.h)) == 0
        p.close()


# ------------------------------------------------------------------------------------------------------------------- mirror
def _mirror_net(hp_extra, N_f=4000):
    from neuralnetwork import NeuralNetwork
    hp = {"layers": BURGERS, "tf_epochs": 6, "tf_lr": 3e-3, "tf_b1": 0.9, "tf_eps": None, "nt_epochs": 0, "nt_lr": 0.8, "nt_ncorr": 50}
    hp.update(hp_extra)

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

    X_f = np.stack(ld.lhs_draw(1, 0, N_f, 0, N_f, *STD), 1)
    return BurgersInformedNN(X_f), X_f


def _hand_loop(net, X_f, X_u, u, draw_every):
    import pinn_cabi
    p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, BURGERS, STD[0], STD[1])
    p.set_pde_params([0.01 / np.pi])
    p.set_collocation(X_f[:, 0], X_f[:, 1])
    p.set_weights(net._w0)
    p.set_data(X_u, u)
    for e in range(6):
        if draw_every and e > 0 and e % draw_every == 0:
            raw_draw(p, 21, e // draw_every, 0, X_f.shape[0], X_f.shape[0])
        p.adam_step(3e-3, 0.9, 0.999, 1e-7, sync=False)
    return p


def test_mirror_resample_every_equals_the_c_abi_loop():
    rng = np.random.default_rng(3)
    X_u = np.stack([rng.uniform(-1, 1, 80), rng.uniform(0, 0.99, 80)], 1)
    u = np.sin(np.pi * X_u[:, :1])
    for extra, every in (({"resample_every": 2, "resample_seed": 21}, 2), ({}, 0)):
        net, X_f = _mirror_net(extra)
        net.tf_optimization(X_u, u)
        hand = _hand_loop(net, X_f, X_u, u, every)
        assert same(net.get_weights(), hand.get_weights()), extra
        assert same(net._native().get_collocation()[0], hand.get_collocation()[0]), extra
        hand.close()
