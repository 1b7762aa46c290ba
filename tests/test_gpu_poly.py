"""GPU: user-defined polynomial residuals (PINN_POLY_INF = 8, PINN_POLY_IDE = 9) on the generic fused kernel -- golden vectors
(tests/golden/make_poly_golden.py), Adam and L-BFGS trajectories, the Burgers spec against the pinned reference run and against
the hard-wired Burgers heads, the per-parameter-block check against the extended-precision oracle, ragged sizes and widths 7 to
256, bitwise reproducibility, the C ABI's error paths, the source reset, and the Python surface."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, assert_matches_reference_run, load_golden

pytestmark = pytest.mark.gpu
sys.path[:0] = [GOLDEN, os.path.dirname(os.path.abspath(__file__))]

CASES = ("ac", "heat", "fisher", "stress")


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


@pytest.fixture(scope="module")
def cabi():
    import pinn_cabi
    pinn_cabi.load()
    return pinn_cabi


def burgers_terms(nu=None):
    """u_t + u u_x - nu u_xx (inference) or u_t + l1 u u_x - e^l2 u_xx (identification)."""
    if nu is not None:
        return [(1.0, 0, (0, 0, 1, 0)), (1.0, 0, (1, 1, 0, 0)), (-nu, 0, (0, 0, 0, 1))]
    return [(1.0, 0, (0, 0, 1, 0)), (1.0, 1, (1, 1, 0, 0)), (-1.0, 4, (0, 0, 0, 1))]


def make(cabi, layers, lb, ub, terms, X_u, u, X_f=None, source=None, ide=False):
    p = cabi.Pinn(cabi.POLY_IDE if ide else cabi.POLY_INF, [int(v) for v in layers], lb, ub)
    p.set_residual(terms)
    p.set_data(X_u, u)
    if not ide:
        p.set_collocation(X_f[:, 0], X_f[:, 1])
    if source is not None:
        p.set_source(source)
    return p


def golden(cabi, name):
    g = load_golden("poly")
    c = {k[len(name) + 1:]: g[k] for k in g.files if k.startswith(name + "_")}
    c["terms"] = [(float(a), int(k), tuple(int(v) for v in e)) for a, k, e in zip(c["coef"], c["kind"], c["exps"])]
    ide = bool(c["identification"])
    return c, make(cabi, c["layers"], c["lb"], c["ub"], c["terms"], c["X_u"], c["u"], c.get("X_f"), c.get("source"), ide)


@pytest.mark.parametrize("name", CASES)
def test_golden_loss_grad_probes_residual(cabi, name):
    c, p = golden(cabi, name)
    assert p.P == c["w"].size
    loss, grad, parts = p.loss_grad(w=c["w"])
    assert abs(loss - c["loss"]) <= 1e-10 * abs(c["loss"])
    assert rel(grad, c["grad"]) < 1e-10
    if bool(c["identification"]):
        assert rel(grad[-2:], c["grad"][-2:]) < 1e-10
    assert np.allclose(parts[[0, 2]], c["parts"], rtol=1e-10) and parts[1] == 0.0
    D = np.stack(p.derivatives(c["X_probe"]), 1)[:, :, 0]
    assert rel(D, c["probe"]) <= 1e-11
    assert rel(p.predict(c["X_probe"]), c["probe"][:, :1]) <= 1e-11
    f = p.residual()
    assert f.shape == c["residual"].shape and rel(f, c["residual"]) <= 1e-10


@pytest.mark.parametrize("name", CASES)
def test_golden_adam_and_lbfgs(cabi, name):
    c, p = golden(cabi, name)
    p.set_weights(c["w"])
    losses = [p.adam_step(1e-3) for _ in range(5)]
    assert rel(losses, c["adam_losses"]) < 1e-8 and rel(p.get_weights(), c["adam_w"]) < 1e-8
    c, p = golden(cabi, name)
    p.set_weights(c["w"])
    r = p.lbfgs(6, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, sync_every=1, want_x_final=True)
    assert r["n_eval"] == len(c["lbfgs_f"])
    assert rel(r["f_hist"], c["lbfgs_f"]) < 1e-7
    assert rel(r["x_final"], c["lbfgs_x_final"]) < 1e-7
    assert rel(p.get_weights(), c["lbfgs_x_eval"][-1]) < 1e-7


def _burgers_handles(cabi, ide):
    g = load_golden("burgers_ide" if ide else "burgers_inf")
    layers = [int(v) for v in g["layers"]]
    if ide:
        return g, make(cabi, layers, g["lb"], g["ub"], burgers_terms(), g["X_u"], g["u"], ide=True)
    return g, make(cabi, layers, g["lb"], g["ub"], burgers_terms(float(g["nu"])), g["X_u"], g["u"], g["X_f"])


def test_burgers_spec_matches_reference_run(cabi):
    g, p = _burgers_handles(cabi, False)
    info = p.kernel_info()
    assert info["grid"] == 2 * info["sms"]                  # the generic kernel (2 CTAs per SM), even on the [2, 20x8, 1] net
    loss, grad, _ = p.loss_grad(w=g["w"])
    assert_matches_reference_run(loss, grad, "burgers_inf_loss", "burgers_inf_grad", tol=1e-10)
    g, p = _burgers_handles(cabi, True)
    for tag in ("", "2"):
        loss, grad, _ = p.loss_grad(w=g["w" + tag])
        assert_matches_reference_run(loss, grad, "burgers_ide_loss" + tag, "burgers_ide_grad" + tag, tol=1e-10)


@pytest.mark.parametrize("ide", [False, True])
def test_burgers_spec_matches_the_hardwired_generic_head(cabi, monkeypatch, ide):
    """Same generic kernel, the polynomial head against the hard-wired Burgers head (PINN_FORCE_GENERIC=1): equal to 1e-13.
    The two heads sum the residual's terms in a different order, so equality is not bitwise in general; the test prints
    which it is."""
    monkeypatch.setenv("PINN_FORCE_GENERIC", "1")
    g, p = _burgers_handles(cabi, ide)
    layers = [int(v) for v in g["layers"]]
    q = cabi.Pinn(cabi.BURGERS_IDE if ide else cabi.BURGERS_INF, layers, g["lb"], g["ub"])
    if not ide:
        q.set_pde_params([float(g["nu"])])
        q.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1])
    q.set_data(g["X_u"], g["u"])
    assert q.kernel_info()["grid"] == 2 * q.kernel_info()["sms"]
    a, b = p.loss_grad(w=g["w"]), q.loss_grad(w=g["w"])
    assert abs(a[0] - b[0]) <= 1e-13 * abs(b[0]) and rel(a[1], b[1]) <= 1e-13
    assert np.allclose(a[2], b[2], rtol=1e-13, atol=0)
    assert rel(p.residual(), q.residual()) <= 1e-13
    print("[poly] Burgers %s spec vs hard-wired head: bitwise %s (loss %r)" %
          ("IDE" if ide else "INF", a[0] == b[0] and np.array_equal(a[1], b[1]), a[0] - b[0]))


def test_stress_spec_per_block_against_longdouble(cabi):
    from oracle import taylor as ty
    from oracle import taylor_poly as tpo
    from test_gpu_precision import check
    c, p = golden(cabi, "stress")
    got = p.loss_grad(w=c["w"])
    args = (c["layers"], c["lb"], c["ub"], c["terms"], c["X_u"], c["u"])
    kw = dict(source=c["source"], identification=True)
    ref = tpo.poly_loss_grad(c["w"], *args, dtype=np.longdouble, magnitudes=True, **kw)
    ref64 = tpo.poly_loss_grad(c["w"], *args, **kw)
    check("poly stress", got, ref, ref64, ty.param_blocks(c["layers"], 2), [0, 2])


def random_case(hidden, n, seed, ide):
    from make_poly_golden import stress_terms
    from oracle import reference_port as rp
    rng = np.random.default_rng(seed)
    layers = [2] + list(hidden) + [1]
    lb, ub = np.array([-1.5, 0.5]), np.array([2.0, 3.0])
    X_u = lb + (ub - lb) * rng.random((max(n // 3, 1), 2)) if not ide else lb + (ub - lb) * rng.random((n, 2))
    u = rng.standard_normal((X_u.shape[0], 1))
    X_f = None if ide else lb + (ub - lb) * rng.random((n, 2))
    terms = stress_terms(rng)[:8] if ide else [(float(v), 0, e) for v, _, e in stress_terms(rng)[:8]]
    w = 0.7 * rp.glorot_normal_flat(layers, rng)
    if ide:
        w = np.concatenate([w, [0.4, -0.3]])
    s = 0.1 * rng.standard_normal(n)
    return layers, lb, ub, terms, X_u, u, X_f, s, w


def _sms(cabi):
    p = cabi.Pinn(cabi.POLY_INF, [2, 4, 1], [0, 0], [1, 1])
    return p.kernel_info()["sms"]


RAGGED = [([20] * 8, 1000), ([20] * 4, 1), ([7, 7], 7), ([9], 9), ([33, 20, 33], 131), ([256, 256], 300), ([128, 7, 200], 77)]


@pytest.mark.parametrize("ide", [False, True])
@pytest.mark.parametrize("hidden,n", RAGGED)
def test_ragged_sizes_and_widths_against_taylor(cabi, hidden, n, ide):
    from oracle import taylor_poly as tpo
    layers, lb, ub, terms, X_u, u, X_f, s, w = random_case(hidden, n, 5 * n + len(hidden), ide)
    p = make(cabi, layers, lb, ub, terms, X_u, u, X_f, s, ide)
    loss, grad, parts = p.loss_grad(w=w)
    f2, g2, parts2 = tpo.poly_loss_grad(w, layers, lb, ub, terms, X_u, u, X_f=X_f, source=s, identification=ide)
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10
    assert np.allclose(parts[[0, 2]], parts2, rtol=1e-10)
    fr = tpo.poly_residual(w, layers, lb, ub, terms, X_u if ide else X_f, source=s, identification=ide)
    assert rel(p.residual(), fr) <= 1e-10


def test_above_grid_times_points_per_cta(cabi):
    from oracle import taylor_poly as tpo
    n = 2 * 16 * _sms(cabi) * 3 + 5
    layers, lb, ub, terms, X_u, u, X_f, s, w = random_case([20] * 3, n, 3, False)
    p = make(cabi, layers, lb, ub, terms, X_u, u, X_f, s, False)
    loss, grad, _ = p.loss_grad(w=w)
    f2, g2, _ = tpo.poly_loss_grad(w, layers, lb, ub, terms, X_u, u, X_f=X_f, source=s)
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10


def test_two_evaluations_are_bit_identical(cabi):
    c, p = golden(cabi, "stress")
    a, b = p.loss_grad(w=c["w"]), p.loss_grad(w=c["w"])
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    c, p = golden(cabi, "heat")
    a, b = p.loss_grad(w=c["w"]), p.loss_grad(w=c["w"])
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_source_is_reset_by_new_residual_points(cabi):
    from oracle import taylor_poly as tpo
    c, p = golden(cabi, "heat")
    args = (c["layers"], c["lb"], c["ub"], c["terms"], c["X_u"], c["u"])
    with_s = p.loss_grad(w=c["w"])[0]
    assert abs(with_s - c["loss"]) <= 1e-10 * c["loss"]
    p.set_collocation(c["X_f"][:, 0], c["X_f"][:, 1])          # the same points again: the source is gone
    no_s = p.loss_grad(w=c["w"])[0]
    ref = tpo.poly_loss_grad(c["w"], *args, X_f=c["X_f"])[0]
    assert abs(no_s - ref) <= 1e-10 * ref and abs(no_s - with_s) > 1e-6 * ref
    assert rel(p.residual(), tpo.poly_residual(c["w"], c["layers"], c["lb"], c["ub"], c["terms"], c["X_f"])) <= 1e-10
    p.set_data(c["X_u"][:10], c["u"][:10])                      # data points of POLY_INF are not residual points
    p.set_source(c["source"])
    assert abs(p.loss_grad(w=c["w"])[0] - tpo.poly_loss_grad(c["w"], c["layers"], c["lb"], c["ub"], c["terms"], c["X_u"][:10],
                                                            c["u"][:10], X_f=c["X_f"], source=c["source"])[0]) <= 1e-10
    f, q = golden(cabi, "stress")                               # POLY_IDE: new data points reset the source
    q.set_data(f["X_u"], f["u"])
    ref = tpo.poly_loss_grad(f["w"], f["layers"], f["lb"], f["ub"], f["terms"], f["X_u"], f["u"], identification=True)[0]
    assert abs(q.loss_grad(w=f["w"])[0] - ref) <= 1e-10 * ref


def test_spec_may_be_replaced(cabi):
    from oracle import taylor_poly as tpo
    c, p = golden(cabi, "ac")
    p.loss_grad(w=c["w"])
    terms = [(1.0, 0, (0, 0, 1, 0)), (-0.01, 0, (0, 0, 0, 1))]
    p.set_residual(terms)
    loss, grad, _ = p.loss_grad(w=c["w"])
    f2, g2, _ = tpo.poly_loss_grad(c["w"], c["layers"], c["lb"], c["ub"], terms, c["X_u"], c["u"], X_f=c["X_f"])
    assert abs(loss - f2) <= 1e-10 * f2 and rel(grad, g2) < 1e-10


def test_error_paths(cabi):
    lb, ub = [0, 0], [1, 1]
    ok = [(1.0, 0, (0, 0, 1, 0))]
    with pytest.raises(cabi.PinnError, match="one GPU"):
        cabi.Pinn(cabi.POLY_INF, [2, 8, 1], lb, ub, world=2, nccl_uid=b"\0" * 128)
    with pytest.raises(cabi.PinnError, match="net \\[2, ..., 1\\]"):
        cabi.Pinn(cabi.POLY_IDE, [2, 8, 2], lb, ub)
    with pytest.raises(cabi.PinnError, match="unknown pde_id"):
        cabi.Pinn(10, [2, 8, 1], lb, ub)
    h = cabi.Pinn(cabi.POLY_INF, [2, 8, 1], lb, ub)
    h.set_data(np.zeros((3, 2)), np.zeros(3))
    h.set_collocation(np.zeros(5), np.zeros(5))
    for call in (lambda: h.loss_grad(w=np.zeros(h.P)), lambda: h.adam_step(1e-3), lambda: h.lbfgs(2), h.residual):
        with pytest.raises(cabi.PinnError, match="pinn_set_residual first"):
            call()
    with pytest.raises(cabi.PinnError, match="outside 1..16"):
        h.set_residual([])
    with pytest.raises(cabi.PinnError, match="outside 1..16"):
        h.set_residual(ok * 17)
    with pytest.raises(cabi.PinnError, match="exponent 4 .*outside 0..3"):
        h.set_residual([(1.0, 0, (4, 0, 0, 0))])
    with pytest.raises(cabi.PinnError, match="outside 0..3"):
        h.set_residual([(1.0, 0, (0, -1, 1, 0))])
    with pytest.raises(cabi.PinnError, match="all four exponents are 0"):
        h.set_residual(ok + [(2.0, 0, (0, 0, 0, 0))])
    with pytest.raises(cabi.PinnError, match="POLY_INF has no trainable lambdas"):
        h.set_residual([(1.0, 1, (1, 0, 0, 0))])
    with pytest.raises(cabi.PinnError, match="not finite"):
        h.set_residual([(float("nan"), 0, (1, 0, 0, 0))])
    with pytest.raises(cabi.PinnError, match="not finite"):
        h.set_residual([(float("inf"), 0, (1, 0, 0, 0))])
    k = cabi.Pinn(cabi.POLY_IDE, [2, 8, 1], lb, ub)
    with pytest.raises(cabi.PinnError, match="kind 5 is outside 0..4"):
        k.set_residual([(1.0, 5, (1, 0, 0, 0))])
    k.set_residual([(1.0, 4, (1, 0, 0, 0))])
    h.set_residual(ok)
    with pytest.raises(cabi.PinnError, match="4 values given but 5 residual points"):
        h.set_source(np.zeros(4))
    with pytest.raises(cabi.PinnError, match="residual points are stored"):
        h.residual(4)
    with pytest.raises(cabi.PinnError, match="zero-copy"):
        h.set_collocation_mapped(None, None, 5)
    with pytest.raises(cabi.PinnError, match="stage matrices"):
        h.set_irk(np.zeros((5, 4)))
    with pytest.raises(cabi.PinnError, match="two snapshots"):
        h.set_snapshot(0, np.zeros(3), np.zeros(3))
    with pytest.raises(cabi.PinnError, match="boundary term"):
        h.set_boundary([0.0])
    with pytest.raises(cabi.PinnError, match="takes no constants"):
        h.set_pde_params([0.01])
    with pytest.raises(cabi.PinnError, match="data points as residual points"):
        k.set_collocation(np.zeros(3), np.zeros(3))
    with pytest.raises(cabi.PinnError, match="only the polynomial residual models"):
        cabi.Pinn(cabi.BURGERS_INF, [2, 8, 1], lb, ub).set_residual(ok)
    with pytest.raises(cabi.PinnError, match="only the polynomial residual models"):
        cabi.Pinn(cabi.BURGERS_INF, [2, 8, 1], lb, ub).set_source([])
    assert list(h.get_params()) == [] and k.P == h.P + 2
    k.set_weights(np.arange(k.P, dtype=float))
    assert list(k.get_params()) == [k.P - 2.0, k.P - 1.0]


def test_python_surface(capsys):
    """Subclasses with a residual string: Fisher-KPP identification (fit(X_u, u) from the lambda_1 / lambda_2 attributes) and the
    heat equation with a source method (inference on x_f, t_f); predict, f_model and get_params."""
    from logger import Logger
    from neuralnetwork import NeuralNetwork
    from oracle import reference_port as rp, reference_port_poly as rpp, taylor_poly as tpo
    from make_poly_golden import HEAT_K, heat_source
    g = load_golden("poly")
    hp = {"layers": [int(v) for v in g["fisher_layers"]], "tf_epochs": 3, "tf_lr": 0.001, "tf_b1": 0.9, "tf_eps": None,
          "nt_epochs": 4, "nt_lr": 0.8, "nt_ncorr": 50, "log_frequency": 1}

    class FisherKPP(NeuralNetwork):
        pde = "poly"
        residual = "u_t - exp(l2)*u_xx - l1*u*(1 - u)"
        lambda_1, lambda_2 = 0.7, -1.5

    pinn = FisherKPP(hp, Logger(hp), g["fisher_ub"], g["fisher_lb"])
    pinn._w0 = np.asarray(g["fisher_w"])[:-2].copy()
    pinn.logger.set_error_fn(lambda: 0.0)
    assert list(pinn.get_params(numpy=True)) == [0.7, -1.5]
    pinn.fit(g["fisher_X_u"], g["fisher_u"])
    out = capsys.readouterr().out
    assert "tf_epoch =      2" in out and "nt_epoch =      3" in out
    terms = [(1.0, 0, (0, 0, 1, 0)), (-1.0, 4, (0, 0, 0, 1)), (-1.0, 1, (1, 0, 0, 0)), (1.0, 1, (2, 0, 0, 0))]
    pb = rpp.PolyProblem(hp["layers"], g["fisher_lb"], g["fisher_ub"], terms, g["fisher_X_u"], g["fisher_u"], identification=True)
    wa, _, _ = rp.adam_train(pb, g["fisher_w"], 3, lr=1e-3)
    tr = rp.lbfgs_fixed_step(lambda z: rp.loss_and_flat_grad(pb, z), wa, max_iter=4, learning_rate=0.8, n_correction=50,
                             tol_fun=np.finfo(float).eps)
    w = pinn.get_weights().numpy()
    assert rel(w, tr.x_eval[-1]) < 1e-7
    Xp = g["fisher_X_probe"]
    assert pinn.predict(Xp).shape == (32, 1) and rel(pinn.predict(Xp), rp.predict(pb, w, Xp)) < 1e-10
    assert rel(pinn.f_model(Xp), pb.f_model(w, Xp)) < 1e-9
    assert pinn.f_model().shape == (g["fisher_X_u"].shape[0], 1) and rel(pinn.f_model(), pb.f_model(w)) < 1e-9
    l1, l2 = pinn.get_params(numpy=True)
    assert l1 == w[-2] and l2 == w[-1]

    class Heat(NeuralNetwork):
        pde = "poly"
        residual = "u_t - k*u_xx"
        k = HEAT_K

        def __init__(self, hp, logger, X_f, ub, lb):
            super().__init__(hp, logger, ub, lb)
            self.x_f, self.t_f = X_f[:, 0:1], X_f[:, 1:2]

        def source(self, x, t):
            return heat_source(x, t, self.k)

    hp = dict(hp, layers=[int(v) for v in g["heat_layers"]], tf_epochs=2, nt_epochs=2)
    heat = Heat(hp, Logger(hp), g["heat_X_f"], g["heat_ub"], g["heat_lb"])
    heat._w0 = np.asarray(g["heat_w"]).copy()
    loss, grads = heat.grad(g["heat_X_u"], g["heat_u"])
    assert abs(loss - g["heat_loss"]) <= 1e-10 * g["heat_loss"] and len(grads) == 6
    assert rel(heat.f_model(), g["heat_residual"]) <= 1e-10
    Xp = g["heat_X_probe"]
    f = tpo.poly_residual(g["heat_w"], hp["layers"], g["heat_lb"], g["heat_ub"], [(1.0, 0, (0, 0, 1, 0)), (-HEAT_K, 0, (0, 0, 0, 1))],
                          Xp, source=heat_source(Xp[:, 0:1], Xp[:, 1:2]))
    assert rel(heat.f_model(Xp), f) <= 1e-10
    assert heat.get_params(numpy=True) == []
