"""GPU: source tables of the polynomial residual models evaluated on the device (pinn_set_source_terms, DESIGN §4.8).

The device's s at Latin-hypercube sets of up to 2 000 000 points stays within the stated bound of the longdouble restatement
(oracle/source_terms.py), and its trig factors are CUDA's sin and cos bit for bit.  A handle with a table equals, bit for bit, a
fresh handle fed the same points plus pinn_set_source(pinn_get_source(...)), after every way the points or the source change.  RAD
on POLY_INF picks what oracle/rad_draw.py picks from pinn_residual on the pool.  Refused calls change nothing, non-finite points
propagate, and the mirror with a string source equals the same calls made by hand."""
import numpy as np
import pytest

from oracle import lhs_draw as ld
from oracle import rad_draw as rd
from oracle import source_terms as st
from test_gpu_lhs_draw import STD, BIG_SEED, BIG_DRAW, create, setup, same, assert_same, observe

pytestmark = pytest.mark.gpu

POLY = dict(pde="POLY_INF", layers=[2, 20, 20, 20, 1], box=STD)
POLY_IDE = dict(pde="POLY_IDE", layers=[2, 20, 20, 1], box=STD)
WIDE = ([-50.0, 0.0], [50.0, 10.0])
TINY = ([0.5, 0.2], [0.501, 0.201])
K = 0.5


def T(a, p=0, q=0, xk=0, om=0.0, ph=0.0, tk=0, nu=0.0, psi=0.0, al=0.0, ga=0.0, be=0.0, de=0.0):
    return (a, p, q, xk, om, ph, tk, nu, psi, al, ga, be, de)


MANUFACTURED = [T(K * np.pi ** 2 - 1, xk=1, om=np.pi, be=-1.0)]                      # heat, u = sin(pi x) e^-t
# every form: powers up to 3, sin and cos in both variables, all four exponent slots, constants
EVERY = [T(1.5, p=3, q=2, xk=1, om=2.0, ph=0.5, tk=2, nu=3.0, psi=-1.0, al=0.01, ga=-0.002, be=0.1, de=-0.01),
         T(-0.75, p=1, q=3, xk=2, om=-1.3, ph=0.25, tk=1, nu=0.7, psi=2.0),
         T(2.0, p=2), T(-1.25, q=1, al=-0.03, be=0.2), T(0.3), T(0.9, xk=1, om=20.0, ph=-3.0, tk=2, nu=15.0, psi=0.1),
         T(-2.5, p=1, q=1, ga=-0.0004, de=-0.02)]
PULSE = [T(3 * np.exp(-10.0), al=60.0, ga=-100.0, be=4.0, de=-4.0)]
OTHER = [T(0.25, p=2, xk=2, om=np.pi, tk=1, nu=2 * np.pi)]


def table(terms):
    import pinn_cabi
    return pinn_cabi.pack_source_terms(terms)


def poly_handle(fam=POLY):
    return setup(create(fam), fam)


# ------------------------------------------------------------------------------------------------------------------ accuracy
@pytest.mark.parametrize("box, n, terms", [(STD, 2000000, EVERY), (STD, 100000, MANUFACTURED), (STD, 100000, PULSE),
                                           (WIDE, 1000000, EVERY), (TINY, 200000, EVERY)])
def test_device_source_meets_the_longdouble_bound(box, n, terms):
    fam = dict(POLY, box=box)
    p = poly_handle(fam)
    p.set_source_terms(terms)
    p.draw_collocation(BIG_SEED, 3, n)
    s = p.get_source()
    x, t = p.get_collocation()
    assert same(x, ld.lhs_draw(BIG_SEED, 3, n, 0, n, *box)[0])
    worst, same_nonfinite = st.check(s, *table(terms), x, t)
    assert same_nonfinite and worst <= 1.0, worst
    p.close()


def test_trig_factors_are_cudas_sin_and_cos_and_exp_is_cudas_exp():
    import torch
    rng = np.random.default_rng(11)
    x = np.concatenate([rng.uniform(-1, 1, 20000), rng.uniform(-1e3, 1e3, 20000), rng.uniform(-2.0 ** 31, 2.0 ** 31, 20000),
                        np.pi / 2 * np.arange(-2000, 2000), [0.0, 2.0 ** 31 - 1, -(2.0 ** 31 - 1), 1e-300, 5e-324]])
    t = np.zeros_like(x)
    want = {1: torch.sin, 2: torch.cos}
    p = poly_handle()
    p.set_collocation(x, t)
    for kind in (1, 2):
        p.set_source_terms([T(1.0, xk=kind, om=1.0)])
        assert same(p.get_source(), want[kind](torch.from_numpy(x).cuda()).cpu().numpy()), kind
    xe = rng.uniform(-700, 700, 50000)
    p.set_collocation(xe, np.zeros_like(xe))
    p.set_source_terms([T(1.0, al=1.0)])
    assert same(p.get_source(), torch.exp(torch.from_numpy(xe).cuda()).cpu().numpy())
    p.close()


# ------------------------------------------------------------------------------------- a handle equals a fresh one fed s
def fresh_array(fam, x, t, s, w=None):
    """A fresh handle fed the points and the source values (and the weights w)."""
    q = poly_handle(fam)
    if w is not None:
        q.set_weights(w)
    q.set_collocation(x, t)
    q.set_source(s)
    return q


def assert_equal_over_adam(p, q, tag):
    """p equals q now and over five asynchronous Adam steps from a fresh optimiser state."""
    assert_same(p, q, tag)
    p.adam_reset()
    for _ in range(5):
        p.adam_step(1e-3, sync=False)
        q.adam_step(1e-3, sync=False)
    assert same(p.get_weights(), q.get_weights()) and same(p.last_loss(), q.last_loss()), tag
    assert same(p.residual(), q.residual()), tag


def test_table_handle_equals_array_handle_after_every_change():
    fam = POLY
    x, t = ld.lhs_draw(4, 0, 30000, 0, 30000, *STD)
    p = poly_handle()
    p.set_source_terms(EVERY)                                   # no points yet: nothing to evaluate
    p.set_collocation(x, t)
    s = p.get_source()
    assert same(s, p.get_source()) and np.any(s != 0.0)
    assert_equal_over_adam(p, fresh_array(fam, x, t, s, p.get_weights()), "after set_collocation")
    for n in (120000, 7000):                                    # larger and smaller LHS sets
        launches = p.launch_count()
        p.draw_collocation(BIG_SEED, BIG_DRAW + n, n)
        assert p.launch_count() == launches + 2                 # the draw and the source
        x2, t2 = p.get_collocation()
        assert_equal_over_adam(p, fresh_array(fam, x2, t2, p.get_source(), p.get_weights()), "after a draw of %d" % n)
    x2, t2 = p.get_collocation()
    # set on stored points, replaced, removed, replaced by an array
    p.set_source_terms(MANUFACTURED)
    w = p.get_weights()
    assert_same(p, fresh_array(fam, x2, t2, p.get_source(), w), "table set on stored points")
    p.set_source_terms(OTHER)
    s_other = p.get_source()
    assert_same(p, fresh_array(fam, x2, t2, s_other, w), "table replaced")
    p.set_source_terms([])
    assert same(p.get_source(), np.zeros_like(x2))
    q = poly_handle()
    q.set_weights(w)
    q.set_collocation(x2, t2)
    assert_same(p, q, "table removed")
    arr = np.cos(x2) * t2
    p.set_source_terms(EVERY)
    p.set_source(arr)
    assert same(p.get_source(), arr)
    assert_same(p, fresh_array(fam, x2, t2, arr, w), "array replaces the table")
    p.set_collocation(x, t)                                     # an array does not follow the points
    assert same(p.get_source(), np.zeros_like(x))
    p.close(); q.close()


def test_table_follows_the_data_points_on_poly_ide():
    import pinn_cabi
    rng = np.random.default_rng(8)
    p, q = create(POLY_IDE), create(POLY_IDE)
    for h in (p, q):
        h.set_residual([(1.0, 0, (0, 0, 1, 0)), (-1.0, 1, (0, 0, 0, 1)), (0.5, 3, (1, 1, 0, 0))])
        h.set_weights(np.concatenate([rng.standard_normal(h.P - 2) * 0.3, [0.2, -1.0]]) if h is p else p.get_weights())
    p.set_source_terms(EVERY)
    for n in (3000, 500):
        X = np.stack([rng.uniform(-1, 1, n), rng.uniform(0, 0.99, n)], 1)
        u = rng.standard_normal((n, 1))
        p.set_data(X, u)
        q.set_data(X, u)
        q.set_source(p.get_source())
        q.adam_reset()
        worst, ok = st.check(p.get_source(), *table(EVERY), X[:, 0], X[:, 1])
        assert ok and worst <= 1.0
        assert_equal_over_adam(p, q, "POLY_IDE after set_data of %d" % n)
    assert p.pde == pinn_cabi.POLY_IDE
    p.close(); q.close()


# ------------------------------------------------------------------------------------------------------------- RAD on POLY_INF
def rad_expected(terms, seed, draw, n, n_pool, k, c, weights=None):
    a = poly_handle()
    if weights is not None:
        a.set_weights(weights)
    a.draw_collocation(seed, draw, n_pool)
    if terms:
        a.set_source_terms(terms)
    f = a.residual()
    px, pt = a.get_collocation()
    a.close()
    i = rd.rad_indices(f, seed, draw, n, k, c)
    return px[i], pt[i]


@pytest.mark.parametrize("terms", [[], MANUFACTURED, EVERY], ids=["sourceless", "manufactured", "every"])
def test_rad_points_equal_the_oracle_on_pinn_residual(terms):
    b = poly_handle()
    if terms:
        b.set_source_terms(terms)
    for n_pool, n, k, c, seed, draw in [(1, 5, 1, 1.0, 3, 0), (7, 40, 4, 1024.0, 5, 1), (1000, 300, 1, 1.0, BIG_SEED, 2),
                                        (1000, 0, 1, 1.0, 6, 7), (1000, 900, 0, 0.0, 6, 8),
                                        (1000000, 100000, 2, 1.0, BIG_SEED, BIG_DRAW)]:
        launches = b.launch_count()
        b.draw_collocation_rad(seed, draw, n, n_pool, k, c)
        assert b.launch_count() == launches + (5 + (1 if terms else 0)) * (n > 0)
        x, t = b.get_collocation()
        wx, wt = rad_expected(terms, seed, draw, n, n_pool, k, c)
        assert same(x, wx) and same(t, wt), (n_pool, n, k, c)
    b.close()


def test_rad_handle_equals_a_fresh_handle_fed_the_points_and_the_table():
    p = poly_handle()
    p.set_source_terms(EVERY)
    p.set_collocation(*ld.lhs_draw(1, 1, 3000, 0, 3000, *STD))
    for _ in range(3):
        p.adam_step(3e-3, sync=False)                           # RAD reads the stepped weights
    w = p.get_weights()
    p.draw_collocation_rad(BIG_SEED, BIG_DRAW, 20011, 50000, 2, 1.0)
    x, t = rad_expected(EVERY, BIG_SEED, BIG_DRAW, 20011, 50000, 2, 1.0, weights=w)
    q = poly_handle()
    q.set_weights(w)
    q.set_collocation(x, t)
    q.set_source_terms(EVERY)
    assert same(p.get_source(), q.get_source())
    assert_same(p, q, "after RAD")
    p.adam_reset()
    for _ in range(5):
        p.adam_step(1e-3, sync=False)
        q.adam_step(1e-3, sync=False)
    assert same(p.get_weights(), q.get_weights()) and same(p.last_loss(), q.last_loss())
    p.close(); q.close()


# --------------------------------------------------------------------------------------------------- refusals and non-finite
def test_refused_calls_change_nothing():
    import ctypes as C
    import pinn_cabi
    x, t = ld.lhs_draw(2, 2, 4000, 0, 4000, *STD)
    p, q = poly_handle(), poly_handle()
    for h in (p, q):
        h.set_collocation(x, t)
        h.set_source_terms(MANUFACTURED)
    p.loss_grad()
    launches = p.launch_count()
    form, par = table(EVERY)
    ip = C.POINTER(C.c_int)
    dp = C.POINTER(C.c_double)
    for k_bad, bad in [("n", None), ("form", 256), ("form", 3 << 4), ("form", 3 << 6), ("form", -1)] + \
                      [("par", (j, v)) for j in range(9) for v in (np.nan, np.inf, -np.inf)]:
        f, pr, n = form.copy(), par.copy(), len(form)
        if k_bad == "n":
            for n in (-1, 17):
                assert p.lib.pinn_set_source_terms(p.h, n, f.ctypes.data_as(ip), pr.ctypes.data_as(dp)) != 0
                assert "n_terms = %d is outside 0..16" % n in p.lib.pinn_last_error().decode()
            continue
        if k_bad == "form":
            f[2] = bad
        else:
            pr[3, bad[0]] = bad[1]
        assert p.lib.pinn_set_source_terms(p.h, n, f.ctypes.data_as(ip), pr.ctypes.data_as(dp)) != 0, (k_bad, bad)
        assert "pinn_set_source_terms: term " in p.lib.pinn_last_error().decode()
    assert p.lib.pinn_set_source_terms(p.h, 2, None, None) != 0
    assert p.launch_count() == launches
    assert_same(p, q, "after refused tables")
    # RAD with an array source, and without a residual spec
    p.set_source(p.get_source())
    q.set_source(q.get_source())
    launches = p.launch_count()
    with pytest.raises(pinn_cabi.PinnError, match="pinn_draw_collocation_rad: POLY_INF.*array.*pinn_set_source_terms"):
        p.draw_collocation_rad(1, 1, 100, 1000)
    assert p.launch_count() == launches
    assert_same(p, q, "after a refused RAD call")
    r = create(POLY)
    r.set_source_terms(MANUFACTURED)
    with pytest.raises(pinn_cabi.PinnError, match="pinn_draw_collocation_rad: POLY_INF has no residual spec"):
        r.draw_collocation_rad(1, 1, 100, 1000)
    assert r.launch_count() == 0
    # models without a source
    b = create(dict(pde="BURGERS_INF", layers=[2, 20, 20, 1], box=STD))
    with pytest.raises(pinn_cabi.PinnError, match="pinn_set_source_terms: only the polynomial"):
        b.set_source_terms(MANUFACTURED)
    with pytest.raises(pinn_cabi.PinnError, match="pinn_get_source: only the polynomial"):
        b.get_source()
    w = np.empty(3)
    assert p.lib.pinn_get_source(p.h, w.ctypes.data_as(dp), 3) != 0 and "4000" in p.lib.pinn_last_error().decode()
    for h in (p, q, r, b):
        h.close()


def test_non_finite_points_propagate_into_the_source_and_the_loss():
    x, t = ld.lhs_draw(3, 1, 2000, 0, 2000, *STD)
    x[5], t[17], x[40], t[41] = np.nan, -np.inf, -np.inf, np.nan
    p = poly_handle()
    p.set_collocation(x, t)
    p.set_source_terms(MANUFACTURED)
    s = p.get_source()
    assert not np.isfinite(s[[5, 17, 40, 41]]).any() and np.isfinite(np.delete(s, [5, 17, 40, 41])).all()
    worst, ok = st.check(s, *table(MANUFACTURED), x, t)
    assert ok and worst <= 1.0
    a, b = observe(p), observe(fresh_array(POLY, x, t, s))
    assert np.isnan(a["loss"]) and same(a["loss"], b["loss"]) and same(a["grad"], b["grad"])
    p.close()


# ------------------------------------------------------------------------------------------------------------------- mirror
def mirror_run(source_key, N_f=4000):
    import pinn_cabi
    from neuralnetwork import NeuralNetwork
    hp = {"layers": POLY["layers"], "tf_epochs": 7, "tf_lr": 3e-3, "tf_b1": 0.9, "tf_eps": None, "nt_epochs": 0, "nt_lr": 0.8,
          "nt_ncorr": 50, "resample_seed": 21}
    hp.update({"resample_every": 3} if source_key == "lhs" else {"rad_every": 3, "rad_pool": 12345, "rad_k": 2, "rad_c": 0.5})

    class Quiet(object):
        def log_train_opt(self, name):
            pass

        def log_train_epoch(self, epoch, loss, custom="", is_iter=False):
            float(loss)

    class Heat(NeuralNetwork):
        pde, residual, source = "poly", "u_t - k*u_xx", "(k*pi**2 - 1)*sin(pi*x)*exp(-t)"

        def __init__(self, X_f):
            super().__init__(hp, Quiet(), np.array(STD[1]), np.array(STD[0]))
            self.k = K
            self.x_f, self.t_f = X_f[:, 0:1], X_f[:, 1:2]

    rng = np.random.default_rng(3)
    X_u = np.stack([rng.uniform(-1, 1, 80), rng.uniform(0, 0.99, 80)], 1)
    u = np.sin(np.pi * X_u[:, :1])
    X_f = np.stack(ld.lhs_draw(1, 0, N_f, 0, N_f, *STD), 1)
    net = Heat(X_f)
    net.tf_optimization(X_u, u)
    p = pinn_cabi.Pinn(pinn_cabi.POLY_INF, POLY["layers"], STD[0], STD[1])
    p.set_residual([(1.0, 0, (0, 0, 1, 0)), (-K, 0, (0, 0, 0, 1))])
    p.set_source_terms(MANUFACTURED)
    p.set_collocation(X_f[:, 0], X_f[:, 1])
    p.set_weights(net._w0)
    p.set_data(X_u, u)
    for e in range(7):
        if e > 0 and e % 3 == 0:
            if source_key == "lhs":
                p.draw_collocation(21, e // 3, N_f)
            else:
                p.draw_collocation_rad(21, e // 3, N_f, 12345, 2, 0.5)
        p.adam_step(3e-3, 0.9, 0.999, 1e-7, sync=False)
    assert same(net.get_weights(), p.get_weights())
    assert same(net._native().get_source(), p.get_source())
    assert same(net.f_model(), p.residual())
    p.close()


@pytest.mark.parametrize("how", ["lhs", "rad"])
def test_mirror_string_source_equals_the_c_abi_loop(how):
    mirror_run(how)

