"""CPU: the two oracles of user-defined polynomial residuals -- oracle.reference_port_poly (nested autograd) against
oracle.taylor_poly (Taylor streams + analytic seeds) on random specs, finite differences, the longdouble run, equality with the
Burgers oracles for the Burgers specs, and the seed formula at u = 0."""
import numpy as np
import pytest

from oracle import reference_port as rp, reference_port_poly as rpp, taylor as ty, taylor_poly as tpo
from conftest import load_golden


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def random_spec(rng, n_terms, ide):
    terms = []
    for _ in range(n_terms):
        e = tuple(int(v) for v in rng.integers(0, 4, 4))
        if not any(e):
            e = (1, 0, 0, 0)
        terms.append((float(rng.uniform(-1, 1)), int(rng.integers(0, 5)) if ide else 0, e))
    return terms


def random_problem(seed, ide, layers=(2, 9, 12, 1), n=40):
    rng = np.random.default_rng(seed)
    layers = list(layers)
    lb, ub = np.array([-0.5, 1.0]), np.array([2.5, 4.0])
    X_u = lb + (ub - lb) * rng.random((n, 2))
    u = rng.standard_normal((n, 1))
    X_f = None if ide else lb + (ub - lb) * rng.random((2 * n, 2))
    s = 0.2 * rng.standard_normal((n if ide else 2 * n, 1))
    w = 0.8 * rp.glorot_normal_flat(layers, rng)
    if ide:
        w = np.concatenate([w, [0.3, -0.2]])
    return layers, lb, ub, random_spec(rng, int(rng.integers(1, 17)), ide), X_u, u, X_f, s, w


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("ide", [False, True])
def test_oracles_agree_on_random_specs(seed, ide):
    layers, lb, ub, terms, X_u, u, X_f, s, w = random_problem(seed, ide)
    pb = rpp.PolyProblem(layers, lb, ub, terms, X_u, u, X_f=X_f, source=s, identification=ide)
    f, g = rp.loss_and_flat_grad(pb, w)
    f2, g2, parts = tpo.poly_loss_grad(w, layers, lb, ub, terms, X_u, u, X_f=X_f, source=s, identification=ide)
    assert abs(f - f2) <= 1e-13 * abs(f) and rel(g2, g) <= 1e-13
    assert abs(sum(parts) - f2) <= 1e-14 * abs(f2)
    fr = tpo.poly_residual(w, layers, lb, ub, terms, X_u if ide else X_f, source=s, identification=ide)
    assert rel(fr, pb.f_model(w)) <= 1e-13


def test_finite_differences():
    layers, lb, ub, terms, X_u, u, X_f, s, w = random_problem(3, True, layers=(2, 6, 1), n=12)
    f0, g, _ = tpo.poly_loss_grad(w, layers, lb, ub, terms, X_u, u, source=s, identification=True)
    rng = np.random.default_rng(0)
    for i in list(rng.choice(w.size - 2, 6, replace=False)) + [w.size - 2, w.size - 1]:
        h = 1e-6 * max(1.0, abs(w[i]))
        wp, wm = w.copy(), w.copy()
        wp[i] += h
        wm[i] -= h
        fp = tpo.poly_loss_grad(wp, layers, lb, ub, terms, X_u, u, source=s, identification=True)[0]
        fm = tpo.poly_loss_grad(wm, layers, lb, ub, terms, X_u, u, source=s, identification=True)[0]
        assert abs((fp - fm) / (2 * h) - g[i]) <= 1e-6 * max(1.0, abs(g[i])), i


def test_longdouble_run_is_close_to_float64():
    layers, lb, ub, terms, X_u, u, X_f, s, w = random_problem(4, True)
    a = tpo.poly_loss_grad(w, layers, lb, ub, terms, X_u, u, source=s, identification=True, dtype=np.longdouble, magnitudes=True)
    b = tpo.poly_loss_grad(w, layers, lb, ub, terms, X_u, u, source=s, identification=True)
    assert a[1].dtype == np.longdouble and len(a) == 4 and a[3].shape == a[1].shape
    assert abs(float(a[0]) - b[0]) <= 1e-13 * abs(b[0]) and rel(a[1].astype(float), b[1]) <= 1e-12
    assert np.all(a[3] >= np.abs(a[1]) * (1 - 1e-12))


def _burgers_terms(nu=None):
    if nu is not None:
        return [(1.0, 0, (0, 0, 1, 0)), (1.0, 0, (1, 1, 0, 0)), (-nu, 0, (0, 0, 0, 1))]
    return [(1.0, 0, (0, 0, 1, 0)), (1.0, 1, (1, 1, 0, 0)), (-1.0, 4, (0, 0, 0, 1))]


def test_burgers_specs_equal_the_burgers_oracles():
    g = load_golden("burgers_inf")
    layers, nu = [int(v) for v in g["layers"]], float(g["nu"])
    X_f = g["X_f"][:800]
    a = tpo.poly_loss_grad(g["w"], layers, g["lb"], g["ub"], _burgers_terms(nu), g["X_u"], g["u"], X_f=X_f)
    b = ty.burgers_loss_grad(g["w"], layers, g["lb"], g["ub"], X_f, g["X_u"], g["u"], nu=nu)
    assert abs(a[0] - b[0]) <= 1e-15 * abs(b[0]) and rel(a[1], b[1]) <= 1e-15
    pb = rpp.PolyProblem(layers, g["lb"], g["ub"], _burgers_terms(nu), g["X_u"], g["u"], X_f=X_f)
    ref = rp.BurgersInference(layers, g["lb"], g["ub"], nu, X_f, g["X_u"], g["u"])
    fa, ga = rp.loss_and_flat_grad(pb, g["w"])
    fb, gb = rp.loss_and_flat_grad(ref, g["w"])
    assert abs(fa - fb) <= 1e-15 * abs(fb) and rel(ga, gb) <= 1e-15
    g = load_golden("burgers_ide")
    layers = [int(v) for v in g["layers"]]
    for tag in ("", "2"):
        a = tpo.poly_loss_grad(g["w" + tag], layers, g["lb"], g["ub"], _burgers_terms(), g["X_u"], g["u"], identification=True)
        b = ty.burgers_loss_grad(g["w" + tag], layers, g["lb"], g["ub"], None, g["X_u"], g["u"], identification=True)
        assert abs(a[0] - b[0]) <= 1e-15 * abs(b[0]) and rel(a[1], b[1]) <= 1e-15
        pb = rpp.PolyProblem(layers, g["lb"], g["ub"], _burgers_terms(), g["X_u"], g["u"], identification=True)
        fa, ga = rp.loss_and_flat_grad(pb, g["w" + tag])
        fb, gb = rp.loss_and_flat_grad(rp.BurgersIdentification(layers, g["lb"], g["ub"], g["X_u"], g["u"]), g["w" + tag])
        assert abs(fa - fb) <= 1e-15 * abs(fb) and rel(ga, gb) <= 1e-15


def test_seed_formula_at_u_zero():
    """u = 0 exactly: d(u^e)/du is 1 for e = 1 and 0 for e = 2, 3 -- the formula takes no quotient by u."""
    terms = [(2.0, 0, (1, 1, 0, 0)), (3.0, 0, (2, 0, 1, 0)), (-1.5, 0, (3, 0, 0, 1)), (0.5, 2, (1, 0, 0, 0))]
    V = tuple(np.array([[v]]) for v in (0.0, 0.7, -1.3, 2.1))
    f, D, f1, f2 = tpo.poly_terms(terms, V, 0.4, -0.6)
    assert np.all(np.isfinite(f)) and all(np.all(np.isfinite(d)) for d in D)
    assert f[0, 0] == 0.0
    assert D[0][0, 0] == 2.0 * 0.7 + 0.5 * -0.6                 # only the e = 1 terms survive at u = 0
    assert D[1][0, 0] == 0.0 and D[2][0, 0] == 0.0 and D[3][0, 0] == 0.0
    assert f2[0, 0] == 0.0 and f1[0, 0] == 0.0
    # against finite differences of f in u around 0
    h = 1e-7
    fp = tpo.poly_terms(terms, (V[0] + h,) + V[1:], 0.4, -0.6)[0]
    fm = tpo.poly_terms(terms, (V[0] - h,) + V[1:], 0.4, -0.6)[0]
    assert abs((fp - fm)[0, 0] / (2 * h) - D[0][0, 0]) <= 1e-7
