"""CPU: the extended-precision oracles of the KdV, Allen-Cahn and polynomial residual heads, as tests/test_gpu_precision_heads.py
uses them -- the magnitudes S are wired (finite, the gradient's shape, |g| <= S entrywise), the term-wise lambda magnitude of the
polynomial head, and the per-block check has teeth: a run whose U_xx or U_xxx path is off by a small factor passes the
whole-vector 1e-10 assertion of test_gpu_kdv_ac.py / test_gpu_poly.py, and check() rejects it."""
import numpy as np
import pytest

from oracle import reference_port as rp, taylor as ty, taylor_kdv_ac as tk, taylor_poly as tpo
from test_gpu_precision import LD, check, points


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def _w(layers, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return scale * (rp.glorot_normal_flat(layers, rng) + 0.05 * rng.standard_normal(rp.num_params(layers)))


def kdv_problem(lam=(0.0, -6.0), layers=(1, 50, 50, 20), lb=-1.0, ub=1.0, n0=61, n1=57, seed=0):
    rng = np.random.default_rng(seed)
    layers = list(layers)
    q = layers[-1]
    x_0, x_1 = (points(rng, [lb, lb], [ub, ub], n)[:, :1] for n in (n0, n1))
    w = np.concatenate([_w(layers, seed + 1), lam])
    args = (layers, np.array([lb]), np.array([ub]), x_0, np.cos(np.pi * x_0), x_1, 0.5 * np.cos(np.pi * x_1), 0.6,
            (rng.standard_normal((q, q)) / q).astype(np.float32), (rng.standard_normal((1, q)) / q).astype(np.float32))
    return w, lambda v, **kw: tk.kdv_ide_disc_loss_grad(v, *args, **kw)


def ac_problem(d=1e-4, k=5.0, layers=(1, 7, 128, 17), lb=-1.0, ub=1.0, n=200, seed=0):
    rng = np.random.default_rng(seed)
    layers = list(layers)
    q = layers[-1] - 1
    x_0 = points(rng, [lb, lb], [ub, ub], n)[:, :1]
    w = _w(layers, seed + 1)
    irk = rng.standard_normal((q + 1, q)) / q
    return w, lambda v, d=d, **kw: tk.ac_disc_loss_grad(v, layers, np.array([lb]), np.array([ub]), x_0, x_0 ** 2 * np.cos(np.pi * x_0),
                                                        0.8, irk, d=d, k=k, **kw)


AC_CONT = [(1.0, 0, (0, 0, 1, 0)), (-1e-4, 0, (0, 0, 0, 1)), (5.0, 0, (3, 0, 0, 0)), (-5.0, 0, (1, 0, 0, 0))]
FISHER = [(1.0, 0, (0, 0, 1, 0)), (-1.0, 4, (0, 0, 0, 1)), (-1.0, 1, (1, 0, 0, 0)), (1.0, 1, (2, 0, 0, 0))]


def poly_problem(terms, ide, layers=(2, 20, 20, 20, 1), lb=(-1.0, 0.0), ub=(1.0, 0.99), n=300, seed=0, bias=0.0, scale=1.0):
    rng = np.random.default_rng(seed)
    layers = list(layers)
    lb, ub = np.array(lb), np.array(ub)
    X_u = points(rng, lb, ub, n if ide else 40)
    u = rng.uniform(-1, 1, (X_u.shape[0], 1))
    X_f = None if ide else points(rng, lb, ub, n)
    w = _w(layers, seed + 1, scale)
    w[-1] += bias
    if ide:
        w = np.concatenate([w, [0.7, -1.5]])
    return w, lambda v, terms=terms, **kw: tpo.poly_loss_grad(v, layers, lb, ub, terms, X_u, u, X_f=X_f, identification=ide, **kw)


# ------------------------------------------------------------------------------------------------------ magnitudes are wired
MAG_CASES = {
    "kdv": lambda: kdv_problem((0.4, 0.5), lb=0.3, ub=3.7),
    "ac": lambda: ac_problem(d=1.0, lb=0.0, ub=1e-2),
    "poly_inf": lambda: poly_problem(AC_CONT, False),
    "poly_ide": lambda: poly_problem(FISHER, True, bias=1.0, scale=0.25),
}


@pytest.mark.parametrize("name", list(MAG_CASES))
def test_magnitudes_are_finite_and_bound_the_gradient(name):
    w, run = MAG_CASES[name]()
    r = run(w, dtype=LD, magnitudes=True)
    assert len(r) == 4
    g, S = r[1], r[3]
    assert g.dtype == LD and S.dtype == LD and S.shape == g.shape == w.shape
    assert np.all(np.isfinite(S)) and np.all(S >= 0)
    assert np.all(np.abs(g) <= S * (1 + 1e-12))
    assert np.all(S[np.abs(g) > 0] > 0)


def test_poly_lambda_magnitude_counts_every_term():
    """S_lambda1 of the polynomial head is sum over points and terms of |2 f / n  d(kappa_k)/d(l1) m_k|.  With Fisher-KPP near
    u = 1, -l1 u + l1 u^2 cancels, and |df/dl1| alone would under-count the rounding of the kernel's sum over the terms."""
    layers, lb, ub = [2, 20, 20, 20, 1], np.array([-1.0, 0.0]), np.array([1.0, 0.99])
    w, run = poly_problem(FISHER, True, bias=1.0, scale=0.25)
    S = run(w, dtype=LD, magnitudes=True)[3]
    rng = np.random.default_rng(0)
    X = points(rng, lb, ub, 300)
    (U, Ux, Ut, Uxx), _ = ty.forward(np.asarray(w[:-2], LD), layers, lb, ub, X, dtype=LD)
    l1, l2 = LD(w[-2]), LD(w[-1])
    f = Ut - np.exp(l2) * Uxx - l1 * U + l1 * U * U
    c = 2 * f / X.shape[0]
    assert S[-2] == pytest.approx(np.sum(np.abs(c) * (np.abs(U) + np.abs(U * U))), rel=1e-15)
    assert S[-1] == pytest.approx(np.sum(np.abs(c * np.exp(l2) * Uxx)), rel=1e-15)
    assert S[-2] > 5 * np.sum(np.abs(c * (U * U - U)))              # the cancellation the term-wise magnitude accounts for


# ------------------------------------------------------------------------------------------------------- the check has teeth
def whole_vector_passes(got, ref64, lam=False):
    """The assertions of tests/test_gpu_kdv_ac.py / test_gpu_poly.py: loss and gradient to 1e-10 in one relative L2 norm."""
    (loss, grad, _), (f2, g2) = got, ref64[:2]
    ok = abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10
    return ok and (not lam or rel(grad[-2:], g2[-2:]) < 1e-10), rel(grad, g2)


def _teeth(tag, got, ref, ref64, blocks, part_idx, lam=False):
    ok, r = whole_vector_passes(got, ref64, lam)
    assert ok, (tag, r)
    with pytest.raises(AssertionError):
        check(tag, got, ref, ref64, blocks, part_idx)
    return r


def _kernel_parts(parts, part_idx):
    out = np.zeros(3)
    out[list(part_idx)] = parts
    return out


def test_check_rejects_an_ac_run_with_d_off_by_1e_5():
    """Allen-Cahn [1, 7, 128, 17], d = 1e-4: the U_xx path scaled by 1 + 1e-5."""
    w, run = ac_problem()
    ref, ref64 = run(w, dtype=LD, magnitudes=True), run(w)
    bad = run(w, d=1e-4 * (1 + 1e-5))
    got = (bad[0], bad[1], _kernel_parts(bad[2], (0, 1)))
    _teeth("teeth/ac_d", got, ref, ref64, ty.param_blocks([1, 7, 128, 17]), (0, 1))


def test_check_rejects_a_kdv_run_with_a_u_xxx_seed_off_by_1e_8():
    """KdV [1, 50, 50, 20], lambda_2 = -6: the net blocks of a run with lambda_2 + 1e-8 (e^{lambda_2} scales the U_xxx seed),
    the lambda entries and the loss of the clean run."""
    w, run = kdv_problem(seed=3)
    ref, ref64 = run(w, dtype=LD, magnitudes=True), run(w)
    wp = w.copy()
    wp[-1] += 1e-8
    g = run(wp)[1]
    g[-2:] = ref64[1][-2:]
    got = (ref64[0], g, _kernel_parts(ref64[2], (0, 1)))
    _teeth("teeth/kdv_lambda2", got, ref, ref64, ty.param_blocks([1, 50, 50, 20], 2), (0, 1), lam=True)


def test_check_rejects_a_poly_run_with_the_u_xx_coefficient_off_by_1e_6():
    """The continuous-time Allen-Cahn spec u_t - 1e-4 u_xx + 5 u^3 - 5 u on POLY_INF: the u_xx coefficient scaled by 1 + 1e-6."""
    w, run = poly_problem(AC_CONT, False)
    ref, ref64 = run(w, dtype=LD, magnitudes=True), run(w)
    terms = [(c * (1 + 1e-6) if e == (0, 0, 0, 1) else c, k, e) for c, k, e in AC_CONT]
    bad = run(w, terms=terms)
    got = (bad[0], bad[1], _kernel_parts(bad[2], (0, 2)))
    _teeth("teeth/poly_ac_uxx", got, ref, ref64, ty.param_blocks([2, 20, 20, 20, 1]), (0, 2))
