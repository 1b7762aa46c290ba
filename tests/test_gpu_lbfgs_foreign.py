"""GPU: the mirror's lbfgs() driven by ARBITRARY closures (utils/custom_lbfgs.py:39 takes any opfunc), i.e. through the
stand-alone device optimiser (pinn_lbfgs_create / pinn_lbfgs_feed), against the oracle port of the reference routine on the
synthetic objectives of tests/lbfgs_compare_worker.py -- the set that takes every exit of the routine (maxIter, maxEval,
optimality at the start and later, no progress, step below tolX, f change below tolX, rejected curvature pairs, history
overflow).  The port itself is pinned to the reference's own lbfgs by tests/test_reference_pin.py."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def run_mirror(fn, x0, **cfgkw):
    from custom_lbfgs import Struct, lbfgs
    cfg = Struct()
    for k, v in cfgkw.items():
        setattr(cfg, k, v)
    xs, logged = [], []

    def opfunc(x):
        xs.append(np.asarray(x.numpy()).copy())
        return fn(np.asarray(x))
    state = Struct()
    ret = lbfgs(opfunc, np.asarray(x0, dtype=np.float64), cfg, state, True, lambda it, f, is_iter: logged.append((it, float(f))))
    return ret, xs, logged, state


def compare(fn, x0, expect_reason, **kw):
    from oracle import reference_port as rp
    port = rp.lbfgs_fixed_step(lambda x: fn(x), np.asarray(x0, dtype=np.float64), max_iter=kw["maxIter"],
                               learning_rate=kw.get("learningRate", 1.0), n_correction=kw.get("nCorrection", 100),
                               tol_fun=kw.get("tolFun", 1e-5), tol_x=kw.get("tolX", 1e-19), max_eval=kw.get("maxEval"))
    assert port.stop_reason == expect_reason
    ret, xs, logged, state = run_mirror(fn, x0, **kw)
    assert state.stop_reason == expect_reason
    assert len(xs) == len(port.x_eval) == port.n_eval                  # same number of opfunc calls, at the same points
    for a, b in zip(xs, port.x_eval):
        assert np.allclose(a, b, rtol=1e-8, atol=1e-13)
    if expect_reason == "initial optimality":
        assert len(ret) == 2                                            # (x, f_hist) only, custom_lbfgs.py:76
        return
    x, f_hist, n_eval = ret
    assert n_eval == port.n_eval and np.allclose(np.asarray(x), port.x_final, rtol=1e-8, atol=1e-13)
    assert np.allclose(f_hist, port.f_hist, rtol=1e-8, atol=1e-300)
    assert [it for it, _ in logged] == [it for it, _ in port.logged]
    assert np.allclose([f for _, f in logged], [f for _, f in port.logged], rtol=1e-8, atol=1e-300)
    assert state.nIter == port.n_iter and state.funcEval == port.n_eval


A = np.diag([1.0, 10.0, 100.0])
quad = lambda x: (0.5 * float(x @ A @ x), A @ x)
_rng = np.random.default_rng(0)
B = _rng.standard_normal((12, 12)); B = np.eye(12) + 0.02 * (B @ B.T)
quad12 = lambda x: (0.5 * float(x @ B @ x), B @ x)
x12 = _rng.standard_normal(12)
lin = lambda x: (float(np.sum(x)), np.ones_like(x))                      # y = 0: every curvature pair rejected (ys <= 1e-10)

CASES = [
    ("quadratic, maxIter", quad, [1.0, 1.0, 1.0], "max iterations", dict(maxIter=4, learningRate=0.05, tolFun=1e-30)),
    ("quadratic, maxEval", quad, [1.0, 1.0, 1.0], "max evaluations", dict(maxIter=40, maxEval=3, learningRate=0.05, tolFun=1e-30)),
    ("zero gradient at start", quad, [0.0, 0.0, 0.0], "initial optimality", dict(maxIter=5)),
    ("optimality after a few steps", quad12, x12, "optimality", dict(maxIter=200, learningRate=1.0, tolFun=1e-6)),
    ("history overflow (nCorrection=3)", quad12, x12, "max iterations", dict(maxIter=15, learningRate=0.5, nCorrection=3, tolFun=1e-30)),
    ("ascent direction", lambda x: (-0.5 * float(x @ x), -x), [1.0, 2.0], "max iterations", dict(maxIter=3, learningRate=0.1, tolFun=1e-30)),
    ("linear objective, no curvature", lin, [0.0, 0.0], "max iterations", dict(maxIter=6, learningRate=0.3, tolFun=1e-30)),
    ("step below tolX", quad, [1e-3, 1e-3, 1e-3], "step below tolX", dict(maxIter=50, learningRate=1e-12, tolFun=1e-30, tolX=1e-9)),
    ("f change below tolX", lambda x: (1.0, np.array([0.3, -0.2])), [0.0, 0.0], "f change below tolX",
     dict(maxIter=50, learningRate=0.5, tolFun=1e-30, tolX=1e-7)),
    ("no progress along direction (it 2)", lambda x: (1.0, np.array([1.0, 0.0])) if x[0] == 0.0 else (0.5, np.array([1e-4, 0.0])),
     [0.0, 0.0], "no progress along direction", dict(maxIter=9, learningRate=1.0, tolFun=1e-9, tolX=1e-5)),
    ("no progress at iteration 1 (the reference crashes here: t unassigned)", lambda x: (1.0, np.array([1e-3, 0.0])), [0.0, 0.0],
     "no progress along direction", dict(maxIter=9, learningRate=1.0, tolFun=1e-9, tolX=1e-5)),
]


def two_valued(first, later):
    """(f, g) = first at the start point (x[0] == 0) and later everywhere else.  The values are dyadic with one nonzero gradient
    entry, so |g|_1, |d t|_1, g.d, y.s and f - f_old are exact in any summation order and land exactly on a threshold."""
    return lambda x: (first[0], np.array(first[1])) if x[0] == 0.0 else (later[0], np.array(later[1]))


TINY = 2.0 ** -20     # g = (-TINY, 0) at the start: the first step is s = (TINY, 0), so y.s = y_0 TINY exactly
# Each stop test and the curvature test with its operands exactly on the threshold (the reference's custom_lbfgs.py decides the
# side, tests/test_reference_pin.py).  The expected reason is the product's; the other side of the comparison ends elsewhere.
BOUNDARY_CASES = [
    ("g1_eq_tolfun_at_start", two_valued((1.0, [0.25, 0.0]), (0.5, [0.25, 0.0])), [0.0, 0.0], "initial optimality",
     dict(maxIter=5, tolFun=0.25)),
    ("g1_eq_tolfun_after_a_step", two_valued((1.0, [0.5, 0.0]), (0.5, [0.25, 0.0])), [0.0, 0.0], "optimality",
     dict(maxIter=5, tolFun=0.25)),
    ("step_eq_tolx", two_valued((4.0, [2.0, 0.0]), (0.0, [2.0, 0.0])), [0.0, 0.0], "step below tolX", dict(maxIter=5, tolX=1.0)),
    ("f_change_eq_tolx", two_valued((1.0, [1.0, 0.0]), (0.75, [1.0, 0.0])), [0.0, 0.0], "max iterations",
     dict(maxIter=2, tolX=0.25)),
    ("gtd_eq_minus_tolx", two_valued((1.0, [0.5, 0.0]), (0.0, [0.5, 0.0])), [0.0, 0.0], "max iterations",
     dict(maxIter=2, tolX=0.25)),
    ("ys_eq_1e-10_rejected", two_valued((1.0, [-TINY, 0.0]), (0.5, [1e-10 / TINY - TINY, 0.0])), [0.0, 0.0],
     "f change below tolX", dict(maxIter=4, tolFun=1e-30)),
    ("ys_2^-31_accepted", two_valued((1.0, [-TINY, 0.0]), (0.5, [2.0 ** -11 - TINY, 0.0])), [0.0, 0.0],
     "f change below tolX", dict(maxIter=4, tolFun=1e-30)),
]
CASES += BOUNDARY_CASES


@pytest.mark.parametrize("name,fn,x0,reason,kw", CASES, ids=[c[0] for c in CASES])
def test_foreign_closure_takes_every_exit_like_the_reference(name, fn, x0, reason, kw):
    compare(fn, x0, reason, **kw)


def test_larger_vector_and_tensor_like_values():
    """P = 5000 entries (the 1024-thread instantiation), f and g returned as objects with .numpy() like eager tensors."""
    from neuralnetwork import _t
    rng = np.random.default_rng(3)
    dvec = 1.0 + rng.random(5000)
    fn = lambda x: (0.5 * float(np.sum(dvec * x * x)), dvec * x)
    wrapped = lambda x: (_t(np.array(fn(x)[0])), _t(fn(x)[1]))
    from oracle import reference_port as rp
    x0 = rng.standard_normal(5000)
    port = rp.lbfgs_fixed_step(fn, x0, max_iter=12, learning_rate=0.6, n_correction=5, tol_fun=1e-30)
    ret, xs, logged, state = run_mirror(wrapped, x0, maxIter=12, learningRate=0.6, nCorrection=5, tolFun=1e-30)
    assert np.allclose(np.asarray(ret[0]), port.x_final, rtol=1e-9, atol=1e-13) and len(xs) == port.n_eval
