"""CPU: what the reference does with NaN and infinite inputs, as tests/test_gpu_nonfinite.py holds the kernels to it.

* For every injection of the GPU matrix, the fp64 Taylor oracle and the nested-autograd port (torch, the reference's tanh) put
  the loss, each loss part and every gradient entry into the same class {finite, +Inf, -Inf, NaN}.  This is what "the
  reference's behaviour" means for each case; test_gpu_nonfinite.FORMULA_DEPENDENT lists the cases where the two disagree.
* The class rule of tests/test_gpu_nonfinite.py has teeth: an oracle run with the kernels' old tanh (|x| clamped by fmin,
  which returns 20 for a NaN, so tanh(NaN) = +-1) standing in for a kernel is rejected on the NaN-coordinate cases, one with
  the select that keeps NaN passes.
* L-BFGS on objectives whose f, g or both turn NaN or +-Inf (stop reason, counts, logged iterations and points pinned; the same
  objectives run against the reference's own lbfgs in tests/lbfgs_compare_worker.py), and Adam with non-finite gradients.
"""
import numpy as np
import pytest

from oracle import reference_port as rp
from oracle import taylor as ty
from test_gpu_nonfinite import (FORMULA_DEPENDENT, H100_SMS, INF, LBFGS_KW, LBFGS_OBJECTIVES, LBFGS_X0, MODELS, NAN, cases,
                                class_mismatch, classes, expected, flat, inject, nonfinite_objective, port_result,
                                same_nan)


def formula_dependent_entries(name, case_name):
    """The [loss, parts, gradient] entries FORMULA_DEPENDENT's reasons name: the head's pressure-column weights for a NaN target
    of the Navier-Stokes model (its bias takes no zero-seeded product), the data part for an infinite head weight."""
    if case_name.startswith("uv"):
        W = dict(ty.param_blocks(MODELS[name]["inputs"]()["layers"]))["W2"]
        return 3 + np.arange(W.start, W.stop)[1::2]
    return np.array([1])


@pytest.mark.parametrize("name", list(MODELS))
def test_taylor_oracle_and_autograd_port_agree_on_every_class(name):
    disagree = {}
    for case in cases(name, H100_SMS):
        d = inject(MODELS[name]["inputs"](), *case[1:])
        with np.errstate(all="ignore"):
            a, b = flat(MODELS[name]["taylor"](d)), flat(port_result(name, d))
        if (name, case[0]) in FORMULA_DEPENDENT:
            diff = np.flatnonzero(classes(a) != classes(b))
            assert diff.size, ("listed as formula-dependent but the classes agree", case[0])
            assert np.array_equal(diff, formula_dependent_entries(name, case[0])), (case[0], diff.tolist())
            continue
        if not np.array_equal(classes(a), classes(b)):
            diff = np.flatnonzero(classes(a) != classes(b))
            disagree[case[0]] = (diff.size, diff[:4].tolist(), classes(a)[diff[:4]].tolist(), classes(b)[diff[:4]].tolist())
    assert not disagree, disagree


def test_the_matrix_covers_every_site():
    """Every model injects into each of its point sets at three positions with three values, its targets, four weight sites
    with three values (plus lambda_1, lambda_2) and its constants; NaN coordinates make the reference's loss NaN."""
    for name, m in MODELS.items():
        cs = cases(name, H100_SMS)
        assert len(cs) == len({c[0] for c in cs})
        n_w = 3 * (4 + (2 if m["n_extra"] else 0))
        assert len(cs) == 9 * len(m["point_sets"]) + len(m["targets"]) + n_w + len(m["consts"]), name
        for case in cs:
            if case[1] in dict(m["point_sets"]) and np.isnan(case[3]):
                assert np.isnan(expected(name, case)[0]), (name, case[0])


# --------------------------------------------------------------------------------------------------------------- the teeth
def old_tanh(z):
    """The kernels' tanh before the fix: |z| clamped with fmin (NaN -> 20), then copysign(tanh(20), z) = +-1 for a NaN."""
    return np.copysign(np.tanh_orig(np.fmin(np.abs(z), 20.0)), z)


def fixed_tanh(z):
    """The fixed clamp, |z| > 20 ? 20 : |z|: a NaN stays NaN."""
    a = np.abs(z)
    return np.copysign(np.tanh_orig(np.where(a > 20.0, 20.0, a)), z)


def _rule_passes(name, case, tanh):
    """class_mismatch of tests/test_gpu_nonfinite.py (the rule the kernels are held to) on an oracle run with `tanh` standing
    in for the kernel."""
    np.tanh = tanh
    try:
        with np.errstate(all="ignore"):
            r = expected(name, case)
    finally:
        np.tanh = np.tanh_orig
    return class_mismatch(name, case, (r[0], r[1], _kernel_parts(name, r[2]))) is None


def _kernel_parts(name, parts):
    out = np.zeros(3)
    out[list(MODELS[name]["part_idx"])] = parts
    return out


@pytest.mark.parametrize("name,case_name", [("burgers_inf", "X_f[first=0,0]=nan"), ("burgers_inf", "X_u[mid=12,1]=nan"),
                                            ("burgers_ide", "X_u[last=202,1]=nan"), ("nls", "X_f[last=36,1]=nan")])
def test_class_rule_rejects_the_old_tanh_on_a_nan_coordinate(monkeypatch, name, case_name):
    case = [c for c in cases(name, H100_SMS) if c[0] == case_name][0]
    monkeypatch.setattr(np, "tanh_orig", np.tanh, raising=False)
    assert not _rule_passes(name, case, old_tanh)
    assert _rule_passes(name, case, fixed_tanh)
    with np.errstate(invalid="ignore"):
        assert np.isnan(fixed_tanh(np.array([NAN]))[0]) and np.abs(old_tanh(np.array([NAN]))[0]) == 1.0
        z = np.array([-INF, -21.0, -20.0, -1e-300, -0.0, 0.0, 3.0, 20.0, INF])
        assert np.array_equal(old_tanh(z), fixed_tanh(z))


# ----------------------------------------------------------------------------------------------------------------- L-BFGS
def run_port(name, k, at, wh):
    kw = dict(LBFGS_KW)
    with np.errstate(all="ignore"):
        return rp.lbfgs_fixed_step(nonfinite_objective(k, at, wh), LBFGS_X0, max_iter=kw["max_iter"], learning_rate=kw["lr"],
                                   n_correction=kw["n_corr"], tol_fun=kw["tol_fun"])


# What the port does on each objective: no stop test fires on a NaN or an infinite f or g (sum |g| <= tolFun, gtd > -tolX,
# |f - f_old| < tolX are all False), so every run takes all 12 iterations, asks for 12 points and logs iterations 1..11.  A
# non-finite g at evaluation j makes the step non-finite, so exactly the first j + 1 points are finite; a non-finite f alone
# changes no point.  (stop reason, iterations, evaluations, logged iterations, finite points asked for)
LBFGS_EXPECT = {name: ("max iterations", 12, 12, list(range(1, 12)), 12 if wh == "f" else at + 1)
                for name, k, at, wh in LBFGS_OBJECTIVES}


@pytest.mark.parametrize("name,k,at,wh", LBFGS_OBJECTIVES, ids=[o[0] for o in LBFGS_OBJECTIVES])
def test_lbfgs_port_on_non_finite_evaluations(name, k, at, wh):
    tr = run_port(name, k, at, wh)
    got = (tr.stop_reason, tr.n_iter, tr.n_eval, [it for it, _ in tr.logged],
           sum(bool(np.all(np.isfinite(x))) for x in tr.x_eval))
    assert got == LBFGS_EXPECT[name], (name, got)
    assert all(np.all(np.isfinite(x)) for x in tr.x_eval[:got[4]])
    # the logged f values are the evaluations themselves; compared NaN-aware (plain == is False wherever one holds a NaN)
    assert same_nan([f for _, f in tr.logged], tr.f_hist[1:12])
    if at == 0 and wh in ("g", "both"):
        # t = min(1, 1 / |g|_1): Python's min returns 1 for a NaN norm, as the device's fmin does, and 0 for an infinite one
        assert tr.t[0] == (1.0 if k == "nan" else 0.0)


def test_min_of_one_and_a_nan_is_one_in_python_as_in_fmin():
    assert min(1.0, NAN) == 1.0 and min(1.0, 1.0 / INF) == 0.0
    assert np.fmin(1.0, NAN) == 1.0


# ------------------------------------------------------------------------------------------------------------------- Adam
@pytest.mark.parametrize("value", [NAN, INF, -INF])
def test_adam_confines_a_non_finite_gradient_entry(value):
    rng = np.random.default_rng(5)
    w, g = rng.standard_normal(64), rng.standard_normal(64)
    bad = [3, 40]
    gb = g.copy(); gb[bad] = value
    st, st0 = rp.adam_init(64), rp.adam_init(64)
    with np.errstate(all="ignore"):
        w1 = rp.adam_update(w, gb, st, 1e-3)
        w2 = rp.adam_update(w1, g, st, 1e-3)
    ref1 = rp.adam_update(w, g, st0, 1e-3)
    ref2 = rp.adam_update(ref1, g, st0, 1e-3)
    ok = np.setdiff1d(np.arange(64), bad)
    assert np.array_equal(w1[ok], ref1[ok]) and np.array_equal(w2[ok], ref2[ok])
    assert np.array_equal(st.m[ok], st0.m[ok]) and np.array_equal(st.v[ok], st0.v[ok])
    # m = (1 - b1) g, v = (1 - b2) g^2: a NaN stays NaN; an infinite g gives m = +-Inf, v = Inf and the update Inf / Inf = NaN
    assert np.all(np.isnan(w1[bad])) and np.all(np.isnan(w2[bad])) and np.all(np.isnan(st.v[bad]) | np.isposinf(st.v[bad]))
    assert np.all(~np.isfinite(st.m[bad]))
