"""CPU: the oracle against the committed golden vectors, and the two oracle formulations against each other."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import reference_port as rp, taylor as ty

EPS = np.finfo(float).eps


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def test_flat_layout_matches_reference_sizes():
    # utils/neuralnetwork.py:40-45 sizes_w / sizes_b for the Burgers net
    layers = [2] + [20] * 8 + [1]
    sizes_w = [int(w * layers[1]) for i, w in enumerate(layers) if i != 1]
    sizes_b = [int(w if i != 0 else layers[1]) for i, w in enumerate(layers) if i != 1]
    offs = rp.param_offsets(layers)
    o = 0
    for (wo, bo), sw, sb in zip(offs, sizes_w, sizes_b):
        assert wo == o and bo == o + sw
        o += sw + sb
    assert o == rp.num_params(layers) == 3021
    assert rp.num_params([2, 100, 100, 100, 100, 2]) == 30802


def test_burgers_inf_golden_both_oracles():
    g = load_golden("burgers_inf")
    layers = list(g["layers"])
    pb = rp.BurgersInference(layers, g["lb"], g["ub"], float(g["nu"]), g["X_f"], g["X_u"], g["u"])
    f, gr = rp.loss_and_flat_grad(pb, g["w"])
    assert abs(f - g["loss"]) <= 1e-13 * abs(g["loss"])
    assert rel(gr, g["grad"]) < 1e-12
    f2, g2, parts = ty.burgers_loss_grad(g["w"], layers, g["lb"], g["ub"], g["X_f"], g["X_u"], g["u"], nu=float(g["nu"]))
    assert abs(f2 - g["loss"]) <= 1e-13 * abs(g["loss"])
    assert rel(g2, g["grad"]) < 1e-12
    assert np.allclose(parts, g["parts"][[0, 1]] if len(g["parts"]) == 2 else g["parts"], rtol=1e-12)
    (U, Ux, Ut, Uxx), _ = ty.forward(g["w"], layers, g["lb"], g["ub"], g["X_f"][:64])
    assert rel(np.hstack([U, Ux, Ut, Uxx]), g["probes"]) < 1e-12


def test_burgers_ide_golden_both_oracles():
    g = load_golden("burgers_ide")
    layers = list(g["layers"])
    pb = rp.BurgersIdentification(layers, g["lb"], g["ub"], g["X_u"], g["u"])
    for wk, fk, gk in (("w", "loss", "grad"), ("w2", "loss2", "grad2")):
        f, gr = rp.loss_and_flat_grad(pb, g[wk])
        f2, g2, _ = ty.burgers_loss_grad(g[wk], layers, g["lb"], g["ub"], None, g["X_u"], g["u"], identification=True)
        assert abs(f - g[fk]) <= 1e-13 * abs(g[fk]) and abs(f2 - g[fk]) <= 1e-13 * abs(g[fk])
        assert rel(gr, g[gk]) < 1e-12 and rel(g2, g[gk]) < 1e-12
    assert g["grad2"].shape == (3023,)


def test_nls_golden_taylor_oracle_and_q1_quirk():
    g = load_golden("nls_inf")
    layers = list(g["layers"])
    x0 = g["x0"]
    for tag, X0 in (("q1", x0), ("x0t0", np.concatenate([x0, 0 * x0], 1))):
        f2, g2, parts = ty.schrodinger_loss_grad(g["w"], layers, g["lb"], g["ub"], g["X_f"], g["tb"], X0, g["uv0"])
        assert abs(f2 - g["loss_" + tag]) <= 1e-13 * abs(g["loss_" + tag])
        assert rel(g2, g["grad_" + tag]) < 1e-12
        assert np.allclose(parts, g["parts_" + tag], rtol=1e-12)
    # quirk Q1 changes only the initial-condition term
    assert g["parts_q1"][0] != g["parts_x0t0"][0]
    assert g["parts_q1"][1] == g["parts_x0t0"][1] and g["parts_q1"][2] == g["parts_x0t0"][2]


def test_adam_tf2_semantics_by_hand():
    # one step: m = (1-b1) g, v = (1-b2) g^2, alpha = lr sqrt(1-b2)/(1-b1) -> w -= lr*g/(|g| + eps*sqrt(1-b2)) approx
    w = np.array([1.0, -2.0]); g = np.array([0.5, -0.25])
    st = rp.adam_init(2)
    w1 = rp.adam_update(w, g, st, lr=0.1, b1=0.9, b2=0.999, eps=None)
    alpha = 0.1 * np.sqrt(1 - 0.999) / (1 - 0.9)
    exp = w - alpha * (0.1 * g) / (np.sqrt(0.001 * g * g) + 1e-7)
    assert np.allclose(w1, exp, rtol=0, atol=1e-15)
    assert st.t == 1


def test_adam_golden_trajectory():
    g = load_golden("burgers_inf")
    pb = rp.BurgersInference(list(g["layers"]), g["lb"], g["ub"], float(g["nu"]), g["X_f"], g["X_u"], g["u"])
    w, losses, _ = rp.adam_train(pb, g["w"], 5, lr=float(g["adam_lr"][0]))
    assert rel(w, g["adam_w"][0]) < 1e-12 and rel(losses, g["adam_losses"][0]) < 1e-12


def _quad(A, b):
    def f(x):
        return float(0.5 * x @ A @ x - b @ x), A @ x - b
    return f


def test_lbfgs_control_flow_quirks():
    rng = np.random.default_rng(0)
    M = rng.standard_normal((6, 6)); A = M @ M.T + 6 * np.eye(6); b = rng.standard_normal(6)
    x0 = rng.standard_normal(6)
    op = _quad(A, b)
    assert rp.lbfgs_fixed_step(op, x0, 0) is None                       # custom_lbfgs.py:43-44
    tr = rp.lbfgs_fixed_step(op, x0, max_iter=8, learning_rate=0.8, n_correction=3, tol_fun=EPS)
    f0, g0 = op(x0)
    assert tr.t[0] == min(1.0, 1.0 / np.abs(g0).sum())                 # :159-161
    assert all(t == 0.8 for t in tr.t[1:])                             # :163 fixed step, no line search
    assert np.allclose(tr.d[0], -g0)
    assert tr.n_iter == 8 and tr.n_eval == 8                           # the last update is NOT evaluated (:176-182)
    assert len(tr.x_eval) == 8 and not np.allclose(tr.x_eval[-1], tr.x_final)
    assert np.allclose(tr.x_final, tr.x_eval[-1] + tr.t[-1] * tr.d[-1])
    assert max(tr.hist_len) <= 3
    assert [it for it, _ in tr.logged] == list(range(1, 8))            # iteration maxIter breaks before the log
    # initial optimality
    xs = np.linalg.solve(A, b)
    tr2 = rp.lbfgs_fixed_step(op, xs, max_iter=5, tol_fun=1e-6)
    assert tr2.stop_reason == "initial optimality" and tr2.n_iter == 0


def test_lbfgs_golden_trace():
    g = load_golden("burgers_inf")
    pb = rp.BurgersInference(list(g["layers"]), g["lb"], g["ub"], float(g["nu"]), g["X_f"], g["X_u"], g["u"])
    tr = rp.lbfgs_fixed_step(lambda x: rp.loss_and_flat_grad(pb, x), g["w"], max_iter=6, learning_rate=0.8,
                             n_correction=50, tol_fun=EPS)
    assert tr.n_iter == int(g["lbfgs_n_iter"]) and tr.n_eval == int(g["lbfgs_n_eval"])
    assert rel(np.array(tr.f_hist), g["lbfgs_f"]) < 1e-9
    assert rel(tr.x_final, g["lbfgs_x_final"]) < 1e-9


def _recorded(fn):
    """fn wrapped so that every (f, g) it returns is kept, for a ScriptedOpfunc replay."""
    fs, gs = [], []

    def op(x):
        f, g = fn(np.asarray(x, dtype=np.float64))
        fs.append(f); gs.append(np.array(g, dtype=np.float64))
        return f, g
    return op, fs, gs


def _steps_agree(a, b, tol):
    """Worst per-iteration ||t a_d - t b_d|| / ||t b_d|| of two traces with the same control flow."""
    assert a.stop_reason == b.stop_reason and a.n_iter == b.n_iter and a.n_eval == b.n_eval
    assert a.logged == b.logged and a.hist_len == b.hist_len and len(a.d) == len(b.d)
    worst = 0.0
    for da, ta, db, tb in zip(a.d, a.t, b.d, b.t):
        sa, sb = (np.asarray(ta * da, dtype=np.longdouble), np.asarray(tb * db, dtype=np.longdouble))
        worst = max(worst, float(np.linalg.norm((sa - sb).astype(np.float64)) / np.linalg.norm(sb.astype(np.float64))))
    assert worst <= tol, worst
    return worst


@pytest.mark.skipif(np.finfo(np.longdouble).eps > 1e-18, reason="np.longdouble has no extended precision on this platform")
def test_lbfgs_longdouble_replay_agrees_with_float64_on_the_exit_objectives():
    """The extended-precision L-BFGS replayed on the evaluations the float64 run saw (the objectives of
    tests/test_gpu_lbfgs_foreign.py, which take every exit of the routine): same control flow, and every step t d within 1e-13
    of the float64 one.  A replay that rounds to a narrower type would not agree; one left in float64 would agree exactly."""
    from test_gpu_lbfgs_foreign import CASES
    exact = 0
    for name, fn, x0, reason, kw in CASES:
        cfg = dict(max_iter=kw["maxIter"], learning_rate=kw.get("learningRate", 1.0), n_correction=kw.get("nCorrection", 100),
                   tol_fun=kw.get("tolFun", 1e-5), tol_x=kw.get("tolX", 1e-19), max_eval=kw.get("maxEval"))
        op, fs, gs = _recorded(fn)
        tr64 = rp.lbfgs_fixed_step(op, np.asarray(x0, dtype=np.float64), **cfg)
        assert tr64.stop_reason == reason, name
        replay = rp.ScriptedOpfunc(fs, gs)
        trld = rp.lbfgs_fixed_step(replay, np.asarray(x0, dtype=np.float64), dtype=np.longdouble, **cfg)
        replay.assert_consumed()
        assert all(d.dtype == np.longdouble for d in trld.d), name
        _steps_agree(tr64, trld, 1e-13)
        exact += all(np.array_equal(a, b.astype(np.float64)) for a, b in zip(tr64.d, trld.d))
    assert exact < len(CASES)


def test_lbfgs_gram_formulation_replay_agrees_with_the_literal_loop():
    """The float64 Gram-matrix restatement of the device kernels (coefficient-space recurrences over s_a.y_b and y_a.y_b) against
    the literal two-loop recursion on the same evaluations: 40 iterations with a 3-pair history (the ring wraps 12 times) on a
    well-conditioned quadratic agree to 1e-12 per step; the two formulations round differently, so they are not identical."""
    rng = np.random.default_rng(5)
    M = rng.standard_normal((40, 40)); A = np.eye(40) + 0.3 * (M @ M.T) / 40; b = rng.standard_normal(40)
    op, fs, gs = _recorded(_quad(A, b))
    x0 = rng.standard_normal(40)
    lit = rp.lbfgs_fixed_step(op, x0, max_iter=40, learning_rate=0.3, n_correction=3, tol_fun=1e-30)
    assert lit.stop_reason == "max iterations" and max(lit.hist_len) == 3
    replay = rp.ScriptedOpfunc(fs, gs)
    gram = rp.lbfgs_fixed_step(replay, x0, max_iter=40, learning_rate=0.3, n_correction=3, tol_fun=1e-30, direction="gram")
    replay.assert_consumed()
    _steps_agree(lit, gram, 1e-12)
    assert any(not np.array_equal(a, b) for a, b in zip(lit.d, gram.d))
    with pytest.raises(AssertionError, match="recorded"):
        replay(x0)


@pytest.mark.skipif(np.finfo(np.longdouble).eps > 1e-18, reason="np.longdouble has no extended precision on this platform")
def test_adam_longdouble_update_agrees_with_float64():
    """Adam in extended precision from the same gradients: m, v and the bias correction carried in np.longdouble agree with the
    float64 update, for the reference's hyperparameters and for eps-dominated and b1 = 0 ones.  The tolerance is set by float64
    itself: 1 - b2^t cancels to about (1 - b2) t, so the bias correction of a float64 Adam is good to only ~1e-16 / ((1 - b2) t)
    -- 1e-11 relative at b2 = 0.99999 and t = 1 -- while a float32 bias correction would be off by ~1e-7."""
    rng = np.random.default_rng(1)
    w0 = rng.standard_normal(500)
    gs = [rng.standard_normal(500) * 10.0 ** rng.uniform(-6, 0, 500) for _ in range(30)]
    for hp in (dict(lr=1e-3), dict(lr=0.05, b1=0.5, b2=0.9, eps=1e-2), dict(lr=1e-2, b1=0.0, b2=0.99999)):
        s64, sld = rp.adam_init(500), rp.adam_init(500)
        w = w0
        for g in gs:
            w64 = rp.adam_update(w, g, s64, **hp)
            wld = rp.adam_update(w, g, sld, dtype=np.longdouble, **hp)
            assert wld.dtype == np.longdouble and sld.m.dtype == np.longdouble
            step = np.abs((wld - w).astype(np.float64))
            assert np.all(np.abs((w64 - wld).astype(np.float64)) <= 1e-10 * step + np.spacing(np.abs(w64))), hp
            w = w64
        assert not np.array_equal(w64, wld.astype(np.float64)), hp


def test_lua_struct_defaults_to_zero():
    s = rp.LuaStruct()
    s.maxIter = 3
    assert s.maxIter == 3 and s.lineSearch == 0 and (s.tolX or 1e-19) == 1e-19    # custom_lbfgs.py:242-246


def test_burgers_disc_golden_both_oracles():
    """Discrete-time IRK model (1d-burgers/inf_disc_burgers.py:61-101): nested autograd with the reference's dummy-gradient
    trick and the closed-form Taylor oracle against the committed vector (upstream q=100 Butcher table)."""
    g = load_golden("burgers_disc")
    layers = [int(v) for v in g["layers"]]
    IRK = g["IRK"].astype(np.float64)
    pb = rp.BurgersDiscreteInference(layers, g["lb"], g["ub"], float(g["nu"]), float(g["dt"]), g["x_0"], g["u_0"], g["x_1"], IRK)
    f, gr = rp.loss_and_flat_grad(pb, g["w"])
    f2, g2, parts = ty.burgers_disc_loss_grad(g["w"], layers, g["lb"], g["ub"], g["x_0"], g["u_0"], g["x_1"], float(g["nu"]),
                                              float(g["dt"]), IRK)
    for fv, gv in ((f, gr), (f2, g2)):
        assert abs(fv - g["loss"]) <= 1e-13 * abs(g["loss"]) and rel(gv, g["grad"]) < 1e-12
    assert np.allclose(parts, g["parts"], rtol=1e-12)
    assert IRK.shape == (101, 100) and abs(IRK[-1].sum() - 1.0) < 1e-5        # last row: the quadrature weights b_j


def test_burgers_ide_disc_golden_both_oracles():
    """Discrete-time identification (1d-burgers/ide_disc_burgers.py:48-203): nested-autograd restatement (dummy-gradient trick)
    and the closed-form Taylor oracle against the golden vector (q = 81 upstream table, float32 like the reference loads it)."""
    g = load_golden("burgers_ide_disc")
    layers = [int(v) for v in g["layers"]]
    assert layers == [1, 50, 50, 50, 81] and g["IRK_alpha"].dtype == np.float32 and g["IRK_alpha"].shape == (81, 81)
    pb = rp.BurgersDiscreteIdentification(layers, g["lb"], g["ub"], float(g["dt"]), g["x_0"], g["u_0"], g["x_1"], g["u_1"],
                                           g["IRK_alpha"], g["IRK_beta"])
    for tag in ("", "2"):
        f, gr = rp.loss_and_flat_grad(pb, g["w" + tag])
        f2, g2, parts = ty.burgers_ide_disc_loss_grad(g["w" + tag], layers, g["lb"], g["ub"], g["x_0"], g["u_0"], g["x_1"], g["u_1"],
                                                      float(g["dt"]), g["IRK_alpha"], g["IRK_beta"])
        for fv, gv in ((f, gr), (f2, g2)):
            assert abs(fv - float(g["loss" + tag])) <= 1e-13 * abs(float(g["loss" + tag]))
            assert np.linalg.norm(gv - g["grad" + tag]) <= 1e-12 * np.linalg.norm(g["grad" + tag])
        assert np.allclose(parts, g["parts" + tag], rtol=1e-13)
    # beta - alpha is rounded in float32 by the reference (numpy arithmetic before TensorFlow sees it): doing it in float64 is
    # a DIFFERENT function at the 1e-10 level, which the pin against the reference's own code detects
    pb64 = rp.BurgersDiscreteIdentification(layers, g["lb"], g["ub"], float(g["dt"]), g["x_0"], g["u_0"], g["x_1"], g["u_1"],
                                             g["IRK_alpha"].astype(np.float64), g["IRK_beta"].astype(np.float64))
    f64, _ = rp.loss_and_flat_grad(pb64, g["w2"])
    assert 1e-14 < abs(f64 - float(g["loss2"])) / float(g["loss2"]) < 1e-8
    U0, U1 = pb.predict(g["w2"], g["x_star"])
    assert np.allclose(U0, g["predict_U0"], rtol=0, atol=1e-13) and np.allclose(U1, g["predict_U1"], rtol=0, atol=1e-13)


def _golden_evaluations():
    """(name, golden loss parts, parameter blocks, f(dtype, magnitudes) -> Taylor oracle result) on the golden inputs of
    all five models."""
    out = []
    g = load_golden("burgers_inf")
    L = [int(v) for v in g["layers"]]
    out.append(("burgers_inf", g["parts"], ty.param_blocks(L),
                lambda dt, m, g=g, L=L: ty.burgers_loss_grad(g["w"], L, g["lb"], g["ub"], g["X_f"], g["X_u"], g["u"],
                                                             nu=float(g["nu"]), dtype=dt, magnitudes=m)))
    g = load_golden("burgers_ide")
    for wk in ("w", "w2"):
        out.append(("burgers_ide_" + wk, g["parts"] if wk == "w" else None, ty.param_blocks(L, 2),
                    lambda dt, m, g=g, wk=wk: ty.burgers_loss_grad(g[wk], L, g["lb"], g["ub"], None, g["X_u"], g["u"],
                                                                   identification=True, dtype=dt, magnitudes=m)))
    g = load_golden("nls_inf")
    Ln = [int(v) for v in g["layers"]]
    for tag, X0 in (("q1", g["x0"]), ("x0t0", np.concatenate([g["x0"], 0 * g["x0"]], 1))):
        out.append(("nls_" + tag, g["parts_" + tag], ty.param_blocks(Ln),
                    lambda dt, m, g=g, X0=X0: ty.schrodinger_loss_grad(g["w"], Ln, g["lb"], g["ub"], g["X_f"], g["tb"], X0,
                                                                       g["uv0"], dtype=dt, magnitudes=m)))
    g = load_golden("burgers_disc")
    Ld = [int(v) for v in g["layers"]]
    out.append(("burgers_disc", g["parts"], ty.param_blocks(Ld),
                lambda dt, m, g=g: ty.burgers_disc_loss_grad(g["w"], Ld, g["lb"], g["ub"], g["x_0"], g["u_0"], g["x_1"],
                                                             float(g["nu"]), float(g["dt"]), g["IRK"].astype(np.float64),
                                                             dtype=dt, magnitudes=m)))
    g = load_golden("burgers_ide_disc")
    Le = [int(v) for v in g["layers"]]
    for tag in ("", "2"):
        out.append(("burgers_ide_disc" + tag, g["parts" + tag], ty.param_blocks(Le, 2),
                    lambda dt, m, g=g, tag=tag: ty.burgers_ide_disc_loss_grad(g["w" + tag], Le, g["lb"], g["ub"], g["x_0"],
                                                                              g["u_0"], g["x_1"], g["u_1"], float(g["dt"]),
                                                                              g["IRK_alpha"], g["IRK_beta"], dtype=dt,
                                                                              magnitudes=m)))
    return out


def test_float64_oracle_still_reproduces_the_golden_files_exactly():
    """The dtype / magnitudes options leave the float64 arithmetic alone: the loss parts stored by make_golden.py (computed by
    this oracle) come back bit for bit, and asking for the magnitudes does not change the gradient."""
    for name, parts, blocks, f in _golden_evaluations():
        loss, grad, pr = f(np.float64, False)
        loss_m, grad_m, pr_m, mag = f(np.float64, True)
        if parts is not None:
            assert np.array_equal(np.array(pr, dtype=np.float64), np.asarray(parts)[:len(pr)]), name
        assert loss_m == loss and np.array_equal(grad_m, grad) and np.array_equal(np.array(pr_m), np.array(pr)), name
        assert grad.dtype == np.float64 and mag.shape == grad.shape and np.all(mag >= np.abs(grad) * (1 - 1e-12)), name
        assert blocks[-1][1].stop == grad.size, name


@pytest.mark.skipif(np.finfo(np.longdouble).eps > 1e-18, reason="np.longdouble has no extended precision on this platform")
def test_longdouble_oracle_agrees_with_float64_per_block():
    """The same sums in 64-bit-mantissa arithmetic.  At the golden (initialisation-scale) weights fp64 is good to ~1e-14 per
    block, so the two must agree to 1e-13 on every W_l, b_l, lambda and loss part; a path that rounds to a narrower type would
    not, and one that stays entirely in float64 fails the last check."""
    for name, _, blocks, f in _golden_evaluations():
        l64, g64, p64 = f(np.float64, False)
        lld, gld, pld, mag = f(np.longdouble, True)
        assert gld.dtype == np.longdouble and mag.dtype == np.longdouble, name
        assert abs(l64 - lld) <= 1e-13 * abs(lld), name
        for a, b in zip(p64, pld):
            assert abs(a - b) <= 1e-13 * abs(b), name
        for bn, sl in blocks:
            err = np.linalg.norm((g64[sl] - gld[sl]).astype(np.longdouble))
            assert err <= 1e-13 * np.linalg.norm(gld[sl]), (name, bn, float(err / np.linalg.norm(gld[sl])))
        # ... and the extended precision is actually used: the two differ somewhere
        assert not np.array_equal(g64, gld.astype(np.float64)), name
