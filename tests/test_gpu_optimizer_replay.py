"""GPU: the device optimisers replayed step by step against an extended-precision oracle fed the same gradients.

The trajectory tests elsewhere compare weights after a whole run at 1e-7 .. 1e-8: Adam moves a weight by about lr per step, so an
error of 1e-7 in the update changes the weights by ~1e-10 relative, and a fixed-step L-BFGS amplifies rounding so much that a
recursion wrong at the 1e-9 level is invisible.  Here every step is checked on its own:

* Adam: before each step the test reads (f_t, g_t) = loss_grad() at the current weights w_t, then steps and reads w_{t+1}.  The
  step's loss and last_loss() must equal f_t bit for bit (both are R[P] + R[P+1] + R[P+2] of the same reduction).  m and v are
  tracked on the host from the recorded g_t in np.longdouble and in float64, each step starting from the device's own w_t:
      |w_dev - w_ld| <= 4 ulp(w_ld) + 1e-13 |D_ld| + 32 |w_64 - w_ld|          per entry, D = the Adam update.
* L-BFGS, through the foreign-closure handle (which exposes every x it asks for), with PINN_LBFGS=serial and =gram: every
  (x_k, f_k, g_k) is recorded, and oracle.reference_port.lbfgs_fixed_step replays the run on exactly those evaluations
  (ScriptedOpfunc) in longdouble, in float64, and in the float64 Gram form.  Control flow must be equal, and per iteration
      ||(x_{k+1} - x_k) - t_k d_k^ld|| <= ||ulp(x_{k+1})|| + 1e-13 ||t_k d_k^ld|| + 32 ||t_k (d_k^64 - d_k^ld)||
  where, for the Gram kernel, d^64 is whichever float64 replay lies further from the longdouble one (their gap is the
  formulation's own conditioning, not a kernel error).  On a nonconvex loss the replay ends at the first curvature test
  y.s > 1e-10 that rounding can decide either way; the synthetic objectives must be replayed to the end.
* pinn_lbfgs on a model handle gives the same f_hist and x_final, bit for bit, as the foreign handle driven by that handle's
  loss_grad: both run the same iteration kernel on the same R, which carries the replay's verdict over to the production path.

Kernel switches are read once per process, so the device work runs in subprocess workers; each test prints the worst
error / bound ratio of its case (run with -s to read them).
"""
import json
import os
import subprocess
import sys
import traceback

import numpy as np
import pytest

from conftest import ROOT, load_golden
from oracle import reference_port as rp
from test_gpu_lbfgs_foreign import BOUNDARY_CASES

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
LD = np.longdouble
FP64_FACTOR = 32.0
EPS = float(np.finfo(float).eps)


def run_worker(func, env, *args):
    """func(*args) of this module in a fresh interpreter with env set; it prints one JSON line."""
    code = "import sys, json; sys.path[:0] = [%r, %r]; import test_gpu_optimizer_replay as m; m.%s(*json.loads(sys.argv[1]))" % (
        ROOT, TESTS, func)
    r = subprocess.run([sys.executable, "-c", code, json.dumps(list(args))], env=dict(os.environ, **env), capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _cabi():
    import pinn_cabi
    pinn_cabi.load()
    return pinn_cabi


def guarded(fn):
    """Run fn() and return its result, or the traceback of what went wrong (one failing case must not hide the others)."""
    try:
        return fn()
    except Exception:
        return {"error": traceback.format_exc()[-2500:]}


def report(tag, res):
    assert "error" not in res, res["error"]
    print("[replay] %-46s worst error/bound %.3g" % (tag, res["worst"]))
    assert not res["bad"], (tag, res["bad"][:5])


def _rand_w(layers, seed):
    rng = np.random.default_rng(seed)
    return rp.glorot_normal_flat(layers, rng) + 0.05 * rng.standard_normal(rp.num_params(layers))


# ------------------------------------------------------------------------------------------------------------- model handles
GENERIC = [2, 24, 12, 24, 1]
WIDE = [2, 128, 128, 128, 1]                     # P = 33 537: more than the single-CTA L-BFGS kernel holds


def make_handle(c, name, n_points=None):
    """(handle, initial weights) of one of the models on its golden inputs; n_points keeps the first points only."""
    if name in ("burgers", "generic", "wide"):
        g = load_golden("burgers_inf")
        layers = {"burgers": [int(v) for v in g["layers"]], "generic": GENERIC, "wide": WIDE}[name]
        p = c.Pinn(c.BURGERS_INF, layers, g["lb"], g["ub"])
        p.set_pde_params([float(g["nu"])]); p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1]); p.set_data(g["X_u"], g["u"])
        return p, (g["w"] if name == "burgers" else _rand_w(layers, 11))
    if name == "ide":
        g = load_golden("burgers_ide")
        n = n_points or g["X_u"].shape[0]
        p = c.Pinn(c.BURGERS_IDE, [int(v) for v in g["layers"]], g["lb"], g["ub"])
        p.set_data(g["X_u"][:n], g["u"][:n])
        return p, g["w2"]
    if name == "nls":
        g = load_golden("nls_inf")
        p = c.Pinn(c.NLS_INF, [int(v) for v in g["layers"]], g["lb"], g["ub"])
        p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1]); p.set_boundary(g["tb"]); p.set_data(g["x0"], g["uv0"])
        return p, g["w"]
    if name == "disc":
        g = load_golden("burgers_disc")
        p = c.Pinn(c.BURGERS_DISC, [int(v) for v in g["layers"]], g["lb"], g["ub"])
        p.set_pde_params([float(g["nu"]), float(g["dt"])]); p.set_irk(g["IRK"].astype(np.float64))
        p.set_boundary(g["x_1"]); p.set_data(g["x_0"], g["u_0"])
        return p, g["w"]
    if name == "ide_disc":
        g = load_golden("burgers_ide_disc")
        p = c.Pinn(c.BURGERS_IDE_DISC, [int(v) for v in g["layers"]], g["lb"], g["ub"])
        p.set_pde_params([float(g["dt"])]); p.set_irk(c.irk_ide_disc(g["IRK_alpha"], g["IRK_beta"]))
        p.set_snapshot(0, g["x_0"], g["u_0"]); p.set_snapshot(1, g["x_1"], g["u_1"])
        return p, g["w2"]
    raise ValueError(name)


# ---------------------------------------------------------------------------------------------------------------------- Adam
class AdamReplay(object):
    """Host replay of the device Adam, one step at a time, from the device's own weights and the gradient it reduced.

    m and v are carried in np.longdouble and in float64 from the recorded gradients; ``check`` applies the per-entry rule of the
    module docstring and returns the worst ratio.  ``reset`` mirrors pinn_adam_reset (m, v and t restart); weights set between
    steps need nothing, because every step starts from the device's w_t."""

    def __init__(self, P, lr, b1=0.9, b2=0.999, eps=1e-7):
        self.P, self.hp = P, dict(lr=lr, b1=b1, b2=b2, eps=eps)
        self.reset()

    def reset(self):
        self.s64, self.sld = rp.adam_init(self.P), rp.adam_init(self.P)

    def check(self, w_t, g_t, w_next):
        w_ld = rp.adam_update(np.asarray(w_t, dtype=LD), g_t, self.sld, dtype=LD, **self.hp)
        w_64 = rp.adam_update(np.asarray(w_t, dtype=np.float64), g_t, self.s64, **self.hp)
        err = np.abs(np.asarray(w_next, dtype=LD) - w_ld)
        bound = (4.0 * np.spacing(np.abs(w_ld.astype(np.float64))) + 1e-13 * np.abs(w_ld - np.asarray(w_t, dtype=LD))
                 + FP64_FACTOR * np.abs(np.asarray(w_64, dtype=LD) - w_ld))
        ratio = (err / bound).astype(np.float64)
        return float(np.max(ratio)), [int(i) for i in np.flatnonzero(~(ratio <= 1.0))]


def adam_replay(p, w0, hp, script):
    """Run `script` on handle p from w0: ("steps", n) single Adam steps, ("reset",) pinn_adam_reset, ("set", scale) set_weights to
    scale * the current weights.  Every step is replayed by AdamReplay; the step's loss and last_loss() must equal loss_grad()'s."""
    rep = AdamReplay(p.P, **hp)
    p.set_weights(w0)
    p.adam_reset()
    worst, bad, step, eps_dominated, launches = 0.0, [], 0, False, set()
    for op in script:
        if op[0] == "reset":
            p.adam_reset(); rep.reset()
            continue
        if op[0] == "set":
            p.set_weights(op[1] * p.get_weights())
            continue
        for _ in range(op[1]):
            step += 1
            w_t = p.get_weights()
            f_t, g_t, _ = p.loss_grad()
            n0 = p.launch_count()
            loss = p.adam_step(**hp)
            launches.add(p.launch_count() - n0)
            if loss != f_t or p.last_loss() != f_t:
                bad.append(("loss", step, loss, p.last_loss(), f_t))
            r, idx = rep.check(w_t, g_t, p.get_weights())
            worst = max(worst, r)
            if idx:
                bad.append(("w", step, idx[:8], r))
            eps_dominated |= bool(np.any(np.sqrt(rep.s64.v) < hp["eps"]))
    return {"worst": worst, "bad": bad, "eps_dominated": eps_dominated, "launches_per_step": sorted(launches)}


REF_HP = dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-7)
EPS_HP = dict(lr=0.05, b1=0.5, b2=0.9, eps=1e-2)       # eps dominates sqrt(v) on the small-gradient entries
B1_0_HP = dict(lr=1e-3, b1=0.0, b2=0.99999, eps=1e-7)  # no momentum, and 1 - b2^t as small as it gets
SCRIPT = [("steps", 20), ("reset",), ("steps", 6), ("set", 1.01), ("steps", 6)]
# (name, model, hyperparameters, script); every path runs the reference's hyperparameters with a reset and a set_weights
ADAM_CASES = [
    ("burgers", "burgers", REF_HP, SCRIPT),
    ("burgers_eps", "burgers", EPS_HP, [("steps", 25)]),
    ("burgers_b1_0", "burgers", B1_0_HP, [("steps", 25)]),
    ("ide", "ide", REF_HP, SCRIPT),
    ("ide_eps", "ide", EPS_HP, [("steps", 25)]),
    ("nls", "nls", REF_HP, SCRIPT),
    ("generic", "generic", REF_HP, SCRIPT),
    ("generic_b1_0", "generic", B1_0_HP, [("steps", 25)]),
    ("disc", "disc", REF_HP, SCRIPT),
    ("ide_disc", "ide_disc", REF_HP, SCRIPT),
    ("ide_disc_eps", "ide_disc", EPS_HP, [("steps", 25)]),
]
# Burgers runs through three different reductions + Adam: the v2 kernel's in-kernel tail, reduce_tail after v2, and v1
ADAM_PATHS = {"v2_tail": {"PINN_BURGERS_KERNEL": "v2"}, "v2_no_tail": {"PINN_BURGERS_KERNEL": "v2", "PINN_FUSED_TAIL": "0"},
              "v1": {"PINN_BURGERS_KERNEL": "v1"}}
RING_STEPS = 4096 + 104


def adam_worker(path):
    c = _cabi()
    out = {}
    for name, model, hp, script in ADAM_CASES:
        if path != "v2_tail" and model not in ("burgers", "ide"):
            continue                                   # the switches only change the specialised Burgers kernels
        p, w0 = make_handle(c, model)
        out[name] = guarded(lambda: adam_replay(p, w0, hp, script))
        out[name]["kernel"] = p.kernel_info()
        p.close()
    if path == "v2_tail":
        out["ring"] = guarded(lambda: adam_ring(c))
    print(json.dumps(out))


def adam_ring(c):
    """More steps than the 4096-entry loss ring holds, replayed step by step; then adam_steps(n) on a second handle must give
    the same bits as n single steps."""
    p, w0 = make_handle(c, "ide", n_points=200)
    res = adam_replay(p, w0, REF_HP, [("steps", RING_STEPS)])
    w_single, last = p.get_weights(), p.last_loss()
    q, _ = make_handle(c, "ide", n_points=200)
    q.set_weights(w0)
    q.adam_steps(RING_STEPS, **REF_HP)
    q.sync()
    if not (np.array_equal(q.get_weights(), w_single) and q.last_loss() == last):
        res["bad"].append(("adam_steps", float(np.max(np.abs(q.get_weights() - w_single))), q.last_loss(), last))
    p.close(); q.close()
    return res


@pytest.fixture(scope="module")
def adam_runs():
    runs = {path: run_worker("adam_worker", env, path) for path, env in ADAM_PATHS.items()}
    k = {path: runs[path]["burgers"]["kernel"] for path in runs}
    assert k["v2_tail"] != k["v1"]                    # two different Burgers kernels actually ran
    return runs


@pytest.mark.parametrize("path", list(ADAM_PATHS))
@pytest.mark.parametrize("case", [c[0] for c in ADAM_CASES])
def test_adam_step_by_step_against_longdouble(adam_runs, path, case):
    run = adam_runs[path]
    if case not in run:
        pytest.skip("the path switch does not apply to this model")
    report("adam/%s/%s" % (path, case), run[case])
    if case.endswith("_eps"):
        assert run[case]["eps_dominated"]            # the case exercises what it is meant to
    # the path ran as named: one launch per step when the v2 kernel reduces and applies Adam in its own last CTAs, two (fused
    # kernel + reduce_tail) with PINN_FUSED_TAIL=0, with v1 and with every other kernel
    model = {c[0]: c[1] for c in ADAM_CASES}[case]
    assert run[case]["launches_per_step"] == [1 if path == "v2_tail" and model in ("burgers", "ide") else 2], run[case]


def test_adam_loss_ring_wraps_and_batched_steps_match(adam_runs):
    report("adam/ring_%d_steps" % RING_STEPS, adam_runs["v2_tail"]["ring"])
    assert adam_runs["v2_tail"]["ring"]["launches_per_step"] == [1]


# -------------------------------------------------------------------------------------------------------------------- L-BFGS
def drive_foreign(c, fn, x0, max_iter, lr=1.0, n_corr=100, tol_fun=1e-5, tol_x=1e-19, max_eval=0.0):
    """Run the foreign-closure handle on fn; record every x it asks for and every (f, g) it is fed."""
    h = c.Lbfgs(x0, max_iter, lr, n_corr, tol_fun, tol_x, max_eval)
    xs, fs, gs, logged = [np.array(x0, dtype=np.float64)], [], [], []
    while True:
        f, g = fn(xs[-1])
        fs.append(float(f)); gs.append(np.array(g, dtype=np.float64))
        x, st, it, ev, li, lf = h.feed(f, g)
        if li is not None:
            logged.append((li, lf))
        if st != 0:
            break
        xs.append(x)
    run = dict(xs=xs, fs=fs, gs=gs, x_final=x, reason=c.LBFGS_REASONS[st], n_iter=it, n_eval=ev, logged=logged, f_hist=h.f_hist())
    h.close()
    return run


def lbfgs_replay(run, x0, mode, max_iter, lr=1.0, n_corr=100, tol_fun=1e-5, tol_x=1e-19, max_eval=0.0):
    """Replay a recorded foreign run in longdouble and float64 (+ the float64 Gram form for the Gram kernel) and apply the
    per-iteration rule of the module docstring."""
    cfg = dict(max_iter=max_iter, learning_rate=lr, n_correction=n_corr or 100, tol_fun=tol_fun, tol_x=tol_x,
               max_eval=max_eval or None)
    trs = {}
    for key, kw in (("ld", dict(dtype=LD)), ("lit", {}), ("gram", dict(direction="gram"))):
        if key == "gram" and mode != "gram":
            continue
        op = rp.ScriptedOpfunc(run["fs"], run["gs"])
        trs[key] = rp.lbfgs_fixed_step(op, x0, **cfg, **kw)
        op.assert_consumed()
    ld, bad = trs["ld"], []
    pts = run["xs"] + ([run["x_final"]] if run["reason"] == "max iterations" else [])
    nrm = lambda v: float(np.sqrt(np.sum(np.square(np.asarray(v, dtype=LD)))))
    worst, ratios, undetermined, s_prev = 0.0, [], None, None
    for k in range(min(len(ld.d), len(pts) - 1)):
        if k >= 1:
            # the curvature test y.s > 1e-10 of iteration k + 1 is decided by rounding when the kernel's y.s may lie on the
            # other side of the threshold: within |y| |s_dev - s_ld| (the step it took differs from the replay's) plus the
            # rounding of the dot product.  The replay cannot know which branch the kernel took; it stops there.
            ys, ys_abs = ld.curv[k - 1]
            # One nonzero product and a step equal to the replay's: the kernel's y.s is the replay's, even on the threshold.
            y = np.asarray(run["gs"][k], dtype=LD) - np.asarray(run["gs"][k - 1], dtype=LD)
            exact = s_prev == 0.0 and np.count_nonzero(y * (LD(ld.t[k - 1]) * ld.d[k - 1])) <= 1
            if not exact and abs(float(ys) - 1e-10) <= nrm(y) * s_prev + 1e-12 * float(ys_abs):
                undetermined = k + 1
                break
        s_ld = LD(ld.t[k]) * ld.d[k]
        s_dev = np.asarray(pts[k + 1], dtype=LD) - np.asarray(pts[k], dtype=LD)
        gap = max(nrm(tr.t[k] * tr.d[k] - s_ld) for key, tr in trs.items() if key != "ld")
        bound = nrm(np.spacing(np.abs(pts[k + 1]))) + 1e-13 * nrm(s_ld) + FP64_FACTOR * gap
        s_prev = nrm(s_dev - s_ld)
        r = s_prev / bound
        ratios.append(r)
        worst = max(worst, r)
        if not r <= 1.0:
            bad.append(("step", k + 1, r))
    if undetermined is None:                          # the whole run is determined: control flow and step count must agree
        for key, tr in trs.items():
            got = (tr.stop_reason, tr.n_iter, tr.n_eval, tr.logged)
            if got != (run["reason"], run["n_iter"], run["n_eval"], [tuple(v) for v in run["logged"]]):
                bad.append(("control flow", key, got[:3], (run["reason"], run["n_iter"], run["n_eval"])))
        if len(pts) != len(ld.d) + 1:
            bad.append(("steps", len(pts) - 1, len(ld.d)))
    if run["f_hist"] != run["fs"]:
        bad.append(("f_hist", len(run["f_hist"]), len(run["fs"])))
    return {"worst": worst, "bad": bad, "n_iter": run["n_iter"], "reason": run["reason"], "checked": len(ratios),
            "undetermined_at": undetermined, "ratios": ratios[:: max(1, len(ratios) // 50)]}


def diag_quadratic(n, top=1e6):
    lam = np.logspace(0.0, np.log10(top), n)
    return lambda x: (0.5 * float(np.sum(lam * x * x)), lam * x)


def repeating(fn, at):
    """fn, except that at the evaluations listed in `at` the previous gradient comes back (y = 0: the pair is rejected).  The
    evaluation count lives in the closure: each worker process drives a case once."""
    state = {"n": 0, "g": None}

    def op(x):
        f, g = fn(x)
        if state["n"] in at:
            g = state["g"]
        state["n"] += 1
        state["g"] = g
        return f, g
    return op


def _x0(n, seed=0):
    return np.random.default_rng(seed).standard_normal(n)


A3 = np.array([1.0, 2.0, 4.0])
quad3 = lambda x: (0.5 * float(np.sum(A3 * x * x)), A3 * x)
X3 = np.array([0.5, 0.125, 0.0625])                    # g = (0.5, 0.25, 0.25): |g|_1 = 1 exactly
# (name, objective, x0, max_iter, options); the Burgers PINN case is built in the worker
LBFGS_CASES = [
    ("diag_n3072", diag_quadratic(3072), _x0(3072), 40, dict(lr=0.5, n_corr=10, tol_fun=1e-30)),
    ("diag_n3073", diag_quadratic(3073), _x0(3073), 40, dict(lr=0.5, n_corr=10, tol_fun=1e-30)),
    ("diag_n8192", diag_quadratic(8192), _x0(8192), 40, dict(lr=0.5, n_corr=10, tol_fun=1e-30)),
    ("diag_n8193", diag_quadratic(8193), _x0(8193), 40, dict(lr=0.5, n_corr=10, tol_fun=1e-30)),
    ("diag_n32768", diag_quadratic(32768), _x0(32768), 40, dict(lr=0.5, n_corr=10, tol_fun=1e-30)),
    ("gram_n40000", diag_quadratic(40000), _x0(40000), 25, dict(lr=0.5, n_corr=8, tol_fun=1e-30)),
    ("gram_n100000", diag_quadratic(100000), _x0(100000), 25, dict(lr=0.5, n_corr=8, tol_fun=1e-30)),
    ("ncorr1", diag_quadratic(500, 1e3), _x0(500, 1), 40, dict(lr=0.5, n_corr=1, tol_fun=1e-30)),
    ("ncorr128", diag_quadratic(700), _x0(700, 2), 160, dict(lr=0.5, n_corr=128, tol_fun=1e-30)),
    ("ncorr0_means_100", diag_quadratic(700), _x0(700, 3), 120, dict(lr=0.5, n_corr=0, tol_fun=1e-30)),
    ("rejected_pairs_full_history", repeating(diag_quadratic(300, 1e3), (9, 13, 14)), _x0(300, 4), 20,
     dict(lr=0.5, n_corr=4, tol_fun=1e-30)),
    ("first_step_g1_exactly_1", quad3, X3, 6, dict(lr=0.5, tol_fun=1e-30)),
    ("first_step_g1_below_1", quad3, 0.999 * X3, 6, dict(lr=0.5, tol_fun=1e-30)),
    ("first_step_g1_above_1", quad3, 1.001 * X3, 6, dict(lr=0.5, tol_fun=1e-30)),
]
# every stop test and the curvature test exactly on its threshold (test_gpu_lbfgs_foreign.BOUNDARY_CASES), in both kernels
_KW = {"maxIter": "max_iter", "learningRate": "lr", "nCorrection": "n_corr", "tolFun": "tol_fun", "tolX": "tol_x"}
LBFGS_CASES += [(name, fn, np.array(x0), kw["maxIter"], {_KW[k]: v for k, v in kw.items() if k != "maxIter"})
                for name, fn, x0, _, kw in BOUNDARY_CASES]
GRAM_ONLY = ("gram_n40000", "gram_n100000")
# the golden Burgers PINN (the problem of profiles/run_lbfgs_stability.py) after ADAM_EPOCHS Adam steps at lr 0.03, then
# BURGERS_ITERS fixed steps of 0.8 with a 50-pair history
ADAM_EPOCHS, BURGERS_ITERS = 2000, 600


def burgers_lbfgs_case(c):
    g = load_golden("burgers_accuracy")
    p = c.Pinn(c.BURGERS_INF, [2] + [20] * 8 + [1], g["lb"], g["ub"])
    p.set_pde_params([0.01 / np.pi]); p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1]); p.set_data(g["X_u"], g["u"])
    p.set_weights(g["w0"])
    p.adam_steps(ADAM_EPOCHS, 0.03)
    p.sync()
    x0 = p.get_weights()
    kw = dict(lr=0.8, n_corr=50, tol_fun=EPS)
    run = drive_foreign(c, lambda x: p.loss_grad(x)[:2], x0, BURGERS_ITERS, **kw)
    p.close()
    return run, x0, kw


def lbfgs_worker(mode):
    c = _cabi()
    out = {}
    for name, fn, x0, max_iter, kw in LBFGS_CASES:
        if mode == "serial" and name in GRAM_ONLY:
            continue
        out[name] = guarded(lambda: lbfgs_replay(drive_foreign(c, fn, x0, max_iter, **kw), x0, mode, max_iter, **kw))

    def burgers():
        run, x0, kw = burgers_lbfgs_case(c)
        res = lbfgs_replay(run, x0, mode, BURGERS_ITERS, **kw)
        res["f"] = run["fs"][:: 25] + run["fs"][-1:]
        above = [j for j, f in enumerate(run["fs"]) if not f <= 1.0]
        res["first_above_1"] = above[0] if above else None          # evaluation j follows iteration j's step
        res["f_last_checked"] = run["fs"][min(res["checked"], len(run["fs"]) - 1)]
        return res
    out["burgers_pinn"] = guarded(burgers)
    try:
        c.Lbfgs(np.zeros(32 * 1024 + 1), 5).close()
        out["refuses_32769"] = "accepted"
    except c.PinnError as e:
        out["refuses_32769"] = str(e)
    out["coupled"] = {name: guarded(lambda: coupled_vs_foreign(c, name)) for name in COUPLED
                      if mode == "gram" or name != "wide"}
    print(json.dumps(out))


@pytest.fixture(scope="module")
def lbfgs_runs():
    return {mode: run_worker("lbfgs_worker", {"PINN_LBFGS": mode}, mode) for mode in ("serial", "gram")}


@pytest.mark.parametrize("mode", ["serial", "gram"])
@pytest.mark.parametrize("case", [c[0] for c in LBFGS_CASES] + ["burgers_pinn"])
def test_lbfgs_iteration_by_iteration_against_longdouble(lbfgs_runs, mode, case):
    run = lbfgs_runs[mode]
    if case not in run:
        pytest.skip("the literal kernel holds at most 32768 entries")
    res = run[case]
    report("lbfgs/%s/%s" % (mode, case), res)
    if case != "burgers_pinn":
        assert res["undetermined_at"] is None and res["checked"] == res["n_iter"], res
        return
    # a nonconvex objective: once |y.s| is lost in rounding the curvature test is a coin toss and the replay ends there
    print("[replay] lbfgs/%s/burgers_pinn: %d iterations (%s), loss first above 1 after iteration %s, replay checked %d "
          "(loss there %.3g), curvature test decided by rounding at %s; loss every 25 iterations: %s"
          % (mode, res["n_iter"], res["reason"], res["first_above_1"], res["checked"], res["f_last_checked"],
             res["undetermined_at"], " ".join("%.3g" % f for f in res["f"])))
    # the case is there to examine the divergence: the run must diverge, and the replay must check the kernel's steps past it
    assert res["first_above_1"] is not None and res["checked"] > res["first_above_1"], res


def test_serial_kernel_refuses_more_than_32768_entries_and_gram_accepts_them(lbfgs_runs):
    assert "vector too large for the single-CTA L-BFGS kernel (32768 entries)" in lbfgs_runs["serial"]["refuses_32769"]
    assert lbfgs_runs["gram"]["refuses_32769"] == "accepted"


# ----------------------------------------------------------------------------------------------- coupled path == foreign path
COUPLED = ("burgers", "ide", "nls", "disc", "generic", "wide")
COUPLED_ITERS = 30


def coupled_vs_foreign(c, name):
    p, w0 = make_handle(c, name)
    kw = dict(learning_rate=0.8, n_correction=10, tol_fun=EPS)
    p.set_weights(w0)
    r = p.lbfgs(COUPLED_ITERS, want_x_final=True, **kw)
    run = drive_foreign(c, lambda x: p.loss_grad(x)[:2], w0, COUPLED_ITERS, lr=0.8, n_corr=10, tol_fun=EPS)
    kernel = p.kernel_info()
    p.close()
    same = (r["n_iter"] == run["n_iter"] and r["n_eval"] == run["n_eval"] and r["reason_str"] == run["reason"]
            and r["f_hist"] == run["f_hist"] and np.array_equal(r["x_final"], run["x_final"]))
    return {"same": bool(same), "n_iter": r["n_iter"], "reason": r["reason_str"], "kernel": kernel,
            "max_dx": float(np.max(np.abs(r["x_final"] - run["x_final"])))}


def coupled_v1_worker(mode):
    c = _cabi()
    print(json.dumps({"burgers": guarded(lambda: coupled_vs_foreign(c, "burgers"))}))


@pytest.fixture(scope="module")
def coupled_v1_runs():
    return {mode: run_worker("coupled_v1_worker", {"PINN_LBFGS": mode, "PINN_BURGERS_KERNEL": "v1"}, mode)
            for mode in ("serial", "gram")}


@pytest.mark.parametrize("mode", ["serial", "gram"])
@pytest.mark.parametrize("name", list(COUPLED) + ["burgers_v1"])
def test_pinn_lbfgs_equals_the_foreign_handle_bit_for_bit(lbfgs_runs, coupled_v1_runs, mode, name):
    if name == "wide" and mode == "serial":
        pytest.skip("P = 33 537 runs in Gram mode only")
    res = coupled_v1_runs[mode]["burgers"] if name == "burgers_v1" else lbfgs_runs[mode]["coupled"][name]
    assert "error" not in res, res["error"]
    assert res["n_iter"] == COUPLED_ITERS and res["reason"] == "max iterations", res
    assert res["same"], res
    if name == "burgers_v1":
        assert res["kernel"] != lbfgs_runs[mode]["coupled"]["burgers"]["kernel"]
