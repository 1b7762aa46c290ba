"""GPU: the generic and Navier-Stokes fused kernels over the tiling sweep of tests/tiling_regimes.py, against the
extended-precision oracle, block by block.

The hand-picked shapes of the other precision files reach only part of the regimes the kernels' launch and item formulas
produce (column-group splits, K tails, bias-row positions, ragged point groups, the per-CTA point counts, the discrete-time
head's N-bar tail and wide-head switch; tests/test_tiling_regimes_cpu.py prints the fraction).  sweep(sms) reaches every one of
them at the SM count of the card the test runs on.  Here:

* the SM count the handle reports is checked first: the sweep is built for it, each shape's point split is the one
  tiling_regimes assumed (test_gpu_precision_load's load formulas agree), and every generic handle runs 2 x SMs CTAs and every
  Navier-Stokes handle SMs CTAs;
* every generic sweep shape is evaluated in the DMMA and the DFMA form (PINN_GENERIC_DFMA=0/1, each in its own process) and
  every Navier-Stokes shape once, and held per parameter block to check() of test_gpu_precision.py: REL 1e-12 plus 32 x the
  fp64 oracle's own error, against oracle.taylor, oracle.taylor_kdv_ac and oracle.taylor_ns;
* the two forms must differ bitwise on at least one shape (both ran);
* the probes (pinn_derivatives, pinn_predict) of every sweep net are held per stream to the oracle's forward streams at
  PROBE_TOL; the sweep has nets whose widest layer is 128 and 129, 1-D and 2-D, so both mlp_forward_generic instantiations run.

Each check prints the worst error/bound per shape and form (run with -s)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import tiling_regimes as tr
from conftest import ROOT
from oracle import taylor as ty, taylor_kdv_ac as tk, taylor_ns as tn
from test_gpu_precision import DOMAINS, FP64_FACTOR, LD, PROBE_TOL, _cabi, _norm, _ratio, _rand_w, _sms, check, points
from test_gpu_precision_heads import DOMAINS_1D, KDV_PROBE_TOL, points_1d
from test_gpu_precision_load import generic_load, ns_load

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
NS_BOXES = {"upstream": ((1.0, -2.0, 0.0), (8.0, 2.0, 20.0)), "small box": ((0.0, 0.0, 0.0), (1e-2, 2e-2, 1e-3))}


# ---------------------------------------------------------------------------------------------------------- shape inputs
def inputs(shape):
    """The arrays of a sweep shape, drawn from its seed.  Continuous heads take nu = 1 / e^{lambda_2} = 1, the discrete-time
    heads an O(1) coefficient on their highest derivative, so the u_xx / u_xxx paths are visible on domains with sc != 1."""
    head, layers, c = shape["head"], shape["layers"], shape["counts"]
    rng = np.random.default_rng(shape["seed"])
    if head == "ns":
        from test_gpu_ns import ns_inputs
        lb, ub = NS_BOXES[shape["dom"]]
        _, lb, ub, X, uv, w = ns_inputs(layers[1:-1], c["n"], shape["seed"], lb, ub)
        return dict(lb=lb, ub=ub, X=X, uv=uv, w=w)
    w = _rand_w(layers, shape["seed"])
    if head in ("disc", "kdv"):
        lb, ub = DOMAINS_1D[shape["dom"]]
        d = dict(lb=np.array([lb]), ub=np.array([ub]))
        x_0 = points_1d(rng, shape["dom"], c["n_0"])
        xi0 = (x_0 - lb) / (ub - lb)
        if head == "disc":
            q = layers[-1] - 1
            d.update(w=w, x_0=x_0, u_0=-np.sin(np.pi * xi0), x_1=np.array([[lb], [ub]]), nu=1.0, dt=0.3,
                     irk=rng.standard_normal((q + 1, q)) / q)
        else:
            q = layers[-1]
            x_1 = points_1d(rng, shape["dom"], c["n_1"])
            d.update(w=np.concatenate([w, [1.0, 0.0]]), x_0=x_0, u_0=np.cos(np.pi * xi0), x_1=x_1,
                     u_1=0.5 * np.cos(np.pi * (x_1 - lb) / (ub - lb) + 0.3), dt=0.6,
                     alpha=(rng.standard_normal((q, q)) / q).astype(np.float32),
                     beta=(rng.standard_normal((1, q)) / q).astype(np.float32))
        return d
    lb, ub = (np.array(v) for v in DOMAINS[shape["dom"]])
    d = dict(lb=lb, ub=ub)
    if head == "nls":
        tb = np.concatenate([[lb[1], ub[1]], rng.uniform(lb[1], ub[1], max(c["n_b"] - 2, 0))])[:c["n_b"], None]
        x0 = np.concatenate([[lb[0], ub[0]], rng.uniform(lb[0], ub[0], max(c["n_0"] - 2, 0))])[:c["n_0"], None]
        d.update(w=w, X_f=points(rng, lb, ub, c["n_f"]), tb=tb, X0=np.concatenate([x0, 0 * x0 + lb[1]], 1),
                 uv0=rng.standard_normal((c["n_0"], 2)))
        return d
    d.update(X_u=points(rng, lb, ub, c["n_u"]), u=rng.uniform(-1, 1, (c["n_u"], 1)))
    if head == "ide":
        d.update(w=np.concatenate([w, [0.5, 0.0]]), X_f=np.zeros((0, 2)))
    else:
        d.update(w=w, X_f=points(rng, lb, ub, c["n_f"]))
    return d


def oracle(shape, d, dtype, magnitudes):
    head, layers = shape["head"], shape["layers"]
    kw = dict(dtype=dtype, magnitudes=magnitudes)
    if head in ("inf", "ide"):
        return ty.burgers_loss_grad(d["w"], layers, d["lb"], d["ub"], d["X_f"], d["X_u"], d["u"],
                                    nu=None if head == "ide" else 1.0, identification=head == "ide", **kw)
    if head == "nls":
        return ty.schrodinger_loss_grad(d["w"], layers, d["lb"], d["ub"], d["X_f"], d["tb"], d["X0"], d["uv0"], **kw)
    if head == "disc":
        return ty.burgers_disc_loss_grad(d["w"], layers, d["lb"], d["ub"], d["x_0"], d["u_0"], d["x_1"], d["nu"], d["dt"],
                                         d["irk"], **kw)
    if head == "kdv":
        return tk.kdv_ide_disc_loss_grad(d["w"], layers, d["lb"], d["ub"], d["x_0"], d["u_0"], d["x_1"], d["u_1"], d["dt"],
                                         d["alpha"], d["beta"], **kw)
    return tn.ns_ide_loss_grad(d["w"], layers, d["lb"], d["ub"], d["X"], d["uv"], **kw)


def handle(c, shape, d):
    head, layers = shape["head"], shape["layers"]
    pde = {"inf": c.BURGERS_INF, "ide": c.BURGERS_IDE, "nls": c.NLS_INF, "disc": c.BURGERS_DISC, "kdv": c.KDV_IDE_DISC,
           "ns": c.NS_IDE}[head]
    p = c.Pinn(pde, layers, d["lb"], d["ub"])
    if head == "inf":
        p.set_pde_params([1.0]); p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1]); p.set_data(d["X_u"], d["u"])
    elif head == "ide":
        p.set_data(d["X_u"], d["u"])
    elif head == "nls":
        p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1]); p.set_boundary(d["tb"]); p.set_data(d["X0"], d["uv0"])
    elif head == "disc":
        p.set_pde_params([d["nu"], d["dt"]]); p.set_irk(d["irk"]); p.set_boundary(d["x_1"]); p.set_data(d["x_0"], d["u_0"])
    elif head == "kdv":
        p.set_pde_params([d["dt"]]); p.set_irk(c.irk_ide_disc(d["alpha"], d["beta"]))
        p.set_snapshot(0, d["x_0"], d["u_0"]); p.set_snapshot(1, d["x_1"], d["u_1"])
    else:
        p.set_data(d["X"], d["uv"])
    return p


def blocks_and_parts(shape):
    """(parameter blocks, the kernel's parts slot of each oracle part, the parts slot that must be 0 or None)."""
    head, layers = shape["head"], shape["layers"]
    lam = 2 if head in ("ide", "kdv", "ns") else 0
    part_idx, zero = {"inf": ((0, 2), 1), "ide": ((0, 2), 1), "nls": ((0, 1, 2), None), "disc": ((0, 1), 2),
                      "kdv": ((0, 1), 2), "ns": ((0, 2), 1)}[head]
    return ty.param_blocks(layers, lam), part_idx, zero


_ORACLE = {}


def reference(sms, shape):
    key = (sms, shape["name"])
    if key not in _ORACLE:
        d = inputs(shape)
        _ORACLE[key] = (oracle(shape, d, LD, True), oracle(shape, d, np.float64, False))
    return _ORACLE[key]


# ------------------------------------------------------------------------------------------------------------ loads
def assert_sweep_loads(sms):
    """The sweep for this card's SM count, and the point split of every shape as tiling_regimes assumed it (the load formulas
    of test_gpu_precision_load agree with it); the sweep reaches every cell at this count."""
    S = tr.sweep(sms)
    U = tr.universe()
    for kind, split, load in (("generic", tr.generic_split, generic_load), ("ns", tr.ns_split, ns_load)):
        reached = set()
        for s in S[kind]:
            n = tr.n_total(s)
            sp, ld = split(n, sms), load(n, sms)
            assert (sp["pts"], sp["grid"]) == (ld["points per CTA"], ld["grid"]), (s["name"], sp, ld)
            print("[load] %-44s n %5d, %2d points per CTA, grid %3d of %3d, last CTA %2d points"
                  % (s["name"], n, sp["pts"], sp["grid"], sp["n_cta"], ld["last CTA points"]))
            reached |= tr.shape_cells(s, sms)
        assert reached == U[kind], (kind, sorted(U[kind] - reached, key=repr)[:5])
    return S


# ------------------------------------------------------------------------------------------------------------ workers
def run_worker(func, env):
    """func() of this module in a fresh interpreter with env set (PINN_GENERIC_DFMA is read once per process); it prints one
    JSON line."""
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_tiling_sweep as m; m.%s()" % (ROOT, TESTS, func)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def generic_worker():
    c, sms = _cabi(), _sms()
    out = {"sms": sms}
    for shape in tr.sweep(sms)["generic"]:
        d = inputs(shape)
        p = handle(c, shape, d)
        info = p.kernel_info()
        assert info["dyn_smem"] == 0 and info["grid"] == 2 * sms, (shape["name"], info)     # the generic kernel, C = 2 x SMs
        loss, grad, parts = p.loss_grad(w=d["w"])
        out[shape["name"]] = [loss, grad.tolist(), parts.tolist()]
        p.close()
    print(json.dumps(out))


@pytest.fixture(scope="module")
def sweep_runs():
    sms = _sms()
    S = assert_sweep_loads(sms)                                   # before anything is evaluated
    runs = {form: run_worker("generic_worker", {"PINN_GENERIC_DFMA": flag}) for form, flag in (("dmma", "0"), ("dfma", "1"))}
    assert runs["dmma"]["sms"] == runs["dfma"]["sms"] == sms
    return sms, S, runs


def _check_all(tag, sms, shapes, got_of):
    failed = []
    for shape in shapes:
        ref, ref64 = reference(sms, shape)
        blocks, part_idx, zero = blocks_and_parts(shape)
        loss, grad, parts = got_of(shape)
        try:
            check("%s/%s" % (tag, shape["name"]), (loss, np.asarray(grad), np.asarray(parts)), ref, ref64, blocks, part_idx)
            assert zero is None or parts[zero] == 0.0, ("parts", zero, parts)
        except AssertionError as e:
            failed.append((shape["name"], tr.n_total(shape), str(e)[:400]))
    assert not failed, failed


@pytest.mark.parametrize("form", ["dmma", "dfma"])
def test_generic_sweep_per_block(sweep_runs, form):
    sms, S, runs = sweep_runs
    _check_all(form, sms, S["generic"], lambda s: runs[form][s["name"]])


def test_both_forms_ran(sweep_runs):
    sms, S, runs = sweep_runs
    assert any(runs["dmma"][s["name"]][1] != runs["dfma"][s["name"]][1] for s in S["generic"])


def test_navier_stokes_sweep_per_block():
    c, sms = _cabi(), _sms()
    S = assert_sweep_loads(sms)
    got = {}
    for shape in S["ns"]:
        d = inputs(shape)
        p = handle(c, shape, d)
        assert p.kernel_info()["grid"] == sms                     # one CTA per SM
        got[shape["name"]] = p.loss_grad(w=d["w"])
        p.close()
    _check_all("ns", sms, S["ns"], lambda s: got[s["name"]])


# ------------------------------------------------------------------------------------------------------------ probes
def _stream_ratio(got, ref, ref64, tol):
    return _ratio(_norm(got - ref), tol * _norm(ref) + FP64_FACTOR * _norm(ref64 - ref))


def test_probes_on_every_sweep_net():
    c, sms = _cabi(), _sms()
    S = tr.sweep(sms)
    failed = []
    for shape in S["generic"] + S["ns"]:
        head, layers = shape["head"], shape["layers"]
        d = inputs(shape)
        rng = np.random.default_rng(shape["seed"] + 1)
        lam = 2 if head in ("ide", "kdv", "ns") else 0
        w_net = d["w"][:len(d["w"]) - lam]
        if head == "ns":
            X = d["lb"] + (d["ub"] - d["lb"]) * rng.random((64, 3))
            ref, ref64 = (tn.forward_ns(w_net, layers, d["lb"], d["ub"], X, dtype=t)[0] for t in (LD, np.float64))
        elif head in ("disc", "kdv"):
            X = points_1d(rng, shape["dom"], 64)
            fwd = tk.forward_third if head == "kdv" else ty.forward
            ref, ref64 = (fwd(w_net, layers, d["lb"], d["ub"], X, dtype=t)[0] for t in (LD, np.float64))
        else:
            X = points(rng, d["lb"], d["ub"], 64)
            ref, ref64 = (ty.forward(w_net, layers, d["lb"], d["ub"], X, dtype=t)[0] for t in (LD, np.float64))
        p = c.Pinn({"inf": c.BURGERS_INF, "ide": c.BURGERS_IDE, "nls": c.NLS_INF, "disc": c.BURGERS_DISC,
                    "kdv": c.KDV_IDE_DISC, "ns": c.NS_IDE}[head], layers, d["lb"], d["ub"])
        p.set_weights(d["w"])
        got, pred = p.derivatives(X), p.predict(X)
        p.close()
        rows = []
        if head == "ns":
            for k, m in enumerate(tn.STREAMS):
                for o in range(2):
                    rows.append(("stream %d/%d" % (k, o), _stream_ratio(got[:, k, o], ref[k][:, o], ref64[k][:, o],
                                                                        1e-13 if sum(m) <= 1 else 1e-12)))
            for o in range(2):
                rows.append(("predict/%d" % o, _stream_ratio(pred[:, o], ref[0][:, o], ref64[0][:, o], PROBE_TOL[0])))
        else:
            tol = KDV_PROBE_TOL if head == "kdv" else PROBE_TOL
            for s in range(4):
                if head == "disc" and s == 2:
                    rows.append(("t stream is 0", 0.0 if np.all(got[s] == 0.0) else np.inf))     # 1-D nets have no t stream
                    continue
                for o in range(layers[-1]):
                    rows.append(("stream %d/%d" % (s, o), _stream_ratio(got[s][:, o], ref[s][:, o], ref64[s][:, o], tol[s])))
            for o in range(layers[-1]):
                rows.append(("predict/%d" % o, _stream_ratio(pred[:, o], ref[0][:, o], ref64[0][:, o], PROBE_TOL[0])))
        worst = max(rows, key=lambda r: r[1])
        print("[precision] %-46s worst error/bound %.3g (%s), max width %d" % ("probes/" + shape["name"], worst[1], worst[0],
                                                                                max(layers[1:])))
        if not worst[1] <= 1.0:
            failed.append((shape["name"], [r for r in rows if not r[1] <= 1.0][:4]))
    assert not failed, failed
