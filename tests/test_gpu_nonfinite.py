"""GPU: every kernel against the oracles on NaN and infinite inputs.

The reference (TF 2.0, fp64) lets NaN and +-Inf propagate: a NaN point coordinate, target, weight or constant makes the loss
NaN, and an infinite coordinate saturates its point (a = +-1, s = 0), keeping the loss finite while Inf * 0 turns that
coordinate's row of W_0 into NaN.  What the kernels return decides what the L-BFGS stop tests, the loss ring and the Logger see,
so here:

* each case injects one NaN or +-Inf into one input of a model: a point coordinate (the first point, a point inside the second
  CTA's range, the last point of a ragged set), a target, one entry of W_0, a middle W_l, a bias, the head, lambda_1, lambda_2,
  and the constants (nu, dt, d, k, one IRK / alpha entry, one source value);
* the class {finite, +Inf, -Inf, NaN} of the loss, of each loss part and of every gradient entry must equal the fp64 Taylor
  oracle's, elementwise (tests/test_nonfinite_cpu.py pins that oracle to the nested-autograd port on every case here);
* every block the oracle leaves entirely finite must pass test_gpu_precision.check() against the longdouble oracle: a saturated
  +-Inf point must be handled correctly, not only stay finite;
* after each injection the finite input is restored on the same handle, and loss_grad must equal that handle's own evaluation
  before the injection bit for bit (no state is poisoned).

The same rules are applied to the probes (predict, derivatives, residual), Adam, L-BFGS (foreign-closure handle and pinn_lbfgs)
and the zero-copy collocation path.  Kernel switches are read once per process, so the device work runs in subprocess workers.
"""
import json
import os
import subprocess
import sys
import traceback

import numpy as np
import pytest

from conftest import ROOT, load_golden
from oracle import reference_port as rp, taylor as ty, taylor_kdv_ac as tk, taylor_ns as tn, taylor_poly as tpo
from test_gpu_precision import BURGERS, FP64_FACTOR, LD, NLS, NU0, PROBE_TOL, _norm, _ratio, check, points
from test_gpu_precision_load import burgers_load, generic_load, nls_load, ns_load, ns_probe_chunks

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
NAN, INF = float("nan"), float("inf")
H100_SMS = 132                                    # positions used where no device is asked (tests/test_nonfinite_cpu.py)


def classes(v):
    """0 finite, 1 +Inf, 2 -Inf, 3 NaN, elementwise."""
    v = np.asarray(v, dtype=np.float64)
    return np.where(np.isnan(v), 3, np.where(np.isposinf(v), 1, np.where(np.isneginf(v), 2, 0)))


def _w(layers, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return scale * (rp.glorot_normal_flat(layers, rng) + 0.05 * rng.standard_normal(rp.num_params(layers)))


# ---------------------------------------------------------------------------------------------------------------- the models
# Each model: inputs() -> d (every array the handle and the oracles take), handle(c, d) -> a handle on those inputs, feed(p, d)
# sets every input of d on an existing handle, taylor(d, dtype, magnitudes), port(d) (the nested-autograd problem), n_extra
# (lambda entries), part_idx (the kernel's parts slot of each oracle part), the point sets (field, load family) with the column
# injected at (first, mid, last), the targets and the constants.
STD = (np.array([-1.0, 0.0]), np.array([1.0, 0.99]))
SHIFTED_1D = (np.array([0.3]), np.array([3.7]))
W33 = [2, 33, 17, 1]                              # widths that are not multiples of 8
DISC_NET = [1, 20, 20]
TERMS = {True: [(1.0, 0, (0, 0, 1, 0)), (1.0, 1, (1, 1, 0, 0)), (-1.0, 2, (0, 0, 0, 1)), (0.5, 0, (3, 0, 0, 0))],
         False: [(1.0, 0, (0, 0, 1, 0)), (1.0, 0, (1, 1, 0, 0)), (-0.1, 0, (0, 0, 0, 1)), (0.5, 0, (3, 0, 0, 0))]}   # by ide


def burgers_inputs(layers, ide):
    rng = np.random.default_rng(11 if ide else 10)
    lb, ub = STD
    w = load_golden("burgers_inf")["w"] if layers == BURGERS else _w(layers, 12)
    d = dict(layers=layers, lb=lb, ub=ub, X_u=points(rng, lb, ub, 203 if ide else 45), ide=ide)
    d["u"] = rng.uniform(-1, 1, (d["X_u"].shape[0], 1))
    if ide:
        d["w"] = np.concatenate([w, [1.0, -5.0]])
    else:
        d.update(w=w, X_f=points(rng, lb, ub, 203), nu=np.array([NU0]))
    return d


def burgers_feed(p, d):
    if not d["ide"]:
        p.set_pde_params([d["nu"][0]]); p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1])
    p.set_data(d["X_u"], d["u"])


def burgers_taylor(d, dtype=np.float64, magnitudes=False):
    return ty.burgers_loss_grad(d["w"], d["layers"], d["lb"], d["ub"], d.get("X_f"), d["X_u"], d["u"],
                                nu=None if d["ide"] else d["nu"][0], identification=d["ide"], dtype=dtype, magnitudes=magnitudes)


def burgers_port(d):
    if d["ide"]:
        return rp.BurgersIdentification(d["layers"], d["lb"], d["ub"], d["X_u"], d["u"])
    return rp.BurgersInference(d["layers"], d["lb"], d["ub"], float(d["nu"][0]), d["X_f"], d["X_u"], d["u"])


def nls_inputs():
    rng = np.random.default_rng(20)
    lb, ub = np.array([-5.0, 0.0]), np.array([5.0, np.pi / 2])
    x0 = rng.uniform(lb[0], ub[0], (11, 1))
    return dict(layers=NLS, lb=lb, ub=ub, w=load_golden("nls_inf")["w"], X_f=points(rng, lb, ub, 37),
                tb=rng.uniform(lb[1], ub[1], (9, 1)), X0=np.concatenate([x0, 0 * x0 + lb[1]], 1), uv0=rng.standard_normal((11, 2)))


def nls_feed(p, d):
    p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1]); p.set_boundary(d["tb"]); p.set_data(d["X0"], d["uv0"])


def nls_taylor(d, dtype=np.float64, magnitudes=False):
    return ty.schrodinger_loss_grad(d["w"], NLS, d["lb"], d["ub"], d["X_f"], d["tb"], d["X0"], d["uv0"], dtype=dtype,
                                    magnitudes=magnitudes)


def poly_inputs(ide):
    rng = np.random.default_rng(31 if ide else 30)
    lb, ub = STD
    n_res = 203
    X_u = points(rng, lb, ub, n_res if ide else 45)
    w = _w(W33, 32)
    d = dict(layers=W33, lb=lb, ub=ub, ide=ide, X_u=X_u, u=rng.uniform(-1, 1, (X_u.shape[0], 1)),
             X_f=None if ide else points(rng, lb, ub, n_res), source=rng.standard_normal(n_res),
             w=np.concatenate([w, [0.6, -0.4]]) if ide else w)
    return d


def poly_feed(p, d):
    p.set_data(d["X_u"], d["u"])
    if not d["ide"]:
        p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1])
    p.set_source(d["source"])                     # after the collocation points: storing them resets the source


def poly_taylor(d, dtype=np.float64, magnitudes=False):
    return tpo.poly_loss_grad(d["w"], W33, d["lb"], d["ub"], TERMS[d["ide"]], d["X_u"], d["u"], X_f=d["X_f"], source=d["source"],
                              identification=d["ide"], dtype=dtype, magnitudes=magnitudes)


def poly_port(d):
    from oracle import reference_port_poly as rpp
    return rpp.PolyProblem(W33, d["lb"], d["ub"], TERMS[d["ide"]], d["X_u"], d["u"], X_f=d["X_f"], source=d["source"],
                           identification=d["ide"])


Q = 8


def disc_inputs(kind):
    rng = np.random.default_rng({"disc": 40, "ide_disc": 41, "kdv": 42, "ac": 43}[kind])
    lb, ub = SHIFTED_1D
    q1 = Q if kind in ("ide_disc", "kdv") else Q + 1
    layers = DISC_NET + [q1]
    x_0 = np.concatenate([[lb[0], ub[0]], rng.uniform(lb[0], ub[0], 59)])[:, None]
    xi = (x_0 - lb[0]) / (ub[0] - lb[0])
    d = dict(kind=kind, layers=layers, lb=lb, ub=ub, w=_w(layers, 44), x_0=x_0, u_0=np.cos(np.pi * xi))
    if kind in ("ide_disc", "kdv"):
        x_1 = np.concatenate([[lb[0]], rng.uniform(lb[0], ub[0], 36)])[:, None]
        d.update(w=np.concatenate([d["w"], [0.4, -1.0]]), dt=np.array([0.6]), x_1=x_1, u_1=0.5 * np.cos(np.pi * x_1),
                 alpha=(rng.standard_normal((Q, Q)) / Q).astype(np.float32), beta=(rng.standard_normal((1, Q)) / Q).astype(np.float32))
    elif kind == "disc":
        d.update(nu=np.array([1.0]), dt=np.array([0.3]), x_1=np.array([[lb[0]], [ub[0]]]), IRK=rng.standard_normal((Q + 1, Q)) / Q)
    else:
        d.update(dt=np.array([0.8]), dk=np.array([1e-4, 5.0]), IRK=rng.standard_normal((Q + 1, Q)) / Q)
    return d


def disc_feed(p, d, c):
    kind = d["kind"]
    if kind in ("ide_disc", "kdv"):
        p.set_pde_params([d["dt"][0]]); p.set_irk(c.irk_ide_disc(d["alpha"], d["beta"]))
        p.set_snapshot(0, d["x_0"], d["u_0"]); p.set_snapshot(1, d["x_1"], d["u_1"])
    elif kind == "disc":
        p.set_pde_params([d["nu"][0], d["dt"][0]]); p.set_irk(d["IRK"]); p.set_boundary(d["x_1"]); p.set_data(d["x_0"], d["u_0"])
    else:
        p.set_pde_params([d["dt"][0], d["dk"][0], d["dk"][1]]); p.set_irk(d["IRK"]); p.set_data(d["x_0"], d["u_0"])


def disc_taylor(d, dtype=np.float64, magnitudes=False):
    kind, a = d["kind"], (d["w"], d["layers"], d["lb"], d["ub"])
    if kind == "disc":
        return ty.burgers_disc_loss_grad(*a, d["x_0"], d["u_0"], d["x_1"], d["nu"][0], d["dt"][0], d["IRK"], dtype=dtype,
                                         magnitudes=magnitudes)
    if kind == "ac":
        return tk.ac_disc_loss_grad(*a, d["x_0"], d["u_0"], d["dt"][0], d["IRK"], d=d["dk"][0], k=d["dk"][1], dtype=dtype,
                                    magnitudes=magnitudes)
    fn = ty.burgers_ide_disc_loss_grad if kind == "ide_disc" else tk.kdv_ide_disc_loss_grad
    return fn(*a, d["x_0"], d["u_0"], d["x_1"], d["u_1"], d["dt"][0], d["alpha"], d["beta"], dtype=dtype, magnitudes=magnitudes)


def disc_port(d):
    from oracle import reference_port_kdv_ac as rka
    kind, a = d["kind"], (d["layers"], d["lb"], d["ub"])
    if kind == "disc":
        return rp.BurgersDiscreteInference(*a, float(d["nu"][0]), float(d["dt"][0]), d["x_0"], d["u_0"], d["x_1"], d["IRK"])
    if kind == "ac":
        return rka.AllenCahnDiscreteInference(*a, float(d["dt"][0]), d["x_0"], d["u_0"], d["IRK"], d=float(d["dk"][0]),
                                              k=float(d["dk"][1]))
    cls = rp.BurgersDiscreteIdentification if kind == "ide_disc" else rka.KdVDiscreteIdentification
    return cls(*a, float(d["dt"][0]), d["x_0"], d["u_0"], d["x_1"], d["u_1"], d["alpha"], d["beta"])


NS_NET = [3, 20, 20, 2]


def ns_inputs():
    rng = np.random.default_rng(50)
    lb, ub = np.array([1.0, -2.0, 0.0]), np.array([8.0, 2.0, 20.0])
    X = lb + (ub - lb) * rng.random((203, 3))
    return dict(layers=NS_NET, lb=lb, ub=ub, X=X, uv=rng.standard_normal((203, 2)),
                w=np.concatenate([_w(NS_NET, 51), [0.6, 0.05]]))


def ns_taylor(d, dtype=np.float64, magnitudes=False):
    return tn.ns_ide_loss_grad(d["w"], NS_NET, d["lb"], d["ub"], d["X"], d["uv"], dtype=dtype, magnitudes=magnitudes)


def ns_port(d):
    from oracle import reference_port_ns as rns
    return rns.NavierStokesIdentification(NS_NET, d["lb"], d["ub"], d["X"], d["uv"])


def _model(pde, inputs, feed, taylor, port, n_extra, part_idx, point_sets, targets, consts):
    return dict(pde=pde, inputs=inputs, feed=feed, taylor=taylor, port=port, n_extra=n_extra, part_idx=part_idx,
                point_sets=point_sets, targets=targets, consts=consts)


def _disc_model(kind):
    ide = kind in ("ide_disc", "kdv")
    pde = {"disc": "BURGERS_DISC", "ide_disc": "BURGERS_IDE_DISC", "kdv": "KDV_IDE_DISC", "ac": "AC_DISC"}[kind]
    consts = {"disc": [("nu", 0), ("dt", 0), ("IRK", (3, 2))], "ide_disc": [("dt", 0), ("alpha", (2, 5))],
              "kdv": [("dt", 0), ("alpha", (2, 5))], "ac": [("dt", 0), ("dk", 0), ("dk", 1), ("IRK", (3, 2))]}[kind]
    sets = [("x_0", "generic")] + ([("x_1", "generic")] if kind != "ac" else [])
    targets = [("u_0", (30, 0))] + ([("u_1", (20, 0))] if ide else [])
    return _model(pde, lambda: disc_inputs(kind), lambda c, p, d: disc_feed(p, d, c), disc_taylor, disc_port, 2 if ide else 0,
                  (0, 1), sets, targets, consts)


MODELS = {
    "burgers_inf": _model("BURGERS_INF", lambda: burgers_inputs(BURGERS, False), lambda c, p, d: burgers_feed(p, d),
                          burgers_taylor, burgers_port, 0, (0, 2), [("X_f", "burgers"), ("X_u", "burgers")], [("u", (20, 0))],
                          [("nu", 0)]),
    "burgers_ide": _model("BURGERS_IDE", lambda: burgers_inputs(BURGERS, True), lambda c, p, d: burgers_feed(p, d),
                          burgers_taylor, burgers_port, 2, (0, 2), [("X_u", "burgers")], [("u", (20, 0))], []),
    "nls": _model("NLS_INF", nls_inputs, lambda c, p, d: nls_feed(p, d), nls_taylor,
                  lambda d: rp.SchrodingerInference(NLS, d["lb"], d["ub"], d["X_f"], d["tb"], d["X0"], d["uv0"]), 0, (0, 1, 2),
                  [("X_f", "nls"), ("X0", "nls"), ("tb", "nls")], [("uv0", (5, 1))], []),
    "w33_inf": _model("BURGERS_INF", lambda: burgers_inputs(W33, False), lambda c, p, d: burgers_feed(p, d), burgers_taylor,
                      burgers_port, 0, (0, 2), [("X_f", "generic"), ("X_u", "generic")], [("u", (20, 0))], [("nu", 0)]),
    "w33_ide": _model("BURGERS_IDE", lambda: burgers_inputs(W33, True), lambda c, p, d: burgers_feed(p, d), burgers_taylor,
                      burgers_port, 2, (0, 2), [("X_u", "generic")], [("u", (20, 0))], []),
    "poly_inf": _model("POLY_INF", lambda: poly_inputs(False), lambda c, p, d: poly_feed(p, d), poly_taylor, poly_port, 0, (0, 2),
                       [("X_f", "generic"), ("X_u", "generic")], [("u", (20, 0))], [("source", 101)]),
    "poly_ide": _model("POLY_IDE", lambda: poly_inputs(True), lambda c, p, d: poly_feed(p, d), poly_taylor, poly_port, 2, (0, 2),
                       [("X_u", "generic")], [("u", (20, 0))], [("source", 101)]),
    "disc": _disc_model("disc"),
    "ide_disc": _disc_model("ide_disc"),
    "kdv": _disc_model("kdv"),
    "ac": _disc_model("ac"),
    "ns": _model("NS_IDE", ns_inputs, lambda c, p, d: p.set_data(d["X"], d["uv"]), ns_taylor, ns_port, 2, (0, 2),
                 [("X", "ns")], [("uv", (100, 1))], []),
}


def _units_per_cta(family, n, sms):
    if family == "burgers":
        return 8 * burgers_load(n, sms, "v2")["tiles per CTA"]
    if family == "nls":
        return nls_load(n, sms)["points per CTA"]
    if family == "ns":
        return ns_load(n, sms)["points per CTA"]
    return generic_load(n, sms)["points per CTA"]


def cases(name, sms):
    """(case name, field, index, value) of every injection into model `name`.  Point sets: NaN, +Inf and -Inf at the first point
    (column 0), inside the second CTA's range (column 1) and at the last point of the ragged set (the last column)."""
    m, d = MODELS[name], MODELS[name]["inputs"]()
    out = []
    for field, family in m["point_sets"]:
        n, ncol = d[field].shape
        mid = min(n - 2, (3 * _units_per_cta(family, n, sms)) // 2)
        for pos, tag, col in ((0, "first", 0), (mid, "mid", min(1, ncol - 1)), (n - 1, "last", ncol - 1)):
            for v in (NAN, INF, -INF):
                out.append(("%s[%s=%d,%d]=%s" % (field, tag, pos, col, v), field, (pos, col), v))
    for field, idx in m["targets"]:
        out.append(("%s%s=nan" % (field, list(idx)), field, idx, NAN))
    blocks = ty.param_blocks(d["layers"], m["n_extra"])
    dense = [b for b in blocks if b[0].startswith("W")]
    mid_l = len(dense) // 2
    sites = [("W0[0]", blocks[0][1].start), ("W%d[3]" % mid_l, dict(blocks)["W%d" % mid_l].start + 3),
             ("b%d[1]" % mid_l, dict(blocks)["b%d" % mid_l].start + 1), ("head[0]", dense[-1][1].start)]
    if m["n_extra"]:
        sites += [("lambda1", blocks[-2][1].start), ("lambda2", blocks[-1][1].start)]
    for tag, i in sites:
        for v in (NAN, INF, -INF):
            out.append(("w:%s=%s" % (tag, v), "w", (i,), v))
    for field, idx in m["consts"]:
        out.append(("%s[%s]=nan" % (field, idx), field, idx if isinstance(idx, tuple) else (idx,), NAN))
    return out


def inject(d, field, idx, value):
    d = dict(d)
    a = np.array(d[field])
    a[idx] = value
    d[field] = a
    return d


# Cases where the Taylor oracle (forward-mode streams) and the nested-autograd port (reverse mode, as TF runs the reference) put
# some values into different classes: the value depends on how a formula is written.  At those entries a kernel may return
# either oracle's class; everywhere else the rule is unchanged.  tests/test_nonfinite_cpu.py pins that this list is complete.
_NS_HEAD_INF = ("the data part: forward-mode streams give u = psi_y = Inf * a_y, so the squared error is +Inf; reverse mode "
                "sends the Inf back through every hidden unit with both signs, and the sum over them is NaN")
FORMULA_DEPENDENT = {
    ("ns", "uv[100, 1]=nan"): "the pressure column of the head: its derivative does not involve the NaN target and is finite "
                              "in the streams; reverse mode differentiates u = psi_y through a product with the zero seed of the "
                              "p column, and 0 * NaN = NaN",
    ("ns", "w:head[0]=inf"): _NS_HEAD_INF,
    ("ns", "w:head[0]=-inf"): _NS_HEAD_INF,
}


def expected(name, case):
    """The fp64 Taylor oracle on the injected inputs."""
    m = MODELS[name]
    with np.errstate(all="ignore"):
        return m["taylor"](inject(m["inputs"](), *case[1:]))


def port_result(name, d):
    """Loss, flat gradient and parts of the nested-autograd port."""
    import torch
    prob = MODELS[name]["port"](d)
    wt = torch.as_tensor(np.asarray(d["w"], dtype=np.float64)).clone().requires_grad_(True)
    parts = prob.loss_parts(wt)
    loss = sum(parts[1:], parts[0])
    (g,) = torch.autograd.grad(loss, wt)
    return float(loss.detach()), g.numpy().copy(), tuple(float(p.detach()) for p in parts)


def flat(r):
    """[loss, parts..., gradient] of an oracle result."""
    return np.concatenate([[r[0]], np.asarray(r[2], np.float64), np.asarray(r[1], np.float64)])


# -------------------------------------------------------------------------------------------------------------- the matrix
# (worker env, models); every run also reports which kernel each handle ran
RUNS = {
    "burgers_v2": ({"PINN_BURGERS_KERNEL": "v2"}, ["burgers_inf", "burgers_ide"]),
    "burgers_v2_no_tail": ({"PINN_BURGERS_KERNEL": "v2", "PINN_FUSED_TAIL": "0"}, ["burgers_inf", "burgers_ide"]),
    "burgers_v1": ({"PINN_BURGERS_KERNEL": "v1"}, ["burgers_inf", "burgers_ide"]),
    "nls_and_ns": ({}, ["nls", "ns"]),
    "forced_generic": ({"PINN_FORCE_GENERIC": "1"}, ["burgers_inf", "burgers_ide", "nls"]),
    "generic_dmma": ({"PINN_GENERIC_DFMA": "0"}, ["w33_inf", "w33_ide", "poly_inf", "poly_ide", "disc", "ide_disc", "kdv", "ac"]),
    "generic_dfma": ({"PINN_GENERIC_DFMA": "1"}, ["w33_inf", "w33_ide", "poly_inf", "poly_ide", "disc", "ide_disc", "kdv", "ac"]),
}
MATRIX = [(run, name) for run, (_, names) in RUNS.items() for name in names]


def run_worker(func, env, *args):
    """func(*args) of this module in a fresh interpreter with env set; it prints one JSON line."""
    code = "import sys, json; sys.path[:0] = [%r, %r]; import test_gpu_nonfinite as m; m.%s(*json.loads(sys.argv[1]))" % (
        ROOT, TESTS, func)
    r = subprocess.run([sys.executable, "-c", code, json.dumps(list(args))], env=dict(os.environ, **env), capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _cabi():
    import pinn_cabi
    pinn_cabi.load()
    return pinn_cabi


def _sms(c):
    p = c.Pinn(c.BURGERS_INF, BURGERS, [-1, 0], [1, 1])
    s = p.kernel_info()["sms"]
    p.close()
    return s


def guarded(fn):
    """Run fn() and return its result, or the traceback of what went wrong (one failing case must not hide the others)."""
    try:
        return fn()
    except Exception:
        return {"error": traceback.format_exc()[-2500:]}


def _res(r):
    return [r[0], r[1].tolist(), r[2].tolist()]


def _same(a, b):
    """Bitwise equality of two loss_grad results (NaN payloads included)."""
    return all(np.array_equal(np.asarray(x, np.float64).view(np.int64), np.asarray(y, np.float64).view(np.int64))
               for x, y in zip(a, b))


def make_handle(c, name, d):
    m = MODELS[name]
    p = c.Pinn(getattr(c, m["pde"]), d["layers"], d["lb"], d["ub"])
    if name.startswith("poly"):
        p.set_residual(TERMS[d["ide"]])
    m["feed"](c, p, d)
    return p


def matrix_worker(run):
    c = _cabi()
    sms = _sms(c)
    out = {"sms": sms}
    for name in RUNS[run][1]:
        def one(name=name):
            m, d = MODELS[name], MODELS[name]["inputs"]()
            p = make_handle(c, name, d)
            clean = p.loss_grad(w=d["w"])
            res = {"kernel": p.kernel_info(), "cases": {}, "poisoned": []}
            for case in cases(name, sms):
                di = inject(d, *case[1:])
                if case[1] != "w":
                    m["feed"](c, p, di)
                res["cases"][case[0]] = _res(p.loss_grad(w=di["w"]))
                if case[1] != "w":
                    m["feed"](c, p, d)
                if not _same(p.loss_grad(w=d["w"]), clean):
                    res["poisoned"].append(case[0])
            p.close()
            return res
        out[name] = guarded(one)
    if run.startswith("generic"):
        # the gradient of a [2, 128, 128, 1] net on 2000 points: its bits differ between the DMMA and the DFMA form (another
        # summation order), which shows that the switch took effect
        lb, ub = STD
        p = c.Pinn(c.BURGERS_INF, [2, 128, 128, 1], lb, ub)
        X = points(np.random.default_rng(90), lb, ub, 2000)
        p.set_pde_params([1.0]); p.set_collocation(X[:, 0], X[:, 1]); p.set_data(X[:50], np.zeros((50, 1)))
        out["form_probe"] = p.loss_grad(w=_w([2, 128, 128, 1], 91))[1].tolist()
        p.close()
    print(json.dumps(out))


@pytest.fixture(scope="module")
def matrix_runs():
    return {run: run_worker("matrix_worker", env, run) for run, (env, _) in RUNS.items()}


_LD_CACHE = {}


def finite_blocks_check(tag, name, case, got):
    """check() of test_gpu_precision on the blocks (and loss, parts) the fp64 oracle leaves entirely finite."""
    m = MODELS[name]
    d = inject(m["inputs"](), *case[1:])
    with np.errstate(all="ignore"):
        ref64 = m["taylor"](d)
        blocks = [(b, sl) for b, sl in ty.param_blocks(d["layers"], m["n_extra"]) if np.all(np.isfinite(ref64[1][sl]))]
        if not blocks:
            return 0.0
        key = (name, case[0])
        if key not in _LD_CACHE:
            _LD_CACHE[key] = m["taylor"](d, LD, True)
        ref = _LD_CACHE[key]
    loss, grad, parts = got
    # a non-finite loss or part is held by the class rule; the bound applies to the finite ones
    fin = lambda v: float(v) if np.isfinite(float(ref64[0])) else 0.0
    l_got, l_ld, l_64 = (fin(v) for v in (loss, ref[0], ref64[0]))
    p_ld, p_64, p_got = list(ref[2]), list(ref64[2]), np.array(parts, dtype=np.float64)
    for i, k in enumerate(m["part_idx"]):
        if not np.isfinite(float(ref64[2][i])):
            p_ld[i], p_64[i], p_got[k] = 0.0, 0.0, 0.0
    return check(tag, (l_got, grad, p_got), (LD(l_ld), ref[1], tuple(p_ld), ref[3]), (l_64, ref64[1], tuple(p_64)), blocks,
                 m["part_idx"])


def class_mismatch(name, case, got):
    """None when the class of every entry of got = (loss, grad, parts[3]) equals the fp64 oracle's, else what differs.  At the
    entries where a FORMULA_DEPENDENT case's two oracles disagree, either oracle's class is accepted."""
    m = MODELS[name]
    loss, grad, parts = got[0], np.asarray(got[1], dtype=np.float64), np.asarray(got[2], dtype=np.float64)
    kern, orc = classes(np.concatenate([[loss], parts[list(m["part_idx"])], grad])), classes(flat(expected(name, case)))
    if (name, case[0]) in FORMULA_DEPENDENT and kern.shape == orc.shape:
        with np.errstate(all="ignore"):
            alt = classes(flat(port_result(name, inject(m["inputs"](), *case[1:]))))
        orc = np.where(kern == alt, alt, orc)
    if kern.shape != orc.shape or not np.array_equal(kern, orc):
        diff = np.flatnonzero(kern != orc)
        return "class: %d entries differ, first %s (kernel %s, oracle %s; index 0 = loss, then the parts, then the gradient)" % (
            diff.size, diff[:4].tolist(), kern[diff[:4]].tolist(), orc[diff[:4]].tolist())
    return None


def class_and_bound(tag, name, case, got):
    """The rule of the module docstring for one evaluation; returns a description of what is wrong, or None."""
    why = class_mismatch(name, case, got)
    if why:
        return why
    try:
        finite_blocks_check(tag, name, case, (got[0], np.asarray(got[1], np.float64), np.asarray(got[2], np.float64)))
    except AssertionError as e:
        return "bound: %s" % (e,)
    return None


@pytest.mark.parametrize("run,name", MATRIX, ids=["%s/%s" % rn for rn in MATRIX])
def test_injected_value_matches_the_oracle_class_and_bound(matrix_runs, run, name):
    res = matrix_runs[run][name]
    assert "error" not in res, res["error"]
    if run.startswith("burgers_v"):
        assert res["kernel"] != matrix_runs["forced_generic"]["burgers_inf"]["kernel"]     # a specialised kernel ran
    if run == "forced_generic" or run.startswith("generic"):
        assert res["kernel"]["dyn_smem"] == 0                                              # the generic kernel ran
    assert not res["poisoned"], ("restoring the finite input did not restore the result", res["poisoned"])
    bad = {}
    for case in cases(name, matrix_runs[run]["sms"]):
        why = class_and_bound("%s/%s/%s" % (run, name, case[0]), name, case, res["cases"][case[0]])
        if why:
            bad[case[0]] = why
    assert not bad, (len(bad), bad)


def test_specialised_kernels_report_their_kernel(matrix_runs):
    k = {run: matrix_runs[run]["burgers_inf"]["kernel"] for run in ("burgers_v2", "burgers_v1", "forced_generic")}
    assert k["burgers_v2"] != k["burgers_v1"] and k["burgers_v2"] != k["forced_generic"]
    assert matrix_runs["nls_and_ns"]["nls"]["kernel"]["dyn_smem"] > 0                      # the specialised Schrodinger kernel
    assert matrix_runs["forced_generic"]["nls"]["kernel"]["dyn_smem"] == 0
    ns, gen = matrix_runs["nls_and_ns"]["ns"]["kernel"], matrix_runs["forced_generic"]["burgers_inf"]["kernel"]
    assert (ns["regs"], ns["block"]) != (gen["regs"], gen["block"])                    # the Navier-Stokes kernel, not generic
    assert matrix_runs["generic_dmma"]["form_probe"] != matrix_runs["generic_dfma"]["form_probe"]   # two forms really ran


# ---------------------------------------------------------------------------------------------------- real loads, then smaller
def load_worker():
    """Burgers v2 at ~100k collocation points and Schrodinger at ~20k: NaN at the last point and at the first point of the
    second CTA's range.  Then, on the same handle, the base set (finite) again: bitwise equal to a fresh handle on it."""
    c = _cabi()
    sms = _sms(c)
    out = {"sms": sms}

    def burgers():
        d = MODELS["burgers_inf"]["inputs"]()
        n = 100003
        X = points(np.random.default_rng(60), d["lb"], d["ub"], n)
        boundary = 8 * burgers_load(n, sms, "v2")["tiles per CTA"]
        r = {"cta_boundary": boundary}
        for tag, pos in (("last", n - 1), ("boundary", boundary)):
            Xb = X.copy(); Xb[pos, 0] = NAN
            big = dict(d, X_f=Xb)
            p = make_handle(c, "burgers_inf", big)
            r[tag] = _res(p.loss_grad(w=d["w"]))
            burgers_feed(p, d)
            small = p.loss_grad(w=d["w"])
            q = make_handle(c, "burgers_inf", d)
            r[tag + "_then_small_same"] = _same(small, q.loss_grad(w=d["w"]))
            r["kernel"] = p.kernel_info()
            p.close(); q.close()
        return r

    def nls():
        d = MODELS["nls"]["inputs"]()
        n = 20150
        X = points(np.random.default_rng(61), d["lb"], d["ub"], n)
        boundary = nls_load(n, sms)["points per CTA"]
        r = {"cta_boundary": boundary}
        for tag, pos in (("last", n - 1), ("boundary", boundary)):
            Xb = X.copy(); Xb[pos, 1] = NAN
            p = make_handle(c, "nls", dict(d, X_f=Xb))
            r[tag] = _res(p.loss_grad(w=d["w"]))
            nls_feed(p, d)
            small = p.loss_grad(w=d["w"])
            q = make_handle(c, "nls", d)
            r[tag + "_then_small_same"] = _same(small, q.loss_grad(w=d["w"]))
            r["kernel"] = p.kernel_info()
            p.close(); q.close()
        return r
    out["burgers"] = guarded(burgers)
    out["nls"] = guarded(nls)
    print(json.dumps(out))


def test_nan_at_real_loads_and_a_smaller_set_afterwards():
    out = run_worker("load_worker", {"PINN_BURGERS_KERNEL": "v2"})
    for name in ("burgers", "nls"):
        res = out[name]
        assert "error" not in res, res["error"]
        assert res["kernel"]["dyn_smem"] > 0                                              # the specialised kernel
        assert res["cta_boundary"] >= 8
        for tag in ("last", "boundary"):
            loss, grad, parts = res[tag]
            # a NaN collocation coordinate reaches every block through the residual mean (the oracle on the small set shows the
            # same for the first, mid and last positions; tests/test_nonfinite_cpu.py pins it)
            assert np.isnan(loss) and np.all(np.isnan(grad)), (name, tag, loss, int(np.sum(np.isnan(grad))), len(grad))
            assert res[tag + "_then_small_same"], (name, tag)


# ------------------------------------------------------------------------------------------------------------------ the probes
def probe_rule(got, ref, ref64, tol):
    """Classes equal elementwise; the finite rows of each column within tol (the rule of test_gpu_precision's probe test)."""
    got, ref64 = np.asarray(got, np.float64).reshape(len(got), -1), np.asarray(ref64, np.float64).reshape(len(got), -1)
    ref = np.asarray(ref).reshape(len(got), -1)
    if not np.array_equal(classes(got), classes(np.asarray(ref, np.float64))):
        return "class: %d entries differ" % int(np.sum(classes(got) != classes(np.asarray(ref, np.float64))))
    rows = np.all(np.isfinite(np.asarray(ref, np.float64)), axis=1)
    for o in range(ref.shape[1]):
        g, r, r64 = got[rows, o], ref[rows, o], ref64[rows, o]
        if not _ratio(_norm(g - r), tol * _norm(r) + FP64_FACTOR * _norm(r64 - r)) <= 1.0:
            return "bound in column %d" % o
    return None


PROBE_MODELS = ("burgers_inf", "nls", "disc", "poly_inf")


def probe_worker():
    c = _cabi()
    out = {}
    for name in PROBE_MODELS:
        def one(name=name):
            d = MODELS[name]["inputs"]()
            X = np.array(d["X_f"] if "X_f" in d else d["x_0"])
            X[0, 0], X[5, -1], X[9, 0], X[-1, 0] = NAN, INF, -INF, NAN
            res = {}
            for tag, w in (("points", d["w"]), ("nan_weight", inject(d, "w", (7,), NAN)["w"])):
                p = make_handle(c, name, d)
                p.set_weights(w)
                res[tag] = [X.tolist(), p.predict(X).tolist(), [s.tolist() for s in p.derivatives(X)]]
                p.close()
            if name in ("burgers_inf", "poly_inf"):           # residual() on stored points, one of them NaN
                di = inject(d, "X_f", (4, 1), NAN)
                p = make_handle(c, name, di)
                p.set_weights(d["w"])
                res["residual"] = p.residual().tolist()
                p.close()
            return res
        out[name] = guarded(one)

    def ns():
        d = MODELS["ns"]["inputs"]()
        layers = [3, 256, 256, 2]
        w = np.concatenate([_w(layers, 70), [0.6, 0.05]])
        n = ns_probe_chunks(11000, 256)["chunk"] + 77
        X = d["lb"] + (d["ub"] - d["lb"]) * np.random.default_rng(71).random((n, 3))
        X[3, 0], X[n - 40, 1], X[n - 30, 2] = NAN, INF, -INF
        p = c.Pinn(c.NS_IDE, layers, d["lb"], d["ub"])
        p.set_weights(w)
        r = {"n": n, "derivatives": p.derivatives(X).tolist(), "predict": p.predict(X).tolist()}
        p.close()
        return r
    out["ns"] = guarded(ns)
    print(json.dumps(out))


def test_probes_on_non_finite_points_and_weights():
    out = run_worker("probe_worker", {})
    bad = []
    for name in PROBE_MODELS:
        res = out[name]
        assert "error" not in res, res["error"]
        d = MODELS[name]["inputs"]()
        for tag in ("points", "nan_weight"):
            X, pred, streams = np.array(res[tag][0]), np.array(res[tag][1]), res[tag][2]
            w = d["w"] if tag == "points" else inject(d, "w", (7,), NAN)["w"]
            wn = w[:rp.num_params(d["layers"])]
            with np.errstate(all="ignore"):
                ref, _ = ty.forward(wn, d["layers"], d["lb"], d["ub"], X, dtype=LD)
                ref64, _ = ty.forward(wn, d["layers"], d["lb"], d["ub"], X)
            for s, tol in enumerate(PROBE_TOL):
                if d["layers"][0] == 1 and s == 2:
                    continue                                  # 1-D nets have no t stream
                why = probe_rule(streams[s], ref[s], ref64[s], tol)
                if why:
                    bad.append((name, tag, "stream %d" % s, why))
            why = probe_rule(pred, ref[0], ref64[0], PROBE_TOL[0])
            if why:
                bad.append((name, tag, "predict", why))
        if "residual" in res:
            di = inject(d, "X_f", (4, 1), NAN)
            with np.errstate(all="ignore"):
                if name == "poly_inf":
                    ref = tpo.poly_residual(d["w"], W33, d["lb"], d["ub"], TERMS[False], di["X_f"], source=d["source"], dtype=LD)
                    ref64 = tpo.poly_residual(d["w"], W33, d["lb"], d["ub"], TERMS[False], di["X_f"], source=d["source"])
                else:
                    (U, Ux, Ut, Uxx), _ = ty.forward(d["w"], BURGERS, d["lb"], d["ub"], di["X_f"], dtype=LD)
                    ref = Ut + U * Ux - LD(NU0) * Uxx
                    (U, Ux, Ut, Uxx), _ = ty.forward(d["w"], BURGERS, d["lb"], d["ub"], di["X_f"])
                    ref64 = Ut + U * Ux - NU0 * Uxx
            why = probe_rule(res["residual"], ref, ref64, PROBE_TOL[3])
            if why:
                bad.append((name, "residual", why))
    res = out["ns"]
    assert "error" not in res, res["error"]
    assert ns_probe_chunks(res["n"], 256)["chunks"] >= 2
    d = MODELS["ns"]["inputs"]()
    layers = [3, 256, 256, 2]
    w = np.concatenate([_w(layers, 70), [0.6, 0.05]])[:-2]
    X = d["lb"] + (d["ub"] - d["lb"]) * np.random.default_rng(71).random((res["n"], 3))
    n = res["n"]
    X[3, 0], X[n - 40, 1], X[n - 30, 2] = NAN, INF, -INF
    got = np.array(res["derivatives"])
    # every row's class from the fp64 oracle; the longdouble bound on rows around the injected ones (rows are independent)
    with np.errstate(all="ignore"):
        O64, _ = tn.forward_ns(w, layers, d["lb"], d["ub"], X)
    ref64 = np.stack([np.asarray(o, np.float64).reshape(n, -1) for o in O64], 1)
    if not np.array_equal(classes(got), classes(ref64)):
        bad.append(("ns", "class", int(np.sum(classes(got) != classes(ref64)))))
    if not np.array_equal(classes(np.array(res["predict"])), classes(ref64[:, 0, :])):          # (psi, p)
        bad.append(("ns", "predict class"))
    rows = np.r_[0:8, n - 45:n]
    with np.errstate(all="ignore"):
        O, _ = tn.forward_ns(w, layers, d["lb"], d["ub"], X[rows], dtype=LD)
    for k in range(13):
        why = probe_rule(got[rows, k], np.asarray(O[k]).reshape(len(rows), -1), ref64[rows, k], 1e-12)
        if why:
            bad.append(("ns", "stream %d" % k, why))
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------- Adam
def adam_worker():
    """One Adam step after an evaluation with a NaN collocation coordinate and after one with a +Inf data coordinate; then
    adam_reset, the finite points and the first weights again: one step bitwise equal to a fresh handle's."""
    c = _cabi()
    out = {}
    d = MODELS["burgers_inf"]["inputs"]()
    for tag, case in (("nan_point", ("", "X_f", (7, 0), NAN)), ("inf_data", ("", "X_u", (3, 1), INF)),
                      ("nan_weight", ("", "w", (100,), NAN))):
        def one(case=case):
            di = inject(d, *case[1:])
            p = make_handle(c, "burgers_inf", di)
            p.set_weights(di["w"])
            p.adam_reset()
            f, g, _ = p.loss_grad()
            loss = p.adam_step(1e-3)
            r = {"w_t": di["w"].tolist(), "f": f, "g": g.tolist(), "loss": loss, "last": p.last_loss(),
                 "w_next": p.get_weights().tolist()}
            p.adam_reset(); burgers_feed(p, d); p.set_weights(d["w"])
            p.adam_step(1e-3)
            q = make_handle(c, "burgers_inf", d)
            q.set_weights(d["w"])
            q.adam_step(1e-3)
            r["restored_same"] = bool(np.array_equal(p.get_weights(), q.get_weights()) and p.last_loss() == q.last_loss())
            p.close(); q.close()
            return r
        out[tag] = guarded(one)
    print(json.dumps(out))


def test_adam_step_after_a_non_finite_evaluation():
    from test_gpu_optimizer_replay import AdamReplay
    out = run_worker("adam_worker", {})
    for tag, res in out.items():
        assert "error" not in res, res["error"]
        w_t, g, w_next = (np.array(res[k]) for k in ("w_t", "g", "w_next"))
        same = lambda a, b: a == b or (np.isnan(a) and np.isnan(b))
        assert same(res["loss"], res["f"]) and same(res["last"], res["f"]), (tag, res["loss"], res["last"], res["f"])
        rep = AdamReplay(w_t.size, 1e-3)
        with np.errstate(all="ignore"):
            w_64 = rp.adam_update(w_t, g, rp.adam_init(w_t.size), 1e-3)
        assert np.array_equal(classes(w_next), classes(w_64)), (tag, int(np.sum(classes(w_next) != classes(w_64))))
        fin = np.isfinite(w_64)
        if fin.any():
            with np.errstate(all="ignore"):
                worst, idx = rep.check(np.where(fin, w_t, 0.0), np.where(fin, g, 0.0), np.where(fin, w_next, 0.0))
            assert not idx, (tag, worst, idx[:8])
        assert res["restored_same"], tag


# -------------------------------------------------------------------------------------------------------------------- L-BFGS
def nonfinite_objective(kind, at, where):
    """A quadratic on 40 entries whose f ('f'), g ('g') or both become `kind` (nan, inf, -inf) at evaluation `at`; 'g' puts the
    value into three entries."""
    lam = np.logspace(0.0, 2.0, 40)
    state = {"n": 0}

    def op(x):
        f, g = 0.5 * float(np.sum(lam * x * x)), lam * x
        if state["n"] == at:
            v = float(kind)
            if where in ("f", "both"):
                f = v
            if where in ("g", "both"):
                g = g.copy(); g[[0, 17, 39]] = v
        state["n"] += 1
        return f, g
    return op


LBFGS_OBJECTIVES = [("%s_%s_at%d" % (k, wh, at), k, at, wh) for k in ("nan", "inf", "-inf") for at in (0, 1, 4)
                    for wh in ("f", "g", "both")]
LBFGS_X0 = np.random.default_rng(80).standard_normal(40)
LBFGS_KW = dict(max_iter=12, lr=0.5, n_corr=5, tol_fun=1e-30)


def same_nan(a, b):
    """NaN-aware equality of nested lists / tuples of floats and ints."""
    if isinstance(a, (list, tuple)) or isinstance(b, (list, tuple)):
        return len(a) == len(b) and all(same_nan(x, y) for x, y in zip(a, b))
    return a == b or (isinstance(a, float) and isinstance(b, float) and np.isnan(a) and np.isnan(b))


def port_trace(fs, gs, x0, max_iter, lr, n_corr, tol_fun, direction="literal"):
    op = rp.ScriptedOpfunc(fs, gs)
    with np.errstate(all="ignore"):
        tr = rp.lbfgs_fixed_step(op, x0, max_iter=max_iter, learning_rate=lr, n_correction=n_corr, tol_fun=tol_fun,
                                 direction=direction)
    op.assert_consumed()
    return tr


def lbfgs_worker(mode):
    from test_gpu_optimizer_replay import coupled_vs_foreign, drive_foreign
    c = _cabi()
    out = {}
    for name, k, at, wh in LBFGS_OBJECTIVES:
        def one(k=k, at=at, wh=wh):
            run = drive_foreign(c, nonfinite_objective(k, at, wh), LBFGS_X0, **LBFGS_KW)
            return {key: (np.array(v).tolist() if key in ("xs", "gs", "x_final") else v) for key, v in run.items()}
        out[name] = guarded(one)

    def coupled():
        """pinn_lbfgs on a model handle with a NaN weight == the foreign handle fed that handle's loss_grad; then the finite
        weights on the same handle == a fresh handle's run."""
        from test_gpu_optimizer_replay import make_handle as opt_handle
        p, w0 = opt_handle(c, "burgers")
        wn = w0.copy(); wn[100] = NAN
        kw = dict(learning_rate=0.8, n_correction=10, tol_fun=float(np.finfo(float).eps))
        p.set_weights(wn)
        r = p.lbfgs(6, want_x_final=True, **kw)
        run = drive_foreign(c, lambda x: p.loss_grad(x)[:2], wn, 6, lr=0.8, n_corr=10, tol_fun=kw["tol_fun"])
        same = (r["n_iter"] == run["n_iter"] and r["n_eval"] == run["n_eval"] and r["reason_str"] == run["reason"]
                and same_nan(r["f_hist"], run["f_hist"]) and same_nan(r["x_final"].tolist(), run["x_final"].tolist()))
        p.set_weights(w0)
        r2 = p.lbfgs(6, want_x_final=True, **kw)
        q, _ = opt_handle(c, "burgers")
        q.set_weights(w0)
        r3 = q.lbfgs(6, want_x_final=True, **kw)
        after = r2["f_hist"] == r3["f_hist"] and np.array_equal(r2["x_final"], r3["x_final"]) and r2["n_iter"] == r3["n_iter"]
        p.close(); q.close()
        return {"same": bool(same), "reason": r["reason_str"], "n_iter": r["n_iter"], "f_hist": r["f_hist"],
                "after_nan_same_as_fresh": bool(after)}
    out["coupled"] = guarded(coupled)
    print(json.dumps(out))


@pytest.fixture(scope="module")
def lbfgs_runs():
    return {mode: run_worker("lbfgs_worker", {"PINN_LBFGS": mode}, mode) for mode in ("serial", "gram")}


@pytest.mark.parametrize("mode", ["serial", "gram"])
def test_lbfgs_on_non_finite_evaluations_takes_the_reference_path(lbfgs_runs, mode):
    bad = {}
    for name, k, at, wh in LBFGS_OBJECTIVES:
        run = lbfgs_runs[mode][name]
        assert "error" not in run, run["error"]
        kw = dict(LBFGS_KW)
        tr = port_trace(run["fs"], [np.array(g) for g in run["gs"]], LBFGS_X0, kw.pop("max_iter"), **kw,
                        direction="gram" if mode == "gram" else "literal")
        got = (run["reason"], run["n_iter"], run["n_eval"], [tuple(v) for v in run["logged"]])
        want = (tr.stop_reason, tr.n_iter, tr.n_eval, tr.logged)
        if not same_nan(list(got[:3]), list(want[:3])) or not same_nan(got[3], want[3]):
            bad[name] = ("control flow", got, want)
            continue
        # the points asked for: classes equal, and the finite ones where the port puts them (to the replay's rounding)
        want_x = [x.tolist() for x in tr.x_eval]
        if len(run["xs"]) != len(want_x) or not all(np.array_equal(classes(a), classes(b)) for a, b in zip(run["xs"], want_x)):
            bad[name] = ("points", len(run["xs"]), len(want_x))
            continue
        for a, b in zip(run["xs"], want_x):
            a, b = np.array(a), np.array(b)
            f = np.isfinite(b)
            if not np.all(np.abs(a[f] - b[f]) <= 1e-12 * (1 + np.abs(b[f]))):
                bad[name] = ("point value", float(np.max(np.abs(a[f] - b[f]))))
                break
        if not same_nan(run["f_hist"], run["fs"]):
            bad[name] = ("f_hist", run["f_hist"][:4], run["fs"][:4])
    assert not bad, bad


@pytest.mark.parametrize("mode", ["serial", "gram"])
def test_pinn_lbfgs_with_a_nan_weight_equals_the_foreign_handle(lbfgs_runs, mode):
    res = lbfgs_runs[mode]["coupled"]
    assert "error" not in res, res["error"]
    assert res["same"], res
    assert res["after_nan_same_as_fresh"], res
    assert np.isnan(res["f_hist"][0])


# ------------------------------------------------------------------------------------------------------- zero-copy collocation
def zero_copy_worker():
    import ctypes as C
    c = _cabi()
    d = MODELS["burgers_inf"]["inputs"]()
    n = d["X_f"].shape[0]
    hx, hx_ptr = c.host_alloc(n); ht, ht_ptr = c.host_alloc(n)
    dp = C.POINTER(C.c_double)
    hx[:] = d["X_f"][:, 0]; ht[:] = d["X_f"][:, 1]
    p = make_handle(c, "burgers_inf", d)
    p.set_collocation_mapped(C.cast(hx_ptr, dp), C.cast(ht_ptr, dp), n)
    before = p.loss_grad(w=d["w"])
    hx[n - 1] = NAN                                    # written in place into the pinned batch
    mapped_nan = p.loss_grad(w=d["w"])
    q = make_handle(c, "burgers_inf", inject(d, "X_f", (n - 1, 0), NAN))
    copied_nan = q.loss_grad(w=d["w"])
    hx[n - 1] = d["X_f"][n - 1, 0]
    after = p.loss_grad(w=d["w"])
    p.close(); q.close()
    print(json.dumps({"mapped_nan": _res(mapped_nan), "copied_nan": _res(copied_nan), "restored_same": _same(before, after)}))


def test_zero_copy_batch_with_a_nan_written_in_place():
    out = run_worker("zero_copy_worker", {})
    m, c = out["mapped_nan"], out["copied_nan"]
    assert np.isnan(m[0]) and np.array_equal(classes(m[1]), classes(c[1])) and np.array_equal(classes(m[2]), classes(c[2]))
    assert out["restored_same"]
