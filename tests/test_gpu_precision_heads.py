"""GPU: the KdV identification (pde 5), Allen-Cahn inference (pde 6) and polynomial residual (pde 8, 9) heads of the generic
fused kernel against their extended-precision Taylor oracles, block by block, in the DMMA and the DFMA form; and the per-stream
probes of KdV (u_xxx), Navier-Stokes (13 streams) and the polynomial residual against longdouble.

The rule, the helpers and the tolerances are those of test_gpu_precision.py (see its docstring): every parameter block, lambda_1,
lambda_2, the loss and every loss part satisfy ||g_B - g*_B|| <= REL ||S_B|| + FP64_FACTOR ||g64_B - g*_B||.  The whole-vector
tests of test_gpu_kdv_ac.py and test_gpu_poly.py use domains with sc = 2 / (ub - lb) near 1 and small coefficients on the
highest derivative (d = 1e-4, e^{lambda_2} = e^{-3}), which hide the U_xx and U_xxx paths; here every non-unit domain is crossed
with an O(1) coefficient on the highest-order stream.  Each test prints the worst error/bound it saw (run with -s)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from oracle import taylor as ty, taylor_kdv_ac as tk, taylor_poly as tpo
from test_gpu_precision import FP64_FACTOR, LD, DOMAINS, PROBE_TOL, _cabi, _norm, _ratio, _rand_w, _sms, cached, check, points

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
DOMAINS_1D = {"std": (-1.0, 1.0), "shifted": (0.3, 3.7), "small": (0.0, 1e-2), "large": (-50.0, 50.0)}   # small: sc = 200


def run_worker(func, env):
    """func() of this module in a fresh interpreter with env set (PINN_GENERIC_DFMA is read once per process); it prints one
    JSON line."""
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_precision_heads as m; m.%s()" % (ROOT, TESTS, func)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def n_points(n, sms):
    """A count, or a total at the generic kernel's points-per-CTA switches: with C = 2 x SM count CTAs, pinn_api.cu gives each
    CTA ceil(n / C) points rounded up to a multiple of 16 from 16 on, and to an even count below that."""
    if isinstance(n, int):
        return n
    C = 2 * sms
    return {"2C": 2 * C, "16C-1": 16 * C - 1, "16C": 16 * C, "16C+1": 16 * C + 1, "16C-3": 16 * C - 3, "16C-2": 16 * C - 2,
            "2C-3": 2 * C - 3}[n]


def points_1d(rng, dom, n):
    """n points of the 1-D domain, the first ones on lb and ub exactly."""
    lb, ub = DOMAINS_1D[dom]
    return points(rng, [lb, lb], [ub, ub], n)[:, :1]


# ------------------------------------------------------------------------------------------------------ KdV identification
# (name, domain, (lambda_1, lambda_2), weight scale, q, hidden, n_0 + n_1).  Every value of every axis appears at least once;
# every non-unit domain is crossed with e^{lambda_2} = O(1), the coefficient of U_xxx.  A total is split into an odd n_0 and
# the rest; (1, 1) is one point per snapshot.
KDV_CASES = [
    ("std_upstream", "std", (0.0, -6.0), 1.0, 36, [50] * 4, (199, 201)),
    ("std_k1_w8_one_each", "std", (1.0, 0.0), 8.0, 1, [7], (1, 1)),
    ("shifted_k1_q512", "shifted", (1.0, 0.0), 1.0, 512, [50] * 4, (17, 9)),
    ("shifted_neg_w4_2C", "shifted", (-0.7, 1.0), 4.0, 36, [128, 128], "2C"),
    ("small_k1", "small", (1.0, 0.0), 1.0, 36, [50] * 4, (33, 31)),
    ("small_neg_w025_16Cm1", "small", (-0.7, 1.0), 0.25, 1, [7], "16C-1"),
    ("small_upstream_w4_q512", "small", (0.0, -6.0), 4.0, 512, [7], (5, 3)),
    ("large_k1_w8_16C", "large", (1.0, 0.0), 8.0, 36, [50] * 4, "16C"),
    ("large_neg_16Cp1", "large", (-0.7, 1.0), 1.0, 1, [256], "16C+1"),
    ("large_k1_w025_h256", "large", (1.0, 0.0), 0.25, 36, [256, 256], (1, 1)),
]


def kdv_inputs(case, sms):
    name, dom, lam, scale, q, hidden, n = case
    rng = np.random.default_rng(KDV_CASES.index(case) + 500)
    if isinstance(n, tuple):
        n0, n1 = n
    else:
        tot = n_points(n, sms)
        n0 = (tot // 2) | 1
        n1 = tot - n0
    layers = [1] + list(hidden) + [q]
    lb, ub = DOMAINS_1D[dom]
    x_0, x_1 = points_1d(rng, dom, n0), points_1d(rng, dom, n1)
    xi0, xi1 = (x_0 - lb) / (ub - lb), (x_1 - lb) / (ub - lb)
    return dict(layers=layers, lb=np.array([lb]), ub=np.array([ub]), w=np.concatenate([_rand_w(layers, 600 + q, scale), lam]),
                x_0=x_0, u_0=np.cos(np.pi * xi0), x_1=x_1, u_1=0.5 * np.cos(np.pi * xi1 + 0.3), dt=0.6,
                alpha=(rng.standard_normal((q, q)) / q).astype(np.float32), beta=(rng.standard_normal((1, q)) / q).astype(np.float32))


def kdv_oracle(d, dtype, magnitudes):
    return tk.kdv_ide_disc_loss_grad(d["w"], d["layers"], d["lb"], d["ub"], d["x_0"], d["u_0"], d["x_1"], d["u_1"], d["dt"],
                                     d["alpha"], d["beta"], dtype=dtype, magnitudes=magnitudes)


def kdv_handle(c, d):
    p = c.Pinn(c.KDV_IDE_DISC, d["layers"], d["lb"], d["ub"])
    p.set_pde_params([d["dt"]]); p.set_irk(c.irk_ide_disc(d["alpha"], d["beta"]))
    p.set_snapshot(0, d["x_0"], d["u_0"]); p.set_snapshot(1, d["x_1"], d["u_1"])
    return p


# ------------------------------------------------------------------------------------------------------ Allen-Cahn inference
# (name, domain, d, k, weight scale, q + 1, hidden, N_0).  The kernel's point block is [x_0 | pad to even | lb, ub]: odd N_0
# take the pad, and "2C-3", "16C-3", "16C-2", "16C-1" put n0p + 2 at 2C, 16C, 16C and 16C + 2 (the points-per-CTA switch).
# Every non-unit domain is crossed with d = 1, the coefficient of U_xx; the slope half of the periodic pair scales with sc.
AC_CASES = [
    ("std_upstream", "std", 1e-4, 5.0, 1.0, 101, [200] * 4, 200),
    ("std_d0_k0_w8_one_point", "std", 0.0, 0.0, 8.0, 2, [20, 20], 1),
    ("shifted_d1", "shifted", 1.0, 5.0, 1.0, 101, [50, 50], 37),
    ("shifted_d1_k0_w4_16Cm2", "shifted", 1.0, 0.0, 4.0, 2, [20, 20], "16C-2"),
    ("small_d1_q512", "small", 1.0, 5.0, 1.0, 512, [32, 32], 45),
    ("small_d1_w025_16Cm1", "small", 1.0, 0.0, 0.25, 2, [16, 16], "16C-1"),
    ("small_d1em4_w8_2Cm3", "small", 1e-4, 5.0, 8.0, 101, [20, 20], "2C-3"),
    ("large_d1_w4_16Cm3", "large", 1.0, 5.0, 4.0, 2, [64, 64], "16C-3"),
    ("large_d1_q512_one_point", "large", 1.0, 0.0, 1.0, 512, [256], 1),
    ("large_d0_even", "large", 0.0, 5.0, 0.25, 101, [256, 256], 64),
]


def ac_inputs(case, sms):
    name, dom, dd, k, scale, q1, hidden, n = case
    rng = np.random.default_rng(AC_CASES.index(case) + 700)
    layers = [1] + list(hidden) + [q1]
    lb, ub = DOMAINS_1D[dom]
    x_0 = points_1d(rng, dom, n_points(n, sms))
    xi = (x_0 - lb) / (ub - lb)
    return dict(layers=layers, lb=np.array([lb]), ub=np.array([ub]), w=_rand_w(layers, 800 + q1, scale), x_0=x_0,
                u_0=xi ** 2 * np.cos(np.pi * xi), dt=0.8, d=dd, k=k, irk=rng.standard_normal((q1, q1 - 1)) / (q1 - 1))


def ac_oracle(d, dtype, magnitudes):
    return tk.ac_disc_loss_grad(d["w"], d["layers"], d["lb"], d["ub"], d["x_0"], d["u_0"], d["dt"], d["irk"], d=d["d"], k=d["k"],
                                dtype=dtype, magnitudes=magnitudes)


def ac_handle(c, d):
    p = c.Pinn(c.AC_DISC, d["layers"], d["lb"], d["ub"])
    p.set_pde_params([d["dt"], d["d"], d["k"]]); p.set_irk(d["irk"]); p.set_data(d["x_0"], d["u_0"])
    return p


# --------------------------------------------------------------------------------------------------- polynomial residual head
# Every single-stream monomial alone (4 streams x exponents 1..3) on both ids, so each exercises exactly one pick_pow /
# pick_dpow select; u_t^3 and u_xx^3 on the small domain (sc = (200, 2000)).
MONO_DOMAIN = {(0, 1): "std", (0, 2): "shifted", (0, 3): "large", (1, 1): "shifted", (1, 2): "large", (1, 3): "small",
               (2, 1): "large", (2, 2): "std", (2, 3): "small", (3, 1): "small", (3, 2): "shifted", (3, 3): "small"}
STREAMS = ("u", "ux", "ut", "uxx")
FISHER = [(1.0, 0, (0, 0, 1, 0)), (-1.0, 4, (0, 0, 0, 1)), (-1.0, 1, (1, 0, 0, 0)), (1.0, 1, (2, 0, 0, 0))]
# (name, identification, domain, terms, (lambda_1, lambda_2), weight scale, n residual points, n data points, source, data weight)
POLY_CASES = [("%s_%s%d" % ("ide" if ide else "inf", STREAMS[j], e), ide, MONO_DOMAIN[j, e],
               [(1.0, 0, tuple(e if i == j else 0 for i in range(4)))], (0.0, 0.0), 1.0, 301 if ide else 400,
               301 if ide else 31, e == 2, 1.0) for j in range(4) for e in (1, 2, 3) for ide in (False, True)]
POLY_CASES += [
    ("inf_four_stream_product_src", False, "shifted", [(0.8, 0, (1, 1, 1, 1))], (0.0, 0.0), 1.0, 500, 40, True, 1.0),
    ("ide_four_stream_product_w4", True, "large", [(-0.6, 0, (1, 2, 1, 1))], (0.0, 0.0), 4.0, 257, 257, False, 1.0),
    ("ide_kind1_pos", True, "shifted", [(1.0, 1, (1, 1, 0, 0))], (0.8, 0.3), 1.0, 200, 200, False, 1.0),
    ("ide_kind1_neg_w025", True, "small", [(1.0, 1, (1, 1, 0, 0))], (-0.8, 0.3), 0.25, 1, 1, True, 1.0),
    ("ide_kind2_pos_src", True, "small", [(-1.0, 2, (0, 0, 0, 1))], (0.3, 0.9), 1.0, 200, 200, True, 1.0),
    ("ide_kind2_neg", True, "large", [(-1.0, 2, (0, 0, 0, 1))], (0.3, -0.9), 1.0, 99, 99, False, 1.0),
    ("ide_kind3_pos_w8", True, "std", [(0.5, 3, (2, 0, 0, 0))], (0.7, 0.0), 8.0, 200, 200, False, 1.0),
    ("ide_kind3_neg", True, "shifted", [(0.5, 3, (2, 0, 0, 0))], (-0.7, 0.0), 1.0, 64, 64, True, 1.0),
    ("ide_kind4_pos", True, "large", [(-1.0, 4, (0, 0, 0, 1))], (0.0, 0.6), 1.0, 200, 200, True, 1.0),
    ("ide_kind4_neg_w4", True, "small", [(-1.0, 4, (0, 0, 0, 1))], (0.0, -0.6), 4.0, 150, 150, False, 1.0),
    # Fisher-KPP with u near 1: -l1 u + l1 u^2 cancels in df/dl1
    ("ide_fisher_kpp_near_u1", True, "shifted", FISHER, (0.7, -1.5), 0.25, 300, 300, False, 1.0),
    ("inf_data_weight_src", False, "small", [(1.0, 0, (0, 0, 1, 0)), (-1.0, 0, (0, 0, 0, 1)), (0.3, 0, (3, 0, 0, 0))],
     (0.0, 0.0), 1.0, 700, 60, True, 3.5),
    ("inf_data_weight_no_src_w025", False, "large", [(1.0, 0, (0, 0, 1, 0)), (1.0, 0, (1, 1, 0, 0)), (-1.0, 0, (0, 0, 0, 1))],
     (0.0, 0.0), 0.25, 333, 1, False, 0.2),
]
POLY_NET = [2, 20, 20, 20, 1]


def poly_inputs(case):
    name, ide, dom, terms, lam, scale, n_res, n_data, src, dw = case
    rng = np.random.default_rng(POLY_CASES.index(case) + 900)
    lb, ub = (np.array(v) for v in DOMAINS[dom])
    w = _rand_w(POLY_NET, 950 + len(terms), scale)
    if name.startswith("ide_fisher"):
        w[-1] += 1.0                                            # the output bias: u = 1 + O(0.25)
    X_u = points(rng, lb, ub, n_data)
    u = rng.uniform(-1, 1, (n_data, 1))
    X_f = None if ide else points(rng, lb, ub, n_res)
    return dict(ide=ide, lb=lb, ub=ub, terms=terms, w=np.concatenate([w, lam]) if ide else w, X_u=X_u, u=u, X_f=X_f,
                source=rng.standard_normal(n_res) if src else None, dw=dw)


def poly_oracle(d, dtype, magnitudes):
    return tpo.poly_loss_grad(d["w"], POLY_NET, d["lb"], d["ub"], d["terms"], d["X_u"], d["u"], X_f=d["X_f"], source=d["source"],
                              identification=d["ide"], data_weight=d["dw"], dtype=dtype, magnitudes=magnitudes)


def poly_handle(c, d):
    p = c.Pinn(c.POLY_IDE if d["ide"] else c.POLY_INF, POLY_NET, d["lb"], d["ub"])
    p.set_residual(d["terms"])
    p.set_data(d["X_u"], d["u"], weight=d["dw"])
    if not d["ide"]:
        p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1])
    if d["source"] is not None:
        p.set_source(d["source"])
    return p


# ------------------------------------------------------------------------------------------------------------- the two forms
HEADS = {"kdv": (KDV_CASES, kdv_inputs, kdv_oracle, kdv_handle),
         "ac": (AC_CASES, ac_inputs, ac_oracle, ac_handle),
         "poly": (POLY_CASES, lambda case, sms: poly_inputs(case), poly_oracle, poly_handle)}


def heads_worker():
    c, sms = _cabi(), _sms()
    out = {"sms": sms}
    for head, (cases, inputs, _, handle) in HEADS.items():
        for case in cases:
            d = inputs(case, sms)
            p = handle(c, d)
            assert p.kernel_info()["dyn_smem"] == 0                         # the generic kernel
            loss, grad, parts = p.loss_grad(w=d["w"])
            out[head + "/" + case[0]] = [loss, grad.tolist(), parts.tolist()]
            p.close()
    print(json.dumps(out))


@pytest.fixture(scope="module")
def runs():
    r = {form: run_worker("heads_worker", {"PINN_GENERIC_DFMA": flag}) for form, flag in (("dmma", "0"), ("dfma", "1"))}
    assert r["dmma"]["kdv/std_upstream"][1] != r["dfma"]["kdv/std_upstream"][1]   # two different summation orders actually ran
    return r


def _check_head(runs, form, head, case):
    cases, inputs, oracle, _ = HEADS[head]
    run = runs[form]
    d = inputs(case, run["sms"])
    ref = cached(head + "/" + case[0], lambda: (oracle(d, LD, True), oracle(d, np.float64, False)))
    loss, grad, parts = run[head + "/" + case[0]]
    ide = head == "kdv" or (head == "poly" and d["ide"])
    part_idx, zero = ((0, 2), 1) if head == "poly" else ((0, 1), 2)
    check("%s/%s/%s" % (form, head, case[0]), (loss, np.array(grad), np.array(parts)), ref[0], ref[1],
          ty.param_blocks(d["layers"] if head != "poly" else POLY_NET, 2 if ide else 0), part_idx)
    assert parts[zero] == 0.0


@pytest.mark.parametrize("form", ["dmma", "dfma"])
@pytest.mark.parametrize("case", KDV_CASES, ids=[c[0] for c in KDV_CASES])
def test_kdv_head_per_block(runs, form, case):
    _check_head(runs, form, "kdv", case)


@pytest.mark.parametrize("form", ["dmma", "dfma"])
@pytest.mark.parametrize("case", AC_CASES, ids=[c[0] for c in AC_CASES])
def test_ac_head_per_block(runs, form, case):
    _check_head(runs, form, "ac", case)


@pytest.mark.parametrize("form", ["dmma", "dfma"])
@pytest.mark.parametrize("case", POLY_CASES, ids=[c[0] for c in POLY_CASES])
def test_poly_head_per_block(runs, form, case):
    _check_head(runs, form, "poly", case)


# ------------------------------------------------------------------------------------------------------------------- probes
def _stream_ratio(got, ref, ref64, tol):
    return _ratio(_norm(got - ref), tol * _norm(ref) + FP64_FACTOR * _norm(ref64 - ref))


# KdV handles' pinn_derivatives: (u, u_x, u_xxx, u_xx).  u_xxx is held to u_xx's 1e-12.
KDV_PROBE_TOL = (PROBE_TOL[0], PROBE_TOL[1], 1e-12, PROBE_TOL[3])


@pytest.mark.parametrize("dom", ["std", "small", "large"])
def test_kdv_probes_per_stream(dom):
    c = _cabi()
    rng = np.random.default_rng(1000 + len(dom))
    layers = [1, 50, 50, 50, 8]
    lb, ub = (np.array([v]) for v in DOMAINS_1D[dom])
    X = points_1d(rng, dom, 200)
    w = np.concatenate([_rand_w(layers, 11, 4.0), [0.3, -1.0]])
    p = c.Pinn(c.KDV_IDE_DISC, layers, lb, ub)
    p.set_weights(w)
    got, pred = p.derivatives(X), p.predict(X)
    p.close()
    ref, _ = tk.forward_third(w[:-2], layers, lb, ub, X, dtype=LD)
    ref64, _ = tk.forward_third(w[:-2], layers, lb, ub, X)
    worst = 0.0
    for s, sname in enumerate(("u", "u_x", "u_xxx", "u_xx")):
        for o in range(layers[-1]):
            r = _stream_ratio(got[s][:, o], ref[s][:, o], ref64[s][:, o], KDV_PROBE_TOL[s])
            worst = max(worst, r)
            assert r <= 1.0, (dom, sname, o, _norm(got[s][:, o] - ref[s][:, o]) / _norm(ref[s][:, o]))
    r = _stream_ratio(pred, ref[0], ref64[0], PROBE_TOL[0])
    assert r <= 1.0, (dom, "predict")
    print("[precision] %-40s worst error/bound %.3g" % ("probes/kdv_" + dom, max(worst, r)))


# Navier-Stokes probe streams (oracle.taylor_ns.STREAMS): derivative order 0, 1 -> 1e-13, 2 and 3 -> 1e-12
NS_LB, NS_UB = np.array([0.0, 0.0, 0.0]), np.array([1e-2, 2e-2, 1e-3])


def test_ns_probes_per_stream_on_the_small_box():
    from oracle import taylor_ns as tn
    c = _cabi()
    rng = np.random.default_rng(1100)
    layers = [3, 20, 20, 20, 2]
    X = NS_LB + (NS_UB - NS_LB) * rng.random((200, 3))
    X[:8] = np.array([[(NS_LB, NS_UB)[(i >> b) & 1][b] for b in range(3)] for i in range(8)])    # the 8 corners
    w = np.concatenate([_rand_w(layers, 12), [0.6, 0.05]])
    p = c.Pinn(c.NS_IDE, layers, NS_LB, NS_UB)
    p.set_weights(w)
    got = p.derivatives(X)
    p.close()
    ref, _ = tn.forward_ns(w[:-2], layers, NS_LB, NS_UB, X, dtype=LD)
    ref64, _ = tn.forward_ns(w[:-2], layers, NS_LB, NS_UB, X)
    worst = 0.0
    for k, m in enumerate(tn.STREAMS):
        tol = 1e-13 if sum(m) <= 1 else 1e-12
        for o in range(2):
            r = _stream_ratio(got[:, k, o], ref[k][:, o], ref64[k][:, o], tol)
            worst = max(worst, r)
            assert r <= 1.0, (k, m, o, _norm(got[:, k, o] - ref[k][:, o]) / _norm(ref[k][:, o]))
    print("[precision] %-40s worst error/bound %.3g" % ("probes/ns_small_box", worst))


# pinn_residual of the polynomial head: f on the host from the probe's streams (DESIGN 4.4d), cubic terms on the small domain
POLY_PROBE_TERMS = [(1.0, 0, (0, 0, 0, 3)), (-0.5, 3, (0, 0, 3, 0)), (0.7, 0, (3, 1, 0, 0)), (1.0, 2, (0, 1, 0, 1))]


@pytest.mark.parametrize("ide", [False, True])
def test_poly_residual_probe_with_cubic_terms(ide):
    c = _cabi()
    rng = np.random.default_rng(1200 + ide)
    lb, ub = (np.array(v) for v in DOMAINS["small"])
    X = points(rng, lb, ub, 300)
    terms = POLY_PROBE_TERMS if ide else [(a, 0, e) for a, _, e in POLY_PROBE_TERMS]
    w = _rand_w(POLY_NET, 13, 1.0)
    if ide:
        w = np.concatenate([w, [0.4, -0.3]])
    s = rng.standard_normal(300)
    p = c.Pinn(c.POLY_IDE if ide else c.POLY_INF, POLY_NET, lb, ub)
    p.set_residual(terms)
    if ide:
        p.set_data(X, np.zeros(300))
    else:
        p.set_data(X[:5], np.zeros(5)); p.set_collocation(X[:, 0], X[:, 1])
    p.set_source(s)
    p.set_weights(w)
    got = p.residual()
    p.close()
    ref = tpo.poly_residual(w, POLY_NET, lb, ub, terms, X, source=s, identification=ide, dtype=LD)
    ref64 = tpo.poly_residual(w, POLY_NET, lb, ub, terms, X, source=s, identification=ide)
    r = _stream_ratio(got, ref, ref64, PROBE_TOL[3])
    print("[precision] %-40s worst error/bound %.3g" % ("probes/poly_residual_" + ("ide" if ide else "inf"), r))
    assert r <= 1.0, _norm(got - ref) / _norm(ref)
