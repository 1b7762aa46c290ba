"""GPU: the fused kernels against an extended-precision (np.longdouble) restatement of the Taylor oracle, block by block.

Every other GPU test compares one relative L2 norm over the whole gradient with an fp64 code at 1e-10, on x in [-1, 1] (where
the input scale factor 2/(ub0 - lb0) is exactly 1) and with nu = 0.01/pi (which hides the u_xx path 300-fold).  Here:

* the reference is oracle.taylor in 64-bit-mantissa arithmetic (g*), and the fp64 oracle on the same inputs (g64) measures how
  well fp64 itself can do there;
* each parameter block B (W_l, b_l, lambda_1, lambda_2), the loss and every loss part must satisfy
      ||g_B - g*_B|| <= REL * ||S_B|| + FP64_FACTOR * ||g64_B - g*_B||
  where S_B is the magnitude of the block's final contraction over the points (sum |H|^T |Z-bar|; for a loss, the loss itself):
  REL * ||S_B|| is the rounding of a sum over the points in another order, and the second term widens the bound only where fp64 is
  ill-conditioned (large weights saturate tanh and 1 - a^2 cancels);
* the domains include shifted, tiny and wide ones, points on lb / ub and the corners, nu (kappa) from 0 to O(1), and weights
  from 0.25x to 8x the initialisation scale.

Each test prints the worst ||g_B - g*_B|| / bound it saw (run with -s to read them).

Held per block here: the specialised Burgers kernels (v2, v1), the Schrodinger kernel, the generic kernel's continuous-time
Burgers heads and its discrete-time Burgers heads (pde 3, 4).  tests/test_gpu_precision_heads.py holds the generic kernel's
KdV (pde 5), Allen-Cahn (pde 6) and polynomial residual (pde 8, 9) heads to the same rule with these helpers, and
tests/test_gpu_ns.py the Navier-Stokes kernel.  tests/test_gpu_precision_load.py holds the specialised Burgers and Schrodinger
kernels, the generic kernel's Burgers and Schrodinger heads, the Navier-Stokes kernel and the probes at the per-CTA loads they
run at (up to 2M points), on shuffled copies of a base set.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, load_golden
from oracle import reference_port as rp, taylor as ty

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
LD = np.longdouble
REL, FP64_FACTOR = 1e-12, 32.0
NU0 = 0.01 / np.pi
BURGERS = [2] + [20] * 8 + [1]
NLS = [2, 100, 100, 100, 100, 2]
DOMAINS = {                                   # (lb, ub) of (x, t)
    "std": ([-1.0, 0.0], [1.0, 0.99]),
    "shifted": ([0.3, -0.5], [3.7, 2.0]),
    "small": ([0.0, 0.0], [1e-2, 1e-3]),      # sc = (200, 2000): u_xx is scaled by 4e4
    "large": ([-50.0, 0.0], [50.0, 10.0]),
}


# ---------------------------------------------------------------------------------------------------------------- comparison
def _norm(v):
    v = np.asarray(v, dtype=LD)
    return float(np.sqrt(np.sum(v * v)))


def _ratio(err, bound):
    return 0.0 if err == 0 else (err / bound if bound > 0 else np.inf)


def check(tag, got, ref, ref64, blocks, part_idx):
    """got = kernel (loss, grad, parts[3]); ref = longdouble (loss, grad, parts, magnitudes); ref64 = fp64 (loss, grad, parts).
    part_idx[i]: the kernel's parts slot holding the oracle's part i."""
    loss, grad, parts = got
    l_ld, g_ld, p_ld, mag = ref
    l_64, g_64, p_64 = ref64[:3]
    rows = []
    for name, sl in blocks:
        err = _norm(grad[sl] - g_ld[sl])
        rows.append((name, err, _ratio(err, REL * _norm(mag[sl]) + FP64_FACTOR * _norm(g_64[sl] - g_ld[sl]))))
    scalars = [("loss", loss, l_ld, l_64)] + [("part%d" % i, parts[k], p_ld[i], p_64[i]) for i, k in enumerate(part_idx)]
    for name, a, b, c in scalars:
        err = abs(float(LD(a) - b))
        rows.append((name, err, _ratio(err, REL * abs(float(b)) + FP64_FACTOR * abs(float(LD(c) - b)))))
    worst = max(rows, key=lambda r: r[2])
    print("[precision] %-40s worst error/bound %.3g (%s)" % (tag, worst[2], worst[0]))
    bad = [(n, "%.3g" % e, "%.3g" % r) for n, e, r in rows if not r <= 1.0]
    assert not bad, (tag, bad)
    return worst[2]


def points(rng, lb, ub, n):
    """n points in the box, the first ones on its corners and edges (x = lb0, ub0 and t = lb1, ub1 exactly)."""
    lb, ub = np.asarray(lb, float), np.asarray(ub, float)
    X = lb + (ub - lb) * rng.random((n, 2))
    mid = 0.5 * (lb + ub)
    edge = np.array([[lb[0], lb[1]], [ub[0], ub[1]], [lb[0], ub[1]], [ub[0], lb[1]],
                     [lb[0], mid[1]], [ub[0], mid[1]], [mid[0], lb[1]], [mid[0], ub[1]]])
    k = min(n, len(edge))
    X[:k] = edge[:k]
    return X


def run_worker(func, env):
    """Run func() of this module in a fresh interpreter with env set (the kernel switches are read once per process); it prints
    one JSON line."""
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_precision as m; m.%s()" % (ROOT, TESTS, func)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _cabi():
    import pinn_cabi
    pinn_cabi.load()
    return pinn_cabi


@pytest.fixture(scope="module")
def cabi():
    return _cabi()


def _sms():
    c = _cabi()
    p = c.Pinn(c.BURGERS_INF, BURGERS, [-1, 0], [1, 1])
    s = p.kernel_info()["sms"]
    p.close()
    return s


# ------------------------------------------------------------------------------------------------- specialised Burgers kernel
# (name, identification, domain, nu or (lambda_1, lambda_2), weight scale, n_f, n_u); identification evaluates on n_u points.
# Every value of every axis appears at least once; every non-unit domain is crossed with nu = 1 (kappa = e^0 = 1).
# "S" stands for 8 * (SM count) - 1: one point short of a full tile per SM.
BURGERS_CASES = [
    ("inf_std", False, "std", NU0, 1.0, 4736, 100),
    ("inf_std_nu0_w8", False, "std", 0.0, 8.0, 20000, 100),
    ("inf_std_data_only", False, "std", NU0, 0.25, 0, 100),
    ("inf_shifted_nu1", False, "shifted", 1.0, 1.0, 4736, 100),
    ("inf_shifted_nu1_w8_one_point", False, "shifted", 1.0, 8.0, 1, 1),
    ("inf_shifted_nu0_w4", False, "shifted", 0.0, 4.0, "S", 0),
    ("inf_small_nu1", False, "small", 1.0, 1.0, "S", 0),
    ("inf_small_nu1_w025", False, "small", 1.0, 0.25, 4736, 100),
    ("inf_small_nu0_data_only", False, "small", 0.0, 1.0, 0, 100),
    ("inf_large_nu1_w4", False, "large", 1.0, 4.0, 20000, 100),
    ("inf_large_nu1_one_point", False, "large", 1.0, 1.0, 1, 1),
    ("ide_std", True, "std", (1.0, -5.0), 1.0, 0, 2000),
    ("ide_std_neg_w025", True, "std", (-0.7, 1.0), 0.25, 0, 1),
    ("ide_shifted_k1_w4", True, "shifted", (0.0, 0.0), 4.0, 0, 4736),
    ("ide_small_k1", True, "small", (0.0, 0.0), 1.0, 0, "S"),
    ("ide_small_neg_w8", True, "small", (-0.7, 1.0), 8.0, 0, 100),
    ("ide_large_k1_w8", True, "large", (0.0, 0.0), 8.0, 0, 20000),
    ("ide_large_std_lambda", True, "large", (1.0, -5.0), 0.25, 0, 1),
]


def burgers_inputs(case, sms):
    name, ide, dom, pde, scale, n_f, n_u = case
    n_f = 8 * sms - 1 if n_f == "S" else n_f
    n_u = 8 * sms - 1 if n_u == "S" else n_u
    rng = np.random.default_rng(BURGERS_CASES.index(case) + 100)
    lb, ub = (np.array(v) for v in DOMAINS[dom])
    X_f, X_u = points(rng, lb, ub, n_f), points(rng, lb, ub, n_u)
    u = rng.uniform(-1, 1, (n_u, 1))
    w = scale * load_golden("burgers_inf")["w"]
    if ide:
        w = np.concatenate([w, pde])
    return dict(ide=ide, lb=lb, ub=ub, nu=None if ide else pde, X_f=X_f, X_u=X_u, u=u, w=w)


def burgers_oracle(d, dtype, magnitudes):
    """Taylor oracle on burgers_inputs(); an empty set contributes nothing (the oracle's means need >= 1 point)."""
    X_u, u, dw = d["X_u"], d["u"], 1.0
    if X_u.shape[0] == 0:
        X_u, u, dw = d["lb"][None, :], np.zeros((1, 1)), 0.0
    return ty.burgers_loss_grad(d["w"], BURGERS, d["lb"], d["ub"], d["X_f"], X_u, u, nu=d["nu"], identification=d["ide"],
                                n_f_global=None if d["ide"] else max(d["X_f"].shape[0], 1), data_weight=dw, dtype=dtype,
                                magnitudes=magnitudes)


def burgers_worker():
    c, sms = _cabi(), _sms()
    out = {"sms": sms}
    for case in BURGERS_CASES:
        d = burgers_inputs(case, sms)
        p = c.Pinn(c.BURGERS_IDE if d["ide"] else c.BURGERS_INF, BURGERS, d["lb"], d["ub"])
        if not d["ide"]:
            p.set_pde_params([d["nu"]])
            p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1])
        p.set_data(d["X_u"], d["u"])
        loss, grad, parts = p.loss_grad(w=d["w"])
        out[case[0]] = [loss, grad.tolist(), parts.tolist()]
        out["kernel"] = p.kernel_info()
        p.close()
    print(json.dumps(out))


@pytest.fixture(scope="module")
def burgers_runs():
    runs = {k: run_worker("burgers_worker", {"PINN_BURGERS_KERNEL": k}) for k in ("v2", "v1")}
    assert runs["v2"]["kernel"] != runs["v1"]["kernel"]          # two different kernels actually ran
    return runs


_ORACLE_CACHE = {}


def cached(key, fn):
    if key not in _ORACLE_CACHE:
        _ORACLE_CACHE[key] = fn()
    return _ORACLE_CACHE[key]


@pytest.mark.parametrize("kernel", ["v2", "v1"])
@pytest.mark.parametrize("case", BURGERS_CASES, ids=[c[0] for c in BURGERS_CASES])
def test_burgers_kernel_per_block(burgers_runs, kernel, case):
    run = burgers_runs[kernel]
    d = burgers_inputs(case, run["sms"])
    ref = cached(case[0], lambda: (burgers_oracle(d, LD, True), burgers_oracle(d, np.float64, False)))
    loss, grad, parts = run[case[0]]
    blocks = ty.param_blocks(BURGERS, 2 if d["ide"] else 0)
    check(kernel + "/" + case[0], (loss, np.array(grad), np.array(parts)), ref[0], ref[1], blocks, (0, 2))
    assert parts[1] == 0.0


# ---------------------------------------------------------------------------------------------------- Schrodinger kernel
# (name, domain (lb, ub), weight scale, n_f, n_0, n_b, Q1 initial-condition mode (x, x))
NLS_OWN = ([-5.0, 0.0], [5.0, np.pi / 2])
NLS_OTHER = ([-0.7, 0.25], [1.3, 0.5])
NLS_CASES = [
    ("own_q1", NLS_OWN, 1.0, 17, 50, 50, True),
    ("own_w3", NLS_OWN, 3.0, 1800, 50, 50, False),
    ("other_q1_w3", NLS_OTHER, 3.0, 15, 3, 2, True),
    ("other", NLS_OTHER, 1.0, 1800, 50, 50, False),
    ("other_one_point_each", NLS_OTHER, 1.0, 1, 1, 1, False),
]


@pytest.mark.parametrize("case", NLS_CASES, ids=[c[0] for c in NLS_CASES])
def test_schrodinger_kernel_per_block(cabi, case):
    name, (lb, ub), scale, n_f, n_0, n_b, q1 = case
    lb, ub = np.array(lb), np.array(ub)
    rng = np.random.default_rng(NLS_CASES.index(case) + 200)
    X_f = points(rng, lb, ub, n_f)
    tb = np.concatenate([[lb[1], ub[1]], rng.uniform(lb[1], ub[1], max(n_b - 2, 0))])[:n_b, None]
    x0 = np.concatenate([[lb[0], ub[0]], rng.uniform(lb[0], ub[0], max(n_0 - 2, 0))])[:n_0, None]
    X0 = x0 if q1 else np.concatenate([x0, 0 * x0 + lb[1]], 1)
    uv0 = rng.standard_normal((n_0, 2))
    w = scale * load_golden("nls_inf")["w"]
    p = cabi.Pinn(cabi.NLS_INF, NLS, lb, ub)
    assert p.kernel_info()["dyn_smem"] > 0                                  # the specialised kernel
    p.set_collocation(X_f[:, 0], X_f[:, 1]); p.set_boundary(tb); p.set_data(X0, uv0)
    got = p.loss_grad(w=w)
    p.close()
    args = (w, NLS, lb, ub, X_f, tb, X0, uv0)
    ref = ty.schrodinger_loss_grad(*args, dtype=LD, magnitudes=True)
    ref64 = ty.schrodinger_loss_grad(*args)
    check("nls/" + name, got, ref, ref64, ty.param_blocks(NLS), (0, 1, 2))


# ---------------------------------------------------------------------------- generic kernel: shape edges, discrete-time heads
def _rand_w(layers, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return scale * (rp.glorot_normal_flat(layers, rng) + 0.05 * rng.standard_normal(rp.num_params(layers)))


MAXL_NET = [2] + [12] * 14 + [1]                  # 15 Dense layers = 16 sizes, the most pinn_create accepts
# (name, pde, layers, domain, n_f, n_u): continuous-time nets on the shifted domain with nu = 1 (kappa = 1)
GENERIC_CASES = [
    ("width1", "inf", [2, 1, 1], "shifted", 300, 20),
    ("width1_ide", "ide", [2, 1, 1], "shifted", 0, 300),
    ("h128x128", "inf", [2, 128, 128, 1], "shifted", 2000, 50),
    ("maxl", "inf", MAXL_NET, "large", 700, 30),
    ("w8k_pm1", "inf", [2, 31, 33, 1], "small", 1000, 40),
    ("w8k_pm1_ide", "ide", [2, 15, 17, 9, 7, 1], "shifted", 0, 500),
]
# (name, identification, q): discrete-time heads on x in [0.3, 3.7]; q = 1 and the widest head (q + 1 = 512, or q = 512)
DISC_CASES = [("disc_q1", False, 1), ("disc_q511", False, 511), ("ide_disc_q1", True, 1), ("ide_disc_q512", True, 512)]
DISC_LB, DISC_UB = np.array([0.3]), np.array([3.7])


def generic_inputs(case):
    name, pde, layers, dom, n_f, n_u = case
    rng = np.random.default_rng(GENERIC_CASES.index(case) + 300)
    lb, ub = (np.array(v) for v in DOMAINS[dom])
    w = _rand_w(layers, GENERIC_CASES.index(case))
    if pde == "ide":
        w = np.concatenate([w, [0.3, 0.0]])
    return dict(ide=pde == "ide", layers=layers, lb=lb, ub=ub, X_f=points(rng, lb, ub, n_f), X_u=points(rng, lb, ub, n_u),
                u=rng.uniform(-1, 1, (n_u, 1)), w=w)


def disc_inputs(case):
    name, ide, q = case
    rng = np.random.default_rng(q + (1000 if ide else 0))
    layers = [1, 50, 50, q if ide else q + 1] if q > 1 else [1, 20, q if ide else q + 1]
    w = _rand_w(layers, q, 1.0)
    d = dict(ide=ide, q=q, layers=layers)
    x0 = np.concatenate([[DISC_LB[0], DISC_UB[0]], rng.uniform(DISC_LB[0], DISC_UB[0], 117)])[:, None]
    if ide:
        x1 = np.concatenate([[DISC_LB[0]], rng.uniform(DISC_LB[0], DISC_UB[0], 60)])[:, None]
        d.update(w=np.concatenate([w, [0.4, -1.0]]), dt=0.8, x_0=x0, u_0=np.sin(x0), x_1=x1, u_1=0.5 * np.cos(x1),
                 alpha=(rng.standard_normal((q, q)) / q).astype(np.float32), beta=(rng.standard_normal((1, q)) / q).astype(np.float32))
    else:
        d.update(w=w, nu=1.0, dt=0.3, x_0=x0, u_0=-np.sin(x0), x_1=np.array([[DISC_LB[0]], [DISC_UB[0]]]),
                 IRK=rng.standard_normal((q + 1, q)) / q)
    return d


def disc_oracle(d, dtype, magnitudes):
    lb, ub = DISC_LB, DISC_UB
    if d["ide"]:
        return ty.burgers_ide_disc_loss_grad(d["w"], d["layers"], lb, ub, d["x_0"], d["u_0"], d["x_1"], d["u_1"], d["dt"],
                                             d["alpha"], d["beta"], dtype=dtype, magnitudes=magnitudes)
    return ty.burgers_disc_loss_grad(d["w"], d["layers"], lb, ub, d["x_0"], d["u_0"], d["x_1"], d["nu"], d["dt"], d["IRK"],
                                     dtype=dtype, magnitudes=magnitudes)


def generic_oracle(d, dtype, magnitudes):
    return ty.burgers_loss_grad(d["w"], d["layers"], d["lb"], d["ub"], d["X_f"], d["X_u"], d["u"], nu=None if d["ide"] else 1.0,
                                identification=d["ide"], dtype=dtype, magnitudes=magnitudes)


def generic_worker():
    c = _cabi()
    out = {}
    for case in GENERIC_CASES:
        d = generic_inputs(case)
        p = c.Pinn(c.BURGERS_IDE if d["ide"] else c.BURGERS_INF, d["layers"], d["lb"], d["ub"])
        assert p.kernel_info()["dyn_smem"] == 0                             # the generic kernel
        if not d["ide"]:
            p.set_pde_params([1.0]); p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1])
        p.set_data(d["X_u"], d["u"])
        loss, grad, parts = p.loss_grad(w=d["w"])
        out[case[0]] = [loss, grad.tolist(), parts.tolist()]
        p.close()
    for case in DISC_CASES:
        d = disc_inputs(case)
        if d["ide"]:
            p = c.Pinn(c.BURGERS_IDE_DISC, d["layers"], DISC_LB, DISC_UB)
            p.set_pde_params([d["dt"]]); p.set_irk(c.irk_ide_disc(d["alpha"], d["beta"]))
            p.set_snapshot(0, d["x_0"], d["u_0"]); p.set_snapshot(1, d["x_1"], d["u_1"])
        else:
            p = c.Pinn(c.BURGERS_DISC, d["layers"], DISC_LB, DISC_UB)
            p.set_pde_params([d["nu"], d["dt"]]); p.set_irk(d["IRK"]); p.set_boundary(d["x_1"]); p.set_data(d["x_0"], d["u_0"])
        loss, grad, parts = p.loss_grad(w=d["w"])
        out[case[0]] = [loss, grad.tolist(), parts.tolist()]
        p.close()
    print(json.dumps(out))


@pytest.fixture(scope="module")
def generic_runs():
    runs = {form: run_worker("generic_worker", {"PINN_GENERIC_DFMA": flag}) for form, flag in (("dmma", "0"), ("dfma", "1"))}
    assert runs["dmma"]["h128x128"][1] != runs["dfma"]["h128x128"][1]      # two different summation orders actually ran
    return runs


@pytest.mark.parametrize("form", ["dmma", "dfma"])
@pytest.mark.parametrize("case", GENERIC_CASES, ids=[c[0] for c in GENERIC_CASES])
def test_generic_kernel_shape_edges_per_block(generic_runs, form, case):
    d = generic_inputs(case)
    ref = cached("generic/" + case[0], lambda: (generic_oracle(d, LD, True), generic_oracle(d, np.float64, False)))
    loss, grad, parts = generic_runs[form][case[0]]
    check(form + "/" + case[0], (loss, np.array(grad), np.array(parts)), ref[0], ref[1],
          ty.param_blocks(d["layers"], 2 if d["ide"] else 0), (0, 2))


@pytest.mark.parametrize("form", ["dmma", "dfma"])
@pytest.mark.parametrize("case", DISC_CASES, ids=[c[0] for c in DISC_CASES])
def test_discrete_time_heads_per_block(generic_runs, form, case):
    d = disc_inputs(case)
    ref = cached("disc/" + case[0], lambda: (disc_oracle(d, LD, True), disc_oracle(d, np.float64, False)))
    loss, grad, parts = generic_runs[form][case[0]]
    check(form + "/" + case[0], (loss, np.array(grad), np.array(parts)), ref[0], ref[1],
          ty.param_blocks(d["layers"], 2 if d["ide"] else 0), (0, 1))
    assert parts[2] == 0.0


def test_seventeen_layer_sizes_are_rejected(cabi):
    with pytest.raises(cabi.PinnError, match="need 3..16 layer sizes"):
        cabi.Pinn(cabi.BURGERS_INF, [2] + [12] * 15 + [1], [0.3, -0.5], [3.7, 2.0])
    p = cabi.Pinn(cabi.BURGERS_INF, MAXL_NET, [0.3, -0.5], [3.7, 2.0])
    assert p.P == rp.num_params(MAXL_NET)
    p.close()


# ------------------------------------------------------------------------------------------------------------------- probes
# per-stream relative tolerances of pinn_derivatives (u, u_x, u_t, u_xx): the thread-per-point forward sums in the oracle's order,
# so only tanh and the input scaling round differently; u_xx carries the most cancellation
PROBE_TOL = (1e-13, 1e-13, 1e-13, 1e-12)
PROBE_CASES = [
    ("burgers_shifted", BURGERS, "shifted", 1.0), ("burgers_small_w4", BURGERS, "small", 4.0),
    ("burgers_large", BURGERS, "large", 1.0), ("nls_other", NLS, NLS_OTHER, 1.0), ("disc", [1, 50, 50, 8], "disc", 1.0),
]


@pytest.mark.parametrize("case", PROBE_CASES, ids=[c[0] for c in PROBE_CASES])
def test_probes_per_stream(cabi, case):
    name, layers, dom, scale = case
    rng = np.random.default_rng(PROBE_CASES.index(case) + 400)
    if dom == "disc":
        lb, ub = DISC_LB, DISC_UB
        X = np.concatenate([[lb[0], ub[0]], rng.uniform(lb[0], ub[0], 198)])[:, None]
        w, pde = _rand_w(layers, 7, scale), cabi.BURGERS_DISC
    else:
        lb, ub = (np.array(v) for v in (DOMAINS[dom] if isinstance(dom, str) else dom))
        X = points(rng, lb, ub, 200)
        w = scale * load_golden("nls_inf" if layers == NLS else "burgers_inf")["w"]
        pde = cabi.NLS_INF if layers == NLS else cabi.BURGERS_INF
    p = cabi.Pinn(pde, layers, lb, ub)
    p.set_weights(w)
    got = p.derivatives(X)
    pred = p.predict(X)
    p.close()
    ref, _ = ty.forward(w, layers, lb, ub, X, dtype=LD)
    ref64, _ = ty.forward(w, layers, lb, ub, X)
    worst = 0.0
    for s, (tol, sname) in enumerate(zip(PROBE_TOL, ("u", "u_x", "u_t", "u_xx"))):
        for o in range(layers[-1]):
            if dom == "disc" and s == 2:
                assert np.all(got[s][:, o] == 0.0)                          # 1-D nets have no t stream
                continue
            err = _norm(got[s][:, o] - ref[s][:, o])
            r = _ratio(err, tol * _norm(ref[s][:, o]) + FP64_FACTOR * _norm(ref64[s][:, o] - ref[s][:, o]))
            worst = max(worst, r)
            assert r <= 1.0, (name, sname, o, err / _norm(ref[s][:, o]))
    r = _ratio(_norm(pred - ref[0]), PROBE_TOL[0] * _norm(ref[0]) + FP64_FACTOR * _norm(ref64[0] - ref[0]))
    assert r <= 1.0, (name, "predict")
    print("[precision] %-40s worst error/bound %.3g" % ("probes/" + name, max(worst, r)))


@pytest.mark.parametrize("model", ["burgers", "nls"])
def test_probes_on_one_column_input(cabi, model):
    """Quirk Q1: an (n, 1) input to a 2-D net is broadcast to (x, t := x) by the reference's Lambda.  predict takes it as it is
    (the probe kernel reads t := x), derivatives broadcasts it on the host; both equal the oracle on (x, x).  x spans the box's
    x range, so t := x lies outside the t range on purpose."""
    layers, pde, (lb, ub) = (BURGERS, cabi.BURGERS_INF, DOMAINS["shifted"]) if model == "burgers" else (NLS, cabi.NLS_INF, NLS_OTHER)
    lb, ub = np.array(lb), np.array(ub)
    x = np.random.default_rng(450).uniform(lb[0], ub[0], (200, 1))
    w = load_golden("nls_inf" if model == "nls" else "burgers_inf")["w"]
    p = cabi.Pinn(pde, layers, lb, ub)
    p.set_weights(w)
    pred, got = p.predict(x), p.derivatives(x)
    with pytest.raises(cabi.PinnError, match="columns"):
        p.derivatives(np.zeros((4, 3)))
    p.close()
    XX = np.concatenate([x, x], 1)
    ref, _ = ty.forward(w, layers, lb, ub, XX, dtype=LD)
    ref64, _ = ty.forward(w, layers, lb, ub, XX)
    bound = lambda s, o, tol: tol * _norm(ref[s][:, o]) + FP64_FACTOR * _norm(ref64[s][:, o] - ref[s][:, o])
    for o in range(layers[-1]):
        assert _ratio(_norm(pred[:, o] - ref[0][:, o]), bound(0, o, PROBE_TOL[0])) <= 1.0, (model, "predict", o)
        for s, tol in enumerate(PROBE_TOL):
            assert _ratio(_norm(got[s][:, o] - ref[s][:, o]), bound(s, o, tol)) <= 1.0, (model, "derivatives", s, o)


# ------------------------------------------------------------------------------- L-BFGS kernel instantiation switch points
# pinn_api.cu picks lbfgs_iterate<12,256> for P <= 3072, <8,1024> for P <= 8192 and <32,1024> above
@pytest.mark.parametrize("layers", [[2, 13, 43, 54, 1], [2, 52, 54, 1], [2, 31, 104, 45, 1], [2, 32, 104, 44, 1]],
                         ids=["P3072", "P3073", "P8192", "P8193"])
def test_lbfgs_at_the_instantiation_switch_points(cabi, layers):
    g = load_golden("burgers_inf")
    nu = float(g["nu"])
    w = _rand_w(layers, 9)
    assert w.size in (3072, 3073, 8192, 8193)
    p = cabi.Pinn(cabi.BURGERS_INF, layers, g["lb"], g["ub"])
    p.set_pde_params([nu]); p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1]); p.set_data(g["X_u"], g["u"]); p.set_weights(w)
    op = lambda x: ty.burgers_loss_grad(x, layers, g["lb"], g["ub"], g["X_f"], g["X_u"], g["u"], nu=nu)[:2]
    tr = rp.lbfgs_fixed_step(op, w, max_iter=5, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps)
    r = p.lbfgs(5, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, want_x_final=True)
    p.close()
    assert r["n_iter"] == tr.n_iter == 5 and r["n_eval"] == tr.n_eval
    rel = lambda a, b: np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b))
    assert rel(r["f_hist"], tr.f_hist) < 1e-7 and rel(r["x_final"], tr.x_final) < 1e-7
