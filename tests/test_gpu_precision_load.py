"""GPU: the fused kernels against the extended-precision oracle, block by block, at the per-CTA loads they run at.

tests/test_gpu_precision.py and tests/test_gpu_precision_heads.py hold every kernel per parameter block on small sets: one to a
few work units (tiles, rounds, point groups, M tiles) per CTA.  The loops over those units, the prefetches and ring phases, the
accumulators carried across hundreds of tiles, the scratch sized for a larger set and the chunked probes only run at real sizes.
Here each kernel is held to the same rule (check(), REL = 1e-12 plus FP64_FACTOR times the fp64 oracle's own error) at those
sizes:

* Burgers v2 / v1 at ~100k points (~95 tiles per CTA) and v2 at 2 000 100 (~1 894 tiles per CTA, ~474 ring phases per chain
  warp), identification at 100k, and a 250k shard of a 2M set with data weight 0;
* the Schrodinger kernel at the upstream 20 150 points (10 rounds per CTA) and at >= 50 rounds per CTA;
* the generic kernel's Burgers and Schrodinger heads at 16C - 1, 16C + 1 (C = 2 x SM count CTAs) and ~100k points, in the DMMA
  and the DFMA form;
* the Navier-Stokes kernel at 5 000 (38 points, three M tiles per CTA) and 50 000 points;
* the probes (derivatives, predict, pinn_residual) at ~1M points, and the Navier-Stokes probe across >= 3 chunks.

Shuffled replication keeps the oracle affordable: every loss is a mean over each point set (Navier-Stokes: a sum), so a set of R
copies of B distinct points has the base set's loss, gradient and magnitudes (x R for Navier-Stokes).  The copies are shuffled
under one permutation, so no tile, round, CTA or chunk boundary lines up with a copy boundary: a kernel that reads one block
twice and skips its neighbour changes the multiset and fails (tests/test_precision_load_cpu.py shows it).  Every case derives
its load from the SM count with the distribution formulas of pinn_api.cu (restated below) and asserts that it reaches it.
After the largest evaluation of each family the base set is evaluated on the same handle, into the larger scratch.

Each test prints the worst error/bound it saw and the load it reached (run with -s)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, load_golden
from oracle import taylor as ty, taylor_ns as tn
from test_gpu_precision import (BURGERS, DOMAINS, FP64_FACTOR, LD, NLS, NLS_OTHER, NLS_OWN, NU0, PROBE_TOL, _cabi, _norm,
                                _ratio, _rand_w, _sms, cached, check, points)

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
NLS_SMALL = ([0.0, 0.0], [1e-2, 1e-3])           # sc = (200, 2000): u_xx (coefficient 1/2) is scaled by 4e4


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------------------------- loads
# Restatements of the distribution formulas; tests/test_precision_load_cpu.py pins them at 132 SMs.
def burgers_load(n_total, sms, kernel):
    """pinn_api.cu: burgers_launch_eval (grid = min(units, SMs)); v2 splits the tiles of 8 points evenly over the CTAs and each CTA's tiles
    over its 4 chain warps (burgers_fused_v2.cuh:361-365); v1 stripes rounds of 32 points over the CTAs (burgers_fused.cuh:315)."""
    if kernel == "v2":
        tiles = _cdiv(n_total, 8)
        grid = min(tiles, sms)
        per = _cdiv(tiles, grid)
        return {"grid": grid, "tiles per CTA": per, "rounds per chain warp": _cdiv(per, 4)}
    rounds = _cdiv(n_total, 32)
    grid = min(rounds, sms)
    return {"grid": grid, "rounds per CTA": _cdiv(rounds, grid)}


def nls_load(n_total, sms):
    """pinn_api.cu: nls_launch_eval: one CTA per SM, ceil(n / SMs) points rounded up to whole 16-point rounds."""
    pts = _cdiv(_cdiv(n_total, sms), 16) * 16
    return {"points per CTA": pts, "rounds per CTA": pts // 16, "last CTA points": n_total - (_cdiv(n_total, pts) - 1) * pts}


def generic_load(n_total, sms):
    """pinn_api.cu: generic_launch_eval with C = 2 x SMs CTAs (pinn_api.cu: pinn_create): ceil(n / C) points rounded up to a multiple of 16 from 16
    on, to an even count below; only CTAs that own points are launched."""
    per = _cdiv(n_total, 2 * sms)
    pts = _cdiv(per, 16) * 16 if per >= 16 else _cdiv(per, 2) * 2
    grid = _cdiv(n_total, pts)
    return {"points per CTA": pts, "8-point groups per CTA": _cdiv(pts, 8), "grid": grid,
            "last CTA points": n_total - (grid - 1) * pts}


def ns_load(n_total, sms):
    """pinn_api.cu: ns_launch_eval: one CTA per SM, ceil(n / SMs) points each, in M tiles of 16 points."""
    pts = _cdiv(n_total, sms)
    grid = _cdiv(n_total, pts)
    return {"points per CTA": pts, "M tiles per CTA": _cdiv(pts, 16), "grid": grid, "last CTA points": n_total - (grid - 1) * pts}


def ns_probe_chunks(n, maxw):
    """pinn_api.cu: ns_probe: chunks of (32 Mi) / (2 x 13 x maxw) points."""
    chunk = min((32 << 20) // (2 * 13 * maxw), n)
    return {"chunk": chunk, "chunks": _cdiv(n, chunk), "last chunk": n - (_cdiv(n, chunk) - 1) * chunk}


def assert_load(tag, load, key, minimum):
    print("[load] %-40s %s" % (tag, ", ".join("%s %d" % kv for kv in load.items())))
    assert load[key] >= minimum, (tag, key, load[key], minimum)


# ------------------------------------------------------------------------------------------------------------- replication
def replicate(n_base, R, seed):
    """Base-row index of every row of R copies of n_base points under one random permutation: big = base[idx]."""
    return np.random.default_rng(seed).permutation(np.tile(np.arange(n_base), R))


def scaled(ref, R):
    """An oracle result (loss, grad, parts[, magnitudes]) of a sum over the points, for R copies of its set."""
    return tuple(tuple(R * v for v in x) if isinstance(x, tuple) else R * x for x in ref)


def probe_check(tag, streams):
    """streams: (name, got, ref, ref64, tol), arrays of rows x outputs, ref and ref64 already mapped row by row; every output
    column satisfies the rule of test_gpu_precision.test_probes_per_stream, ||got - ref|| <= tol ||ref|| + FP64_FACTOR
    ||ref64 - ref||."""
    worst = 0.0
    for name, got, ref, ref64, tol in streams:
        got, ref, ref64 = (np.asarray(v).reshape(len(v), -1) for v in (got, ref, ref64))
        for o in range(ref.shape[1]):
            r = _ratio(_norm(got[:, o] - ref[:, o]), tol * _norm(ref[:, o]) + FP64_FACTOR * _norm(ref64[:, o] - ref[:, o]))
            worst = max(worst, r)
            assert r <= 1.0, (tag, name, o, "%.3g" % r)
    print("[precision] %-40s worst error/bound %.3g" % (tag, worst))
    return worst


def run_worker(func, env):
    """func() of this module in a fresh interpreter with env set (the kernel switches are read once per process); it prints one
    JSON line."""
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_precision_load as m; m.%s()" % (ROOT, TESTS, func)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _result(p, w):
    loss, grad, parts = p.loss_grad(w=w)
    return [loss, grad.tolist(), parts.tolist()]


def _got(r):
    return r[0], np.array(r[1]), np.array(r[2])


# ------------------------------------------------------------------------------------------------- specialised Burgers kernel
# key: (identification, domain, nu or (lambda_1, lambda_2), replicated base points, distinct data points, data weight,
#       collocation count of one copy in n_global).  Inference replicates the collocation set, identification the data set.
BURGERS_BASES = {
    "std": (False, "std", NU0, 20000, 100, 1.0, None),
    "small": (False, "small", 1.0, 20000, 100, 1.0, None),
    "ide_shifted": (True, "shifted", (1.0, 0.0), 20000, 0, 1.0, None),
    "shard_large": (False, "large", 1.0, 12500, 100, 0.0, 100000),     # a 250k shard of 2M points, data on another rank
}
# (name, base, copies, {kernel: the least tiles (v2) / rounds (v1) per CTA the case must reach})
BURGERS_LOAD = [
    ("inf_std_100k", "std", 5, {"v2": 90, "v1": 23}),
    ("inf_small_nu1_100k", "small", 5, {"v2": 90, "v1": 23}),
    ("ide_shifted_k1_100k", "ide_shifted", 5, {"v2": 90, "v1": 23}),
    ("inf_std_2M", "std", 100, {"v2": 1800}),
    ("inf_small_nu1_2M", "small", 100, {"v2": 1800}),
    ("shard_large_nu1_250k", "shard_large", 20, {"v2": 230}),
]
BURGERS_UNIT = {"v2": "tiles per CTA", "v1": "rounds per CTA"}


def burgers_set(base, R):
    """The base set (R = 0) or R shuffled copies of it."""
    ide, dom, pde, nb, nd, dw, nfg = BURGERS_BASES[base]
    seed = list(BURGERS_BASES).index(base) + 1300
    rng = np.random.default_rng(seed)
    lb, ub = (np.array(v) for v in DOMAINS[dom])
    Xb, ub_ = points(rng, lb, ub, nb), rng.uniform(-1, 1, (nb, 1))
    Xd, ud = points(rng, lb, ub, nd), rng.uniform(-1, 1, (nd, 1))
    idx = replicate(nb, R, seed) if R else np.arange(nb)
    w = load_golden("burgers_inf")["w"]
    d = dict(ide=ide, lb=lb, ub=ub, nu=None if ide else pde, w=np.concatenate([w, pde]) if ide else w, dw=dw,
             n_global=(nfg or nb) * max(R, 1))
    if ide:
        d.update(X_f=np.zeros((0, 2)), X_u=Xb[idx], u=ub_[idx])
    else:
        d.update(X_f=Xb[idx], X_u=Xd, u=ud)
    return d


def burgers_ref(base):
    def run():
        d = burgers_set(base, 0)
        args = (d["w"], BURGERS, d["lb"], d["ub"], d["X_f"], d["X_u"], d["u"])
        kw = dict(nu=d["nu"], identification=d["ide"], n_f_global=None if d["ide"] else d["n_global"], data_weight=d["dw"])
        return ty.burgers_loss_grad(*args, dtype=LD, magnitudes=True, **kw), ty.burgers_loss_grad(*args, **kw)
    return cached("load/burgers/" + base, run)


def burgers_handle(c, d):
    p = c.Pinn(c.BURGERS_IDE if d["ide"] else c.BURGERS_INF, BURGERS, d["lb"], d["ub"])
    assert p.kernel_info()["dyn_smem"] > 0                                  # the specialised kernel
    if not d["ide"]:
        p.set_pde_params([d["nu"]])
        p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1], n_global=d["n_global"])
    p.set_data(d["X_u"], d["u"], weight=d["dw"])
    return p


def burgers_worker():
    c, sms = _cabi(), _sms()
    kernel = "v1" if os.environ.get("PINN_BURGERS_KERNEL") == "v1" else "v2"
    out = {"sms": sms}
    for name, base, R, need in BURGERS_LOAD:
        if kernel not in need:
            continue
        d = burgers_set(base, R)
        p = burgers_handle(c, d)
        out["n_cta"], out["kernel"] = p.kernel_info()["grid"], p.kernel_info()
        out[name] = _result(p, d["w"])
        if name == "inf_std_2M":
            out[name + "/again"] = _result(p, d["w"])
            b = burgers_set(base, 0)                      # the base set on the same handle, after the largest set
            p.set_collocation(b["X_f"][:, 0], b["X_f"][:, 1]); p.set_data(b["X_u"], b["u"])
            out[name + "/base"] = _result(p, b["w"])
        p.close()
    print(json.dumps(out))


def burgers_tail_worker():
    """inf_std_2M with the stand-alone tail kernel (PINN_FUSED_TAIL=0)."""
    c = _cabi()
    d = burgers_set("std", 100)
    p = burgers_handle(c, d)
    out = {"inf_std_2M": _result(p, d["w"])}
    p.close()
    print(json.dumps(out))


@pytest.fixture(scope="module")
def burgers_runs():
    runs = {k: run_worker("burgers_worker", {"PINN_BURGERS_KERNEL": k}) for k in ("v2", "v1")}
    assert runs["v2"]["kernel"] != runs["v1"]["kernel"]          # two different kernels actually ran
    return runs


BURGERS_PARAMS = [(case, k) for case in BURGERS_LOAD for k in case[3]]


@pytest.mark.parametrize("case,kernel", BURGERS_PARAMS, ids=["%s-%s" % (c[0], k) for c, k in BURGERS_PARAMS])
def test_burgers_kernel_at_load(burgers_runs, case, kernel):
    name, base, R, need = case
    run = burgers_runs[kernel]
    assert run["n_cta"] == run["sms"]
    d = burgers_set(base, R)
    n_total = d["X_u"].shape[0] + d["X_f"].shape[0]
    assert_load(kernel + "/" + name, burgers_load(n_total, run["sms"], kernel), BURGERS_UNIT[kernel], need[kernel])
    ref = burgers_ref(base)
    check(kernel + "/" + name, _got(run[name]), ref[0], ref[1], ty.param_blocks(BURGERS, 2 if d["ide"] else 0), (0, 2))
    assert run[name][2][1] == 0.0


def test_burgers_2M_is_reproducible_and_the_tail_kernel_agrees_bitwise(burgers_runs):
    a, b = burgers_runs["v2"]["inf_std_2M"], burgers_runs["v2"]["inf_std_2M/again"]
    assert a == b                                                   # two evaluations, bit for bit
    tail = run_worker("burgers_tail_worker", {"PINN_BURGERS_KERNEL": "v2", "PINN_FUSED_TAIL": "0"})["inf_std_2M"]
    assert tail == a                                                # the in-kernel tail and the tail kernel, bit for bit


def test_burgers_base_set_after_2M(burgers_runs):
    ref = burgers_ref("std")
    check("v2/inf_std_base_after_2M", _got(burgers_runs["v2"]["inf_std_2M/base"]), ref[0], ref[1], ty.param_blocks(BURGERS),
          (0, 2))


# ---------------------------------------------------------------------------------------------------- Schrodinger kernels
# key: (domain, replicated collocation points, n_0, n_b, Q1 initial-condition mode (x, x)).  An odd n_0 takes the inert
# alignment point.
NLS_BASES = {
    "own": (NLS_OWN, 2000, 50, 50, False),
    "other_q1_odd": (NLS_OTHER, 2000, 49, 50, True),
    "small": (NLS_SMALL, 2000, 51, 1, False),
}


def nls_set(dom, n_c, n0, nb, q1, layers, seed, R):
    """Collocation base set of n_c points (R = 0) or R shuffled copies of it; the initial-condition and boundary sets are not
    replicated."""
    lb, ub = (np.array(v) for v in dom)
    rng = np.random.default_rng(seed)
    Xb = points(rng, lb, ub, n_c)
    tb = np.concatenate([[lb[1], ub[1]], rng.uniform(lb[1], ub[1], max(nb - 2, 0))])[:nb, None]
    x0 = np.concatenate([[lb[0], ub[0]], rng.uniform(lb[0], ub[0], max(n0 - 2, 0))])[:n0, None]
    X0 = x0 if q1 else np.concatenate([x0, 0 * x0 + lb[1]], 1)
    uv0 = rng.standard_normal((n0, 2))
    w = load_golden("nls_inf")["w"] if layers == NLS else _rand_w(layers, seed)
    idx = replicate(n_c, R, seed) if R else np.arange(n_c)
    return dict(layers=layers, lb=lb, ub=ub, X_f=Xb[idx], tb=tb, X0=X0, uv0=uv0, w=w,
                n_total=(n0 + 1) // 2 * 2 + 2 * nb + len(idx))


def nls_ref(key, d):
    def run():
        args = (d["w"], d["layers"], d["lb"], d["ub"], d["X_f"], d["tb"], d["X0"], d["uv0"])
        return ty.schrodinger_loss_grad(*args, dtype=LD, magnitudes=True), ty.schrodinger_loss_grad(*args)
    return cached("load/nls/" + key, run)


def nls_handle(c, d):
    p = c.Pinn(c.NLS_INF, d["layers"], d["lb"], d["ub"])
    p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1]); p.set_boundary(d["tb"]); p.set_data(d["X0"], d["uv0"])
    return p


# (name, base, copies, the least 16-point rounds per CTA)
NLS_LOAD = [("own_upstream", "own", 10, 10), ("own_rounds", "own", 53, 50),
            ("other_q1_odd_upstream", "other_q1_odd", 10, 10), ("other_q1_odd_rounds", "other_q1_odd", 53, 50),
            ("small_upstream", "small", 10, 10), ("small_rounds", "small", 53, 50)]


@pytest.mark.parametrize("case", NLS_LOAD, ids=[c[0] for c in NLS_LOAD])
def test_schrodinger_kernel_at_load(case):
    name, base, R, rounds = case
    c, sms = _cabi(), _sms()
    dom, n_c, n0, nb, q1 = NLS_BASES[base]
    seed = list(NLS_BASES).index(base) + 1400
    d = nls_set(dom, n_c, n0, nb, q1, NLS, seed, R)
    assert_load("nls/" + name, nls_load(d["n_total"], sms), "rounds per CTA", rounds)
    ref = nls_ref(base, nls_set(dom, n_c, n0, nb, q1, NLS, seed, 0))
    p = nls_handle(c, d)
    info = p.kernel_info()
    assert info["dyn_smem"] > 0 and info["grid"] == sms                     # the specialised kernel, one CTA per SM
    got = p.loss_grad(w=d["w"])
    if rounds >= 50:                                                        # the base set into the larger scratch
        b = nls_set(dom, n_c, n0, nb, q1, NLS, seed, 0)
        p.set_collocation(b["X_f"][:, 0], b["X_f"][:, 1])
        got_base = p.loss_grad(w=d["w"])
    p.close()
    check("nls/" + name, got, ref[0], ref[1], ty.param_blocks(NLS), (0, 1, 2))
    if rounds >= 50:
        check("nls/" + base + "_base_after_" + name, got_base, ref[0], ref[1], ty.param_blocks(NLS), (0, 1, 2))


# ------------------------------------------------------------------------------------------- generic kernel, continuous heads
W40X8, MIXED, W256 = [2] + [40] * 8 + [1], [2, 37, 5, 64, 13, 1], [2, 256, 256, 1]
# (name, head, layers, domain, total, base size (None: distinct points), inf: least distinct data points / nls: (n_0, n_b, Q1))
# "16C-1", "16C+1": totals on each side of 16 points per CTA; "100k": 100 000 replicated points plus the data / auxiliary set.
# Inference puts n_d data points in front of the collocation set, n_d not a multiple of 8: the data / collocation boundary falls
# inside an 8-point group.  Every non-unit domain runs with an O(1) coefficient on u_xx (nu = 1, e^{lambda_2} = 1, 1/2).
GENERIC_LOAD = [
    ("inf_w40x8_16Cm1", "inf", W40X8, "shifted", "16C-1", None, 37),
    ("ide_w40x8_100k", "ide", W40X8, "small", "100k", 2000, None),
    ("ide_mixed_16Cp1", "ide", MIXED, "large", "16C+1", None, None),
    ("inf_mixed_w4_100k", "inf", MIXED, "small", "100k", 2000, 101),
    ("inf_w256_16Cp1", "inf", W256, "large", "16C+1", 400, 37),
    ("inf_w256_100k", "inf", W256, "std", "100k", 400, 101),
    ("ide_w256_100k", "ide", W256, "shifted", "100k", 400, None),
    ("nls_30_20_16Cm1", "nls", [2, 30, 20, 2], NLS_OWN, "16C-1", None, (49, 1, False)),
    ("nls_16x5_q1_16Cp1", "nls", [2] + [16] * 5 + [2], NLS_OTHER, "16C+1", None, (50, 50, True)),
    ("nls_256_100k", "nls", [2, 256, 2], NLS_SMALL, "100k", 2000, (51, 50, False)),
    ("nls_100x4_forced_100k", "nls", NLS, NLS_OWN, "100k", 1000, (50, 1, True)),
]


def generic_set(case, sms, base=False):
    """The case's set, or (base=True) its base set with the distinct points unchanged."""
    name, head, layers, dom, total, B, extra = case
    seed = GENERIC_LOAD.index(case) + 1500
    if head == "nls":
        n0, nb, q1 = extra
        aux = (n0 + 1) // 2 * 2 + 2 * nb
        T = 100000 + aux if total == "100k" else {"16C-1": 32 * sms - 1, "16C+1": 32 * sms + 1}[total]
        n_c = T - aux
        B = B or n_c
        assert n_c % B == 0
        d = nls_set(dom, B, n0, nb, q1, layers, seed, 0 if base else n_c // B)
        d.update(head=head, base_key="generic/" + name)
        return d
    rng = np.random.default_rng(seed)
    lb, ub = (np.array(v) for v in DOMAINS[dom])
    ide = head == "ide"
    T = (100000 if ide else 100000 + extra) if total == "100k" else {"16C-1": 32 * sms - 1, "16C+1": 32 * sms + 1}[total]
    if ide:
        n_d, B = 0, B or T
        assert T % B == 0
    else:
        B = B or T - extra
        n_d = extra + (T - extra) % B                 # the rest of the total in distinct data points
        assert n_d % 8
    w = _rand_w(layers, seed, 4.0 if "_w4" in name else 1.0)
    Xb, ub_ = points(rng, lb, ub, B), rng.uniform(-1, 1, (B, 1))
    Xd, ud = points(rng, lb, ub, n_d), rng.uniform(-1, 1, (n_d, 1))
    R = (T - n_d) // B
    idx = np.arange(B) if base else replicate(B, R, seed)
    d = dict(head=head, layers=layers, lb=lb, ub=ub, base_key="generic/" + name, n_total=n_d + len(idx))
    if ide:
        d.update(ide=True, w=np.concatenate([w, [0.5, 0.0]]), X_f=np.zeros((0, 2)), X_u=Xb[idx], u=ub_[idx])
    else:
        d.update(ide=False, w=w, X_f=Xb[idx], X_u=Xd, u=ud)
    return d


def generic_ref(d):
    """The oracle pair of a base set."""
    if d["head"] == "nls":
        return nls_ref(d["base_key"], d)

    def run():
        args = (d["w"], d["layers"], d["lb"], d["ub"], d["X_f"], d["X_u"], d["u"])
        kw = dict(nu=None if d["ide"] else 1.0, identification=d["ide"])
        return ty.burgers_loss_grad(*args, dtype=LD, magnitudes=True, **kw), ty.burgers_loss_grad(*args, **kw)
    return cached("load/" + d["base_key"], run)


def generic_handle(c, d):
    if d["head"] == "nls":
        return nls_handle(c, d)
    p = c.Pinn(c.BURGERS_IDE if d["ide"] else c.BURGERS_INF, d["layers"], d["lb"], d["ub"])
    if not d["ide"]:
        p.set_pde_params([1.0]); p.set_collocation(d["X_f"][:, 0], d["X_f"][:, 1])
    p.set_data(d["X_u"], d["u"])
    return p


def generic_worker():
    c, sms = _cabi(), _sms()
    out = {"sms": sms}
    for case in GENERIC_LOAD:
        d = generic_set(case, sms)
        p = generic_handle(c, d)
        info = p.kernel_info()
        assert info["dyn_smem"] == 0 and info["grid"] == 2 * sms            # the generic kernel, two CTAs per SM
        out[case[0]] = _result(p, d["w"])
        if case[4] == "100k":                                               # the base set into the larger scratch
            b = generic_set(case, sms, base=True)
            if b["head"] == "nls" or not b["ide"]:
                p.set_collocation(b["X_f"][:, 0], b["X_f"][:, 1])
            else:
                p.set_data(b["X_u"], b["u"])
            out[case[0] + "/base"] = _result(p, d["w"])
        p.close()
    print(json.dumps(out))


@pytest.fixture(scope="module")
def generic_runs():
    runs = {form: run_worker("generic_worker", {"PINN_GENERIC_DFMA": flag, "PINN_FORCE_GENERIC": "1"})
            for form, flag in (("dmma", "0"), ("dfma", "1"))}
    assert runs["dmma"]["inf_w256_100k"][1] != runs["dfma"]["inf_w256_100k"][1]   # two different summation orders ran
    return runs


@pytest.mark.parametrize("form", ["dmma", "dfma"])
@pytest.mark.parametrize("case", GENERIC_LOAD, ids=[c[0] for c in GENERIC_LOAD])
def test_generic_kernel_at_load(generic_runs, form, case):
    run = generic_runs[form]
    d = generic_set(case, run["sms"])
    load = generic_load(d["n_total"], run["sms"])
    if case[4] == "100k":
        assert_load("%s/%s" % (form, case[0]), load, "8-point groups per CTA", 32)
    else:                                                   # one short of / one past 16 points per CTA, ragged last CTA
        assert_load("%s/%s" % (form, case[0]), load, "points per CTA", 16)
        assert load["points per CTA"] == (16 if case[4] == "16C-1" else 32) and load["last CTA points"] in (15, 1)
    ref = generic_ref(generic_set(case, run["sms"], base=True))
    nls = d["head"] == "nls"
    blocks = ty.param_blocks(d["layers"], 2 if not nls and d["ide"] else 0)
    part_idx = (0, 1, 2) if nls else (0, 2)
    check("%s/%s" % (form, case[0]), _got(run[case[0]]), ref[0], ref[1], blocks, part_idx)
    if case[4] == "100k":
        check("%s/%s_base_after" % (form, case[0]), _got(run[case[0] + "/base"]), ref[0], ref[1], blocks, part_idx)


# --------------------------------------------------------------------------------------------------------- Navier-Stokes
NS_NET = [20] * 8
# (name, lb, ub, weight scale, base points, copies, the least M tiles per CTA)
NS_LOAD = [("upstream_5000", (1.0, -2.0, 0.0), (8.0, 2.0, 20.0), 1.0, 500, 10, 3),
           ("small_box_50000", (0.0, 0.0, 0.0), (1e-2, 2e-2, 1e-3), 1.0, 500, 100, 20),
           ("w4_5000", (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0), 4.0, 500, 10, 3)]


@pytest.mark.parametrize("case", NS_LOAD, ids=[c[0] for c in NS_LOAD])
def test_navier_stokes_kernel_at_load(case):
    from test_gpu_ns import ns_inputs
    name, lb, ub, scale, B, R, tiles = case
    c, sms = _cabi(), _sms()
    layers, lb, ub, X, uv, w = ns_inputs(NS_NET, B, NS_LOAD.index(case) + 1600, lb, ub, scale=scale)
    idx = replicate(B, R, NS_LOAD.index(case) + 1600)
    assert_load("ns/" + name, ns_load(B * R, sms), "M tiles per CTA", tiles)
    ref = cached("load/ns/" + name, lambda: (tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv, dtype=LD, magnitudes=True),
                                             tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv)))
    p = c.Pinn(c.NS_IDE, layers, lb, ub)
    assert p.kernel_info()["grid"] == sms
    p.set_data(X[idx], uv[idx])
    got = p.loss_grad(w=w)
    p.set_data(X, uv)                                           # the base set into the larger scratch
    got_base = p.loss_grad(w=w)
    p.close()
    blocks = ty.param_blocks(layers, 2)
    check("ns/" + name, got, scaled(ref[0], R), scaled(ref[1], R), blocks, (0, 2))
    check("ns/" + name + "_base_after", got_base, ref[0], ref[1], blocks, (0, 2))


# ------------------------------------------------------------------------------------------------------------------- probes
def test_burgers_probes_and_residuals_at_1M():
    """derivatives / predict and pinn_residual of Burgers inference and identification on 100 shuffled copies of 10 000 points;
    every row against the longdouble streams of its base point."""
    c = _cabi()
    lb, ub = (np.array(v) for v in DOMAINS["small"])
    Xb = points(np.random.default_rng(1700), lb, ub, 10000)
    idx = replicate(10000, 100, 1700)
    X = Xb[idx]
    w = 4.0 * load_golden("burgers_inf")["w"]
    lam = (0.7, 0.2)
    ref = [v[idx] for v in ty.forward(w, BURGERS, lb, ub, Xb, dtype=LD)[0]]
    ref64 = [v[idx] for v in ty.forward(w, BURGERS, lb, ub, Xb)[0]]
    p = c.Pinn(c.BURGERS_INF, BURGERS, lb, ub)
    p.set_weights(w)
    got, pred = p.derivatives(X), p.predict(X)
    p.set_pde_params([1.0]); p.set_collocation(X[:, 0], X[:, 1]); p.set_data(Xb[:5], np.zeros(5))
    f_inf = p.residual()
    p.close()
    q = c.Pinn(c.BURGERS_IDE, BURGERS, lb, ub)
    q.set_data(X, np.zeros(len(X)))
    q.set_weights(np.concatenate([w, lam]))
    f_ide = q.residual()
    q.close()
    f = lambda s, l1, kap: s[2] + l1 * s[0] * s[1] - kap * s[3]
    names = ("u", "u_x", "u_t", "u_xx")
    probe_check("probes/burgers_1M", [(n, got[k], ref[k], ref64[k], PROBE_TOL[k]) for k, n in enumerate(names)] +
                [("predict", pred, ref[0], ref64[0], PROBE_TOL[0])])
    probe_check("probes/burgers_residual_1M", [
        ("f inf", f_inf, f(ref, 1, 1), f(ref64, 1, 1), PROBE_TOL[3]),
        ("f ide", f_ide, f(ref, LD(lam[0]), np.exp(LD(lam[1]))), f(ref64, lam[0], np.exp(lam[1])), PROBE_TOL[3])])


def test_schrodinger_probes_and_residual_at_1M():
    c = _cabi()
    lb, ub = (np.array(v) for v in NLS_OTHER)
    Xb = points(np.random.default_rng(1701), lb, ub, 2000)
    idx = replicate(2000, 500, 1701)
    X = Xb[idx]
    w = load_golden("nls_inf")["w"]
    ref = [v[idx] for v in ty.forward(w, NLS, lb, ub, Xb, dtype=LD)[0]]
    ref64 = [v[idx] for v in ty.forward(w, NLS, lb, ub, Xb)[0]]
    p = c.Pinn(c.NLS_INF, NLS, lb, ub)
    p.set_weights(w)
    got, pred = p.derivatives(X), p.predict(X)
    p.set_collocation(X[:, 0], X[:, 1])
    fr = p.residual()
    p.close()

    def f(s):
        (u, v), (ut, vt), (uxx, vxx) = s[0].T, s[2].T, s[3].T
        h2 = u * u + v * v
        return np.stack([ut + 0.5 * vxx + h2 * v, vt - 0.5 * uxx - h2 * u], 1)
    names = ("u", "u_x", "u_t", "u_xx")
    probe_check("probes/nls_1M", [(n, got[k], ref[k], ref64[k], PROBE_TOL[k]) for k, n in enumerate(names)] +
                [("predict", pred, ref[0], ref64[0], PROBE_TOL[0]), ("f", fr, f(ref), f(ref64), PROBE_TOL[3])])


# (name, hidden, lb, ub, base points, copies): widths 256 (chunks of 5 041 points) and 20 (chunks of 64 527 points)
NS_PROBE = [("w256_upstream", [256, 256], (1.0, -2.0, 0.0), (8.0, 2.0, 20.0), 500, 32),
            ("w20_small_box", [20] * 8, (0.0, 0.0, 0.0), (1e-2, 2e-2, 1e-3), 500, 400)]


@pytest.mark.parametrize("case", NS_PROBE, ids=[c[0] for c in NS_PROBE])
def test_navier_stokes_probes_across_chunks(case):
    from test_gpu_ns import ns_inputs
    name, hidden, lb, ub, B, R = case
    c = _cabi()
    layers, lb, ub, Xb, uvb, w = ns_inputs(hidden, B, NS_PROBE.index(case) + 1800, lb, ub)
    idx = replicate(B, R, NS_PROBE.index(case) + 1800)
    X = Xb[idx]
    load = ns_probe_chunks(len(X), max(hidden))
    assert_load("ns_probe/" + name, load, "chunks", 4)
    assert load["last chunk"] < load["chunk"]                               # a ragged last chunk
    O = [v[idx] for v in tn.forward_ns(w[:-2], layers, lb, ub, Xb, dtype=LD)[0]]
    O64 = [v[idx] for v in tn.forward_ns(w[:-2], layers, lb, ub, Xb)[0]]
    p = c.Pinn(c.NS_IDE, layers, lb, ub)
    p.set_weights(w)
    got, pred = p.derivatives(X), p.predict(X)
    p.set_data(X, uvb[idx])
    fr = p.residual()
    p.close()
    streams = [("stream %d" % k, got[:, k], O[k], O64[k], 1e-13 if sum(m) <= 1 else 1e-12) for k, m in enumerate(tn.STREAMS)]
    f = lambda S, l1, l2: np.stack(tn.ns_terms(S, l1, l2), 1)
    probe_check("probes/ns_" + name, streams + [
        ("predict", pred, O[0], O64[0], PROBE_TOL[0]),
        ("f", fr, f(O, LD(w[-2]), LD(w[-1])), f(O64, w[-2], w[-1]), 1e-12)])
