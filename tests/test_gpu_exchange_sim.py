"""GPU: the multi-GPU evaluation tail run by W simulated ranks on one H100, and sharded evaluations held to the whole-set oracle.

tests/exchange_harness.cu launches the product's pinn::reduce_tail, pinn::fused_tail and pinn::adam_update unchanged, one stream
and one set of buffers per rank, with the exchange buffers of the other ranks as plain device allocations instead of IPC
mappings (tests/exchange_order.py drives it).  Checked here:

* the exchanged R on every rank equals the host restatement of the summation order bit for bit, on partials whose sums cancel
  heavily (so a different order changes bits), for W in {2, 3, 5, 8}, the Burgers, Schrodinger, a small generic and 32k +- 1
  entry vectors, and per-rank CTA counts that differ from rank to rank; both forms of the tail give the same bits;
* Adam inside the exchange equals adam_update on the same R and state, bit for bit; the step counter and the loss ring follow;
* a sequence of evaluations enqueued without a host synchronisation, mixing both forms, Adam steps, plain evaluations and
  evaluations skipped through run_flag, advances the exchange sequence and the Adam step only for the evaluations that ran, with
  alternating parities, and each equals a one-shot run of the same partials;
* a NaN or +-Inf in one rank's entry gives that entry the class of the reference sum on every rank and changes no other entry;
* sharded Burgers inference (v2, v1 and the generic kernel) and Schrodinger (specialised and generic) evaluations, exchanged by
  the harness, are held per parameter block to the longdouble oracle of the whole set (test_gpu_precision.check), and five
  sharded Adam steps track a whole-set handle;
* the five models that cannot be sharded count a W-fold (part of the) loss when composed the same way, and pinn_create refuses
  world > 1 for them.

Every rank's grid is sized so that all ranks' CTAs are resident at once (the tail CTAs of one rank spin on the others' flags);
a schedule in which the streams did not overlap would end in the exchange's bounded wait with err = 1, not in a hang.  The
harness runs in a subprocess with a timeout.  Run with -s to read the worst error/bound ratios and the wall times.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import exchange_order as xo
from conftest import ROOT, load_golden

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
UTILS = os.path.join(ROOT, "pinns-tf2.0_b200", "utils")
ADAM = (1e-3, 0.9, 0.999, 1e-7)
ADAM_BIG = (0.05, 0.99, 0.999, 0.1)


def _geom(p_net):
    return p_net, (p_net, p_net + 1, p_net + 2), (p_net + 8 + 15) // 16 * 16


# name -> (p_net, extra_src, stride): R = [p_net columns 1:1 | three loss parts gathered from extra_src]
SIZES = {
    "burgers": (3021, (3024, 3023, 3025), 3040),            # the Burgers kernel's map (pinn_api.cu: burgers_launch_eval)
    "nls": (30802, (30802, 30803, 30804), 30816),           # 963 virtual blocks: more than 2 x SMs, the walk runs
    "small": _geom(17),                                     # n_out = 20 < 32: one partly filled block
    "32k-1": _geom(32764), "32k": _geom(32765), "32k+1": _geom(32766),
}
# (size, per-rank CTA counts): W in {2, 3, 5, 8}; the fused form runs n_cta CTAs, so the counts cover grid < nb, = nb, > nb and 1
ARITH_CASES = [(s, n) for s in SIZES for n in ([264, 1], [9, 132, 5], [1, 5, 8, 9, 132], [5, 8, 9, 132, 264, 1, 16, 7])]
ARITH_CASES += [("burgers", [95, 1, 132]), ("small", [1, 5, 9])]


def run_worker(func, lib, arg=None, env=None, timeout=900):
    """func(arg) of this module in a fresh interpreter (the kernel switches are read per process); it prints one JSON line."""
    code = "import sys; sys.path[:0] = [%r, %r, %r]; import test_gpu_exchange_sim as m; m.%s(%r)" % (ROOT, TESTS, UTILS, func, arg)
    t0 = time.time()
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, XH_LIB=lib, **(env or {})), capture_output=True,
                       text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    print("[exchange] %-28s %s wall %.1f s" % (func, arg if arg is not None else "", time.time() - t0))
    return out


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return xo.compile_harness(str(tmp_path_factory.mktemp("exchange_harness")))


def _harness(world, size, max_cta=1, n_slots=1, n_snap=1):
    p_net, extra, stride = SIZES[size]
    return xo.Harness(os.environ["XH_LIB"], world, p_net, extra, stride, max_cta=max_cta, n_slots=n_slots, n_snap=n_snap)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same(a, b):
    return bool(np.array_equal(_bits(a), _bits(b)))


# ------------------------------------------------------------------------------------------------- a, b: bit-exact arithmetic
def arith_worker(_):
    out = {}
    for ci, (size, n_ctas) in enumerate(ARITH_CASES):
        W = len(n_ctas)
        h = _harness(W, size, max_cta=max(n_ctas), n_snap=2)
        parts = xo.cancelling_ranks(np.random.default_rng(ci), n_ctas, h.stride)
        ref = xo.tail_sum(parts, h.cols)
        for k in range(W):
            h.load(k, 0, parts[k])
        h.enqueue(0, "reduce", snap=0)
        h.enqueue(0, "fused", snap=1)
        h.sync()
        res = dict(W=W, nb=h.nb, reduce_grid=h.reduce_grid(), sms=h.sms, occ=[h.occ_reduce, h.occ_fused], bad=[])
        for snap, form in ((0, "reduce"), (1, "fused")):
            for k in range(W):
                s = h.read(k, snap)
                if not _same(s["R"], ref):
                    res["bad"].append("%s rank %d: %d entries differ from the restatement" % (form, k, np.count_nonzero(_bits(s["R"]) != _bits(ref))))
                if s["err"] != 0 or s["step"][1:] != [0, 0] or s["xseq"] != snap + 1:
                    res["bad"].append("%s rank %d: err %d step %s xseq %d" % (form, k, s["err"], s["step"], s["xseq"]))
        h.close()
        out["%s/%s" % (size, n_ctas)] = res
    print(json.dumps(out))


@pytest.fixture(scope="module")
def arith(lib):
    return run_worker("arith_worker", lib)


@pytest.mark.parametrize("case", ARITH_CASES, ids=["%s-W%d-%s" % (s, len(n), "_".join(map(str, n))) for s, n in ARITH_CASES])
def test_exchange_is_bit_exact_and_both_forms_agree(arith, case):
    r = arith["%s/%s" % case]
    assert not r["bad"], r["bad"]
    if case[0] == "nls":
        assert r["reduce_grid"] < r["nb"]                                   # the virtual-block walk ran


# ------------------------------------------------------------------------------------------------- c: Adam inside the exchange
ADAM_CASES = [("burgers", ADAM), ("nls", ADAM_BIG), ("32k+1", ADAM), ("small", ADAM_BIG)]


def _state(rng, P):
    return rng.standard_normal(P), 0.1 * rng.standard_normal(P), rng.random(P) * 1e-2


def adam_worker(_):
    out = {}
    for ci, (size, hp) in enumerate(ADAM_CASES):
        n_ctas = [9, 132, 5]
        W = len(n_ctas)
        h = _harness(W, size, max_cta=max(n_ctas), n_snap=4)
        rng = np.random.default_rng(50 + ci)
        parts = xo.cancelling_ranks(rng, n_ctas, h.stride)
        w, m, v = _state(rng, h.P)
        for k in range(W):
            h.load(k, 0, parts[k])

        def reset():
            for k in range(W):
                h.set_state(k, w, m, v, 4)

        reset(); h.enqueue(0, "reduce", adam=hp, snap=0)
        reset(); h.enqueue(0, "fused", adam=hp, snap=1)
        reset(); h.enqueue(0, "reduce", snap=2); h.enqueue(0, "adam_update", adam=hp, snap=3)
        h.sync()
        bad = []
        ref = xo.tail_sum(parts, h.cols)
        P = h.P
        loss = (ref[P] + ref[P + 1]) + ref[P + 2]
        for k in range(W):
            s = [h.read(k, i) for i in range(4)]
            for i in (0, 1, 3):
                for key in ("w", "m", "v"):
                    if not _same(s[i][key], s[3][key]):
                        bad.append("rank %d snap %d: %s differs from adam_update" % (k, i, key))
                if s[i]["step"] != [5, 0, 0] or not _same(s[i]["ring"][4], loss) or s[i]["err"] != 0:
                    bad.append("rank %d snap %d: step %s ring %r loss %r err %d" % (k, i, s[i]["step"], s[i]["ring"][4], loss, s[i]["err"]))
                if not _same(s[i]["R"], ref):
                    bad.append("rank %d snap %d: R differs from the restatement" % (k, i))
            if _same(s[0]["w"], w):
                bad.append("rank %d: the weights did not move" % k)
        h.close()
        out[size] = bad
    print(json.dumps(out))


@pytest.fixture(scope="module")
def adam(lib):
    return run_worker("adam_worker", lib)


@pytest.mark.parametrize("case", ADAM_CASES, ids=[c[0] for c in ADAM_CASES])
def test_adam_inside_the_exchange_equals_adam_update(adam, case):
    assert adam[case[0]] == []


# ------------------------------------------------------------------------------------------------------------- d: sequences
# (form, Adam step, skipped through run_flag): ten evaluations enqueued back to back, then one synchronisation
SEQUENCE = [("reduce", True, False), ("fused", False, False), ("reduce", False, True), ("fused", True, False),
            ("fused", True, True), ("reduce", True, False), ("fused", False, False), ("reduce", True, True),
            ("fused", True, False), ("reduce", False, False)]
SEQ_CTAS = [[9, 1, 132], [5, 8, 9], [1, 1, 1], [132, 9, 5], [8, 264, 1], [1, 5, 8], [264, 132, 9], [9, 9, 9], [5, 1, 264],
            [132, 132, 132]]


def sequence_worker(size):
    W, n = 3, len(SEQUENCE)
    h = _harness(W, size, max_cta=264, n_slots=n, n_snap=n)
    rng = np.random.default_rng(77)
    parts = [xo.cancelling_ranks(rng, SEQ_CTAS[e], h.stride) for e in range(n)]
    w0, m0, v0 = _state(rng, h.P)
    for k in range(W):
        h.set_state(k, w0, m0, v0, 0)
        for e, (_, _, skip) in enumerate(SEQUENCE):
            h.load(k, e, parts[e][k], run_flag=1 if skip else 0)
    for e, (form, ad, _) in enumerate(SEQUENCE):
        h.enqueue(e, form, adam=ADAM if ad else None, snap=e)
    h.sync()
    snaps = [[h.read(k, e) for e in range(n)] for k in range(W)]
    flags = [h.flags(k) for k in range(W)]
    h.close()
    bad, ran, steps = [], 0, 0
    for e, (form, ad, skip) in enumerate(SEQUENCE):
        ran += 0 if skip else 1
        steps += 1 if (ad and not skip) else 0
        for k in range(W):
            s = snaps[k][e]
            if s["xseq"] != ran or s["step"] != [steps, 0, 0] or s["err"] != 0:
                bad.append("eval %d rank %d: xseq %d step %s err %d (want %d, %d)" % (e, k, s["xseq"], s["step"], s["err"], ran, steps))
            if skip:
                prev = snaps[k][e - 1]
                if not all(_same(s[key], prev[key]) for key in ("R", "w", "m", "v", "ring")):
                    bad.append("eval %d rank %d: a skipped evaluation changed the state" % (e, k))
        if skip:
            continue
        # one-shot: a fresh set of ranks with the state before this evaluation and the same partials
        one = _harness(W, size, max_cta=264)
        for k in range(W):
            before = snaps[k][e - 1] if e else dict(w=w0, m=m0, v=v0, step=[0])
            one.set_state(k, before["w"], before["m"], before["v"], before["step"][0])
            one.load(k, 0, parts[e][k])
        one.enqueue(0, form, adam=ADAM if ad else None)
        one.sync()
        ref = xo.tail_sum(parts[e], one.cols)
        for k in range(W):
            o, s = one.read(k), snaps[k][e]
            if not all(_same(s[key], o[key]) for key in ("R", "w", "m", "v")) or not _same(s["R"], ref):
                bad.append("eval %d rank %d: differs from the one-shot run" % (e, k))
            if ad and not _same(s["ring"][(steps - 1) % xo.RING], o["ring"][(o["step"][0] - 1) % xo.RING]):
                bad.append("eval %d rank %d: loss ring entry differs" % (e, k))
        one.close()
    # parities alternate: every published evaluation s wrote parity s & 1, so the two parities hold the last two sequence numbers
    for k in range(W):
        if not (np.all(flags[k][ran & 1] == ran) and np.all(flags[k][(ran - 1) & 1] == ran - 1)):
            bad.append("rank %d: flags %s" % (k, [sorted(set(flags[k][p].ravel().tolist())) for p in (0, 1)]))
    print(json.dumps(dict(bad=bad, ran=ran, adam_steps=steps)))


@pytest.mark.parametrize("size", ["burgers", "32k+1"])
def test_enqueued_sequence_with_skips_equals_one_shot_runs(lib, size):
    r = run_worker("sequence_worker", lib, size)
    assert r["bad"] == [], r["bad"]
    assert r["ran"] == 7 and r["adam_steps"] == 4


# ---------------------------------------------------------------------------------------------------------- e: non-finite
def nonfinite_worker(size):
    n_ctas = [9, 132, 5]
    W = len(n_ctas)
    h = _harness(W, size, max_cta=max(n_ctas), n_snap=4)
    rng = np.random.default_rng(91)
    base = xo.cancelling_ranks(rng, n_ctas, h.stride)
    P = h.P
    # (entry of R, [(rank, cta, value)])
    inserts = [(5, [(0, 0, np.nan)]), (40, [(1, 3, np.inf)]), (41, [(2, 4, -np.inf)]), (h.n_out - 1, [(0, 8, -np.inf)]),
               (P + 1, [(1, 131, np.inf)]), (70, [(0, 8, np.inf), (2, 0, -np.inf)])]
    mod = [p.copy() for p in base]
    for i, hits in inserts:
        for k, b, val in hits:
            mod[k][b, h.cols[i]] = val
    for k in range(W):
        h.load(k, 0, base[k])
    h.enqueue(0, "reduce", snap=0); h.enqueue(0, "fused", snap=1)
    for k in range(W):
        h.load(k, 0, mod[k])
    h.enqueue(0, "reduce", snap=2); h.enqueue(0, "fused", snap=3)
    h.sync()
    with np.errstate(invalid="ignore"):
        ref = xo.tail_sum(mod, h.cols)
    touched = np.zeros(h.n_out, bool)
    touched[[i for i, _ in inserts]] = True
    bad = []
    for k in range(W):
        for snap in (2, 3):
            s, clean = h.read(k, snap), h.read(k, snap - 2)
            if not _same(s["R"][~touched], clean["R"][~touched]) or s["err"] != 0:
                bad.append("rank %d snap %d: an entry without a non-finite value changed" % (k, snap))
            for i, _ in inserts:
                got, want = s["R"][i], ref[i]
                if not ((np.isnan(got) and np.isnan(want)) or got == want):
                    bad.append("rank %d snap %d entry %d: %r, the reference sum is %r" % (k, snap, i, got, want))
    h.close()
    print(json.dumps(dict(bad=bad, classes=[str(float(ref[i])) for i, _ in inserts])))


@pytest.mark.parametrize("size", ["burgers", "32k+1"])
def test_non_finite_entry_takes_the_reference_class_on_every_rank(lib, size):
    r = run_worker("nonfinite_worker", lib, size)
    assert r["bad"] == [], r["bad"]
    assert r["classes"] == ["nan", "inf", "-inf", "-inf", "inf", "nan"]


# ------------------------------------------------------------------------------------- f: sharded models against the oracle
# (W, N): N never divisible by W; with W = 8 and N = 45 every shard (5 or 6 rows) is smaller than a tile
SHARDS = [(2, 4737), (3, 20000), (8, 45)]
NLS_SHARDS = [(2, 1801), (3, 1000), (8, 45)]
KERNELS = {"burgers_v2": ("burgers", {"PINN_BURGERS_KERNEL": "v2"}), "burgers_v1": ("burgers", {"PINN_BURGERS_KERNEL": "v1"}),
           "burgers_generic": ("burgers", {"PINN_FORCE_GENERIC": "1"}), "nls": ("nls", {}),
           "nls_generic": ("nls", {"PINN_FORCE_GENERIC": "1"})}


def burgers_problem(N):
    import test_gpu_precision as tp
    rng = np.random.default_rng(N)
    lb, ub = (np.array(v) for v in tp.DOMAINS["shifted"])
    return dict(lb=lb, ub=ub, X_f=tp.points(rng, lb, ub, N), X_u=tp.points(rng, lb, ub, 100), u=rng.uniform(-1, 1, (100, 1)),
                w=load_golden("burgers_inf")["w"], nu=1.0)


def nls_problem(N):
    import test_gpu_precision as tp
    rng = np.random.default_rng(N + 1)
    lb, ub = (np.array(v) for v in tp.NLS_OTHER)
    tb = np.concatenate([[lb[1], ub[1]], rng.uniform(lb[1], ub[1], 48)])[:, None]
    x0 = np.concatenate([[lb[0], ub[0]], rng.uniform(lb[0], ub[0], 48)])[:, None]
    return dict(lb=lb, ub=ub, X_f=tp.points(rng, lb, ub, N), tb=tb, X0=np.concatenate([x0, 0 * x0 + lb[1]], 1),
                uv0=rng.standard_normal((50, 2)), w=load_golden("nls_inf")["w"])


def _handle(c, model, d, lo, hi, N, weight):
    import test_gpu_precision as tp
    if model == "burgers":
        p = c.Pinn(c.BURGERS_INF, tp.BURGERS, d["lb"], d["ub"])
        p.set_pde_params([d["nu"]])
        p.set_collocation(d["X_f"][lo:hi, 0], d["X_f"][lo:hi, 1], n_global=N)
        p.set_data(d["X_u"], d["u"], weight=weight)
    else:
        p = c.Pinn(c.NLS_INF, tp.NLS, d["lb"], d["ub"])
        p.set_collocation(d["X_f"][lo:hi, 0], d["X_f"][lo:hi, 1], n_global=N)
        p.set_boundary(d["tb"]); p.set_data(d["X0"], d["uv0"], weight=weight)
    return p


def _exchange(vecs, adam_state=None, hp=None):
    """The ranks' [grad | parts] vectors as one-CTA partials through the harness: R on every rank (and the state after an
    Adam step when adam_state = (w, m, v, step0))."""
    W, n = len(vecs), len(vecs[0])
    stride = (n + 15) // 16 * 16
    h = xo.Harness(os.environ["XH_LIB"], W, n, (), stride)
    for k, vec in enumerate(vecs):
        row = np.zeros((1, stride)); row[0, :n] = vec
        h.load(k, 0, row)
        if adam_state is not None:
            h.set_state(k, *adam_state)
    h.enqueue(0, "reduce", adam=hp)
    h.sync()
    out = [h.read(k) for k in range(W)]
    h.close()
    assert all(o["err"] == 0 for o in out)
    return out


def _same_on_all(out, key):
    return all(_same(o[key], out[0][key]) for o in out)


def sharded_worker(kernel):
    import pinn_cabi as c
    import sharding
    c.load()
    model, _ = KERNELS[kernel]
    res = {}
    for W, N in (SHARDS if model == "burgers" else NLS_SHARDS):
        d = burgers_problem(N) if model == "burgers" else nls_problem(N)
        hs = []
        for r in range(W):
            lo, hi = sharding.shard_rows(N, r, W)
            hs.append(_handle(c, model, d, lo, hi, N, sharding.data_weight(r)))
        info = hs[0].kernel_info()
        vecs = []
        for p in hs:
            loss, grad, parts = p.loss_grad(w=d["w"])
            vecs.append(np.concatenate([grad, parts]))
        out = _exchange(vecs)
        R = out[0]["R"]
        entry = dict(R=R.tolist(), identical=_same_on_all(out, "R"), kernel=info)
        if W == 3:                                       # five sharded Adam steps against a whole-set handle
            s = _handle(c, model, d, 0, N, N, 1.0)
            hp = ADAM_BIG if model == "nls" else ADAM
            P = hs[0].P
            w, m, v, step = d["w"].copy(), np.zeros(P), np.zeros(P), 0
            s.set_weights(d["w"])
            losses, whole = [], []
            identical = True
            for _ in range(5):
                vecs = []
                for p in hs:
                    _, grad, parts = p.loss_grad(w=w)
                    vecs.append(np.concatenate([grad, parts]))
                out = _exchange(vecs, (w, m, v, step), hp)
                identical &= all(_same_on_all(out, key) for key in ("w", "m", "v", "ring"))
                w, m, v, step = out[0]["w"], out[0]["m"], out[0]["v"], out[0]["step"][0]
                losses.append(float(out[0]["ring"][(step - 1) % xo.RING]))
                whole.append(s.adam_step(*hp))
            ws = s.get_weights()
            s.close()
            entry.update(adam_identical=bool(identical), adam_steps=step,
                         adam_rel_w=float(np.linalg.norm(w - ws) / np.linalg.norm(ws)),
                         adam_rel_loss=max(abs(a - b) / abs(b) for a, b in zip(losses, whole)))
        for p in hs:
            p.close()
        res["%d/%d" % (W, N)] = entry
    print(json.dumps(res))


_SHARD_RUNS = {}


def _sharded(lib, kernel):
    if kernel not in _SHARD_RUNS:
        _SHARD_RUNS[kernel] = run_worker("sharded_worker", lib, kernel, env=KERNELS[kernel][1])
    return _SHARD_RUNS[kernel]


_ORACLE = {}


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("shard", [0, 1, 2], ids=["W2", "W3", "W8_small_shards"])
def test_sharded_evaluation_against_the_whole_set_oracle(lib, kernel, shard):
    import test_gpu_precision as tp
    from oracle import taylor as ty
    model = KERNELS[kernel][0]
    W, N = (SHARDS if model == "burgers" else NLS_SHARDS)[shard]
    r = _sharded(lib, kernel)["%d/%d" % (W, N)]
    assert r["identical"]
    if kernel.endswith("generic"):
        assert r["kernel"]["dyn_smem"] == 0
    else:
        assert r["kernel"]["dyn_smem"] > 0
    if kernel == "burgers_v1":                                            # the switch took: another kernel ran
        assert r["kernel"] != _sharded(lib, "burgers_v2")["%d/%d" % (W, N)]["kernel"]
    R = np.array(r["R"])
    if model == "burgers":
        d = burgers_problem(N)
        layers, part_idx = tp.BURGERS, (0, 2)
        fn = lambda dt, mg: ty.burgers_loss_grad(d["w"], layers, d["lb"], d["ub"], d["X_f"], d["X_u"], d["u"], nu=d["nu"],
                                                 dtype=dt, magnitudes=mg)
    else:
        d = nls_problem(N)
        layers, part_idx = tp.NLS, (0, 1, 2)
        fn = lambda dt, mg: ty.schrodinger_loss_grad(d["w"], layers, d["lb"], d["ub"], d["X_f"], d["tb"], d["X0"], d["uv0"],
                                                     dtype=dt, magnitudes=mg)
    key = (model, N)
    if key not in _ORACLE:
        _ORACLE[key] = (fn(tp.LD, True), fn(np.float64, False))
    P = len(R) - 3
    parts = R[P:]
    got = ((parts[0] + parts[1]) + parts[2], R[:P], parts)
    tp.check("sharded %s W=%d N=%d" % (kernel, W, N), got, _ORACLE[key][0], _ORACLE[key][1], ty.param_blocks(layers), part_idx)
    if W == 3:
        assert r["adam_identical"] and r["adam_steps"] == 5
        assert r["adam_rel_w"] < 1e-10 and r["adam_rel_loss"] < 1e-10, (r["adam_rel_w"], r["adam_rel_loss"])
        print("[exchange] sharded %s Adam x5: rel w %.2g, rel loss %.2g" % (kernel, r["adam_rel_w"], r["adam_rel_loss"]))


# --------------------------------------------------------------------------------------------- the models that cannot shard
def unshardable_worker(_):
    import pinn_cabi as c
    import sharding
    import test_gpu_precision as tp
    import test_gpu_precision_heads as th
    c.load()
    ide = tp.burgers_inputs(tp.BURGERS_CASES[11], 132)                   # ide_std: 2000 data points
    disc, ide_disc = tp.disc_inputs(tp.DISC_CASES[0]), tp.disc_inputs(tp.DISC_CASES[2])
    kdv, ac = th.kdv_inputs(th.KDV_CASES[1], 132), th.ac_inputs(th.AC_CASES[2], 132)

    def make(pde, weight):
        if pde == c.BURGERS_IDE:
            p = c.Pinn(pde, tp.BURGERS, ide["lb"], ide["ub"]); p.set_data(ide["X_u"], ide["u"], weight=weight)
            return p, ide["w"]
        if pde == c.BURGERS_DISC:
            p = c.Pinn(pde, disc["layers"], tp.DISC_LB, tp.DISC_UB)
            p.set_pde_params([disc["nu"], disc["dt"]]); p.set_irk(disc["IRK"]); p.set_boundary(disc["x_1"])
            p.set_data(disc["x_0"], disc["u_0"], weight=weight)
            return p, disc["w"]
        if pde in (c.BURGERS_IDE_DISC, c.KDV_IDE_DISC):
            d = ide_disc if pde == c.BURGERS_IDE_DISC else kdv
            lb, ub = (tp.DISC_LB, tp.DISC_UB) if pde == c.BURGERS_IDE_DISC else (d["lb"], d["ub"])
            p = c.Pinn(pde, d["layers"], lb, ub)
            p.set_pde_params([d["dt"]]); p.set_irk(c.irk_ide_disc(d["alpha"], d["beta"]))
            p.set_snapshot(0, d["x_0"], d["u_0"]); p.set_snapshot(1, d["x_1"], d["u_1"])     # no data weight to set
            return p, d["w"]
        p = c.Pinn(pde, ac["layers"], ac["lb"], ac["ub"])
        p.set_pde_params([ac["dt"], ac["d"], ac["k"]]); p.set_irk(ac["irk"]); p.set_data(ac["x_0"], ac["u_0"], weight=weight)
        return p, ac["w"]

    out = {}
    for pde in (c.BURGERS_IDE, c.BURGERS_DISC, c.BURGERS_IDE_DISC, c.KDV_IDE_DISC, c.AC_DISC):
        p, w = make(pde, 1.0)
        whole = p.loss_grad(w=w)[2]
        p.close()
        for W in (2, 3):
            vecs = []
            for r in range(W):
                p, w = make(pde, sharding.data_weight(r))
                loss, grad, parts = p.loss_grad(w=w)
                vecs.append(np.concatenate([grad, parts]))
                p.close()
            o = _exchange(vecs)
            out["%d/%d" % (pde, W)] = dict(whole=whole.tolist(), sharded=o[0]["R"][-3:].tolist())
    print(json.dumps(out))


UNSHARDABLE = {1: "Burgers identification", 3: "Burgers discrete", 4: "Burgers discrete identification", 5: "KdV",
               6: "Allen-Cahn"}


@pytest.fixture(scope="module")
def unshardable(lib):
    return run_worker("unshardable_worker", lib)


@pytest.mark.parametrize("pde", sorted(UNSHARDABLE), ids=[UNSHARDABLE[k] for k in sorted(UNSHARDABLE)])
def test_models_without_a_sharded_loss_are_refused(unshardable, pde):
    """Composed under the sharding contract (collocation rows with the global 1/N, replicated terms weighted by
    sharding.data_weight), these models do not give the whole-set loss: Burgers identification counts its residual on every
    rank, the discrete-time heads count everything on every rank.  So pinn_create refuses world > 1 for them."""
    import pinn_cabi as c
    for W in (2, 3):
        r = unshardable["%d/%d" % (pde, W)]
        whole, sharded = np.array(r["whole"]), np.array(r["sharded"])
        if pde == c.BURGERS_IDE:
            np.testing.assert_allclose(sharded[[0, 2]], [whole[0], W * whole[2]], rtol=1e-12)
        else:
            np.testing.assert_allclose(sharded.sum(), W * whole.sum(), rtol=1e-12)
    with pytest.raises(c.PinnError, match="world must be 1"):
        c.Pinn(pde, [2, 20, 1] if pde == c.BURGERS_IDE else [1, 20, 3], [-1.0, 0.0], [1.0, 1.0], rank=1, world=2)
