"""GPU: what a handle returns depends on its CURRENT inputs only, never on how it got there.

A pinn_t lives for a whole training run: it is re-fed per fit, its collocation set is resampled per step, Adam and L-BFGS run on
it in turn.  Between calls the host side of pinn_api.cu keeps point storage in two regions with their own capacities (the data
block right-aligned in its region), auxiliary blocks re-assembled from host copies, grow-only scratch keyed on one number, device
counters of the evaluation tail, the L-BFGS history and Gram buffers, the source and the polynomial spec.  Every other GPU test
feeds a fresh handle once, in one order.  Here a handle is driven through a seeded HISTORY of setter and evaluation calls and is
then compared with a FRESH handle fed the same final inputs in canonical order.  Same kernel, same grid (a function of the current
counts and the SM count), same summation order: loss, parts, gradient, residual, probes, constants and weights must be equal
BIT FOR BIT, so there is no tolerance and many histories are affordable.  So that both handles cannot be wrong the same way, the
first history of every family also holds the fresh handle to the fp64 Taylor oracle at the 1e-10 of that family's own GPU file.

The sizes come from a ladder that crosses every capacity rule of pinn_api.cu (restated in CapModel; tests/test_handle_state_cpu.py
asserts at 132 SMs that the ladder reaches what it claims, runs the same histories on the CPU oracle stand-in and shows that four
broken stand-ins are rejected).  The optimiser tests compare handles with each other: L-BFGS between two Adam phases must not
disturb the moments, the step count or the tail's counters; a second L-BFGS run must not see the first one's history; adam_reset
must give a fresh trajectory; a resampled collocation batch must give the same step whichever path and capacity history brought
it; a refused call must leave the handle as it was.  A failure message names the family and the seed: generate(FAMILIES[name],
seed, sms) replays it."""
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import itertools

from conftest import ROOT

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
EPS = float(np.finfo(float).eps)
SEEDS = tuple(range(10))

BURGERS = [2] + [20] * 8 + [1]
STD = ([-1.0, 0.0], [1.0, 0.99])
SHIFTED = ([0.3, -0.5], [3.7, 2.0])
# kind: which setters the family takes.  env: kernel switches that are read once per process, so the family runs in a worker.
FAMILIES = {
    "burgers_inf": dict(pde="BURGERS_INF", kind="inf", layers=BURGERS, box=STD, mapped=True),
    "burgers_inf_v1": dict(pde="BURGERS_INF", kind="inf", layers=BURGERS, box=STD, env={"PINN_BURGERS_KERNEL": "v1"}),
    "burgers_ide": dict(pde="BURGERS_IDE", kind="ide", layers=BURGERS, box=STD),
    "burgers_ide_v1": dict(pde="BURGERS_IDE", kind="ide", layers=BURGERS, box=STD, env={"PINN_BURGERS_KERNEL": "v1"}),
    "nls": dict(pde="NLS_INF", kind="nls", layers=[2, 100, 100, 100, 100, 2], box=([-5.0, 0.0], [5.0, np.pi / 2])),
    "nls_generic": dict(pde="NLS_INF", kind="nls", layers=[2, 100, 100, 100, 100, 2], box=([-5.0, 0.0], [5.0, np.pi / 2]),
                        env={"PINN_FORCE_GENERIC": "1"}),
    "generic_w24": dict(pde="BURGERS_INF", kind="inf", layers=[2, 24, 24, 24, 1], box=SHIFTED),
    "generic_w24_dfma": dict(pde="BURGERS_INF", kind="inf", layers=[2, 24, 24, 24, 1], box=SHIFTED, env={"PINN_GENERIC_DFMA": "1"}),
    "generic_w256": dict(pde="BURGERS_IDE", kind="ide", layers=[2, 256, 40, 1], box=SHIFTED),
    "burgers_disc": dict(pde="BURGERS_DISC", kind="disc", layers=[1, 30, 30, 9], box=([-1.0], [1.0])),
    "ac_disc": dict(pde="AC_DISC", kind="disc", layers=[1, 30, 30, 9], box=([-1.0], [1.0])),
    "burgers_ide_disc": dict(pde="BURGERS_IDE_DISC", kind="ide_disc", layers=[1, 30, 30, 8], box=([-1.0], [1.0])),
    "kdv_ide_disc": dict(pde="KDV_IDE_DISC", kind="ide_disc", layers=[1, 30, 30, 8], box=([-0.5], [2.0])),
    "ns": dict(pde="NS_IDE", kind="ns", layers=[3, 24, 256, 2], box=([1.0, -2.0, 0.0], [8.0, 2.0, 20.0])),
    "poly_inf": dict(pde="POLY_INF", kind="inf", poly=True, layers=[2, 20, 20, 20, 1], box=STD),
    "poly_ide": dict(pde="POLY_IDE", kind="ide", poly=True, layers=[2, 20, 20, 20, 1], box=STD),
}
for _name, _fam in FAMILIES.items():
    _fam["name"] = _name

# canonical order of the slots of a state; a state maps slot -> the setter call (method, args, kwargs) that fills it
CANON = ("params", "irk", "spec", "coll", "data", "snap0", "snap1", "boundary", "source", "weights")
SPECS_INF = [
    [(1.0, 0, (0, 0, 1, 0)), (1.0, 0, (1, 1, 0, 0)), (-0.02, 0, (0, 0, 0, 1))],
    [(1.0, 0, (0, 0, 1, 0)), (-1e-2, 0, (0, 0, 0, 1)), (5.0, 0, (3, 0, 0, 0)), (-5.0, 0, (1, 0, 0, 0)), (0.3, 0, (1, 0, 1, 0)),
     (0.1, 0, (2, 1, 0, 0))],
    [(1.0, 0, (0, 0, 1, 0)), (-0.1, 0, (0, 0, 0, 1))],
]
SPECS_IDE = [
    [(1.0, 0, (0, 0, 1, 0)), (1.0, 1, (1, 1, 0, 0)), (-1.0, 4, (0, 0, 0, 1))],
    [(1.0, 0, (0, 0, 1, 0)), (-1.0, 4, (0, 0, 0, 1)), (-1.0, 1, (1, 0, 0, 0)), (1.0, 1, (2, 0, 0, 0)), (0.2, 2, (1, 1, 0, 0))],
    [(1.0, 0, (0, 0, 1, 0)), (-0.5, 3, (0, 0, 0, 1))],
]


def has_lambdas(fam):
    return fam["kind"] in ("ide", "ide_disc", "ns")


def slots_of(fam):
    s = {"inf": ["params", "coll", "data"], "ide": ["data"], "nls": ["coll", "data", "boundary"],
         "disc": ["params", "irk", "data", "boundary"], "ide_disc": ["params", "irk", "snap0", "snap1"], "ns": ["data"]}[fam["kind"]]
    s = [v for v in s if not (v == "boundary" and fam["pde"] == "AC_DISC")]
    if fam.get("poly"):
        s = [v for v in s if v != "params"] + ["spec", "source"]
    return s + ["weights"]


def residual_slot(fam):
    """The slot holding the residual points (None: the discrete-time models have no residual probe)."""
    return {"inf": "coll", "nls": "coll", "ide": "data", "ns": "data"}.get(fam["kind"])


# ------------------------------------------------------------------------------------------------------------------ ladder
def ladder(fam, sms):
    """Sizes per slot.  1024 is the initial capacity of the data region; need + need/4 + 1024 (data) and need + need/8 + 1024
    (collocation) are odd for 1025 and 8 * 132 + 1, even for 1500 and 2400; 8 x SMs and 32 x SMs points are the chains-per-CTA
    switch points of the Burgers kernel, 16 x 2 x SMs the step of the generic kernel's points per CTA from 16 to 32, 16 x SMs
    that of the Schrodinger kernel; 0 and 1 are the smallest sets the header allows."""
    base = [1, 2, 7, 8, 9, 100, 255, 1023, 1024, 1025, 8 * sms, 8 * sms + 1, 1500, 2400, 16 * sms + 1, 32 * sms - 1, 32 * sms + 1,
            6000, 9000]
    small = [1, 2, 7, 8, 9, 50, 51, 100, 255, 600, 1023, 1025, 1500]
    kind = fam["kind"]
    if kind == "inf":
        return {"coll": base, "data": [0, 0] + base[:-1], "mapped": base + [12000]}
    if kind == "ide":
        return {"data": base}
    if kind == "nls":
        return {"coll": base, "data": small, "boundary": [0, 1, 2, 7, 50, 51, 100, 600]}
    if kind == "disc":
        return {"data": small, "boundary": [1, 2, 7, 50, 51, 300, 1100, 2300]}
    if kind == "ide_disc":
        return {"snap0": small, "snap1": small}
    return {"data": [1, 7, 9, sms - 1, sms, sms + 1, 300, 1000, 16 * sms + 3, 5000]}


class CapModel(object):
    """The capacity rules of pinn_api.cu (ensure_points, upload_points, pinn_set_collocation[_mapped], and Scratch::reserve
    in generic_launch_eval), restated for the continuous-time inference handles, so that a history can be asked what it
    exercised."""

    def __init__(self, sms):
        self.sms, self.dcap, self.ccap, self.alloc = sms, 0, 0, False
        self.n_d = self.n_c = 0
        self.mapped = False
        self.g_pts = 0
        self.events = set()

    def _ensure(self, need_d, need_c):
        if need_d <= self.dcap and need_c <= self.ccap and self.alloc:
            return
        keep_c = 0 if self.mapped else min(self.n_c, self.ccap)
        if self.alloc:
            if need_d > self.dcap and keep_c:
                self.events.add("data region regrown with a device collocation block present")
            if need_c > self.ccap and self.n_d:
                self.events.add("collocation region regrown with a data block present")
        if need_d > self.dcap:
            self.dcap = need_d + need_d // 4 + 1024
        if need_c > self.ccap:
            self.ccap = need_c + need_c // 8 + 1024
        self.dcap = max(self.dcap, 1024)
        self.alloc = True

    def step(self, method, n):
        if method == "set_collocation":
            self._ensure(self.n_d, n)
            if self.mapped:
                self.events.add("mapped -> copied")
            self.n_c, self.mapped = n, False
        elif method == "set_collocation_mapped":
            self._ensure(self.n_d, 0)
            if self.n_c and not self.mapped:
                self.events.add("copied -> mapped")
            self.n_c, self.mapped = n, True
        elif method == "set_data":
            if n < self.n_d:
                self.events.add("data block shrunk")
            if self.mapped and n > self.dcap:
                self.events.add("data region regrown under a mapped batch")
            self._ensure(n, self.n_c)
            self.n_d = n
            self.events.add("dcap - n %s" % ("odd" if (self.dcap - n) % 2 else "even"))
        elif method == "eval" and self.n_c + self.n_d:
            per = -(-(self.n_c + self.n_d) // (2 * self.sms))
            pts = -(-per // 16) * 16 if per >= 16 else -(-per // 2) * 2
            if pts > self.g_pts:
                if self.g_pts:
                    self.events.add("scratch regrown for more points per CTA")
                self.g_pts = pts
            elif pts < self.g_pts:
                self.events.add("points per CTA below the scratch's")


def coverage(fam, steps, sms):
    """Events of CapModel over a history, plus the orders and switches the generator drew."""
    m, ev, seen = CapModel(sms), set(), []
    for slot, method, args, kw in steps:
        if slot == "eval":
            m.step("eval", 0)
            continue
        seen.append(method)
        if slot in ("coll", "data"):
            n = len(args[0])
            m.step(method, n)
            if slot == "data":
                ev.add("in_dim %d" % (1 if np.ndim(args[0]) == 1 or np.shape(args[0])[1] == 1 else 2))
                ev.add("weight %g" % kw.get("weight", 1.0))
                ev.add("data n = 0" if n == 0 else "data n > 0")
            if slot == "coll" and kw.get("n_global") not in (None, n):
                ev.add("n_global > n")
    first = [s for s in seen if s in ("set_data", "set_collocation", "set_collocation_mapped", "set_boundary")]
    if first:
        ev.add("first: " + first[0])
    return ev | m.events


# --------------------------------------------------------------------------------------------------------------- generator
def _rng(fam, seed, salt=0):
    return np.random.default_rng([seed, zlib.crc32(fam["name"].encode()), salt])


def _box(fam, rng, n, cols=None):
    lb, ub = (np.asarray(v, float) for v in fam["box"])
    X = lb + (ub - lb) * rng.random((n, lb.size))
    return X if cols is None else X[:, :cols]


def draw(fam, slot, rng, n, state, variants=True):
    """One setter call (slot, method, args, kwargs) with n points; `variants` lets it pick the zero-copy call, the (N,1)
    broadcast, a data weight, n_global > n."""
    kind, q = fam["kind"], fam["layers"][-1]
    pick = (lambda *v: v[int(rng.integers(len(v)))]) if variants else (lambda *v: v[0])
    if slot == "params":
        p = {"BURGERS_INF": [pick(0.01 / np.pi, 0.05, 1.0)], "BURGERS_DISC": [pick(0.01 / np.pi, 0.1), pick(0.8, 0.3)],
             "AC_DISC": [pick(0.8, 0.4), pick(1e-4, 1e-2), pick(5.0, 2.0)]}.get(fam["pde"], [pick(0.6, 0.2)])
        return (slot, "set_pde_params", (p,), {})
    if slot == "irk":
        if kind == "ide_disc":
            import pinn_cabi
            a, b = (rng.standard_normal((q, q)) / q).astype(np.float32), (rng.standard_normal((1, q)) / q).astype(np.float32)
            return (slot, "set_irk", (pinn_cabi.irk_ide_disc(a, b),), {"_tables": (a, b)})
        return (slot, "set_irk", (rng.standard_normal((q, q - 1)) / (q - 1),), {})
    if slot == "spec":
        specs = SPECS_IDE if kind == "ide" else SPECS_INF
        return (slot, "set_residual", (specs[int(rng.integers(len(specs)))],), {})
    if slot == "source":
        n_res = len(state[residual_slot(fam)][1][0])
        return (slot, "set_source", (rng.standard_normal(n_res),), {})
    if slot == "weights":
        wr, L = np.random.default_rng(int(rng.integers(1 << 31))), fam["layers"]      # one draw, whatever the net's size
        w = np.concatenate([np.concatenate([wr.standard_normal(a * b) * np.sqrt(2.0 / (a + b)), 0.05 * wr.standard_normal(b)])
                            for a, b in zip(L[:-1], L[1:])])
        if has_lambdas(fam):
            w = np.concatenate([w, [rng.uniform(0.3, 1.0), rng.uniform(-3.0, -1.0)]])
        return (slot, "set_weights", (w,), {})
    if slot == "coll":
        X = _box(fam, rng, n)
        kw = {"n_global": n + pick(0, 0, 17, 3 * n)} if n else {}
        method = "set_collocation_mapped" if fam.get("mapped") and n and pick(0, 1, 1) else "set_collocation"
        return (slot, method, (X[:, 0].copy(), X[:, 1].copy()), kw)
    if slot == "boundary":
        return (slot, "set_boundary", (_box(fam, rng, n)[:, -1:].copy(),), {})
    if slot in ("snap0", "snap1"):
        x = _box(fam, rng, n)
        u = (1.0 if slot == "snap0" else 0.5) * np.cos(np.pi * x)
        if slot == "snap0" and pick(0, 1):
            return (slot, "set_data", (x, u), {})                      # pinn_set_data == snapshot 0
        return (slot, "set_snapshot", (int(slot[-1]), x, u), {})
    assert slot == "data"
    if kind == "ns":
        return (slot, "set_data", (_box(fam, rng, n), rng.standard_normal((n, 2))), {})
    if kind == "disc":
        x = _box(fam, rng, n)
        return (slot, "set_data", (x, x ** 2 * np.cos(np.pi * x)), {})
    X = _box(fam, rng, n, cols=pick(2, 2, 1) if kind in ("inf", "nls") else 2)
    u = rng.uniform(-1, 1, (n, q))
    kw = {"weight": pick(1.0, 1.0, 0.0, 3.0)} if kind in ("inf", "nls") else {}
    return (slot, "set_data", (X, u), kw)


def track(fam, state, step):
    """What a setter call leaves in the handle: its own slot, as the call that a fresh handle is fed with."""
    slot, method, args, kw = step
    if method == "set_collocation_mapped":
        method = "set_collocation"                                     # the same batch, copied
    if slot == "snap0" and method == "set_data":
        method, args = "set_snapshot", (0,) + tuple(args)
    state[slot] = (method, args, kw)
    if fam.get("poly") and slot == residual_slot(fam):
        state.pop("source", None)                                      # new residual points: the source is zero again


def evaluable(fam, state):
    return all(s in state for s in slots_of(fam) if s != "source")


def generate(fam, seed, sms):
    """-> (steps, final state).  Round 0 and the last round call every setter in a random order, the rounds between a random
    subset; evaluations are interleaved so that scratch is sized by intermediate states ("eval" steps whose args[1] is True
    are checkpoints: the handle is compared with a fresh one there too)."""
    rng, lad, slots = _rng(fam, seed), ladder(fam, sms), slots_of(fam)
    steps, state = [], {}
    evals = ["loss_grad", "predict", "derivatives"] + (["residual"] if residual_slot(fam) else []) + \
            (["probe_chunks"] if fam["kind"] == "ns" else [])
    n_rounds = 3 + int(rng.integers(3))
    for r in range(n_rounds):
        last = r == n_rounds - 1
        todo = [s for s in slots if r == 0 or last or rng.random() < 0.55]
        if fam.get("poly") and not last and rng.random() < 0.5 and "source" in todo:
            todo.remove("source")
        if last and fam.get("poly") and rng.random() < 0.4:
            todo.remove("source")                                      # final state: the source that the points reset
        todo = [todo[i] for i in rng.permutation(len(todo))]
        if r == 0:                                                     # the point setters' first order: every one, over the seeds
            pts = [s for s in todo if s in lad]
            perms = list(itertools.permutations(sorted(pts)))
            it = iter(perms[seed % len(perms)])
            todo = [next(it) if s in lad else s for s in todo]
        if "source" in todo and residual_slot(fam) in todo:            # a source is computed for the points it follows
            todo.remove("source")
            i = todo.index(residual_slot(fam))
            todo.insert(i + 1 + int(rng.integers(len(todo) - i)), "source")
        for slot in todo:
            if slot == "source" and residual_slot(fam) not in state:
                continue
            sizes, n = lad["mapped"] if slot == "coll" and fam.get("mapped") else lad.get(slot), 0
            if sizes:
                n = sizes[int(rng.integers(len(sizes)))]
                if slot in state and rng.random() < 0.25:              # the same count again: only the contents change
                    n = len(state[slot][1][-1])
                if last and n == 0:                                    # the oracle of the final state needs every mean defined
                    n = [v for v in sizes if v][int(rng.integers(len(sizes) - sizes.count(0)))]
            step = draw(fam, slot, rng, n, state)
            if slot == "coll" and step[1] == "set_collocation" and n > 9000:
                step = draw(fam, slot, rng, 9000, state)               # only a mapped batch exceeds every copied set
            steps.append(step)
            track(fam, state, step)
            if evaluable(fam, state) and rng.random() < 0.4:
                steps.append(("eval", evals[int(rng.integers(len(evals)))], (None, False), {}))
        if not last and evaluable(fam, state):
            steps.append(("eval", "loss_grad", (None, bool(rng.random() < 0.35)), {}))
    return steps, state


def fixed_state(fam, seed, sizes):
    """A complete state with the given size per point slot, every setter in its plain form."""
    rng, state = _rng(fam, seed, 1), {}
    for slot in [s for s in CANON if s in slots_of(fam)]:
        track(fam, state, draw(fam, slot, rng, sizes.get(slot, 0), state, variants=False))
    return state


# ---------------------------------------------------------------------------------------------------------------- backend
class GpuBackend(object):
    """The handles of libpinn_b200.so through the ctypes binding."""

    def __init__(self):
        import pinn_cabi
        pinn_cabi.load()
        self.cabi = pinn_cabi
        self.Error = pinn_cabi.PinnError
        self._sms = None

    def create(self, fam):
        p = self.cabi.Pinn(getattr(self.cabi, fam["pde"]), fam["layers"], fam["box"][0], fam["box"][1])
        p._pinned = []
        return p

    def sms(self):
        if self._sms is None:
            p = self.cabi.Pinn(self.cabi.BURGERS_INF, BURGERS, [-1, 0], [1, 1])
            self._sms = p.kernel_info()["sms"]
            p.close()
        return self._sms

    def set_mapped(self, p, x, t, n_global=None):
        dp = C.POINTER(C.c_double)
        bufs = []
        for v in (x, t):
            arr, ptr = self.cabi.host_alloc(len(v))
            arr[:] = v
            p._pinned.append(ptr)
            bufs.append(C.cast(ptr, dp))
        p.set_collocation_mapped(bufs[0], bufs[1], len(x), n_global)

    def close(self, p):
        p.close()                                                      # synchronises the stream: no launch reads the buffers now
        for ptr in p._pinned:
            p.lib.pinn_host_free(ptr)
        p._pinned = []


def apply(backend, p, step):
    slot, method, args, kw = step
    kw = {k: v for k, v in kw.items() if not k.startswith("_")}
    if method == "set_collocation_mapped":
        backend.set_mapped(p, *args, **kw)
    else:
        getattr(p, method)(*args, **kw)


def feed_canonical(backend, fam, state):
    p = backend.create(fam)
    for slot in CANON:
        if slot in state:
            apply(backend, p, (slot,) + tuple(state[slot]))
    return p


def probe_points(fam, n=64):
    return _box(fam, np.random.default_rng(7), n)


def run_eval(backend, p, fam, name):
    if name == "loss_grad":
        return p.loss_grad()
    if name == "predict":
        return p.predict(probe_points(fam))
    if name == "derivatives":
        return p.derivatives(probe_points(fam))
    if name == "probe_chunks":            # Navier-Stokes probe over three chunks of (32 Mi) / (2 x 13 x maxw) points, then one
        maxw = max(fam["layers"][1:-1])
        return p.derivatives(probe_points(fam, 2 * ((32 << 20) // (26 * maxw)) + 50))
    return p.residual()


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def same(a, b):
    a, b = bits(a), bits(b)
    return a.shape == b.shape and bool(np.all(a == b))


def observe(backend, p, fam):
    """Everything a caller can read back from a handle, as a dict of arrays."""
    loss, grad, parts = p.loss_grad()
    d = p.derivatives(probe_points(fam))
    out = {"loss": loss, "grad": grad, "parts": parts, "weights": p.get_weights(), "params": p.get_params(),
           "predict": p.predict(probe_points(fam)), "derivatives": d if fam["kind"] == "ns" else np.stack(d)}
    if residual_slot(fam):
        out["residual"] = p.residual()
    return out


def assert_same(backend, fam, p, q, tag):
    a, b = observe(backend, p, fam), observe(backend, q, fam)
    bad = [k for k in a if not same(a[k], b[k])]
    assert not bad, "%s: %s differ between the handle with a history and the fresh one (loss %r vs %r)" % (
        tag, bad, a["loss"], b["loss"])


# ----------------------------------------------------------------------------------------------------------- oracle guard
def oracle_loss_grad(fam, state):
    """fp64 Taylor oracle of the state: (loss, gradient)."""
    from oracle import taylor as ty, taylor_kdv_ac as tk, taylor_ns as tn, taylor_poly as tpo
    layers, (lb, ub) = fam["layers"], (np.asarray(v, float) for v in fam["box"])
    w = state["weights"][1][0]
    kind, pde = fam["kind"], fam["pde"]
    if kind in ("inf", "ide"):
        X_u, u = state["data"][1]
        X_u = np.concatenate([X_u, X_u], 1) if X_u.shape[1] == 1 else X_u
        kw = {}
        if kind == "inf":
            x, t = state["coll"][1]
            kw = dict(n_f_global=state["coll"][2].get("n_global"), data_weight=state["data"][2].get("weight", 1.0))
            X_f = np.stack([x, t], 1)
        if fam.get("poly"):
            src = state["source"][1][0] if "source" in state else None
            r = tpo.poly_loss_grad(w, layers, lb, ub, state["spec"][1][0], X_u, u, X_f=None if kind == "ide" else X_f, source=src,
                                   identification=kind == "ide", **kw)
        elif kind == "ide":
            r = ty.burgers_loss_grad(w, layers, lb, ub, None, X_u, u, identification=True)
        else:
            r = ty.burgers_loss_grad(w, layers, lb, ub, X_f, X_u, u, nu=state["params"][1][0][0], **kw)
    elif kind == "nls":
        x, t = state["coll"][1]
        X0, uv0 = state["data"][1]
        X0 = np.concatenate([X0, X0], 1) if X0.shape[1] == 1 else X0
        r = ty.schrodinger_loss_grad(w, layers, lb, ub, np.stack([x, t], 1), state["boundary"][1][0], X0, uv0,
                                     n_f_global=state["coll"][2].get("n_global"), aux_weight=state["data"][2].get("weight", 1.0))
    elif kind == "disc":
        x_0, u_0 = state["data"][1]
        c = state["params"][1][0]
        if pde == "AC_DISC":
            r = tk.ac_disc_loss_grad(w, layers, lb, ub, x_0, u_0, c[0], state["irk"][1][0], d=c[1], k=c[2])
        else:
            r = ty.burgers_disc_loss_grad(w, layers, lb, ub, x_0, u_0, state["boundary"][1][0], c[0], c[1], state["irk"][1][0])
    elif kind == "ide_disc":
        (_, x_0, u_0), (_, x_1, u_1) = state["snap0"][1], state["snap1"][1]
        a, b = state["irk"][2]["_tables"]
        f = tk.kdv_ide_disc_loss_grad if pde == "KDV_IDE_DISC" else ty.burgers_ide_disc_loss_grad
        r = f(w, layers, lb, ub, x_0, u_0, x_1, u_1, state["params"][1][0][0], a, b)
    else:
        r = tn.ns_ide_loss_grad(w, layers, lb, ub, *state["data"][1])
    return float(r[0]), np.asarray(r[1], float)


def assert_matches_oracle(fam, state, p, tag):
    loss, grad, _ = p.loss_grad()
    f2, g2 = oracle_loss_grad(fam, state)
    assert abs(loss - f2) <= 1e-10 * abs(f2), (tag, loss, f2)
    assert np.linalg.norm(grad - g2) <= 1e-10 * np.linalg.norm(g2), tag


# -------------------------------------------------------------------------------------------------------------- histories
def run_history(backend, fam, seed, guard=False):
    """Drive one handle through history `seed`; compare it with a fresh handle at the checkpoints and at the end."""
    steps, final = generate(fam, seed, backend.sms())
    tag = "%s, seed %d" % (fam["name"], seed)
    p, state, n_cmp = backend.create(fam), {}, 0
    try:
        for i, step in enumerate(steps):
            if step[0] != "eval":
                apply(backend, p, step)
                track(fam, state, step)
                continue
            run_eval(backend, p, fam, step[1])
            if step[2][1]:
                q = feed_canonical(backend, fam, state)
                assert_same(backend, fam, p, q, "%s, checkpoint after step %d of %d" % (tag, i, len(steps)))
                backend.close(q)
                n_cmp += 1
        assert sorted(state) == sorted(final)
        q = feed_canonical(backend, fam, final)
        assert_same(backend, fam, p, q, tag + ", final state")
        if guard:
            assert_matches_oracle(fam, final, q, tag)
        backend.close(q)
    finally:
        backend.close(p)
    return len(steps), n_cmp + 1


def run_family(name, seeds=SEEDS, backend=None):
    backend = backend or GpuBackend()
    fam = FAMILIES[name]
    tot = [run_history(backend, fam, s, guard=(s == seeds[0])) for s in seeds]
    print("[handle state] %-18s %d histories, %d calls, %d comparisons with a fresh handle: no mismatch" % (
        name, len(tot), sum(t[0] for t in tot), sum(t[1] for t in tot)))


def run_worker(call, env):
    """`call` of this module in a fresh interpreter with env set (the kernel switches are read once per process)."""
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_handle_state as m; m.%s" % (ROOT, TESTS, call)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-1500:] + r.stderr[-3000:])
    print(r.stdout.strip())


@pytest.mark.parametrize("name", list(FAMILIES))
def test_history_leaves_the_handle_equal_to_a_fresh_one(name):
    if FAMILIES[name].get("env"):
        run_worker("run_family(%r)" % name, FAMILIES[name]["env"])
    else:
        run_family(name)


# --------------------------------------------------------------------------------------------------- optimiser sequencing
OPT_SIZES = {"inf": {"coll": 3000, "data": 100}, "ide": {"data": 1500}, "nls": {"coll": 3000, "data": 51, "boundary": 50},
             "ns": {"data": 700}}
LR = 1e-3


def adam_phase(p):
    """Two synchronous steps, three enqueued by one call, one asynchronous: the per-step losses that can be read, then the ring's
    last slot (host step count against the device's)."""
    out = [p.adam_step(LR), p.adam_step(LR)]
    p.adam_steps(3, LR)
    out.append(p.last_loss())
    p.adam_step(LR, sync=False)
    out.append(p.last_loss())
    return out


def check_adam_lbfgs_adam(name, early, backend=None):
    """Adam, L-BFGS, Adam on handle A == Adam, set_weights(A's weights after L-BFGS), Adam on handle B; then adam_reset and the
    first weights give the first phase again.  early: the L-BFGS run meets its tolerance inside a sync_every batch, so the
    batch's trailing launches are skipped through run_flag."""
    backend = backend or GpuBackend()
    fam = FAMILIES[name]
    state = fixed_state(fam, 3, OPT_SIZES[fam["kind"]])
    w0 = state["weights"][1][0]
    A, B = feed_canonical(backend, fam, state), feed_canonical(backend, fam, state)
    la1 = adam_phase(A)
    wa1 = A.get_weights()
    kw = dict(max_iter=6, tol_fun=EPS)
    if early:
        # |g|_1 at the point a 6-iteration run evaluates last: a long run with that tolerance stops there (iteration 5) or before
        S = feed_canonical(backend, fam, state)
        S.set_weights(wa1)
        S.lbfgs(6, learning_rate=0.5, n_correction=20, tol_fun=EPS, sync_every=1)
        kw = dict(max_iter=40, tol_fun=float(np.sum(np.abs(S.loss_grad()[1]))) * (1 + 1e-9))
        backend.close(S)
    r = A.lbfgs(learning_rate=0.5, n_correction=20, sync_every=4, **kw)
    if early:
        assert r["n_iter"] <= 5 and r["reason"] != 1, r["reason_str"]
    wl = A.get_weights()
    la2 = adam_phase(A)
    assert same(adam_phase(B), la1) and same(B.get_weights(), wa1), name
    B.set_weights(wl)
    lb2 = adam_phase(B)
    assert same(la2, lb2), "%s: Adam after L-BFGS (%s) differs from Adam after set_weights: %r vs %r" % (name, r["reason_str"], la2, lb2)
    assert same(A.get_weights(), B.get_weights()), name
    A.adam_reset()
    A.set_weights(w0)
    assert same(adam_phase(A), la1) and same(A.get_weights(), wa1), name + ": adam_reset + set_weights is not a fresh start"
    backend.close(A)
    backend.close(B)
    print("[handle state] %-18s Adam / L-BFGS (%s, %d iterations) / Adam / reset: no mismatch" % (name, r["reason_str"], r["n_iter"]))


def lbfgs_run(p, max_iter, n_corr):
    logged = []
    r = p.lbfgs(max_iter, learning_rate=0.5, n_correction=n_corr, tol_fun=EPS, sync_every=3,
                log_fn=lambda it, f: logged.append((it, f)), want_x_final=True)
    return {"counts": [r["n_iter"], r["n_eval"], r["reason"]], "f_hist": r.get("f_hist", []), "x_final": r["x_final"],
            "logged": [v for it, f in logged for v in (it, f)], "weights": p.get_weights()}


# (first run, second run) as (max_iter, n_correction): fewer pairs and more iterations (iteration buffers reallocated, the ring
# overflows), more pairs and fewer iterations (buffers reused)
LBFGS_PAIRS = [((8, 50), (12, 7)), ((12, 7), (6, 50)), ((9, 3), (9, 5))]


def check_lbfgs_twice(name, backend=None, pairs=LBFGS_PAIRS):
    """A second pinn_lbfgs run on a handle == the same run on a fresh handle started from the same weights."""
    backend = backend or GpuBackend()
    fam = FAMILIES[name] if isinstance(name, str) else name
    name = fam["name"]
    state = fixed_state(fam, 4, OPT_SIZES[fam["kind"]])
    for first, second in pairs:
        A = feed_canonical(backend, fam, state)
        lbfgs_run(A, *first)
        w1 = A.get_weights()
        a = lbfgs_run(A, *second)
        B = feed_canonical(backend, fam, state)
        B.set_weights(w1)
        b = lbfgs_run(B, *second)
        bad = [k for k in a if not same(a[k], b[k])]
        assert not bad, "%s: L-BFGS %r after %r differs from the same run on a fresh handle in %s" % (name, second, first, bad)
        backend.close(A)
        backend.close(B)
    print("[handle state] %-18s L-BFGS twice, %d pairs of runs: no mismatch" % (name, len(pairs)))


OPT_FAMILIES = ["burgers_inf", "generic_w24", "nls", "ns"]


@pytest.mark.parametrize("early", [False, True], ids=["max_iter", "tolerance"])
@pytest.mark.parametrize("name", OPT_FAMILIES)
def test_lbfgs_between_two_adam_phases(name, early):
    check_adam_lbfgs_adam(name, early)


def test_lbfgs_between_two_adam_phases_with_the_tail_kernel():
    run_worker("check_adam_lbfgs_adam('burgers_inf', True)", {"PINN_FUSED_TAIL": "0"})


@pytest.mark.parametrize("name", OPT_FAMILIES)
def test_second_lbfgs_run_equals_a_fresh_handle(name):
    check_lbfgs_twice(name)


@pytest.mark.parametrize("name", ["burgers_inf", "generic_w24"])
def test_second_lbfgs_run_equals_a_fresh_handle_gram(name):
    run_worker("check_lbfgs_twice(%r)" % name, {"PINN_LBFGS": "gram"})


def test_lbfgs_with_max_iter_zero_reports_an_empty_history():
    """pinn_lbfgs(max_iter = 0) is a run with no evaluation (custom_lbfgs.py:43-44 returns before creating any state):
    pinn_lbfgs_history reports it, not the run before it, and nothing else moves."""
    backend, fam = GpuBackend(), FAMILIES["burgers_inf"]
    p = feed_canonical(backend, fam, fixed_state(fam, 5, OPT_SIZES["inf"]))
    assert len(p.lbfgs(4, learning_rate=0.5, n_correction=5, tol_fun=EPS)["f_hist"]) > 0
    w = p.get_weights()
    r = p.lbfgs(0)
    assert (r["n_iter"], r["n_eval"], r["reason"], r["f_hist"]) == (0, 0, 0, [])
    assert same(p.get_weights(), w)
    backend.close(p)


def test_resampled_batches_step_alike_whatever_brought_them():
    """One collocation batch per Adam step: copied (A), zero-copy (B), copied after an evaluation of a much larger set (C)."""
    backend, fam = GpuBackend(), FAMILIES["burgers_inf"]
    state = fixed_state(fam, 6, OPT_SIZES["inf"])
    sms = backend.sms()
    A, B, Cc = (feed_canonical(backend, fam, state) for _ in range(3))
    rng = _rng(fam, 6, 2)
    big = _box(fam, rng, 40000)
    Cc.set_collocation(big[:, 0], big[:, 1])
    Cc.loss_grad()
    for k, n in enumerate([2000, 1025, 8 * sms + 1, 9000, 7, 32 * sms + 1, 2000, 1]):
        X = _box(fam, rng, n)
        x, t = X[:, 0].copy(), X[:, 1].copy()
        A.set_collocation(x, t, n_global=2 * n)
        backend.set_mapped(B, x, t, n_global=2 * n)
        Cc.set_collocation(x, t, n_global=2 * n)
        la, lb, lc = A.adam_step(LR), B.adam_step(LR), Cc.adam_step(LR)
        assert same(la, lb) and same(la, lc), "step %d (%d points): losses %r %r %r" % (k, n, la, lb, lc)
        wa = A.get_weights()
        assert same(wa, B.get_weights()) and same(wa, Cc.get_weights()), "step %d (%d points): weights differ" % (k, n)
    for p in (A, B, Cc):
        backend.close(p)


def refused_calls(backend, fam, state, p):
    """Calls the library refuses on a handle in `state`, as thunks."""
    kind, P = fam["kind"], p.P
    x = np.linspace(0.1, 0.9, 5)
    X = np.stack([x, x], 1)
    calls = [lambda: p.set_weights(np.zeros(P + 1)), lambda: p.loss_grad(w=np.zeros(3)), lambda: p.set_data(X, X[:, :1], 1.0) if
             kind in ("disc", "ns") else p.set_data(np.stack([x, x, x], 1), X[:, :1])]
    if kind in ("inf", "nls"):
        calls += [lambda: p.set_collocation(x, x, n_global=4), lambda: p.set_data(X, np.zeros((5, 3)))]
    else:
        calls += [lambda: p.set_collocation(x, x)]
    if fam.get("mapped"):
        dp = C.POINTER(C.c_double)
        calls += [lambda: p.set_collocation_mapped(x.ctypes.data_as(dp), x.ctypes.data_as(dp), 5)]      # pageable memory
    if fam.get("poly"):
        ok = state["spec"][1][0]
        n_res = len(state[residual_slot(fam)][1][0])
        calls += [lambda: p.set_residual([]), lambda: p.set_residual(ok + [(1.0, 0, (4, 0, 0, 0))]),
                  lambda: p.set_residual([(2.0, 0, (1, 0, 0, 0)), (1.0, 0, (0, 0, 0, 0))]),
                  lambda: p.set_residual([(2.0, 5, (1, 0, 0, 0))] + ok), lambda: p.set_source(np.zeros(n_res + 1))]
    if kind in ("disc", "ide_disc"):
        q = fam["layers"][-1]
        calls += [lambda: p.set_irk(np.zeros((q + 3, q + 2))), lambda: p.set_pde_params([0.1] * 5), lambda: p.residual()]
    if kind == "ide_disc":
        calls += [lambda: p.set_snapshot(2, x, x), lambda: p.set_boundary(x)]
    if kind == "ns":
        calls += [lambda: p.set_boundary(x), lambda: p.set_pde_params([0.1])]
    return calls


@pytest.mark.parametrize("name", ["burgers_inf", "nls", "burgers_disc", "kdv_ide_disc", "ns", "poly_inf", "poly_ide"])
def test_refused_calls_leave_the_handle_as_it_was(name):
    backend, fam = GpuBackend(), FAMILIES[name]
    sizes = {"coll": 1500, "data": 255, "boundary": 51, "snap0": 100, "snap1": 51}
    state = fixed_state(fam, 8, sizes)
    p, q = feed_canonical(backend, fam, state), feed_canonical(backend, fam, state)
    p.loss_grad()
    for i, call in enumerate(refused_calls(backend, fam, state, p)):
        with pytest.raises(backend.Error):
            call()
        assert_same(backend, fam, p, q, "%s after refused call %d" % (name, i))
    backend.close(p)
    backend.close(q)
