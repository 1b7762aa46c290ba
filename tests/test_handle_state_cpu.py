"""CPU: the harness of tests/test_gpu_handle_state.py has teeth, and its histories are legal.

* Every generated history of the families the CPU oracle stand-in can serve (Burgers inference and identification, Schrodinger,
  discrete-time Burgers, the polynomial inference head; small nets, the same sizes and call orders as on the GPU) runs on the
  stand-in and ends bit for bit equal to a fresh stand-in fed the final state: each history is a legal call sequence that ends in
  the state it claims.  The histories of the other families are generated and their final states checked for completeness.
* Four stand-ins, each broken the way a handle could be, are each rejected by at least one history of their family: a data block
  whose right-aligned start stays where it was when the block shrinks; a Schrodinger pad point that stays when n_0 becomes even; a
  source that survives new residual points of the same count; a second L-BFGS run that starts with the first run's (s, y) pairs.
* At 132 SMs the size ladder reaches what it claims under the capacity rules restated in CapModel."""
import numpy as np
import pytest

from oracle import reference_port as rp, taylor_poly as tpo
from oracle_backend import OraclePinn
import test_gpu_handle_state as hs

PDE_ID = {"BURGERS_INF": 0, "BURGERS_IDE": 1, "NLS_INF": 2, "BURGERS_DISC": 3, "POLY_INF": 8}
# the GPU families on nets the numpy oracle evaluates in milliseconds; the name (the generator's seed) and the widths of the
# input and the head stay, so sizes and call orders are those of the GPU histories
SMALL = {"burgers_inf": [2, 6, 6, 1], "burgers_ide": [2, 6, 6, 1], "nls": [2, 8, 8, 2], "burgers_disc": [1, 6, 9], "poly_inf": [2, 6, 6, 1]}
CPU_FAMILIES = {k: dict(hs.FAMILIES[k], layers=v) for k, v in SMALL.items()}


class Stand(OraclePinn):
    """OraclePinn with the f_hist of pinn_lbfgs_history.  The oracle takes a mean over every point set, so an empty data or
    boundary set (a term the library drops) evaluates to NaN here, one way or the other."""

    def _eval(self, w):
        try:
            return super()._eval(w)
        except ZeroDivisionError:
            return np.nan, np.full(self.P, np.nan), np.full(3, np.nan)

    def lbfgs(self, max_iter, learning_rate=1.0, n_correction=100, tol_fun=1e-5, tol_x=1e-19, sync_every=1, log_fn=None,
              want_x_final=False):
        fs = []

        def opfunc(x):
            f, g, _ = self._eval(x)
            self.w = np.array(x, float)
            fs.append(f)
            return f, g
        tr = rp.lbfgs_fixed_step(opfunc, self.w, max_iter=max_iter, learning_rate=learning_rate, n_correction=n_correction,
                                 tol_fun=tol_fun, tol_x=tol_x)
        for it, f in tr.logged:
            log_fn(it, f)
        return {"n_iter": tr.n_iter, "n_eval": tr.n_eval, "reason": 1 if tr.stop_reason == "max iterations" else 2,
                "x_final": np.array(tr.x_final), "f_hist": fs}


class PolyStand(Stand):
    """POLY_INF: the residual spec and the source, reset by new collocation points (include/pinn_b200.h)."""
    terms = source = None

    def set_residual(self, terms):
        self.terms = list(terms)

    def set_source(self, s):
        assert len(s) == len(self.X_f)
        self.source = np.array(s, float)

    def set_collocation(self, x, t, n_global=None):
        super().set_collocation(x, t, n_global)
        self.source = None

    def _eval(self, w):
        f, g, (a, b) = tpo.poly_loss_grad(w, self.layers, self.lb, self.ub, self.terms, self.X, self.u, X_f=self.X_f, source=self.source,
                                          n_f_global=self.n_f_global, data_weight=self.weight)
        return f, g, np.array([a, 0.0, b])

    def residual(self, n=None):
        return tpo.poly_residual(self.w, self.layers, self.lb, self.ub, self.terms, self.X_f, source=self.source)


class OracleBackend(object):
    Error = AssertionError

    def __init__(self, cls=Stand):
        self.cls = cls

    def create(self, fam):
        cls = self.cls if not fam.get("poly") or issubclass(self.cls, PolyStand) else PolyStand
        return cls(PDE_ID[fam["pde"]], fam["layers"], fam["box"][0], fam["box"][1])

    def sms(self):
        return 132

    def set_mapped(self, p, x, t, n_global=None):
        p.set_collocation(x, t, n_global)

    def close(self, p):
        OraclePinn.created.clear()


def run_all(name, cls=Stand):
    """Every history of the family on the stand-in `cls`; -> the seeds whose history was rejected."""
    rejected = []
    with np.errstate(all="ignore"):                # a mean over an empty data or boundary set is NaN on the oracle, bit for bit
        for seed in hs.SEEDS:
            try:
                hs.run_history(OracleBackend(cls), CPU_FAMILIES[name], seed)
            except AssertionError:
                rejected.append(seed)
    return rejected


@pytest.mark.parametrize("name", list(CPU_FAMILIES))
def test_every_history_passes_on_the_oracle_stand_in(name):
    assert run_all(name) == []


@pytest.mark.parametrize("name", [k for k in hs.FAMILIES if k not in CPU_FAMILIES])
def test_histories_of_the_other_families_end_in_a_complete_state(name):
    fam = hs.FAMILIES[name]
    for seed in hs.SEEDS:
        steps, final = hs.generate(fam, seed, 132)
        state = {}
        for step in steps:
            if step[0] != "eval":
                hs.track(fam, state, step)
        assert hs.evaluable(fam, final) and sorted(state) == sorted(final), (name, seed)
        for slot in hs.ladder(fam, 132):
            if slot in final:
                assert len(final[slot][1][-1]) > 0, (name, seed, slot)


# ----------------------------------------------------------------------------------------------------------------- mutants
class StaleDataOffset(Stand):
    """set_data writes the block right-aligned but keeps reading from the old start when the block shrinks."""
    CAP = 1 << 14

    def set_data(self, X, u, weight=1.0):
        super().set_data(X, u, weight)
        if not hasattr(self, "_buf"):
            self._buf, self._n = np.zeros((self.CAP, 2)), 0
        n = len(self.X)
        self._buf[self.CAP - n:] = self.X if self.X.shape[1] == 2 else np.concatenate([self.X, self.X], 1)
        start = self.CAP - max(n, self._n)
        self.X, self._n = self._buf[start:start + n].copy(), n


class StalePad(Stand):
    """The alignment point behind an odd n_0 is not removed when n_0 becomes even."""

    def set_data(self, X, u, weight=1.0):
        super().set_data(X, u, weight)
        if len(self.X) % 2:
            self._pad = True
        elif getattr(self, "_pad", False):
            X2 = self.X if self.X.shape[1] == 2 else np.concatenate([self.X, self.X], 1)
            self.X, self.u = np.vstack([X2, [self.lb]]), np.vstack([self.u, np.zeros((1, 2))])


class StaleSource(PolyStand):
    """The source survives new collocation points of the same count."""

    def set_collocation(self, x, t, n_global=None):
        keep = self.source if self.X_f is not None and len(x) == len(self.X_f) else None
        super().set_collocation(x, t, n_global)
        self.source = keep


class StaleLbfgs(Stand):
    """Every run starts with the (s, y) pairs the run before it left.  The loop is the reference's (rp.lbfgs_fixed_step) without
    the stop tests, which the runs of check_lbfgs_twice never meet; with no pairs left over it is a correct run."""

    def lbfgs(self, max_iter, learning_rate=1.0, n_correction=100, log_fn=None, **kw):
        S, Y = [list(v) for v in getattr(self, "_pairs", ([], []))]

        def opfunc(x):
            self.w = np.array(x, float)
            return self._eval(x)[:2]
        x = self.w.copy()
        f, g = opfunc(x)
        fs, h_diag, d, t, g_old = [f], 1.0, None, None, None
        for it in range(1, max_iter + 1):
            if it > 1:
                y, s = g - g_old, d * t
                if y @ s > 1e-10:
                    S, Y = (S + [s])[-n_correction:], (Y + [y])[-n_correction:]
                    h_diag = (y @ s) / (y @ y)
            q, al = -g, []
            for s_, y_ in zip(reversed(S), reversed(Y)):
                al.append((s_ @ q) / (y_ @ s_))
                q = q - al[-1] * y_
            r = q * h_diag
            for s_, y_, a in zip(S, Y, reversed(al)):
                r = r + (a - (y_ @ r) / (y_ @ s_)) * s_
            d, g_old = r, g
            t = min(1.0, 1.0 / np.sum(np.abs(g))) if it == 1 else learning_rate
            x = x + t * d
            if it < max_iter:
                f, g = opfunc(x)
                fs.append(f)
                log_fn(it, f)
        self._pairs = (S, Y)
        return {"n_iter": max_iter, "n_eval": len(fs), "reason": 1, "x_final": x, "f_hist": fs}


MUTANTS = [("burgers_inf", StaleDataOffset), ("nls", StalePad), ("poly_inf", StaleSource)]


@pytest.mark.parametrize("name,cls", MUTANTS, ids=[c.__name__ for _, c in MUTANTS])
def test_a_broken_stand_in_is_rejected_by_a_history_of_its_family(name, cls):
    rejected = run_all(name, cls)
    print("[handle state] %s rejected by the histories of %s with seeds %s" % (cls.__name__, name, rejected))
    assert rejected, "%s survives every history of %s: the ladder or the generator is too weak" % (cls.__name__, name)


def test_a_second_lbfgs_run_that_keeps_the_first_ones_pairs_is_rejected():
    fam = CPU_FAMILIES["burgers_inf"]
    hs.check_lbfgs_twice(fam, OracleBackend(Stand))
    hs.check_lbfgs_twice(fam, OracleBackend(StaleLbfgs), pairs=[((1, 5), (3, 5))])         # one iteration leaves no pair
    for pair in hs.LBFGS_PAIRS:
        with pytest.raises(AssertionError, match="differs from the same run on a fresh handle"):
            hs.check_lbfgs_twice(fam, OracleBackend(StaleLbfgs), pairs=[pair])
    print("[handle state] StaleLbfgs rejected by every pair of runs of check_lbfgs_twice")


# ------------------------------------------------------------------------------------------------------------------ ladder
def events(name):
    fam, ev = hs.FAMILIES[name], set()
    for seed in hs.SEEDS:
        ev |= hs.coverage(fam, hs.generate(fam, seed, 132)[0], 132)
    return ev


def test_the_ladder_reaches_what_it_claims_at_132_sms():
    want = {"dcap - n odd", "dcap - n even", "data region regrown with a device collocation block present",
            "collocation region regrown with a data block present", "data block shrunk", "data n = 0", "data n > 0", "in_dim 1",
            "in_dim 2", "weight 0", "weight 1", "n_global > n", "first: set_data"}
    ev = events("burgers_inf")
    assert want | {"copied -> mapped", "mapped -> copied", "data region regrown under a mapped batch",
                   "first: set_collocation_mapped"} <= ev, sorted(ev)
    for name in ("burgers_inf_v1", "generic_w24", "poly_inf"):
        ev = events(name)
        assert want | {"first: set_collocation", "scratch regrown for more points per CTA", "points per CTA below the scratch's"} <= ev, \
            (name, sorted(ev))
    # every order of the Schrodinger handle's three point setters, and both of the two-setter families
    for name, n in (("nls", 6), ("burgers_inf", 2), ("burgers_disc", 2), ("kdv_ide_disc", 2)):
        fam, orders = hs.FAMILIES[name], set()
        for seed in hs.SEEDS:
            seen = [s[0] for s in hs.generate(fam, seed, 132)[0] if s[0] in hs.ladder(fam, 132)]
            orders.add(tuple(dict.fromkeys(seen)))
        assert len(orders) == n, (name, orders)
    # the Schrodinger pad point appears and disappears, the boundary block empties and fills
    fam, par, nb = hs.FAMILIES["nls"], set(), set()
    for seed in hs.SEEDS:
        ns = [len(s[2][0]) for s in hs.generate(fam, seed, 132)[0] if s[0] == "data"]
        par |= {(a % 2, b % 2) for a, b in zip(ns, ns[1:])}
        bs = [len(s[2][0]) for s in hs.generate(fam, seed, 132)[0] if s[0] == "boundary"]
        nb |= {(a > 0, b > 0) for a, b in zip(bs, bs[1:])}
    assert {(1, 0), (0, 1)} <= par and {(False, True), (True, False)} <= nb
    # the polynomial handles: new points of the same count behind a source, a spec replaced by a shorter one
    for name in ("poly_inf", "poly_ide"):
        fam, same_count, shorter = hs.FAMILIES[name], False, False
        for seed in hs.SEEDS:
            state, n_terms = {}, None
            for s in hs.generate(fam, seed, 132)[0]:
                if s[0] == hs.residual_slot(fam) and "source" in state and len(s[2][-1]) == len(state[s[0]][1][-1]):
                    same_count = True
                if s[0] == "spec":
                    shorter |= n_terms is not None and len(s[2][0]) < n_terms
                    n_terms = len(s[2][0])
                if s[0] != "eval":
                    hs.track(fam, state, s)
        assert same_count and shorter, (name, same_count, shorter)
