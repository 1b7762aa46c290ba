"""CPU: the residual-based adaptive draw of pinn_draw_collocation_rad (DESIGN §4.7) as restated in oracle/rad_draw.py, the golden
file that pins it, the exactness of its integer path, its sampling distribution, the mirror's schedule (hp["rad_every"]) on a
stand-in handle, and the built library's RAD kernels and symbols."""
import bisect
import ctypes
import itertools
import math
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import PKG, load_golden
from oracle import lhs_draw as ld
from oracle import rad_draw as rd


def golden_cases():
    g = load_golden("rad_draw")
    j = 0
    while "case%d_params" % j in g:
        seed, draw, n, k, T = (int(v) for v in g["case%d_params" % j])
        yield j, g["case%d_f" % j], seed, draw, n, k, float(g["case%d_c" % j]), T, g["case%d_idx" % j]
        j += 1


def test_golden_draws_reproduce():
    seen_k, seen_c, count = set(), set(), 0
    for j, f, seed, draw, n, k, c, T, idx in golden_cases():
        Q, T_now = rd.quantise(rd.numerators(f, k), c)
        assert T_now == T, j
        assert np.array_equal(rd.pick(Q, T, seed, draw, n), idx), j
        seen_k.add(k); seen_c.add(c); count += 1
    assert count >= 20 and seen_k == {0, 1, 2, 3, 4} and seen_c == {0.0, 1.0, 1024.0}


# ------------------------------------------------------------------------------------------------- the integer path is exact
def python_int_indices(f, seed, draw, n, k, c):
    """Steps 3-5 in Python floats and ints: no numpy integer arithmetic, no limbs."""
    a = [float(v) for v in rd.numerators(f, k)]
    fin = [v for v in a if math.isfinite(v)]
    amax = max(fin, default=0.0)
    A = [rd.SCALE if not math.isfinite(v) else (math.floor((v / amax) * 2.0 ** 24) if amax > 0.0 else 0) for v in a]
    S = sum(A)
    cq = math.floor(c * float(S) / len(a))
    Q = [v + cq for v in A]
    if sum(Q) == 0:
        Q = [1] * len(a)
    P = list(itertools.accumulate(Q))
    T = P[-1]
    out = []
    for j in range(n):
        w = ld.philox4x32_10(j & 0xFFFFFFFF, j >> 32, draw & 0xFFFFFFFF, draw >> 32, (seed & 0xFFFFFFFF) ^ rd.RAD_SALT[0],
                             (seed >> 32) ^ rd.RAD_SALT[1])
        target = (((int(w[0]) << 32) | int(w[1])) * T) >> 64
        assert 0 <= target < T
        out.append(bisect.bisect_right(P, target))
    return np.array(out)


def test_oracle_equals_a_python_int_reference():
    for j, f, seed, draw, n, k, c, T, idx in golden_cases():
        assert np.array_equal(python_int_indices(f, seed, draw, min(n, 400), k, c), idx[:400]), j


def test_mulhi64_limbs_equal_python_ints():
    rng = np.random.default_rng(1)
    x = rng.integers(0, 1 << 63, 5000, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, 5000, dtype=np.uint64)
    x[:3] = (0, 1, (1 << 64) - 1)
    for T in (1, 2, 3, (1 << 24) * 1000 + 17, 1025 << 53, (1 << 64) - 1):
        assert [int(v) for v in rd.mulhi64(x, T)] == [(int(v) * T) >> 64 for v in x], T


def segmented_indices(f, seed, draw, n, k, c, grid):
    """The device's route (csrc/rad_sample.cuh): segment-local prefixes of A, an exclusive prefix of the segment sums, and
    P_i = base[i / seg] + lp_i + (i + 1) C' formed inside the binary search."""
    a = rd.numerators(f, k)
    n_pool = a.size
    fin = np.isfinite(a)
    # the block maxima of a strided head, reduced in another order
    bmax = [max([v for v in a[b::grid] if np.isfinite(v)], default=0.0) for b in range(grid)]
    amax = max(bmax[::-1])
    A = np.full(n_pool, rd.SCALE, dtype=np.uint64)
    A[fin] = np.floor((a[fin] / amax) * 2.0 ** 24).astype(np.uint64) if amax > 0 else 0
    seg = -(-n_pool // grid)
    lp = np.zeros(n_pool, dtype=np.uint64)
    bsum = []
    for b in range(grid):
        lo, hi = min(b * seg, n_pool), min(b * seg + seg, n_pool)
        lp[lo:hi] = np.cumsum(A[lo:hi], dtype=np.uint64)
        bsum.append(int(A[lo:hi].sum(dtype=np.uint64)))
    base = [0] + list(itertools.accumulate(bsum))[:-1]
    S = sum(bsum)
    cq = math.floor(c * float(S) / n_pool)
    if S == 0 and cq == 0:
        cq = 1
    T = S + n_pool * cq
    out = []
    for target in rd.targets(seed, draw, n, T):
        lo, hi = 0, n_pool - 1
        while lo < hi:
            mid = (lo + hi) // 2
            if base[mid // seg] + int(lp[mid]) + (mid + 1) * cq > int(target):
                hi = mid
            else:
                lo = mid + 1
        out.append(lo)
    return np.array(out)


@pytest.mark.parametrize("grid", [1, 3, 7, 64])
def test_segmented_route_equals_the_definition_for_any_grid(grid):
    for j, f, seed, draw, n, k, c, T, idx in golden_cases():
        if grid <= len(f):
            assert np.array_equal(segmented_indices(f, seed, draw, min(n, 300), k, c, grid), idx[:300]), (j, grid)


def test_sums_do_not_depend_on_the_order():
    rng = np.random.default_rng(7)
    f = rng.standard_normal(100000) * np.exp(rng.standard_normal(100000) * 3)
    Q, T = rd.quantise(rd.numerators(f, 2), 1.0)
    perm = rng.permutation(f.size)
    Qp, Tp = rd.quantise(rd.numerators(f[perm], 2), 1.0)
    assert Tp == T and np.array_equal(Qp, Q[perm])
    cuts = np.sort(rng.choice(np.arange(1, f.size), 37, replace=False))
    assert sum(int(p.sum(dtype=np.uint64)) for p in np.split(Q[perm], cuts)) == T == sum(int(v) for v in Q)


# ------------------------------------------------------------------------------------------------------------ distribution
def test_frequencies_match_the_weights():
    from scipy.stats import chisquare
    rng = np.random.default_rng(11)
    f = rng.standard_normal(40) * np.linspace(0.1, 3.0, 40)
    f[3] = 0.0
    for k, c in ((1, 1.0), (2, 0.0), (4, 0.5)):
        Q, T = rd.quantise(rd.numerators(f, k), c)
        idx = rd.pick(Q, T, 5, 0x100000000 + k, 400000)
        counts = np.bincount(idx, minlength=f.size)
        p = Q.astype(np.float64) / T
        keep = p > 0
        assert np.all(counts[~keep] == 0)
        stat = chisquare(counts[keep], p[keep] / p[keep].sum() * counts.sum())
        assert stat.pvalue > 1e-4, (k, c, stat)


def test_zero_weights_are_never_drawn_and_duplicates_occur():
    f = np.array([0.0, 1.0, 0.0, 2.0, 0.0])
    idx = rd.rad_indices(f, 1, 2, 1000, 1, 0.0)
    assert set(idx.tolist()) == {1, 3}
    assert len(np.unique(rd.rad_indices(np.ones(100), 1, 2, 100, 1, 1.0))) < 100     # with replacement


def test_k0_and_t0_give_a_uniform_draw():
    f = np.array([0.0, np.nan, 1e300, -3.0, 5e-324, np.inf])
    Q, T = rd.quantise(rd.numerators(f, 0), 0.0)
    assert len(set(Q.tolist())) == 1 and T == f.size * rd.SCALE
    Q, T = rd.quantise(rd.numerators(np.zeros(9), 3), 0.0)                            # every A_i = 0 and C' = 0
    assert Q.tolist() == [1] * 9 and T == 9
    Q, T = rd.quantise(rd.numerators(np.full(4, 5e-324), 2), 0.0)                     # r^2 underflows to 0
    assert Q.tolist() == [1] * 4


def test_nonfinite_residuals_take_the_top_weight():
    f = np.array([np.nan, 1.0, -np.inf, 0.5, np.inf, 1e200])
    for k in (1, 2):                                                                    # k = 2: 1e200^2 = Inf too
        Q, T = rd.quantise(rd.numerators(f, k), 1.0)
        assert Q[0] == Q[2] == Q[4] == Q.max()
    pair = np.array([[np.nan, 0.0], [1.0, 1.0], [0.0, -np.inf]])
    Q, _ = rd.quantise(rd.numerators(pair, 1), 0.0)
    assert Q[0] == Q[2] == rd.SCALE and Q[1] == rd.SCALE                                # the finite max also gets 2^24
    Q, T = rd.quantise(rd.numerators(np.array([np.nan, np.nan]), 1), 0.0)              # no finite value: amax = 0
    assert Q.tolist() == [rd.SCALE] * 2


def test_pick_key_differs_from_the_lhs_keys():
    assert tuple(rd.RAD_SALT) not in ((0, 0), tuple(ld.KEY_SALT))
    src = open(os.path.join(PKG, "csrc", "rad_sample.cuh")).read()
    assert "RAD_SALT0 = 0x%08Xu, RAD_SALT1 = 0x%08Xu" % rd.RAD_SALT in src


# ------------------------------------------------------------------------------------------------------- mirror schedule
class StandIn(object):
    """Records every call the mirror makes on its handle (pinn_cabi.Pinn's method names)."""
    log = []

    def __init__(self, pde, layers, lb, ub, device=0, rank=0, world=1, nccl_uid=None):
        self.pde = pde

    def __getattr__(self, name):
        def call(*args, **kw):
            StandIn.log.append((name, args, kw))
            return 0.5 if name == "last_loss" else None
        return call


class QuietLogger(object):
    def log_train_opt(self, name):
        pass

    def log_train_epoch(self, epoch, loss, custom="", is_iter=False):
        float(loss)


@pytest.fixture()
def mirror(monkeypatch):
    import pinn_cabi
    import neuralnetwork
    monkeypatch.setattr(pinn_cabi, "Pinn", StandIn)
    StandIn.log = []
    return neuralnetwork


def _burgers(nn, epochs, n_f=300, **hp_extra):
    hp = {"layers": [2, 8, 8, 1], "tf_epochs": epochs, "tf_lr": 1e-3, "tf_b1": 0.9, "tf_eps": None, "nt_epochs": 0, "nt_lr": 0.8,
          "nt_ncorr": 50}
    hp.update(hp_extra)

    class Burgers(nn.NeuralNetwork):
        def __init__(self):
            super().__init__(hp, QuietLogger(), np.array([1.0, 0.99]), np.array([-1.0, 0.0]))
            self.nu = 0.01 / np.pi
            X_f = np.random.default_rng(0).random((n_f, 2))
            self.x_f, self.t_f = X_f[:, 0:1], X_f[:, 1:2]
    return Burgers()


def _rad_calls():
    return [(a, kw) for name, a, kw in StandIn.log if name == "draw_collocation_rad"]


def test_mirror_without_the_keys_never_draws(mirror):
    net = _burgers(mirror, 5)
    net.tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    assert _rad_calls() == [] and net.rad_every == 0


def test_mirror_rad_draws_before_every_kth_epoch(mirror):
    net = _burgers(mirror, 7, rad_every=3, resample_seed=0xFFFFFFFF00000003)
    net.tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    assert _rad_calls() == [((0xFFFFFFFF00000003, d, 300, 3000, 1, 1.0), {}) for d in (1, 2)]
    names = [name for name, _, _ in StandIn.log if name in ("adam_step", "draw_collocation_rad", "draw_collocation")]
    assert names == ["adam_step"] * 3 + ["draw_collocation_rad"] + ["adam_step"] * 3 + ["draw_collocation_rad", "adam_step"]
    StandIn.log = []
    _burgers(mirror, 3, n_f=50, rad_every=1, rad_pool=777, rad_k=0, rad_c=1024).tf_optimization(np.zeros((5, 2)),
                                                                                               np.zeros((5, 1)))
    assert _rad_calls() == [((0, d, 50, 777, 0, 1024.0), {}) for d in (1, 2)]


def test_mirror_refuses_bad_rad_keys(mirror):
    import pinn_cabi
    with pytest.raises(pinn_cabi.PinnError, match="resample_every.*rad_every"):
        _burgers(mirror, 1, resample_every=2, rad_every=2)
    for bad in ({"rad_every": -1}, {"rad_every": 2.0}, {"rad_k": 5}, {"rad_k": -1}, {"rad_c": -0.5}, {"rad_c": 1025.0},
                {"rad_c": float("nan")}, {"rad_c": float("inf")}, {"rad_c": True}, {"rad_pool": 0}, {"rad_pool": (1 << 29) + 1}):
        with pytest.raises(pinn_cabi.PinnError, match=list(bad)[0]):
            _burgers(mirror, 1, **bad)
    # a sharded run: the weights are whole-pool quantities
    net = _burgers(mirror, 2, rad_every=1)
    net.world = 2
    with pytest.raises(pinn_cabi.PinnError, match="rad_every"):
        net.tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))


@pytest.mark.parametrize("kind", ["identification", "poly"])
def test_mirror_refuses_rad_on_models_the_call_refuses(mirror, kind):
    import pinn_cabi
    hp = {"layers": [2, 8, 1], "tf_epochs": 2, "tf_lr": 1e-3, "tf_b1": 0.9, "tf_eps": None, "nt_epochs": 0, "nt_lr": 0.8,
          "nt_ncorr": 50, "rad_every": 1}

    class Ide(mirror.NeuralNetwork):
        def __init__(self):
            super().__init__(hp, QuietLogger(), np.array([1.0, 1.0]), np.array([-1.0, 0.0]))
            self.lambda_1, self.lambda_2 = 0.0, -6.0

    class Heat(mirror.NeuralNetwork):
        pde, residual = "poly", "u_t - 0.5*u_xx"

        def __init__(self):
            super().__init__(hp, QuietLogger(), np.array([1.0, 1.0]), np.array([-1.0, 0.0]))
            self.x_f, self.t_f = np.zeros((40, 1)), np.zeros((40, 1))

    with pytest.raises(pinn_cabi.PinnError, match="rad_every"):
        (Ide if kind == "identification" else Heat)().tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    assert _rad_calls() == []


# ------------------------------------------------------------------------------------------------------------- library
def test_library_exports_and_binds_the_rad_draw(lib_built):
    import pinn_cabi
    lib = ctypes.CDLL(lib_built)
    assert hasattr(lib, "pinn_draw_collocation_rad") and "pinn_draw_collocation_rad" in pinn_cabi.SIGNATURES


def test_rad_kernels_have_no_stack_and_no_local_memory(lib_built):
    out = subprocess.run(["cuobjdump", "-res-usage", lib_built], capture_output=True, text=True).stdout
    m = re.findall(r"Function (\S*4pinn3rad\S*?):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert sorted(re.search(r"rad\d+(\w+?)_kernel", name).group(1) for name, *_ in m) == ["head", "pick", "quantise"], m
    for name, regs, stack, local in m:
        assert int(stack) == 0 and int(local) == 0, name
    for bad in ("fused_loss_grad", "reduce_tail", "adam_update", "lbfgs_iterate"):
        assert not any(bad in name for name, *_ in m)
