"""CPU: the Latin-hypercube draw of pinn_draw_collocation (DESIGN §4.6) as restated in oracle/lhs_draw.py, the golden file that pins
it, the mirror's draw schedule (hp["resample_every"]) on a stand-in handle, and the built library's draw kernel and symbols."""
import ctypes
import re
import subprocess

import numpy as np
import pytest

from conftest import load_golden
from oracle import lhs_draw as ld

BOXES = [([-1.0, 0.0], [1.0, 0.99]), ([-5.0, 0.0], [5.0, np.pi / 2]), ([0.3, -0.5], [3.7, 2.0])]


@pytest.mark.parametrize("ctr, key, want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_gives_the_random123_known_answers(ctr, key, want):
    assert tuple(int(w) for w in ld.philox4x32_10(*ctr, *key)) == want


def _sizes():
    return sorted(set(list(range(1, 65)) + [v for k in range(1, 9) for v in (4 ** k - 1, 4 ** k, 4 ** k + 1)] + [100000]))


@pytest.mark.parametrize("seed, draw", [(0, 0), (1234, 7), (0xDEADBEEF00000001, 0x1234567800000009)])
def test_permutations_are_bijections_and_differ_between_dimensions(seed, draw):
    for N in _sizes():
        i = np.arange(N, dtype=np.uint64)
        p0, p1 = ld.permute(i, N, 0, seed, draw), ld.permute(i, N, 1, seed, draw)
        for p in (p0, p1):
            assert np.array_equal(np.sort(p), i), N
        if N >= 16:
            assert not np.array_equal(p0, p1), N


def test_mean_walk_stays_below_the_domain_ratio():
    for N in (2, 5, 17, 1025, 100000):
        walks = []
        ld.permute(np.arange(N, dtype=np.uint64), N, 0, 3, 1, walks)
        assert walks[0].min() >= 1 and walks[0].mean() <= 4 ** ld.half_bits(N) / N < 4


@pytest.mark.parametrize("lb, ub", BOXES)
def test_one_point_per_stratum_and_every_value_in_the_box(lb, ub):
    for N in (1, 2, 7, 1000, 4097, 100000):
        x, t = ld.lhs_draw(42, 3, N, 0, N, lb, ub)
        i = np.arange(N, dtype=np.uint64)
        for d, v in enumerate((x, t)):
            p = ld.permute(i, N, d, 42, 3).astype(np.float64)
            w = np.float64(ub[d]) - np.float64(lb[d])
            lo, hi = lb[d] + w * (p / N), lb[d] + w * ((p + 1.0) / N)        # the stratum's ends, rounded as the value is
            assert np.all(lo <= v) and np.all(v <= hi), (N, d)
            assert np.all(lb[d] <= v) and np.all(v <= ub[d]), (N, d)


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_shards_concatenate_to_the_whole_draw(world):
    from sharding import shard_rows
    for N, (lb, ub) in ((4097, BOXES[0]), (100000, BOXES[1]), (7, BOXES[2])):
        x, t = ld.lhs_draw(0xFFFFFFFF00000001, 0x100000002, N, 0, N, lb, ub)
        parts = [ld.lhs_draw(0xFFFFFFFF00000001, 0x100000002, N, lo, hi - lo, lb, ub) for lo, hi in
                 (shard_rows(N, r, world) for r in range(world))]
        assert np.concatenate([p[0] for p in parts]).view(np.uint64).tolist() == x.view(np.uint64).tolist()
        assert np.concatenate([p[1] for p in parts]).view(np.uint64).tolist() == t.view(np.uint64).tolist()


def test_golden_draws_reproduce():
    g = load_golden("lhs_draw")
    k = 0
    while "case%d_params" % k in g:
        seed, draw, N = (int(v) for v in g["case%d_params" % k])
        box = g["case%d_box" % k]
        x, t = ld.lhs_draw(seed, draw, N, 0, N, box[:2], box[2:])
        assert np.array_equal(x.view(np.uint64), g["case%d_x" % k].view(np.uint64)), k
        assert np.array_equal(t.view(np.uint64), g["case%d_t" % k].view(np.uint64)), k
        k += 1
    assert k >= 7 and {int(g["case%d_params" % j][2]) for j in range(k)} == {1, 2, 7, 1000, 4097}


# ------------------------------------------------------------------------------------------------------- mirror schedule
class StandIn(object):
    """Records every call the mirror makes on its handle (pinn_cabi.Pinn's method names)."""
    log = []

    def __init__(self, pde, layers, lb, ub, device=0, rank=0, world=1, nccl_uid=None):
        self.pde, self.layers = pde, list(layers)
        self.n_c = 0

    def __getattr__(self, name):
        def call(*args, **kw):
            StandIn.log.append((name, args, kw))
            if name == "set_collocation":
                self.n_c = len(args[0])
            if name == "draw_collocation":
                from sharding import shard_rows
                lo, hi = shard_rows(args[2], kw.get("rank", 0), kw.get("world", 1))
                self.n_c = hi - lo
            if name == "get_collocation":
                return np.linspace(0.0, 1.0, self.n_c), np.linspace(1.0, 2.0, self.n_c)
            if name == "last_loss":
                return 0.5
            return None
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


def _draws():
    return [(a, kw) for name, a, kw in StandIn.log if name == "draw_collocation"]


def _adam_positions():
    return [i for i, (name, _, _) in enumerate(StandIn.log) if name == "adam_step"]


def test_mirror_without_the_key_never_draws(mirror):
    net = _burgers(mirror, 7)
    net.tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    assert _draws() == [] and len(_adam_positions()) == 7 and net.resample_every == 0


def test_mirror_draws_before_every_kth_epoch(mirror):
    net = _burgers(mirror, 7, resample_every=2, resample_seed=0xFFFFFFFF00000003)
    net.tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    assert _draws() == [((0xFFFFFFFF00000003, d, 300), {"rank": 0, "world": 1}) for d in (1, 2, 3)]
    # the draw for epoch e comes right before that epoch's step: epochs 0, 1 train on the script's X_f
    names = [name for name, _, _ in StandIn.log if name in ("adam_step", "draw_collocation")]
    assert names == ["adam_step", "adam_step", "draw_collocation", "adam_step", "adam_step", "draw_collocation", "adam_step",
                     "adam_step", "draw_collocation", "adam_step"]
    # a second fit starts the schedule again
    StandIn.log = []
    net.tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    assert [a[1] for a, _ in _draws()] == [1, 2, 3]


def test_mirror_draws_this_ranks_rows_of_the_global_set(mirror):
    net = _burgers(mirror, 4, n_f=100, resample_every=3)
    net.rank, net.world, net.n_f_global = 2, 3, 301
    net.tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    assert _draws() == [((0, 1, 301), {"rank": 2, "world": 3})]


def test_mirror_poly_source_follows_each_draw(mirror):
    hp = {"layers": [2, 8, 1], "tf_epochs": 3, "tf_lr": 1e-3, "tf_b1": 0.9, "tf_eps": None, "nt_epochs": 0, "nt_lr": 0.8,
          "nt_ncorr": 50, "resample_every": 1}

    class Heat(mirror.NeuralNetwork):
        pde, residual = "poly", "u_t - 0.5*u_xx"

        def __init__(self):
            super().__init__(hp, QuietLogger(), np.array([1.0, 1.0]), np.array([-1.0, 0.0]))
            self.x_f, self.t_f = np.zeros((40, 1)), np.zeros((40, 1))

        def source(self, x, t):
            return x + 10.0 * t

    Heat().tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    seq = [(name, a) for name, a, _ in StandIn.log if name in ("draw_collocation", "get_collocation", "set_source")]
    assert [s[0] for s in seq] == ["set_source"] + ["draw_collocation", "get_collocation", "set_source"] * 2
    x, t = np.linspace(0.0, 1.0, 40), np.linspace(1.0, 2.0, 40)
    assert np.array_equal(seq[-1][1][0], x + 10.0 * t)


def test_mirror_refuses_the_key_without_a_collocation_set(mirror):
    import pinn_cabi
    hp = {"layers": [2, 8, 1], "tf_epochs": 2, "tf_lr": 1e-3, "tf_b1": 0.9, "tf_eps": None, "nt_epochs": 0, "nt_lr": 0.8,
          "nt_ncorr": 50, "resample_every": 1}

    class Ide(mirror.NeuralNetwork):
        def __init__(self):
            super().__init__(hp, QuietLogger(), np.array([1.0, 1.0]), np.array([-1.0, 0.0]))
            self.lambda_1, self.lambda_2 = 0.0, -6.0

    with pytest.raises(pinn_cabi.PinnError, match="no collocation set"):
        Ide().tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    for bad in ({"resample_every": -1}, {"resample_every": 1.5}, {"resample_seed": -3}, {"resample_seed": 1 << 64}):
        with pytest.raises(pinn_cabi.PinnError, match="resample_"):
            _burgers(mirror, 1, **bad)


# ------------------------------------------------------------------------------------------------------------- library
def test_library_exports_and_binds_the_draw(lib_built):
    import pinn_cabi
    lib = ctypes.CDLL(lib_built)
    for name in ("pinn_draw_collocation", "pinn_get_collocation"):
        assert hasattr(lib, name) and name in pinn_cabi.SIGNATURES


def test_draw_kernel_has_no_stack_and_no_local_memory(lib_built):
    out = subprocess.run(["cuobjdump", "-res-usage", lib_built], capture_output=True, text=True).stdout
    m = re.findall(r"Function (\S*lhs\S*draw_kernel\S*?):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert len(m) == 1, m
    assert int(m[0][2]) == 0 and int(m[0][3]) == 0
    sass = subprocess.run(["cuobjdump", "-sass", lib_built], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
