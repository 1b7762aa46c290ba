"""GPU: continuous-time Navier-Stokes identification (pde id 7) on its 13-stream fused kernel -- golden vectors
(tests/golden/make_ns_golden.py), Adam and L-BFGS trajectories, the Taylor oracle at ragged sizes and widths 7 to 256, the
per-parameter-block check against the extended-precision oracle, the probe kernel (predict / derivatives / residual), bitwise
reproducibility, the C ABI's error paths, and the Python surface with the driver script."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import PKG, ROOT, load_golden

pytestmark = pytest.mark.gpu
sys.path[:0] = [os.path.join(PKG, "2d-navier-stokes"), os.path.dirname(os.path.abspath(__file__))]


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


@pytest.fixture(scope="module")
def cabi():
    import pinn_cabi
    pinn_cabi.load()
    return pinn_cabi


def make(cabi, layers, lb, ub, X, uv):
    p = cabi.Pinn(cabi.NS_IDE, [int(v) for v in layers], lb, ub)
    p.set_data(X, uv)
    return p


def golden(cabi):
    g = load_golden("ns_ide")
    return g, make(cabi, g["layers"], g["lb"], g["ub"], g["X"], g["uv"])


def test_golden_loss_grad_at_two_points(cabi):
    g, p = golden(cabi)
    assert p.P == g["w"].size
    for tag in ("", "2"):
        loss, grad, parts = p.loss_grad(w=g["w" + tag])
        assert abs(loss - g["loss" + tag]) <= 1e-10 * abs(g["loss" + tag])
        assert rel(grad, g["grad" + tag]) < 1e-10
        assert rel(grad[-2:], g["grad" + tag][-2:]) < 1e-10
        assert np.allclose(parts[[0, 2]], g["parts" + tag], rtol=1e-10) and parts[1] == 0.0


def test_adam_and_lbfgs_trajectories(cabi):
    g, p = golden(cabi)
    p.set_weights(g["w2"])
    losses = [p.adam_step(1e-3) for _ in range(3)]
    assert rel(losses, g["adam_losses"]) < 1e-8 and rel(p.get_weights(), g["adam_w"]) < 1e-8
    g, p = golden(cabi)
    p.set_weights(g["w2"])
    r = p.lbfgs(4, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, sync_every=1, want_x_final=True)
    assert r["n_iter"] == 4 and r["n_eval"] == len(g["lbfgs_f"])
    assert rel(r["f_hist"], g["lbfgs_f"]) < 1e-7
    assert rel(r["x_final"], g["lbfgs_x_final"]) < 1e-7
    assert rel(p.get_weights(), g["lbfgs_x_eval"][-1]) < 1e-7


def ns_inputs(hidden, n, seed, lb=(1.0, -2.0, 0.0), ub=(8.0, 2.0, 20.0), lam=(0.6, 0.05), scale=1.0):
    from oracle import reference_port as rp
    rng = np.random.default_rng(seed)
    layers = [3] + list(hidden) + [2]
    lb, ub = np.array(lb), np.array(ub)
    X = lb + (ub - lb) * rng.random((n, 3))
    uv = rng.standard_normal((n, 2))
    w = np.concatenate([scale * rp.glorot_normal_flat(layers, rng) + 0.02 * rng.standard_normal(rp.num_params(layers)), lam])
    return layers, lb, ub, X, uv, w


def _sms(cabi):
    p = cabi.Pinn(cabi.NS_IDE, [3, 4, 2], [0, 0, 0], [1, 1, 1])
    return p.kernel_info()["sms"]


# n = 1, 7 (< 8 points), 9, 131 (< one point per CTA), 5000 (upstream), widths 7 ... 256, depth 1 ... 8
CASES = [([20] * 8, 5000), ([20] * 8, 1), ([7, 7], 7), ([9], 9), ([33, 20, 33], 131), ([256, 256], 300), ([128, 7, 200], 77),
         ([17] * 3, 1000)]


@pytest.mark.parametrize("hidden,n", CASES)
def test_against_taylor_oracle(cabi, hidden, n):
    from oracle import taylor_ns as tn
    layers, lb, ub, X, uv, w = ns_inputs(hidden, n, 7 * n + len(hidden))
    p = make(cabi, layers, lb, ub, X, uv)
    loss, grad, parts = p.loss_grad(w=w)
    f2, g2, parts2 = tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv)
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10
    assert rel(grad[-2:], g2[-2:]) < 1e-10
    assert np.allclose(parts[[0, 2]], parts2, rtol=1e-10) and parts[1] == 0.0


def test_above_grid_times_points_per_cta(cabi):
    """More points than the CTAs' first even share: the last CTA's block is ragged, and an evaluation of a smaller set on the same
    handle reuses the larger scratch."""
    from oracle import taylor_ns as tn
    n = 38 * _sms(cabi) + 5
    layers, lb, ub, X, uv, w = ns_inputs([20] * 4, n, 3)
    p = make(cabi, layers, lb, ub, X, uv)
    loss, grad, _ = p.loss_grad(w=w)
    f2, g2, _ = tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv)
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10
    p.set_data(X[:37], uv[:37])
    loss, grad, _ = p.loss_grad(w=w)
    f2, g2, _ = tn.ns_ide_loss_grad(w, layers, lb, ub, X[:37], uv[:37])
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10


PREC = [("upstream", [20] * 8, 500, (1.0, -2.0, 0.0), (8.0, 2.0, 20.0), 1.0),
        ("small box", [20, 20, 20], 200, (0.0, 0.0, 0.0), (1e-2, 2e-2, 1e-3), 1.0),
        ("wide weights", [33, 33], 300, (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0), 4.0)]


@pytest.mark.parametrize("tag,hidden,n,lb,ub,scale", PREC)
def test_per_block_against_longdouble(cabi, tag, hidden, n, lb, ub, scale):
    from oracle import taylor as ty, taylor_ns as tn
    from test_gpu_precision import check
    layers, lb, ub, X, uv, w = ns_inputs(hidden, n, 17, lb, ub, scale=scale)
    p = make(cabi, layers, lb, ub, X, uv)
    got = p.loss_grad(w=w)
    ref = tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv, dtype=np.longdouble, magnitudes=True)
    ref64 = tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv)
    ref = (ref[0], ref[1], ref[2], ref[3])
    check("ns " + tag, got, ref, ref64, ty.param_blocks(layers, 2), [0, 2])


def test_probes_residual_and_predict(cabi):
    from oracle import taylor_ns as tn
    g, p = golden(cabi)
    p.set_weights(g["w2"])
    D = p.derivatives(g["X_probe"])
    assert D.shape == (64, 13, 2) and rel(D, g["probe"]) <= 1e-11
    for k in range(13):
        assert rel(D[:, k], g["probe"][:, k]) <= 1e-10, k
    assert rel(p.predict(g["X_probe"]), g["probe"][:, 0]) <= 1e-11
    f = p.residual()
    assert f.shape == g["residual"].shape and rel(f, g["residual"]) <= 1e-10
    # a width-256 net probes in chunks of 5 041 points: 11 000 points take two full chunks and a ragged third
    layers, lb, ub, X, uv, w = ns_inputs([256, 256], 11000, 5)
    q = make(cabi, layers, lb, ub, X, uv)
    q.set_weights(w)
    O, _ = tn.forward_ns(w[:-2], layers, lb, ub, X)
    assert rel(q.derivatives(X), np.stack(O, 1)) <= 1e-11
    assert rel(q.residual(), np.stack(tn.ns_terms(O, w[-2], w[-1]), 1)) <= 1e-10


def test_two_evaluations_are_bit_identical(cabi):
    layers, lb, ub, X, uv, w = ns_inputs([20] * 8, 5000, 1)
    p = make(cabi, layers, lb, ub, X, uv)
    a = p.loss_grad(w=w)
    b = p.loss_grad(w=w)
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_get_params_and_error_paths(cabi):
    g, p = golden(cabi)
    p.set_weights(g["w2"])
    assert list(p.get_params()) == list(g["w2"][-2:])
    assert p.kernel_info()["local_bytes"] == 0
    assert p.time_kernel_ms(3) > 0
    lb, ub = [0, 0, 0], [1, 1, 1]
    with pytest.raises(cabi.PinnError, match="net \\[3, ..., 2\\]"):
        cabi.Pinn(cabi.NS_IDE, [2, 8, 2], lb, ub)
    with pytest.raises(cabi.PinnError, match="net \\[3, ..., 2\\]"):
        cabi.Pinn(cabi.NS_IDE, [3, 8, 1], lb, ub)
    with pytest.raises(cabi.PinnError, match="one GPU"):
        cabi.Pinn(cabi.NS_IDE, [3, 8, 2], lb, ub, world=2, nccl_uid=b"\0" * 128)
    with pytest.raises(cabi.PinnError, match="ub > lb"):
        cabi.Pinn(cabi.NS_IDE, [3, 8, 2], lb, [1, 1, 0])
    with pytest.raises(cabi.PinnError, match="width out of range"):
        cabi.Pinn(cabi.NS_IDE, [3, 257, 2], lb, ub)
    with pytest.raises(cabi.PinnError, match="unknown pde_id"):
        cabi.Pinn(8, [3, 8, 2], lb, ub)
    h = cabi.Pinn(cabi.NS_IDE, [3, 8, 2], lb, ub)
    with pytest.raises(cabi.PinnError, match="no points set"):
        h.loss_grad(w=np.zeros(h.P))
    with pytest.raises(cabi.PinnError, match="X \\(n,3\\)"):
        h.set_data(np.zeros((4, 2)), np.zeros((4, 2)))
    with pytest.raises(cabi.PinnError, match="u \\(n,2\\)"):
        h.set_data(np.zeros((4, 3)), np.zeros((4, 1)))
    with pytest.raises(cabi.PinnError, match="data points as residual points"):
        h.set_collocation(np.zeros(3), np.zeros(3))
    with pytest.raises(cabi.PinnError, match="boundary term"):
        h.set_boundary([0.0])
    with pytest.raises(cabi.PinnError, match="stage matrices"):
        h.set_irk(np.zeros((5, 4)))
    with pytest.raises(cabi.PinnError, match="two snapshots"):
        h.set_snapshot(0, np.zeros(3), np.zeros(3))
    with pytest.raises(cabi.PinnError, match="takes no constants"):
        h.set_pde_params([0.01])
    h.set_pde_params([])
    with pytest.raises(cabi.PinnError, match="residual points are stored"):
        h.residual(5)
    with pytest.raises(cabi.PinnError, match="X \\(n,3\\)"):
        h.predict(np.zeros((4, 2)))
    # PINN_FORCE_GENERIC has no effect on these handles
    code = ("import sys; sys.path[:0] = [%r]; import pinn_cabi as c; p = c.Pinn(c.NS_IDE, [3, 20, 2], [0, 0, 0], [1, 1, 1]); "
            "print(p.kernel_info()['block'])" % os.path.join(PKG, "utils"))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PINN_FORCE_GENERIC="1"), capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0 and r.stdout.strip().splitlines()[-1] == "256", r.stderr[-2000:]


def test_python_surface(capsys):
    """A subclass with pde = "ns_ide": fit(X, uv) runs Adam then L-BFGS on the fused kernel from lambda = (0, 0), predict returns
    (u, v, p), f_model (f_u, f_v), get_params the raw lambdas."""
    from logger import Logger
    from neuralnetwork import NeuralNetwork
    from oracle import reference_port as rp, reference_port_ns as rn
    g = load_golden("ns_ide")

    class NavierStokesInformedNN(NeuralNetwork):
        pde = "ns_ide"

    hp = {"layers": [int(v) for v in g["layers"]], "tf_epochs": 3, "tf_lr": 0.001, "tf_b1": 0.9, "tf_eps": None,
          "nt_epochs": 4, "nt_lr": 0.8, "nt_ncorr": 50, "log_frequency": 1}
    pinn = NavierStokesInformedNN(hp, Logger(hp), g["ub"], g["lb"])
    pinn._w0 = np.asarray(g["w"])[:-2].copy()
    pinn.logger.set_error_fn(lambda: 0.0)
    assert list(pinn.get_params(numpy=True)) == [0.0, 0.0] and len(pinn.wrap_training_variables()) == 2 * 9 + 2
    pinn.fit(g["X"], g["uv"])
    out = capsys.readouterr().out
    assert "tf_epoch =      2" in out and "nt_epoch =      3" in out
    pb = rn.NavierStokesIdentification(hp["layers"], g["lb"], g["ub"], g["X"], g["uv"])
    wa, _, _ = rp.adam_train(pb, g["w"], 3, lr=1e-3)
    tr = rp.lbfgs_fixed_step(lambda z: rp.loss_and_flat_grad(pb, z), wa, max_iter=4, learning_rate=0.8, n_correction=50,
                             tol_fun=np.finfo(float).eps)
    w = pinn.get_weights().numpy()
    assert rel(w, tr.x_eval[-1]) < 1e-7
    (u, v, p), (f_u, f_v) = pb.predict(w, g["X_probe"])
    U, V, Pp = pinn.predict(g["X_probe"])
    assert U.shape == (64, 1) and rel(U, u) < 1e-10 and rel(V, v) < 1e-10 and rel(Pp, p) < 1e-10
    F_u, F_v = pinn.f_model(g["X_probe"])
    assert rel(F_u, f_u) < 1e-9 and rel(F_v, f_v) < 1e-9
    R_u, R_v = pinn.f_model()
    assert R_u.shape == (g["X"].shape[0], 1)
    l1, l2 = pinn.get_params(numpy=True)
    assert l1 == w[-2] and l2 == w[-1]


def test_driver_script_at_a_tiny_size():
    hp = {"N_train": 300, "layers": [3, 10, 10, 2], "tf_epochs": 5, "nt_epochs": 5, "log_frequency": 1}
    r = subprocess.run([sys.executable, os.path.join(PKG, "2d-navier-stokes", "ide_cont_navier_stokes.py")],
                       env=dict(os.environ, PINN_NS_HP=json.dumps(hp)), capture_output=True, text=True, timeout=600, cwd=PKG)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "Error l1:" in r.stdout and "Error l2:" in r.stdout
