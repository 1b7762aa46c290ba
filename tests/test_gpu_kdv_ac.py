"""GPU: discrete-time KdV identification (pde id 5, third-order mode) and Allen-Cahn inference (pde id 6, periodic value and
slope pair) on the generic fused kernel -- golden vectors (tests/golden/make_kdv_ac_golden.py), the Taylor oracle at ragged
sizes and widths up to 256, u_xxx from pinn_derivatives, the DMMA and DFMA forms, Adam / L-BFGS trajectories, the C ABI's
error paths, and reference-style classes through the Python surface."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import PKG, ROOT, load_golden

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(PKG, "shims"))


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


@pytest.fixture(scope="module")
def cabi():
    import pinn_cabi
    pinn_cabi.load()
    return pinn_cabi


def make_kdv(cabi, layers, lb, ub, dt, alpha, beta, x_0, u_0, x_1, u_1):
    p = cabi.Pinn(cabi.KDV_IDE_DISC, [int(v) for v in layers], lb, ub)
    p.set_pde_params([float(dt)])
    p.set_irk(cabi.irk_ide_disc(alpha, beta))
    p.set_snapshot(0, x_0, u_0)
    p.set_snapshot(1, x_1, u_1)
    return p


def make_ac(cabi, layers, lb, ub, dt, d, k, irk, x_0, u_0):
    p = cabi.Pinn(cabi.AC_DISC, [int(v) for v in layers], lb, ub)
    p.set_pde_params([float(dt), float(d), float(k)])
    p.set_irk(irk)
    p.set_data(x_0, u_0)
    return p


def golden_handle(cabi, name):
    g = load_golden(name)
    if name == "kdv_ide_disc":
        return g, make_kdv(cabi, g["layers"], g["lb"], g["ub"], g["dt"], g["IRK_alpha"], g["IRK_beta"], g["x_0"], g["u_0"],
                           g["x_1"], g["u_1"])
    return g, make_ac(cabi, g["layers"], g["lb"], g["ub"], g["dt"], g["d"], g["k"], g["IRK"], g["x_0"], g["u_0"])


@pytest.mark.parametrize("name", ["kdv_ide_disc", "ac_disc"])
def test_golden_loss_grad_at_two_points(cabi, name):
    g, p = golden_handle(cabi, name)
    assert p.P == g["w"].size
    for tag in ("", "2"):
        loss, grad, parts = p.loss_grad(w=g["w" + tag])
        assert abs(loss - g["loss" + tag]) <= 1e-10 * abs(g["loss" + tag])
        assert rel(grad, g["grad" + tag]) < 1e-10
        if name == "kdv_ide_disc":
            assert rel(grad[-2:], g["grad" + tag][-2:]) < 1e-10               # d/d lambda_1, d/d lambda_2
        assert np.allclose(parts[:2], g["parts" + tag], rtol=1e-10) and parts[2] == 0.0


@pytest.mark.parametrize("name", ["kdv_ide_disc", "ac_disc"])
def test_adam_and_lbfgs_trajectories(cabi, name):
    g, p = golden_handle(cabi, name)
    p.set_weights(g["w2"])
    losses = [p.adam_step(1e-3) for _ in range(3)]
    assert rel(losses, g["adam_losses"]) < 1e-8 and rel(p.get_weights(), g["adam_w"]) < 1e-8
    g, p = golden_handle(cabi, name)
    p.set_weights(g["w2"])
    r = p.lbfgs(4, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, sync_every=1, want_x_final=True)
    assert r["n_iter"] == 4 and r["n_eval"] == len(g["lbfgs_f"])
    assert rel(r["f_hist"], g["lbfgs_f"]) < 1e-7
    assert rel(r["x_final"], g["lbfgs_x_final"]) < 1e-7
    assert rel(p.get_weights(), g["lbfgs_x_eval"][-1]) < 1e-7


def kdv_inputs(q, n0, n1, hidden, lb=-1.0, ub=1.0, seed=0):
    rng = np.random.default_rng(seed + q + n0)
    from oracle import reference_port as rp
    layers = [1] + hidden + [q]
    w = np.concatenate([rp.glorot_normal_flat(layers, rng) + 0.02 * rng.standard_normal(rp.num_params(layers)), [0.4, -3.0]])
    x_0 = rng.uniform(lb, ub, (n0, 1)); u_0 = np.cos(np.pi * x_0)
    x_1 = rng.uniform(lb, ub, (n1, 1)); u_1 = 0.5 * np.cos(np.pi * x_1)
    alpha = (rng.standard_normal((q, q)) / q).astype(np.float32); beta = (rng.standard_normal((1, q)) / q).astype(np.float32)
    return layers, np.array([lb]), np.array([ub]), w, x_0, u_0, x_1, u_1, 0.6, alpha, beta


def ac_inputs(q, n, hidden, lb=-1.0, ub=1.0, seed=0):
    rng = np.random.default_rng(seed + q + n)
    from oracle import reference_port as rp
    layers = [1] + hidden + [q + 1]
    w = rp.glorot_normal_flat(layers, rng) + 0.02 * rng.standard_normal(rp.num_params(layers))
    x_0 = rng.uniform(lb, ub, (n, 1)); u_0 = x_0 ** 2 * np.cos(np.pi * x_0)
    irk = rng.standard_normal((q + 1, q)) / q
    return layers, np.array([lb]), np.array([ub]), w, x_0, u_0, 0.8, irk


# q up to 512, odd N_0, a single point, widths 7 / 128 / 200 / 256; upstream sizes (KdV [1, 50 x 4, 36] on 199 + 201 points)
KDV_CASES = [(36, 199, 201, [50] * 4), (512, 5, 3, [16]), (7, 33, 1, [7, 7]), (20, 1, 2, [9]), (24, 301, 300, [128, 128]),
             (12, 40, 41, [200, 200]), (9, 60, 11, [256])]
# AC: upstream [1, 200 x 4, 101] on 200 points, q+1 = 512, an odd count, one point, 4001 points (spans many CTAs), width 256
AC_CASES = [(100, 200, [200] * 4), (511, 4, [16]), (16, 37, [7, 128]), (5, 1, [7]), (8, 4001, [20, 20]), (8, 45, [256, 256])]


@pytest.mark.parametrize("q,n0,n1,hidden", KDV_CASES)
def test_kdv_against_taylor_oracle(cabi, q, n0, n1, hidden):
    from oracle import taylor as ty, taylor_kdv_ac as tk
    layers, lb, ub, w, x_0, u_0, x_1, u_1, dt, alpha, beta = kdv_inputs(q, n0, n1, hidden, -0.5, 2.0)
    p = make_kdv(cabi, layers, lb, ub, dt, alpha, beta, x_0, u_0, x_1, u_1)
    loss, grad, parts = p.loss_grad(w=w)
    f2, g2, parts2 = tk.kdv_ide_disc_loss_grad(w, layers, lb, ub, x_0, u_0, x_1, u_1, dt, alpha, beta)
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10
    assert rel(grad[-2:], g2[-2:]) < 1e-10
    assert np.allclose(parts[:2], parts2, rtol=1e-10)


@pytest.mark.parametrize("q,n,hidden", AC_CASES)
def test_ac_against_taylor_oracle(cabi, q, n, hidden):
    from oracle import taylor as ty, taylor_kdv_ac as tk
    layers, lb, ub, w, x_0, u_0, dt, irk = ac_inputs(q, n, hidden, -1.0, 1.5)
    p = make_ac(cabi, layers, lb, ub, dt, 1e-4, 5.0, irk, x_0, u_0)
    loss, grad, parts = p.loss_grad(w=w)
    f2, g2, parts2 = tk.ac_disc_loss_grad(w, layers, lb, ub, x_0, u_0, dt, irk, d=1e-4, k=5.0)
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10
    assert np.allclose(parts[:2], parts2, rtol=1e-10)


def test_derivatives_including_u_xxx(cabi):
    from oracle import taylor as ty, taylor_kdv_ac as tk
    layers, lb, ub, w, x_0, u_0, x_1, u_1, dt, alpha, beta = kdv_inputs(20, 50, 50, [50, 50, 50], -0.5, 2.0)
    p = make_kdv(cabi, layers, lb, ub, dt, alpha, beta, x_0, u_0, x_1, u_1)
    p.set_weights(w)
    X = np.linspace(-0.5, 2.0, 97)[:, None]
    U, Ux, Uxxx, Uxx = p.derivatives(X)
    (T, Tx, Txxx, Txx), _ = tk.forward_third(w[:-2], layers, lb, ub, X)
    for a, b in ((U, T), (Ux, Tx), (Uxx, Txx), (Uxxx, Txxx)):
        assert rel(a, b) <= 1e-11
    assert rel(p.predict(X), T) <= 1e-11
    # AC: no third-order mode, the t block stays zero for a 1-D net; a 200-wide net takes the wide forward
    layers, lb, ub, w, x_0, u_0, dt, irk = ac_inputs(30, 20, [200, 200])
    p = make_ac(cabi, layers, lb, ub, dt, 1e-4, 5.0, irk, x_0, u_0)
    p.set_weights(w)
    U, Ux, Ut, Uxx = p.derivatives(X)
    (T, Tx, _, Txx), _ = ty.forward(w, layers, lb, ub, X)
    assert rel(U, T) <= 1e-11 and rel(Ux, Tx) <= 1e-11 and rel(Uxx, Txx) <= 1e-11 and not Ut.any()


def test_dmma_and_dfma_forms_agree():
    code = r'''
import os, sys, json, numpy as np
ROOT = %r
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "pinns-tf2.0_b200", "utils")]
import pinn_cabi
from test_gpu_kdv_ac import kdv_inputs, ac_inputs, make_kdv, make_ac
out = {}
layers, lb, ub, w, x_0, u_0, x_1, u_1, dt, alpha, beta = kdv_inputs(36, 199, 201, [50] * 4)
p = make_kdv(pinn_cabi, layers, lb, ub, dt, alpha, beta, x_0, u_0, x_1, u_1)
loss, grad, _ = p.loss_grad(w=w)
out["kdv"] = {"loss": loss, "grad": grad.tolist()}
layers, lb, ub, w, x_0, u_0, dt, irk = ac_inputs(20, 301, [200, 200])
p = make_ac(pinn_cabi, layers, lb, ub, dt, 1e-4, 5.0, irk, x_0, u_0)
loss, grad, _ = p.loss_grad(w=w)
out["ac"] = {"loss": loss, "grad": grad.tolist()}
print(json.dumps(out))
''' % ROOT
    res = {}
    for mode in ("0", "1"):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PINN_GENERIC_DFMA=mode), capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        res[mode] = json.loads(r.stdout.strip().splitlines()[-1])
    for name in ("kdv", "ac"):
        a, b = res["0"][name], res["1"][name]
        assert abs(a["loss"] - b["loss"]) <= 1e-12 * abs(b["loss"]) and rel(a["grad"], b["grad"]) < 1e-12
        assert a["grad"] != b["grad"]          # two different summation orders actually ran


def test_get_params_and_error_paths(cabi):
    g, p = golden_handle(cabi, "kdv_ide_disc")
    p.set_weights(g["w2"])
    l1, kappa = p.get_params()
    assert l1 == g["w2"][-2] and abs(kappa - np.exp(g["w2"][-1])) < 1e-15
    g, p = golden_handle(cabi, "ac_disc")
    assert list(p.get_params()) == [float(g["dt"]), float(g["d"]), float(g["k"])]
    lb, ub = np.array([-1.0]), np.array([1.0])
    with pytest.raises(cabi.PinnError, match="AC_DISC takes"):
        p.set_pde_params([0.8, 1e-4])
    with pytest.raises(cabi.PinnError, match="periodic pair"):
        p.set_boundary([0.0])
    with pytest.raises(cabi.PinnError, match="q\\+1 must equal"):
        p.set_irk(np.zeros((5, 4)))
    with pytest.raises(cabi.PinnError, match="set_irk first"):
        h = cabi.Pinn(cabi.AC_DISC, [1, 8, 5], lb, ub)
        h.set_pde_params([0.8, 1e-4, 5.0]); h.set_data(np.zeros((3, 1)), np.zeros((3, 1)))
        h.loss_grad(w=np.zeros(h.P))
    with pytest.raises(cabi.PinnError, match="no points set"):
        h = cabi.Pinn(cabi.AC_DISC, [1, 8, 5], lb, ub)
        h.set_pde_params([0.8, 1e-4, 5.0]); h.set_irk(np.zeros((5, 4)))
        h.loss_grad(w=np.zeros(h.P))
    with pytest.raises(cabi.PinnError, match="1-D input"):
        cabi.Pinn(cabi.AC_DISC, [2, 8, 5], [-1, 0], [1, 1])
    with pytest.raises(cabi.PinnError, match="q\\+1 >= 2"):
        cabi.Pinn(cabi.AC_DISC, [1, 8, 1], lb, ub)
    with pytest.raises(cabi.PinnError, match="width out of range"):
        cabi.Pinn(cabi.KDV_IDE_DISC, [1, 257, 4], lb, ub)
    k = cabi.Pinn(cabi.KDV_IDE_DISC, [1, 8, 4], lb, ub)
    with pytest.raises(cabi.PinnError, match="take \\[dt\\]"):
        k.set_pde_params([0.6, 1.0])
    with pytest.raises(cabi.PinnError, match="q must equal"):
        k.set_irk(np.zeros((10, 5)))
    with pytest.raises(cabi.PinnError, match="set_irk first"):
        k.set_snapshot(0, np.zeros(3), np.zeros(3))
        k.loss_grad(w=np.zeros(k.P))
    with pytest.raises(cabi.PinnError, match="no collocation set"):
        k.set_collocation(np.zeros(3), np.zeros(3))
    with pytest.raises(cabi.PinnError, match="not defined for the discrete-time"):
        k.residual()


def test_width_200_continuous_burgers_net(cabi):
    """Hidden widths up to 256 hold for every generic net, not only the discrete-time ones."""
    from oracle import taylor as ty, taylor_kdv_ac as tk
    rng = np.random.default_rng(200)
    layers = [2, 200, 200, 1]
    lb, ub = np.array([-1.0, 0.0]), np.array([1.0, 0.99])
    X_f = lb + (ub - lb) * rng.random((999, 2)); X_u = lb + (ub - lb) * rng.random((50, 2)); u = rng.uniform(-1, 1, (50, 1))
    P = sum(layers[i] * layers[i + 1] + layers[i + 1] for i in range(len(layers) - 1))
    w = 0.1 * rng.standard_normal(P)
    p = cabi.Pinn(cabi.BURGERS_INF, layers, lb, ub)
    p.set_pde_params([0.01 / np.pi]); p.set_collocation(X_f[:, 0], X_f[:, 1]); p.set_data(X_u, u)
    loss, grad, _ = p.loss_grad(w=w)
    f2, g2, _ = ty.burgers_loss_grad(w, layers, lb, ub, X_f, X_u, u, nu=0.01 / np.pi)
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10
    p.set_weights(w)
    U, Ux, Ut, Uxx = p.derivatives(X_u)
    (T, Tx, Tt, Txx), _ = ty.forward(w, layers, lb, ub, X_u)
    assert rel(np.hstack([U, Ux, Ut, Uxx]), np.hstack([T, Tx, Tt, Txx])) <= 1e-11


def test_kdv_reference_style_class_through_the_surface(capsys):
    """A KdV.py-style class (tape bodies elided): the two-snapshot fit() runs the native loop from lambda = (0, -6),
    predict() returns (U_0, U_1), get_params() the identified (lambda_1, exp(lambda_2))."""
    from logger import Logger
    from neuralnetwork import NeuralNetwork
    g = load_golden("kdv_ide_disc")
    q = int(g["q"])

    class KdVInformedNN(NeuralNetwork):
        pde = "kdv_ide_disc"

        def __init__(self, hp, logger, dt, lb, ub, q, IRK_alpha, IRK_beta):
            super().__init__(hp, logger, ub, lb)
            self.dt, self.q, self.IRK_alpha, self.IRK_beta = dt, q, IRK_alpha, IRK_beta

        def U_0_model(self, x, customDummy=None):
            raise AssertionError("tape body must have been replaced")

        def grad(self, x_0, u_0, x_1, u_1):
            raise AssertionError("tape body must have been replaced")

        def fit(self, x_0, u_0, x_1, u_1):
            raise AssertionError("the four-argument fit must run the native loop")

        def predict(self, x_star):
            raise AssertionError("the two-snapshot predict must run natively")

    hp = {"layers": [int(v) for v in g["layers"]], "tf_epochs": 3, "tf_lr": 0.001, "tf_b1": 0.9, "tf_eps": None,
          "nt_epochs": 4, "nt_lr": 0.8, "nt_ncorr": 50, "log_frequency": 1}
    pinn = KdVInformedNN(hp, Logger(hp), float(g["dt"]), g["lb"], g["ub"], q, g["IRK_alpha"], g["IRK_beta"])
    pinn._w0 = np.asarray(g["w"])[:-2].copy()
    pinn.logger.set_error_fn(lambda: 0.0)
    loss, grads = pinn.grad(g["x_0"], g["u_0"], g["x_1"], g["u_1"])
    assert abs(loss - g["loss"]) <= 1e-10 * abs(g["loss"]) and len(grads) == 2 * 4 + 2
    pinn.fit(g["x_0"], g["u_0"], g["x_1"], g["u_1"])
    out = capsys.readouterr().out
    assert "tf_epoch =      2" in out and "nt_epoch =      3" in out and "l1 = " in out
    U0, U1 = pinn.predict(g["x_star"])
    assert U0.shape == U1.shape == (g["x_star"].shape[0], q)
    # the two-snapshot models on the host use U_xxx from the device
    from oracle import taylor as ty, taylor_kdv_ac as tk
    w = pinn.get_weights().numpy()
    (U, Ux, Uxxx, _), _ = tk.forward_third(w[:-2], hp["layers"], g["lb"], g["ub"], g["x_star"])
    N = w[-2] * U * Ux + np.exp(w[-1]) * Uxxx
    assert rel(U0, U + float(g["dt"]) * N @ g["IRK_alpha"].astype(np.float64).T) < 1e-11
    l1, l2 = pinn.get_params(numpy=True)
    assert l1 == w[-2] and abs(l2 - np.exp(w[-1])) < 1e-15


def test_ac_reference_style_class_through_the_surface(capsys):
    """An AC.py-style class: fit(x_0, u_0) runs Adam then L-BFGS on the fused kernel, predict() returns U1 (all q+1 outputs);
    it has no identified parameters."""
    from logger import Logger
    from neuralnetwork import NeuralNetwork
    from oracle import reference_port as rp, reference_port_kdv_ac as rk
    g = load_golden("ac_disc")
    q = int(g["q"])

    class ACInformedNN(NeuralNetwork):
        pde = "ac_disc"

        def __init__(self, hp, logger, dt, lb, ub, q, IRK_weights):
            super().__init__(hp, logger, ub, lb)
            self.dt, self.q, self.IRK_weights = dt, q, IRK_weights
            self.d, self.k = 1e-4, 5.0

        def loss(self, x_0, u_0):
            raise AssertionError("tape body must have been replaced")

    hp = {"layers": [int(v) for v in g["layers"]], "tf_epochs": 3, "tf_lr": 0.001, "tf_b1": 0.9, "tf_eps": None,
          "nt_epochs": 4, "nt_lr": 0.8, "nt_ncorr": 50, "log_frequency": 1}
    pinn = ACInformedNN(hp, Logger(hp), float(g["dt"]), g["lb"], g["ub"], q, g["IRK"])
    pinn._w0 = np.asarray(g["w2"]).copy()
    pinn.logger.set_error_fn(lambda: 0.0)
    pinn.fit(g["x_0"], g["u_0"])
    out = capsys.readouterr().out
    assert "tf_epoch =      2" in out and "nt_epoch =      3" in out
    # Adam then L-BFGS from w2: the weights the two golden runs reach when chained
    pb = rk.AllenCahnDiscreteInference(hp["layers"], g["lb"], g["ub"], float(g["dt"]), g["x_0"], g["u_0"], g["IRK"])
    tr = rp.lbfgs_fixed_step(lambda z: rp.loss_and_flat_grad(pb, z), g["adam_w"], max_iter=4, learning_rate=0.8,
                             n_correction=50, tol_fun=np.finfo(float).eps)
    assert rel(pinn.get_weights().numpy(), tr.x_eval[-1]) < 1e-7
    X = np.linspace(-1, 1, 17)[:, None]
    U1 = pinn.predict(X)
    assert U1.shape == (17, q + 1) and rel(U1, rp.predict(pb, pinn.get_weights().numpy(), X)) < 1e-11
    assert pinn.get_params() == []
