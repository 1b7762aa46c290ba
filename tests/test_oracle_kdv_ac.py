"""CPU: the discrete-time KdV identification and Allen-Cahn inference oracles -- nested torch autograd (the upstream
formulation, oracle.reference_port_kdv_ac) against the Taylor-mode streams with the third-order mode (oracle.taylor_kdv_ac), finite
differences of U_xxx and of the lambda gradients, and the extended-precision Taylor run against the fp64 one."""
import numpy as np
import pytest
import torch

from oracle import reference_port as rp, reference_port_kdv_ac as rk, taylor as ty, taylor_kdv_ac as tk


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def kdv_case(q, n0, n1, hidden, seed, lb=-1.0, ub=1.0):
    rng = np.random.default_rng(seed)
    layers = [1] + hidden + [q]
    w = np.concatenate([rp.glorot_normal_flat(layers, rng) + 0.05 * rng.standard_normal(rp.num_params(layers)), [0.7, -2.0]])
    x_0 = rng.uniform(lb, ub, (n0, 1)); u_0 = np.cos(np.pi * x_0)
    x_1 = rng.uniform(lb, ub, (n1, 1)); u_1 = 0.8 * np.cos(np.pi * x_1 + 0.3)
    alpha = (rng.standard_normal((q, q)) / q).astype(np.float32)
    beta = (rng.standard_normal((1, q)) / q).astype(np.float32)
    return layers, np.array([lb]), np.array([ub]), w, x_0, u_0, x_1, u_1, 0.6, alpha, beta


def ac_case(q, n, hidden, seed, lb=-1.0, ub=1.0):
    rng = np.random.default_rng(seed)
    layers = [1] + hidden + [q + 1]
    w = rp.glorot_normal_flat(layers, rng) + 0.05 * rng.standard_normal(rp.num_params(layers))
    x_0 = rng.uniform(lb, ub, (n, 1)); u_0 = x_0 ** 2 * np.cos(np.pi * x_0)
    irk = rng.standard_normal((q + 1, q)) / q
    return layers, np.array([lb]), np.array([ub]), w, x_0, u_0, 0.8, irk


KDV_SIZES = [(5, 17, 3, [12, 7]), (1, 6, 4, [8]), (4, 1, 1, [1]), (9, 11, 13, [1, 6]), (16, 40, 30, [20, 20, 20])]
AC_SIZES = [(5, 17, [12, 7]), (1, 6, [8]), (3, 1, [1]), (8, 13, [1, 6]), (16, 40, [20, 20, 20])]


@pytest.mark.parametrize("q,n0,n1,hidden", KDV_SIZES)
def test_kdv_nested_autograd_matches_taylor(q, n0, n1, hidden):
    layers, lb, ub, w, x_0, u_0, x_1, u_1, dt, alpha, beta = kdv_case(q, n0, n1, hidden, q + 7 * n0, -0.5, 2.0)
    pb = rk.KdVDiscreteIdentification(layers, lb, ub, dt, x_0, u_0, x_1, u_1, alpha, beta)
    f, g = rp.loss_and_flat_grad(pb, w)
    f2, g2, parts = tk.kdv_ide_disc_loss_grad(w, layers, lb, ub, x_0, u_0, x_1, u_1, dt, alpha, beta)
    assert abs(f - f2) <= 1e-13 * abs(f) and rel(g2, g) <= 1e-13
    assert abs(g2[-2] - g[-2]) <= 1e-13 * abs(g[-2]) and abs(g2[-1] - g[-1]) <= 1e-13 * abs(g[-1])
    a, b = (float(v.detach()) for v in pb.loss_parts(torch.as_tensor(w)))
    assert np.allclose(parts, [a, b], rtol=1e-13)
    U, U_x, U_xx, U_xxx = (v.detach().numpy() for v in pb.autograd(torch.as_tensor(w[:-2]), torch.as_tensor(x_0)))
    (T, T_x, T_xxx, T_xx), _ = tk.forward_third(w[:-2], layers, lb, ub, x_0)
    for a_, b_ in ((T, U), (T_x, U_x), (T_xx, U_xx), (T_xxx, U_xxx)):
        assert rel(a_, b_) <= 1e-13


@pytest.mark.parametrize("q,n,hidden", AC_SIZES)
def test_ac_nested_autograd_matches_taylor(q, n, hidden):
    layers, lb, ub, w, x_0, u_0, dt, irk = ac_case(q, n, hidden, 3 * q + n, -1.0, 1.5)
    pb = rk.AllenCahnDiscreteInference(layers, lb, ub, dt, x_0, u_0, irk, d=1e-3, k=5.0)
    f, g = rp.loss_and_flat_grad(pb, w)
    f2, g2, parts = tk.ac_disc_loss_grad(w, layers, lb, ub, x_0, u_0, dt, irk, d=1e-3, k=5.0)
    assert abs(f - f2) <= 1e-13 * abs(f) and rel(g2, g) <= 1e-13
    a, b = (float(v.detach()) for v in pb.loss_parts(torch.as_tensor(w)))
    assert np.allclose(parts, [a, b], rtol=1e-13)


def test_third_order_stream_against_finite_differences():
    layers, lb, ub, w, x_0, *_ = kdv_case(6, 9, 1, [10, 10], 1, -1.0, 3.0)
    wn = w[:-2]
    (_, _, _, Uxx), _ = tk.forward_third(wn, layers, lb, ub, x_0)
    (_, _, Uxxx, _), _ = tk.forward_third(wn, layers, lb, ub, x_0)
    h = 1e-4
    (_, _, _, Uxx_p), _ = tk.forward_third(wn, layers, lb, ub, x_0 + h)
    (_, _, _, Uxx_m), _ = tk.forward_third(wn, layers, lb, ub, x_0 - h)
    assert rel((Uxx_p - Uxx_m) / (2 * h), Uxxx) < 1e-6
    # the other streams are those of the second-order mode, bit for bit
    (a, b, _, c), _ = ty.forward(wn, layers, lb, ub, x_0)
    (a3, b3, _, c3), _ = tk.forward_third(wn, layers, lb, ub, x_0)
    assert np.array_equal(a, a3) and np.array_equal(b, b3) and np.array_equal(c, c3)


def test_lambda_gradients_against_finite_differences():
    layers, lb, ub, w, x_0, u_0, x_1, u_1, dt, alpha, beta = kdv_case(5, 21, 19, [12, 12], 2)
    f = lambda v: tk.kdv_ide_disc_loss_grad(v, layers, lb, ub, x_0, u_0, x_1, u_1, dt, alpha, beta)[0]
    _, g, _ = tk.kdv_ide_disc_loss_grad(w, layers, lb, ub, x_0, u_0, x_1, u_1, dt, alpha, beta)
    for i in (-2, -1, 3, len(w) - 5):
        h = 1e-6 * max(1.0, abs(w[i]))
        wp, wm = w.copy(), w.copy()
        wp[i] += h; wm[i] -= h
        fd = (f(wp) - f(wm)) / (2 * h)
        assert abs(fd - g[i]) <= 1e-6 * max(abs(g[i]), 1e-3 * np.linalg.norm(g)), i


def test_longdouble_matches_float64():
    layers, lb, ub, w, x_0, u_0, x_1, u_1, dt, alpha, beta = kdv_case(9, 31, 29, [20, 20], 3)
    f, g, p = tk.kdv_ide_disc_loss_grad(w, layers, lb, ub, x_0, u_0, x_1, u_1, dt, alpha, beta)
    fl, gl, pl = tk.kdv_ide_disc_loss_grad(w, layers, lb, ub, x_0, u_0, x_1, u_1, dt, alpha, beta, dtype=np.longdouble)
    assert gl.dtype == np.longdouble
    assert abs(float(fl) - f) <= 1e-13 * abs(f) and rel(np.asarray(gl, float), g) <= 1e-13
    layers, lb, ub, w, x_0, u_0, dt, irk = ac_case(9, 31, [20, 20], 4)
    f, g, _ = tk.ac_disc_loss_grad(w, layers, lb, ub, x_0, u_0, dt, irk)
    fl, gl, _ = tk.ac_disc_loss_grad(w, layers, lb, ub, x_0, u_0, dt, irk, dtype=np.longdouble)
    assert gl.dtype == np.longdouble
    assert abs(float(fl) - f) <= 1e-13 * abs(f) and rel(np.asarray(gl, float), g) <= 1e-13
