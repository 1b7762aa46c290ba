"""CPU: the Navier-Stokes identification oracles -- nested torch autograd (the upstream formulation, oracle.reference_port_ns)
against the 13 Taylor streams with the hand-derived reverse (oracle.taylor_ns), finite differences, the extended-precision run,
the Taylor-Green data generator, prep_data, and the CUDA kernel's division-free Z-bar formulas restated in numpy."""
import os
import sys

import numpy as np
import pytest
import scipy.io
import torch

from conftest import PKG
from oracle import reference_port as rp, reference_port_ns as rn, taylor_ns as tn

sys.path.insert(0, os.path.join(PKG, "2d-navier-stokes"))
import navierstokesutil as nsu  # noqa: E402


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def ns_case(hidden, n, seed, lb=(1.0, -2.0, 0.0), ub=(8.0, 2.0, 20.0), lam=(0.7, 0.03)):
    rng = np.random.default_rng(seed)
    layers = [3] + hidden + [2]
    lb, ub = np.array(lb), np.array(ub)
    X = lb + (ub - lb) * rng.random((n, 3))
    uv = rng.standard_normal((n, 2))
    w = np.concatenate([rp.glorot_normal_flat(layers, rng) + 0.05 * rng.standard_normal(rp.num_params(layers)), lam])
    return layers, lb, ub, X, uv, w


SIZES = [([7, 7], 13), ([20] * 8, 40), ([33, 33, 33], 17), ([20, 7, 33], 5), ([1, 9], 3)]
BOXES = [((1.0, -2.0, 0.0), (8.0, 2.0, 20.0)), ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), ((0.0, 0.3, 2.0), (1e-2, 0.5, 2.001))]


@pytest.mark.parametrize("hidden,n", SIZES)
@pytest.mark.parametrize("box", range(len(BOXES)))
def test_nested_autograd_matches_taylor(hidden, n, box):
    layers, lb, ub, X, uv, w = ns_case(hidden, n, 11 * n + box, *BOXES[box])
    pb = rn.NavierStokesIdentification(layers, lb, ub, X, uv)
    f, g = rp.loss_and_flat_grad(pb, w)
    f2, g2, parts = tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv)
    assert abs(f - f2) <= 1e-13 * abs(f) and rel(g2, g) <= 1e-13
    assert abs(g2[-2] - g[-2]) <= 1e-13 * np.linalg.norm(g) and abs(g2[-1] - g[-1]) <= 1e-13 * np.linalg.norm(g)
    a, b = (float(v.detach()) for v in pb.loss_parts(torch.as_tensor(w)))
    assert np.allclose(parts, [a, b], rtol=1e-13)
    # the residuals of the upstream formulation from the Taylor streams
    (_, _, _), (f_u, f_v) = pb.predict(w, X)
    O, _ = tn.forward_ns(w[:-2], layers, lb, ub, X)
    t_u, t_v = tn.ns_terms(O, w[-2], w[-1])
    assert rel(t_u, f_u[:, 0]) <= 1e-13 and rel(t_v, f_v[:, 0]) <= 1e-13


def test_against_finite_differences():
    layers, lb, ub, X, uv, w = ns_case([12, 12], 21, 2)
    f = lambda v: tn.ns_ide_loss_grad(v, layers, lb, ub, X, uv)[0]
    _, g, _ = tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv)
    for i in (-2, -1, 0, 3, 40, len(w) - 5):
        h = 1e-6 * max(1.0, abs(w[i]))
        wp, wm = w.copy(), w.copy()
        wp[i] += h; wm[i] -= h
        fd = (f(wp) - f(wm)) / (2 * h)
        assert abs(fd - g[i]) <= 1e-6 * max(abs(g[i]), 1e-3 * np.linalg.norm(g)), i
    # the third-order streams against central differences of the second-order ones
    O, _ = tn.forward_ns(w[:-2], layers, lb, ub, X)
    hx = 1e-5
    for k, (kd, d) in {9: (4, 0), 10: (4, 1), 11: (6, 0), 12: (6, 1), 7: (1, 2), 8: (2, 2)}.items():
        e = np.zeros(3); e[d] = hx
        Op, _ = tn.forward_ns(w[:-2], layers, lb, ub, X + e)
        Om, _ = tn.forward_ns(w[:-2], layers, lb, ub, X - e)
        assert rel((Op[kd] - Om[kd]) / (2 * hx), O[k]) < 1e-6, k


def test_longdouble_matches_float64():
    layers, lb, ub, X, uv, w = ns_case([20, 20], 31, 3)
    f, g, p = tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv)
    fl, gl, pl, ml = tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv, dtype=np.longdouble, magnitudes=True)
    assert gl.dtype == np.longdouble and ml.shape == gl.shape
    assert abs(float(fl) - f) <= 1e-13 * abs(f) and rel(np.asarray(gl, float), g) <= 1e-13


def kernel_zbar(A, B):
    """navier_stokes_fused.cuh zbar_streams, restated: Z-bar_beta = sum_{alpha >= beta} C(alpha, beta) s_(alpha - beta) B_alpha
    with s_gamma = -d^gamma (a^2) written in the stored layer outputs A (no division by s)."""
    a = A[0]
    S = [1.0 - a * a, -2 * a * A[1], -2 * a * A[2], -2 * a * A[3],
         -2 * (a * A[4] + A[1] * A[1]), -2 * (a * A[5] + A[1] * A[2]), -2 * (a * A[6] + A[2] * A[2]),
         -2 * (a * A[7] + A[1] * A[3]), -2 * (a * A[8] + A[2] * A[3]),
         -2 * (a * A[9] + 3 * A[4] * A[1]), -2 * (a * A[10] + A[4] * A[2] + 2 * A[5] * A[1]),
         -2 * (a * A[11] + 2 * A[5] * A[2] + A[6] * A[1]), -2 * (a * A[12] + 3 * A[6] * A[2])]
    s = S[0]
    Z = [sum(S[k] * B[k] for k in range(13)),
         s * B[1] + 2 * S[1] * B[4] + S[2] * B[5] + S[3] * B[7] + 3 * S[4] * B[9] + 2 * S[5] * B[10] + S[6] * B[11],
         s * B[2] + S[1] * B[5] + 2 * S[2] * B[6] + S[3] * B[8] + S[4] * B[10] + 2 * S[5] * B[11] + 3 * S[6] * B[12],
         s * B[3] + S[1] * B[7] + S[2] * B[8],
         s * B[4] + 3 * S[1] * B[9] + S[2] * B[10],
         s * B[5] + 2 * S[1] * B[10] + 2 * S[2] * B[11],
         s * B[6] + S[1] * B[11] + 3 * S[2] * B[12]]
    return Z + [s * B[k] for k in range(7, 13)]


def test_kernel_zbar_formulas_match_the_z_based_reverse():
    rng = np.random.default_rng(5)
    for scale in (0.3, 1.0, 3.0):
        Z = [scale * rng.standard_normal(200) for _ in range(13)]
        B = [rng.standard_normal(200) for _ in range(13)]
        A = tn.tanh_streams(Z)
        ref = tn.zbar(A[0], 1.0 - A[0] ** 2, Z, B)
        got = kernel_zbar(A, B)
        for k in range(13):
            assert rel(got[k], ref[k]) <= 1e-13, (scale, k)


def test_taylor_green_solves_navier_stokes():
    """u = psi_y, v = -psi_x and p of the generator, differentiated exactly (autograd), make f_u and f_v vanish at
    lambda = (1, nu) -- and not at other lambdas."""
    d = nsu.tg_vortex(n_space=50, n_t=7, seed=3)
    k, nu = nsu.TG_K, nsu.TG_NU
    X = np.hstack([np.repeat(d["X_star"], 7, 0), np.tile(d["t"], (50, 1))])
    x, y, t = (torch.tensor(X[:, c:c + 1], requires_grad=True) for c in range(3))
    F = torch.exp(-2 * nu * k * k * t)
    psi = torch.sin(k * x) * torch.sin(k * y) * F / k
    p = 0.25 * (torch.cos(2 * k * x) + torch.cos(2 * k * y)) * F * F
    gr = lambda a, b: torch.autograd.grad(a, b, torch.ones_like(a), create_graph=True)[0]
    u, v = gr(psi, y), -gr(psi, x)
    U = d["U_star"].transpose(0, 2, 1).reshape(-1, 2)
    assert rel(u.detach().numpy()[:, 0], U[:, 0]) < 1e-14 and rel(v.detach().numpy()[:, 0], U[:, 1]) < 1e-14
    assert rel(p.detach().numpy()[:, 0], d["p_star"].reshape(-1)) < 1e-14
    for l1, l2, vanish in ((1.0, nu, True), (0.9, nu, False), (1.0, 2 * nu, False)):
        f_u = gr(u, t) + l1 * (u * gr(u, x) + v * gr(u, y)) + gr(p, x) - l2 * (gr(gr(u, x), x) + gr(gr(u, y), y))
        f_v = gr(v, t) + l1 * (u * gr(v, x) + v * gr(v, y)) + gr(p, y) - l2 * (gr(gr(v, x), x) + gr(gr(v, y), y))
        m = max(float(f_u.detach().abs().max()), float(f_v.detach().abs().max()))
        assert (m <= 1e-12) == vanish, (l1, l2, m)


def test_prep_data_on_a_mat_file(tmp_path):
    path = nsu.write_tg_vortex_mat(str(tmp_path / "tg.mat"), n_space=120, n_t=9, seed=4)
    X, uv, lb, ub, (Xs, us, vs, ps) = nsu.prep_data(path, N_train=200, noise=0.01, seed=99)
    # upstream selection restated directly
    data = scipy.io.loadmat(path)
    Us, Ps, ts, XS = data["U_star"], data["p_star"], data["t"], data["X_star"]
    N, T = XS.shape[0], ts.shape[0]
    x = np.tile(XS[:, 0:1], (1, T)).flatten()[:, None]
    y = np.tile(XS[:, 1:2], (1, T)).flatten()[:, None]
    t = np.tile(ts, (1, N)).T.flatten()[:, None]
    u, v = Us[:, 0, :].flatten()[:, None], Us[:, 1, :].flatten()[:, None]
    rs = np.random.RandomState(99)
    idx = rs.choice(N * T, 200, replace=False)
    u_t, v_t = u[idx], v[idx]
    u_t = u_t + 0.01 * np.std(u_t) * rs.randn(*u_t.shape)
    v_t = v_t + 0.01 * np.std(v_t) * rs.randn(*v_t.shape)
    assert np.array_equal(X, np.hstack([x[idx], y[idx], t[idx]])) and np.array_equal(uv, np.hstack([u_t, v_t]))
    assert np.array_equal(lb, X.min(0)) and np.array_equal(ub, X.max(0))
    assert Xs.shape == (N * T, 3) and np.array_equal(ps, Ps.flatten()[:, None])
    # the default (no path) is the same code path on the in-memory Taylor-Green set
    X2, uv2, *_ = nsu.prep_data(None, N_train=50)
    assert X2.shape == (50, 3) and uv2.shape == (50, 2)
