"""Independent fp64 oracle for the discrete-time KdV identification and Allen-Cahn inference models: forward Taylor-mode
streams with a third-order mode, and the hand-derived reverse sweep.

TEST INFRASTRUCTURE (see oracle/__init__.py).  numpy only; built on the contraction helpers of ``oracle.taylor`` and shares no
derivation with ``oracle.reference_port_kdv_ac`` (nested autograd).  The two must agree to ~1e-13.  Every entry point takes
dtype= (np.longdouble runs the same sums with a 64-bit mantissa on x86-64).

Third-order mode (1-D nets only): the slot of the t stream carries h_xxx instead (input h_xxx = 0), so outputs are
(u, u_x, u_xxx, u_xx).  Per tanh layer, z = hW+b, a = tanh z, s = 1-a^2:
    a_xxx = s z_xxx - 6 a s z_x z_xx - 2 s (1-3a^2) z_x^3
Reverse with adjoints (A, A_x, A_xxx, A_xx):
    Z_xxx = s A_xxx;  Z_xx = s A_xx - 6 a s z_x A_xxx
    Z_x   = s A_x - 4 a s z_x A_xx - A_xxx (6 a s z_xx + 6 s (1-3a^2) z_x^2)
    Z     = s A - 2 a s z_x A_x - A_xx (2 a s z_xx + 2 s (1-3a^2) z_x^2)
            + A_xxx (-2 a s z_xxx - 6 s (1-3a^2) z_x z_xx + 8 a s (2-3a^2) z_x^3)
The other three streams are those of oracle.taylor.forward, operation for operation.
"""
from __future__ import annotations

import numpy as np

from oracle.taylor import _backward_sum, _contraction, _flat, _magnitude, _unpack, forward


def forward_third(w, layers, lb, ub, X, dtype=np.float64):
    """X: (N,1) -> outputs (u, u_x, u_xxx, u_xx), each (N, n_out), and the per-layer stash."""
    if int(layers[0]) != 1:
        raise ValueError("the third-order mode needs a 1-D input")
    X = np.asarray(X, dtype=dtype)
    lb, ub = np.asarray(lb, dtype).reshape(-1), np.asarray(ub, dtype).reshape(-1)
    Ws, bs = _unpack(np.asarray(w, dtype=dtype), layers)
    N = X.shape[0]
    sc = 2.0 / (ub[:1] - lb[:1])
    h = sc * (X[:, :1] - lb[:1]) - 1.0
    hx = np.full((N, 1), sc[0], dtype); hxxx = np.zeros((N, 1), dtype); hxx = np.zeros((N, 1), dtype)
    stash = []
    for l in range(len(Ws) - 1):
        W, b = Ws[l], bs[l]
        z, zx, zxxx, zxx = h @ W + b, hx @ W, hxxx @ W, hxx @ W
        a = np.tanh(z)
        s = 1.0 - a * a
        stash.append((h, hx, hxxx, hxx, a, s, zx, zxxx, zxx))
        hxxx = s * zxxx - 6.0 * a * s * zx * zxx - 2.0 * s * (1.0 - 3.0 * a * a) * zx ** 3
        h, hx, hxx = a, s * zx, s * zxx - 2.0 * a * s * zx * zx
    W, b = Ws[-1], bs[-1]
    stash.append((h, hx, hxxx, hxx))
    return (h @ W + b, hx @ W, hxxx @ W, hxx @ W), stash


def backward_third(w, layers, stash, seeds, dtype=np.float64, magnitudes=False):
    """seeds: adjoints of (u, u_x, u_xxx, u_xx).  Returns the flat parameter gradient (and with magnitudes=True the
    per-entry contraction magnitudes, as oracle.taylor.backward)."""
    Ws, _ = _unpack(np.asarray(w, dtype=dtype), layers)
    g, m = [], []
    h, hx, hxxx, hxx = stash[-1]
    Z, Zx, Zxxx, Zxx = seeds
    g.append(_contraction(h, hx, hxxx, hxx, Z, Zx, Zxxx, Zxx))
    if magnitudes:
        m.append(_magnitude(h, hx, hxxx, hxx, Z, Zx, Zxxx, Zxx))
    WT = Ws[-1].T
    A, Ax, Axxx, Axx = Z @ WT, Zx @ WT, Zxxx @ WT, Zxx @ WT
    for l in range(len(Ws) - 2, -1, -1):
        h, hx, hxxx, hxx, a, s, zx, zxxx, zxx = stash[l]
        c3 = 1.0 - 3.0 * a * a
        Zxxx = s * Axxx
        Zxx = s * Axx - 6.0 * a * s * zx * Axxx
        Zx = s * Ax - 4.0 * a * s * zx * Axx - Axxx * (6.0 * a * s * zxx + 6.0 * s * c3 * zx * zx)
        Z = (s * A - 2.0 * a * s * zx * Ax - Axx * (2.0 * a * s * zxx + 2.0 * s * c3 * zx * zx)
             + Axxx * (-2.0 * a * s * zxxx - 6.0 * s * c3 * zx * zxx + 8.0 * a * s * (2.0 - 3.0 * a * a) * zx ** 3))
        g.append(_contraction(h, hx, hxxx, hxx, Z, Zx, Zxxx, Zxx))
        if magnitudes:
            m.append(_magnitude(h, hx, hxxx, hxx, Z, Zx, Zxxx, Zxx))
        if l > 0:
            WT = Ws[l].T
            A, Ax, Axxx, Axx = Z @ WT, Zx @ WT, Zxxx @ WT, Zxx @ WT
    return (_flat(g), _flat(m)) if magnitudes else _flat(g)


def kdv_ide_disc_loss_grad(w, layers, lb, ub, x_0, u_0, x_1, u_1, dt, IRK_alpha, IRK_beta, dtype=np.float64,
                           magnitudes=False):
    """Discrete-time KdV identification (PINNs/main/discrete_time_identification (KdV)/KdV.py, restated in fp64):
    u_t + l1 u u_x + e^{l2} u_xxx = 0; w = [net, l1, l2], net [1, ..., q]; N = l1 U U_x + e^{l2} U_xxx;
    pred = U + dt N M^T with M_0 = alpha on x_0 and M_1 = -(beta - alpha) on x_1 (the convention of
    oracle.taylor.burgers_ide_disc_loss_grad); loss = sum((pred_0 - u_0)^2) + sum((pred_1 - u_1)^2).
    Upstream (from memory, not pinned): l1 init 0.0, l2 init -6.0, N_0 = 199, N_1 = 201, layers [1, 50 x 4, q]."""
    w = np.asarray(w, dtype=dtype)
    wn, l1, kappa = w[:-2], w[-2], np.exp(w[-1])
    A = np.asarray(IRK_alpha, dtype=dtype)
    # beta - alpha in the tables' own dtype, as for the Burgers identification
    M1 = -np.asarray(np.asarray(IRK_beta).reshape(1, -1) - np.asarray(IRK_alpha), dtype=dtype)
    g, m = np.zeros(wn.size, dtype), 0
    dl1 = dl2 = dtype(0.0)
    ml1 = ml2 = dtype(0.0)
    parts = []
    for x, u, M in ((x_0, u_0, A), (x_1, u_1, M1)):
        (U, Ux, Uxxx, _), st = forward_third(wn, layers, lb, ub, x, dtype)
        Nn = l1 * U * Ux + kappa * Uxxx
        R = 2.0 * (U + dt * Nn @ M.T - u)
        Nbar = dt * R @ M
        r = backward_third(wn, layers, st, (R + Nbar * l1 * Ux, Nbar * l1 * U, kappa * Nbar, np.zeros_like(R)), dtype,
                           magnitudes)
        gs, ms = r if magnitudes else (r, 0)
        g, m = g + gs, m + ms
        dl1 += dtype(np.sum(Nbar * U * Ux))
        dl2 += dtype(np.sum(kappa * Nbar * Uxxx))
        if magnitudes:
            ml1 += np.sum(np.abs(Nbar * U * Ux)); ml2 += np.sum(np.abs(kappa * Nbar * Uxxx))
        parts.append(dtype(np.sum((0.5 * R) ** 2)))
    return (parts[0] + parts[1], np.concatenate([g, [dl1, dl2]]), tuple(parts)) + \
        ((np.concatenate([m, [ml1, ml2]]),) if magnitudes else ())


def ac_disc_loss_grad(w, layers, lb, ub, x_0, u_0, dt, IRK_weights, d=1e-4, k=5.0, dtype=np.float64, magnitudes=False):
    """Discrete-time Allen-Cahn inference (PINNs/main/discrete_time_inference (AC)/AC.py, restated in fp64):
    u_t - d u_xx + k u^3 - k u = 0; net [1, ..., q+1]; U_1 = net(x) (N, q+1); U = U_1[:, :q]; N = k U^3 - k U - d U_xx;
    U_0 = U_1 + dt N IRK^T (IRK: (q+1, q)); with D = U_1(lb) - U_1(ub) over all q+1 outputs,
    loss = sum((U_0 - u_0)^2) + sum(D^2) + sum(D_x^2)  (periodic in value and slope).
    Upstream (from memory, not pinned): d = 1e-4, k = 5, N = 200, dt = 0.8, layers [1, 200 x 4, q+1]."""
    w = np.asarray(w, dtype=dtype)
    IRK = np.asarray(IRK_weights, dtype=dtype)
    q = IRK.shape[1]
    (U1, U1x, _, U1xx), st = forward(w, layers, lb, ub, x_0, dtype)
    U, Uxx = U1[:, :q], U1xx[:, :q]
    Nn = k * U ** 3 - k * U - d * Uxx
    U0 = U1 + dt * Nn @ IRK.T
    R = 2.0 * (U0 - u_0)
    Nbar = dt * R @ IRK
    S = R.copy(); S[:, :q] += Nbar * (3.0 * k * U * U - k)
    Sxx = np.zeros_like(R); Sxx[:, :q] = -d * Nbar
    zr = np.zeros_like(R)
    g, m = _backward_sum(w, layers, st, (S, zr, zr, Sxx), dtype, magnitudes)
    loss0 = dtype(np.sum((U0 - u_0) ** 2))
    xb = np.array([[np.asarray(lb).reshape(-1)[0]], [np.asarray(ub).reshape(-1)[0]]])
    (B, Bx, _, _), stb = forward(w, layers, lb, ub, xb, dtype)
    D, Dx = B[0:1] - B[1:2], Bx[0:1] - Bx[1:2]
    zb = np.zeros_like(B)
    g2, m2 = _backward_sum(w, layers, stb, (2.0 * np.concatenate([D, -D]), 2.0 * np.concatenate([Dx, -Dx]), zb, zb), dtype,
                           magnitudes)
    g, m = g + g2, m + m2
    loss1 = dtype(np.sum(D * D) + np.sum(Dx * Dx))
    return (loss0 + loss1, g, (loss0, loss1)) + ((m,) if magnitudes else ())
