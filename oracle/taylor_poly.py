"""User-defined polynomial residuals on the forward Taylor streams of ``oracle.taylor`` with the analytic seed formula.

TEST INFRASTRUCTURE (see oracle/__init__.py).  numpy only; shares no derivation with ``oracle.reference_port_poly`` (nested
autograd).  Every entry point takes dtype= (np.longdouble: the extended-precision reference of tests/test_gpu_poly.py).

With streams v = (u, u_x, u_t, u_xx) and a term m_k = c_k kappa_k prod_j v_j^e_kj:
    f = sum_k m_k - s
    dL/dv_j = 2 w f sum_k c_k kappa_k e_kj v_j^(e_kj - 1) prod_{i != j} v_i^e_ki   (+ 2 w_d (u - u_d) for j = u)
    dL/dl_i = 2 w f df/dl_i,  d(l_i)/dl_i = 1,  d(e^l_i)/dl_i = e^l_i
The power e - 1 is formed directly, never by dividing by v_j, so u = 0 is an ordinary point.
"""
from __future__ import annotations

import numpy as np

from oracle.taylor import _backward_sum, forward


def _pw(v, e):
    out = np.ones_like(v)
    for _ in range(e):
        out = out * v
    return out


def poly_terms(terms, V, l1=0.0, l2=0.0, dtype=np.float64, magnitudes=False):
    """(f without the source, [df/dv_j for j = u, u_x, u_t, u_xx], df/dl1, df/dl2) on the stream arrays V.
    magnitudes=True appends the term-wise magnitudes of df/dl1 and df/dl2 (sum_k |d kappa_k/dl_i m_k|): the scale of the
    rounding of a sum over the terms, which |df/dl_i| under-counts where terms cancel (Fisher-KPP's -l1 u + l1 u^2 at u = 1)."""
    e1, e2 = np.exp(dtype(l1)), np.exp(dtype(l2))
    kv = (dtype(1), dtype(l1), dtype(l2), e1, e2)
    f = np.zeros_like(V[0])
    D = [np.zeros_like(V[0]) for _ in range(4)]
    f1, f2 = np.zeros_like(V[0]), np.zeros_like(V[0])
    a1, a2 = np.zeros_like(V[0]), np.zeros_like(V[0])
    for c, k, e in terms:
        c = dtype(c)
        q = [_pw(V[j], e[j]) for j in range(4)]
        m = c * q[0] * q[1] * q[2] * q[3]
        f = f + kv[k] * m
        for j in range(4):
            if e[j]:
                other = np.ones_like(V[0])
                for i in range(4):
                    if i != j:
                        other = other * q[i]
                D[j] = D[j] + c * kv[k] * e[j] * _pw(V[j], e[j] - 1) * other
        if k in (1, 3):
            f1 = f1 + (m if k == 1 else e1 * m)
            a1 = a1 + np.abs(m if k == 1 else e1 * m)
        elif k in (2, 4):
            f2 = f2 + (m if k == 2 else e2 * m)
            a2 = a2 + np.abs(m if k == 2 else e2 * m)
    return (f, D, f1, f2) + ((a1, a2) if magnitudes else ())


def poly_loss_grad(w, layers, lb, ub, terms, X_u, u, X_f=None, source=None, identification=False, n_f_global=None,
                   data_weight=1.0, dtype=np.float64, magnitudes=False):
    """Loss, flat gradient and parts (mse_u, mse_f) of PINN_POLY_INF (identification=False: the BURGERS_INF structure on the
    collocation points X_f) or PINN_POLY_IDE (w = [net, l1, l2], residual on X_u, the BURGERS_IDE structure).
    magnitudes=True appends the contraction magnitudes of every gradient entry (oracle.taylor.backward)."""
    w = np.asarray(w, dtype=dtype)
    u = np.asarray(u, dtype=dtype).reshape(-1, 1)
    if identification:
        wn, l1, l2 = w[:-2], w[-2], w[-1]
        X_f = X_u
    else:
        wn, l1, l2 = w, dtype(0), dtype(0)
    nf = X_f.shape[0] if identification else (n_f_global or X_f.shape[0])
    (U, Ux, Ut, Uxx), st = forward(wn, layers, lb, ub, X_f, dtype)
    f, D, f1, f2, *a = poly_terms(terms, (U, Ux, Ut, Uxx), l1, l2, dtype, magnitudes)
    if source is not None:
        f = f - np.asarray(source, dtype=dtype).reshape(-1, 1)
    c = 2.0 * f / nf
    g, m = _backward_sum(wn, layers, st, tuple(c * d for d in D), dtype, magnitudes)
    mse_f = dtype(np.sum(f * f) / nf)
    (Ud, _, _, _), std = forward(wn, layers, lb, ub, X_u, dtype)
    r = Ud - u
    n_u = X_u.shape[0]
    wd = dtype(1.0) if identification else dtype(data_weight)
    zero = np.zeros_like(r)
    g2, m2 = _backward_sum(wn, layers, std, (wd * 2.0 * r / n_u, zero, zero, zero), dtype, magnitudes)
    g, m = g + g2, m + m2
    mse_u = wd * dtype(np.sum(r * r) / n_u)
    if identification:
        g = np.concatenate([g, [np.sum(c * f1), np.sum(c * f2)]])
        if magnitudes:
            m = np.concatenate([m, [np.sum(np.abs(c) * a[0]), np.sum(np.abs(c) * a[1])]])
    return (mse_u + mse_f, g, (mse_u, mse_f)) + ((m,) if magnitudes else ())


def poly_residual(w, layers, lb, ub, terms, X, source=None, identification=False, dtype=np.float64):
    """f (N, 1) on the points X."""
    w = np.asarray(w, dtype=dtype)
    wn, l1, l2 = (w[:-2], w[-2], w[-1]) if identification else (w, 0.0, 0.0)
    (U, Ux, Ut, Uxx), _ = forward(wn, layers, lb, ub, X, dtype)
    f = poly_terms(terms, (U, Ux, Ut, Uxx), l1, l2, dtype)[0]
    return f if source is None else f - np.asarray(source, dtype=dtype).reshape(-1, 1)
