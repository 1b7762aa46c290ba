"""Independent fp64 oracle for the continuous-time Navier-Stokes identification model: 13 forward Taylor streams of a
3-input net and the hand-derived reverse sweep.

TEST INFRASTRUCTURE (see oracle/__init__.py).  numpy only; shares no derivation with ``oracle.reference_port_ns`` (nested
autograd).  The two must agree to ~1e-13.  Every entry point takes dtype= (np.longdouble runs the same sums with a 64-bit
mantissa on x86-64) and magnitudes= (per-entry contraction magnitudes, as oracle.taylor.backward).

Streams (fixed order, shared with the CUDA kernel and the C ABI's probe layout), as multi-indices over (x, y, t):
    0 value, 1 x, 2 y, 3 t, 4 xx, 5 xy, 6 yy, 7 xt, 8 yt, 9 xxx, 10 xxy, 11 xyy, 12 yyy
Input layer: h = 2(X-lb)/(ub-lb)-1; the first-order streams are the unit columns scaled by 2/(ub-lb); the others are 0.
tanh layer, z = hW+b, a = tanh z, s = 1-a^2, sigma2 = -2as, sigma3 = -2s(1-3a^2) (= d sigma2/dz),
sigma4 = 8as(2-3a^2) (= d sigma3/dz):
    a_i   = s z_i
    a_ij  = s z_ij + sigma2 z_i z_j
    a_ijk = s z_ijk + sigma2 (z_ij z_k + z_ik z_j + z_jk z_i) + sigma3 z_i z_j z_k
The reverse differentiates these rules term by term with respect to the z streams (z-based; see backward_ns).
"""
from __future__ import annotations

import numpy as np

from oracle.taylor import _flat, _unpack

# multi-index (x, y, t) of every stream
STREAMS = [(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (2, 0, 0), (1, 1, 0), (0, 2, 0), (1, 0, 1), (0, 1, 1),
           (3, 0, 0), (2, 1, 0), (1, 2, 0), (0, 3, 0)]
NS = len(STREAMS)
_IDX = {m: k for k, m in enumerate(STREAMS)}


def _sid(*dirs):
    """Stream index of the derivative along the given directions (0 = x, 1 = y, 2 = t)."""
    m = [0, 0, 0]
    for d in dirs:
        m[d] += 1
    return _IDX[tuple(m)]


def _dirs(k):
    m = STREAMS[k]
    return tuple(d for d in range(3) for _ in range(m[d]))


FIRST = [k for k in range(NS) if len(_dirs(k)) == 1]
SECOND = [k for k in range(NS) if len(_dirs(k)) == 2]
THIRD = [k for k in range(NS) if len(_dirs(k)) == 3]


def tanh_streams(Z):
    """The 13 output streams of a tanh layer from its 13 pre-activation streams Z."""
    a = np.tanh(Z[0])
    s = 1.0 - a * a
    s2 = -2.0 * a * s
    s3 = -2.0 * s * (1.0 - 3.0 * a * a)
    A = [None] * NS
    A[0] = a
    for k in FIRST:
        A[k] = s * Z[k]
    for k in SECOND:
        i, j = _dirs(k)
        A[k] = s * Z[k] + s2 * Z[_sid(i)] * Z[_sid(j)]
    for k in THIRD:
        i, j, m = _dirs(k)
        zi, zj, zm = Z[_sid(i)], Z[_sid(j)], Z[_sid(m)]
        A[k] = s * Z[k] + s2 * (Z[_sid(i, j)] * zm + Z[_sid(i, m)] * zj + Z[_sid(j, m)] * zi) + s3 * zi * zj * zm
    return A


def zbar(a, s, Z, Ab):
    """Adjoints of the 13 pre-activation streams Z of a tanh layer (a = tanh Z[0], s = 1 - a^2) from the adjoints Ab of its
    outputs: the forward rules differentiated term by term in z."""
    s2 = -2.0 * a * s
    s3 = -2.0 * s * (1.0 - 3.0 * a * a)
    s4 = 8.0 * a * s * (2.0 - 3.0 * a * a)
    Zb = [s * Ab[k] for k in range(NS)]                   # every stream carries s z_k
    for k in FIRST:                                       # a_i = s z_i
        Zb[0] = Zb[0] + s2 * Z[k] * Ab[k]
    for k in SECOND:                                      # a_ij = s z_ij + sigma2 z_i z_j
        i, j = (_sid(d) for d in _dirs(k))
        Zb[0] = Zb[0] + (s2 * Z[k] + s3 * Z[i] * Z[j]) * Ab[k]
        Zb[i] = Zb[i] + s2 * Z[j] * Ab[k]
        Zb[j] = Zb[j] + s2 * Z[i] * Ab[k]
    for k in THIRD:                                       # a_ijk
        di, dj, dm = _dirs(k)
        i, j, q = _sid(di), _sid(dj), _sid(dm)
        ij, iq, jq = _sid(di, dj), _sid(di, dm), _sid(dj, dm)
        Zb[0] = Zb[0] + (s2 * Z[k] + s3 * (Z[ij] * Z[q] + Z[iq] * Z[j] + Z[jq] * Z[i]) + s4 * Z[i] * Z[j] * Z[q]) * Ab[k]
        Zb[ij] = Zb[ij] + s2 * Z[q] * Ab[k]
        Zb[iq] = Zb[iq] + s2 * Z[j] * Ab[k]
        Zb[jq] = Zb[jq] + s2 * Z[i] * Ab[k]
        Zb[i] = Zb[i] + (s2 * Z[jq] + s3 * Z[j] * Z[q]) * Ab[k]
        Zb[j] = Zb[j] + (s2 * Z[iq] + s3 * Z[i] * Z[q]) * Ab[k]
        Zb[q] = Zb[q] + (s2 * Z[ij] + s3 * Z[i] * Z[j]) * Ab[k]
    return Zb


def forward_ns(w, layers, lb, ub, X, dtype=np.float64):
    """X: (N,3) = (x, y, t) -> the 13 output streams, each (N, n_out), and the per-layer stash."""
    if int(layers[0]) != 3:
        raise ValueError("the Navier-Stokes net takes 3 inputs (x, y, t)")
    X = np.asarray(X, dtype=dtype)
    lb, ub = np.asarray(lb, dtype).reshape(-1), np.asarray(ub, dtype).reshape(-1)
    Ws, bs = _unpack(np.asarray(w, dtype=dtype), layers)
    N = X.shape[0]
    sc = 2.0 / (ub - lb)
    H = [np.zeros((N, 3), dtype) for _ in range(NS)]
    H[0] = sc * (X - lb) - 1.0
    for d in range(3):
        H[_sid(d)][:, d] = sc[d]
    stash = []
    for l in range(len(Ws) - 1):
        W, b = Ws[l], bs[l]
        Z = [Hk @ W for Hk in H]
        Z[0] = Z[0] + b
        A = tanh_streams(Z)
        stash.append((H, A[0], 1.0 - A[0] * A[0], Z))
        H = A
    W, b = Ws[-1], bs[-1]
    out = [Hk @ W for Hk in H]
    out[0] = out[0] + b
    stash.append((H,))
    return out, stash


def _contraction(H, Zb):
    return sum(H[k].T @ Zb[k] for k in range(NS)), Zb[0].sum(0)


def backward_ns(w, layers, stash, seeds, dtype=np.float64, magnitudes=False):
    """seeds: adjoints of the 13 output streams, each (N, n_out).  Returns the flat parameter gradient (and with
    magnitudes=True the per-entry magnitudes sum |H|^T |Z-bar|, sum |Z-bar| of the final contractions)."""
    Ws, _ = _unpack(np.asarray(w, dtype=dtype), layers)
    g, m = [], []
    (H,) = stash[-1]
    Zb = list(seeds)
    g.append(_contraction(H, Zb))
    if magnitudes:
        m.append(_contraction([np.abs(v) for v in H], [np.abs(v) for v in Zb]))
    WT = Ws[-1].T
    Ab = [v @ WT for v in Zb]
    for l in range(len(Ws) - 2, -1, -1):
        H, a, s, Z = stash[l]
        Zb = zbar(a, s, Z, Ab)
        g.append(_contraction(H, Zb))
        if magnitudes:
            m.append(_contraction([np.abs(v) for v in H], [np.abs(v) for v in Zb]))
        if l > 0:
            WT = Ws[l].T
            Ab = [v @ WT for v in Zb]
    return (_flat(g), _flat(m)) if magnitudes else _flat(g)


def ns_terms(O, l1, l2):
    """(e-less) residuals from the 13 output streams O (each (N, 2): psi, p): f_u, f_v and the streams they use."""
    P, Q = (lambda k: O[k][:, 0]), (lambda k: O[k][:, 1])
    px, py, pxx, pxy, pyy = P(1), P(2), P(4), P(5), P(6)
    f_u = P(8) + l1 * (py * pxy - px * pyy) + Q(1) - l2 * (P(10) + P(12))
    f_v = -P(7) + l1 * (px * pxy - py * pxx) + Q(2) + l2 * (P(9) + P(11))
    return f_u, f_v


def ns_ide_loss_grad(w, layers, lb, ub, X, uv, dtype=np.float64, magnitudes=False):
    """Continuous-time Navier-Stokes identification (PINNs/main/continuous_time_identification (Navier-Stokes)/NavierStokes.py,
    restated in fp64): w = [net, l1, l2], net [3, ..., 2] -> (psi, p); u = psi_y, v = -psi_x;
        f_u = u_t + l1 (u u_x + v u_y) + p_x - l2 (u_xx + u_yy),  f_v = v_t + l1 (u v_x + v v_y) + p_y - l2 (v_xx + v_yy);
    loss = sum (u - u_d)^2 + sum (v - v_d)^2 + sum f_u^2 + sum f_v^2 on the same points.
    Returns (loss, grad, (data SSE, residual SSE)).  Upstream (from memory, not pinned): l1, l2 init 0.0 (raw, no exp),
    N_train = 5000, layers [3, 20 x 8, 2]."""
    w = np.asarray(w, dtype=dtype)
    wn, l1, l2 = w[:-2], w[-2], w[-1]
    uv = np.asarray(uv, dtype=dtype)
    O, st = forward_ns(wn, layers, lb, ub, X, dtype)
    P = lambda k: O[k][:, 0]
    px, py, pxx, pxy, pyy = P(1), P(2), P(4), P(5), P(6)
    e_u, e_v = py - uv[:, 0], -px - uv[:, 1]
    f_u, f_v = ns_terms(O, l1, l2)
    c_u, c_v = 2.0 * f_u, 2.0 * f_v
    S = [np.zeros_like(O[0]) for _ in range(NS)]
    S[1][:, 0] = -l1 * c_u * pyy + l1 * c_v * pxy - 2.0 * e_v
    S[2][:, 0] = l1 * c_u * pxy - l1 * c_v * pxx + 2.0 * e_u
    S[5][:, 0] = l1 * (c_u * py + c_v * px)
    S[6][:, 0] = -l1 * c_u * px
    S[4][:, 0] = -l1 * c_v * py
    S[8][:, 0] = c_u
    S[7][:, 0] = -c_v
    S[10][:, 0] = S[12][:, 0] = -l2 * c_u
    S[9][:, 0] = S[11][:, 0] = l2 * c_v
    S[1][:, 1] = c_u
    S[2][:, 1] = c_v
    r = backward_ns(wn, layers, st, S, dtype, magnitudes)
    g, mg = r if magnitudes else (r, None)
    t1 = c_u * (py * pxy - px * pyy) + c_v * (px * pxy - py * pxx)
    t2 = -c_u * (P(10) + P(12)) + c_v * (P(9) + P(11))
    g = np.concatenate([g, [np.sum(t1), np.sum(t2)]])
    data = dtype(np.sum(e_u * e_u) + np.sum(e_v * e_v))
    res = dtype(np.sum(f_u * f_u) + np.sum(f_v * f_v))
    out = (data + res, g, (data, res))
    if magnitudes:
        out += (np.concatenate([mg, [np.sum(np.abs(t1)), np.sum(np.abs(t2))]]),)
    return out
