"""numpy restatement of the device RAD draw (pinn_draw_collocation_rad, csrc/rad_sample.cuh; DESIGN §4.7), steps 3-5 of its
definition: from the residual at the pool points to the pool rows of the new collocation set.  The pool itself is
oracle/lhs_draw.py's draw, and the residual is what pinn_residual returns on it.

    r_i  = |f_i| (one residual per point) or sqrt(f_u^2 + f_v^2) (two), each operation rounded
    a_i  = r_i^k, left-to-right rounded products (k = 0: 1)
    A_i  = 2^24 if a_i is not finite, else floor((a_i / amax) * 2^24) (0 when amax, the largest finite a_i, is 0 or absent)
    C'   = floor(c * (double)S / n_pool), S = sum A_i;  Q_i = A_i + C';  every Q_i = 1 when T = sum Q_i = 0
    row j: target = mulhi64(w0 << 32 | w1, T) for the Philox4x32-10 block of counter (lo j, hi j, lo draw, hi draw) under the key
           (lo seed ^ RAD_SALT[0], hi seed ^ RAD_SALT[1]); it takes the least i whose inclusive prefix of Q exceeds target.
Every integer step is exact in uint64, so the indices equal the device's.
"""
import math

import numpy as np

from oracle import lhs_draw as ld

RAD_SALT = (0xBF58476D, 0x1CE4E5B9)        # the pick key is the seed's two words XOR these
SCALE = 1 << 24
MAX_POOL = 1 << 29
MAX_C = 1024.0
_M32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def numerators(f, k):
    """a_i = r_i^k for the residual f: shape (n_pool,) or (n_pool, 1), or (n_pool, 2) (the Schrodinger pair (f_u, f_v))."""
    f = np.asarray(f, dtype=np.float64)
    if f.ndim == 2 and f.shape[1] == 1:
        f = f[:, 0]
    with np.errstate(over="ignore", invalid="ignore"):
        r = np.abs(f) if f.ndim == 1 else np.sqrt(f[:, 0] * f[:, 0] + f[:, 1] * f[:, 1])
        a = np.ones_like(r) if k == 0 else r.copy()
        for _ in range(1, k):
            a = a * r
    return a


def quantise(a, c):
    """(Q as a uint64 array, T as an int) for the numerators a and the constant c."""
    a = np.asarray(a, dtype=np.float64)
    fin = np.isfinite(a)
    amax = float(a[fin].max()) if fin.any() else 0.0
    A = np.full(a.shape, SCALE, dtype=np.uint64)
    if amax > 0.0:
        A[fin] = np.floor((a[fin] / amax) * float(SCALE)).astype(np.uint64)
    else:
        A[fin] = 0
    S = int(A.sum(dtype=np.uint64))
    cq = int(math.floor(float(c) * float(S) / float(a.size)))
    Q = A + np.uint64(cq)
    T = S + a.size * cq
    if T == 0:
        Q[:], T = 1, a.size
    return Q, T


def mulhi64(x, y):
    """High 64 bits of the 128-bit products x * y (x a uint64 array, y an int < 2^64), from 32-bit limbs."""
    x = np.asarray(x, dtype=np.uint64)
    x0, x1 = x & _M32, x >> _S32
    y0, y1 = np.uint64(y & 0xFFFFFFFF), np.uint64(y >> 32)
    p00, p01, p10, p11 = x0 * y0, x0 * y1, x1 * y0, x1 * y1         # each below 2^64
    mid = (p00 >> _S32) + (p01 & _M32) + (p10 & _M32)                # below 3 * 2^32
    return p11 + (p01 >> _S32) + (p10 >> _S32) + (mid >> _S32)


def targets(seed, draw, n, T):
    """mulhi64(r64_j, T) of rows j in [0, n)."""
    seed, draw = int(seed), int(draw)
    j = np.arange(n, dtype=np.uint64)
    w = ld.philox4x32_10(j & _M32, j >> _S32, draw & 0xFFFFFFFF, draw >> 32, (seed & 0xFFFFFFFF) ^ RAD_SALT[0],
                         (seed >> 32) ^ RAD_SALT[1])
    return mulhi64((w[0] << _S32) | w[1], T)


def pick(Q, T, seed, draw, n):
    """Pool indices of rows [0, n): the least i with inclusive prefix P_i > target_j."""
    P = np.cumsum(np.asarray(Q, dtype=np.uint64), dtype=np.uint64)
    assert int(P[-1]) == T
    return np.searchsorted(P, targets(seed, draw, n, T), side="right")


def rad_indices(f, seed, draw, n, k, c):
    """Pool indices that pinn_draw_collocation_rad(seed, draw, n_pool = len(f), n, k, c) stores, given the pool residual f."""
    Q, T = quantise(numerators(f, k), c)
    return pick(Q, T, seed, draw, n)


def rad_draw(f, seed, draw, n, k, c, lb, ub):
    """(x, t) of the new collocation set: the pool is Latin-hypercube draw `draw` of `seed` with len(f) strata over [lb, ub]."""
    n_pool = len(f)
    px, pt = ld.lhs_draw(seed, draw, n_pool, 0, n_pool, lb, ub)
    i = rad_indices(f, seed, draw, n, k, c)
    return px[i], pt[i]
