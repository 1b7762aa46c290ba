"""numpy restatement of the device Latin-hypercube draw (pinn_draw_collocation, csrc/lhs_draw.cuh; DESIGN §4.6).

A draw is a pure function of (seed, draw, N, lb, ub).  Row i of it is
    u_d   = 53-bit uniform from Philox4x32-10, counter (lo(i), hi(i), lo(draw), hi(draw)), key (lo(seed), hi(seed)):
            words 0, 1 give u_x = ((w0 >> 11) << 32 | w1) * 2^-53, words 2, 3 give u_t likewise;
    pi_d  = a balanced Feistel permutation of the 2m-bit domain (4^m >= N, m >= 1), FEISTEL_ROUNDS rounds whose round function is
            word 0 of Philox4x32-10 on (R, round | d << 8, lo(draw), hi(draw)) under the key (lo(seed) ^ KEY_SALT[0],
            hi(seed) ^ KEY_SALT[1]), cycle-walked down to [0, N);
    x_d   = lb_d + (ub_d - lb_d) * ((pi_d(i) + u_d) / N), in fp64, in that order.
Every integer step is done in uint64 arrays masked to 32 bits, so the restatement follows the kernel's instructions exactly and
its values equal the device's bit for bit.
"""
import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57            # Philox4x32 multipliers (Random123)
W0, W1 = 0x9E3779B9, 0xBB67AE85            # Philox4x32 Weyl key increments
KEY_SALT = (0x5851F42D, 0x4C957F2D)        # the permutation key is the seed's two words XOR these
FEISTEL_ROUNDS = 4
_MASK = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint64 arrays (or ints) holding 32-bit words; returns the four output words as uint64 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _MASK for c in (c0, c1, c2, c3))
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    m0, m1 = np.uint64(M0), np.uint64(M1)
    for _ in range(10):
        p0, p1 = m0 * c0, m1 * c2                    # exact: both factors are below 2^32
        c0, c1, c2, c3 = ((p1 >> _S32) ^ c1 ^ np.uint64(k0)), p1 & _MASK, ((p0 >> _S32) ^ c3 ^ np.uint64(k1)), p0 & _MASK
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return c0, c1, c2, c3


def half_bits(N):
    """m of the 2m-bit Feistel domain: the least m >= 1 with 4^m >= N."""
    return max(1, ((int(N) - 1).bit_length() + 1) // 2)


def permute(i, N, d, seed, draw, walks=None):
    """pi_d(i) for the uint64 array i (every entry < N).  walks: an optional list that receives the number of network
    applications per entry."""
    seed, draw = int(seed), int(draw)
    m = half_bits(N)
    half = np.uint64((1 << m) - 1)
    kf0, kf1 = (seed & 0xFFFFFFFF) ^ KEY_SALT[0], (seed >> 32) ^ KEY_SALT[1]
    out = np.array(i, dtype=np.uint64)
    todo = np.arange(out.size)
    count = np.zeros(out.size, dtype=np.int64)
    while todo.size:
        v = out[todo]
        L, R = v >> np.uint64(m), v & half
        for r in range(FEISTEL_ROUNDS):
            f = philox4x32_10(R, r | (d << 8), draw & 0xFFFFFFFF, draw >> 32, kf0, kf1)[0] & half
            L, R = R, L ^ f
        out[todo] = (L << np.uint64(m)) | R
        count[todo] += 1
        todo = todo[out[todo] >= np.uint64(N)]
    if walks is not None:
        walks.append(count)
    return out


def uniforms(i, seed, draw):
    """(u_x, u_t) of rows i: 53-bit uniforms in [0, 1)."""
    seed, draw = int(seed), int(draw)
    i = np.asarray(i, dtype=np.uint64)
    w = philox4x32_10(i & _MASK, i >> _S32, draw & 0xFFFFFFFF, draw >> 32, seed & 0xFFFFFFFF, seed >> 32)
    return tuple((((w[2 * d] >> np.uint64(11)) << _S32) | w[2 * d + 1]).astype(np.float64) * 2.0 ** -53 for d in (0, 1))


def lhs_rows(seed, draw, N, rows, lb, ub):
    """(x, t) of the given rows of draw `draw` of `seed` with N strata per dimension over [lb, ub]."""
    rows = np.asarray(rows, dtype=np.uint64)
    lb, ub = np.asarray(lb, dtype=np.float64), np.asarray(ub, dtype=np.float64)
    u = uniforms(rows, seed, draw)
    out = []
    for d in (0, 1):
        p = permute(rows, N, d, seed, draw)
        out.append(lb[d] + (ub[d] - lb[d]) * ((p.astype(np.float64) + u[d]) / np.float64(N)))
    return out[0], out[1]


def lhs_draw(seed, draw, N, first, n, lb, ub):
    """Rows [first, first + n) of the draw: what pinn_draw_collocation(seed, draw, first, n, N) stores."""
    return lhs_rows(seed, draw, N, np.arange(first, first + n, dtype=np.uint64), lb, ub)
