"""Generate tests/golden/lhs_draw.npz (and no other file):
    PYTHONPATH=. python tests/golden/make_lhs_golden.py

Whole-set Latin-hypercube draws of oracle/lhs_draw.py (the definition pinn_draw_collocation computes, DESIGN §4.6) for a few
seeds and draw indices, some with the high 32 bits set, at N in {1, 2, 7, 1000, 4097}.  The file pins the definition: a later
change to the sampler shows up as a failing test instead of as silently different training runs.  Case k is stored as
case<k>_params = [seed, draw, N] (uint64), case<k>_box = [lb_x, lb_t, ub_x, ub_t], case<k>_x and case<k>_t.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT]
from oracle import lhs_draw as ld  # noqa: E402

OUT = os.environ.get("PINN_GOLDEN_OUT", os.path.dirname(os.path.abspath(__file__)))

BURGERS_BOX = ([-1.0, 0.0], [1.0, 0.99])
NLS_BOX = ([-5.0, 0.0], [5.0, np.pi / 2])
CASES = [
    (0, 0, 1, BURGERS_BOX),
    (1234, 1, 2, BURGERS_BOX),
    (1234, 2, 7, BURGERS_BOX),
    (7, 5, 1000, NLS_BOX),
    (0xDEADBEEF00000001, 3, 1000, BURGERS_BOX),
    (99, 0x1234567800000009, 4097, NLS_BOX),
    (0xFFFFFFFFFFFFFFFF, 0xFFFFFFFF00000000, 1000, ([0.3, -0.5], [3.7, 2.0])),
]


def cases():
    out = {}
    for k, (seed, draw, N, (lb, ub)) in enumerate(CASES):
        x, t = ld.lhs_draw(seed, draw, N, 0, N, lb, ub)
        out["case%d_params" % k] = np.array([seed, draw, N], dtype=np.uint64)
        out["case%d_box" % k] = np.array(list(lb) + list(ub), dtype=np.float64)
        out["case%d_x" % k], out["case%d_t" % k] = x, t
    return out


if __name__ == "__main__":
    path = os.path.join(OUT, "lhs_draw.npz")
    np.savez_compressed(path, **cases())
    print(path)
