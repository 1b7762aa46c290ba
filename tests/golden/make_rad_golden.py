"""Generate tests/golden/rad_draw.npz (and no other file):
    PYTHONPATH=. python tests/golden/make_rad_golden.py

Residual-based adaptive draws of oracle/rad_draw.py (steps 3-5 of the definition pinn_draw_collocation_rad computes, DESIGN §4.7):
from a pool residual to the pool rows of the new set.  The residual vectors hold zeros, ties, NaN, +-Inf, subnormals, values
whose k-th power overflows, an all-zero vector, a one-point pool and Schrodinger pairs; every k in 0..4 meets c in {0, 1, 1024},
and the seeds and draws include ones with their high 32 bits set.  The file pins the definition: a later change to the sampler
shows up as a failing test instead of as silently different training runs.  Case j is stored as case<j>_f (n_pool or
(n_pool, 2) residuals), case<j>_params = [seed, draw, n, k, T] (uint64), case<j>_c and case<j>_idx (the pool rows drawn).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT]
from oracle import rad_draw as rd  # noqa: E402

OUT = os.environ.get("PINN_GOLDEN_OUT", os.path.dirname(os.path.abspath(__file__)))
BIG_SEED, BIG_DRAW = 0xFEDCBA9876543210, 0x100000003


def residuals():
    """name -> residual vector."""
    rng = np.random.default_rng(20231)
    mixed = rng.standard_normal(200) * 10.0 ** rng.integers(-3, 3, 200)
    mixed[:40] = 0.0                                             # zeros
    mixed[40:60] = 0.75                                          # ties
    mixed[60:63] = np.nan
    mixed[63], mixed[64] = np.inf, -np.inf
    mixed[65:70] = 5e-324 * np.arange(1, 6)                      # subnormals
    rng.shuffle(mixed)
    pair = rng.standard_normal((300, 2))
    pair[5] = (np.nan, 0.0)
    pair[6] = (0.0, -np.inf)
    pair[7:30] = 0.0
    return {
        "mixed": mixed,
        "all_zero": np.zeros(50),
        "subnormal": 5e-324 * rng.integers(0, 1000, 64).astype(np.float64),
        "overflow": np.concatenate([[1e100, -1e80, 3e77], rng.standard_normal(40)]),   # r^4 and r^3 overflow to +Inf
        "normal": np.round(rng.standard_normal(2000), 2),        # many ties
        "one": np.array([0.3]),
        "pair": pair,
    }


def cases():
    f = residuals()
    plan = [("mixed", k, c, BIG_SEED, BIG_DRAW, 500) for k in range(5) for c in (0.0, 1.0, 1024.0)]
    plan += [("all_zero", k, c, 3, 1, 80) for k in (0, 2) for c in (0.0, 1.0)]
    plan += [("subnormal", 1, 0.0, 7, 0xFFFFFFFF00000000, 300), ("subnormal", 2, 1.0, 7, 2, 300)]
    plan += [("overflow", k, 0.0, 0xFFFFFFFFFFFFFFFF, 9, 400) for k in (1, 3, 4)]
    plan += [("normal", k, c, 0xDEADBEEF00000001, 0x1234567800000009, 3000) for k, c in ((1, 1.0), (2, 0.0), (4, 1024.0))]
    plan += [("one", k, c, 1, 1, 5) for k, c in ((0, 0.0), (1, 1.0))]
    plan += [("pair", k, c, 99, 0x100000000, 700) for k, c in ((0, 1.0), (1, 1.0), (2, 0.0), (3, 1024.0))]
    out = {}
    for j, (name, k, c, seed, draw, n) in enumerate(plan):
        Q, T = rd.quantise(rd.numerators(f[name], k), c)
        idx = rd.pick(Q, T, seed, draw, n)
        out["case%d_f" % j] = f[name]
        out["case%d_params" % j] = np.array([seed, draw, n, k, T], dtype=np.uint64)
        out["case%d_c" % j] = np.float64(c)
        out["case%d_idx" % j] = idx.astype(np.int64)
    return out


if __name__ == "__main__":
    path = os.path.join(OUT, "rad_draw.npz")
    np.savez_compressed(path, **cases())
    print(path)
