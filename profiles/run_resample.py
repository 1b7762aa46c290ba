"""Cost of a fresh collocation set every Adam step (pinn_draw_collocation, DESIGN §4.6) on the Burgers net [2, 20 x 8, 1] at
N_f = 100 000 and 2 000 000:

  (a) resident:  the Adam step on a collocation set that stays on the device (device events around each step);
  (b) draw:      pinn_draw_collocation + the Adam step, per step (device events around the pair);
  (c) host:      a vectorised numpy Latin hypercube (rng.permutation per dimension) + pinn_set_collocation + the step, host clock
                 around work that ends in a synchronise;
  (d) kernel:    the draw kernel alone (device events), as bytes written per second (16 B per point) against the 3.35 TB/s of
                 HBM3 in NVIDIA's H100 SXM data sheet, and as Philox4x32-10 blocks per second (1 + 2 x rounds x walks per point,
                 the walks counted by the restatement at the same N).

Every shape is warmed up first; each figure is the median of `--steps` (>= 200) steps, (a) and (b) alternated in two rounds.  The
card's name and power limit are read in the same run.  Run from the repository root; prints one JSON object and, with --out DIR,
writes it to DIR/run_resample_h100.json."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.getcwd()
sys.path[:0] = [ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "utils")]
import pinn_cabi  # noqa: E402
from bench import init_weights  # noqa: E402
from oracle import lhs_draw as ld  # noqa: E402

BURGERS = [2] + 8 * [20] + [1]
LB, UB = np.array([-1.0, 0.0]), np.array([1.0, 0.99])
NU = 0.01 / np.pi
HBM_TBS = 3.35
LR = 1e-3


def handle(n_f):
    rng = np.random.default_rng(1234)
    x0 = np.linspace(-1, 1, 100)[:, None]
    p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, BURGERS, LB, UB)
    p.set_pde_params([NU])
    p.set_data(np.hstack([x0, 0 * x0]), -np.sin(np.pi * x0))
    p.set_collocation(*host_lhs(rng, n_f))
    p.set_weights(init_weights(BURGERS))
    return p


def host_lhs(rng, n):
    """The vectorised numpy Latin hypercube a user would write: one permutation of the strata per dimension."""
    k = np.stack([rng.permutation(n), rng.permutation(n)], 1)
    X = LB + (UB - LB) * ((k + rng.random((n, 2))) / n)
    return X[:, 0], X[:, 1]


def device_ms(p, steps, body):
    """Per-step device times (ms) of body(i), CUDA events on the handle's stream around each call."""
    for i in range(steps):
        p.event_record(2 * i)
        body(i)
        p.event_record(2 * i + 1)
    p.sync()
    return [p.event_elapsed_ms(2 * i, 2 * i + 1) for i in range(steps)]


def measure(n_f, steps, draw0):
    p = handle(n_f)
    step = lambda i: p.adam_step(LR, sync=False)                      # noqa: E731
    draw = lambda i: p.draw_collocation(7, draw0 + i, n_f)            # noqa: E731

    def draw_step(i):
        draw(i)
        step(i)
    for body in (step, draw_step, draw):                               # warm-up of every timed body
        device_ms(p, 20, body)
    a, b = [], []
    for _ in range(2):
        a += device_ms(p, steps, step)
        b += device_ms(p, steps, draw_step)
    d = device_ms(p, steps, draw)
    rng = np.random.default_rng(5)
    for _ in range(3):
        p.set_collocation(*host_lhs(rng, n_f))
    c = []
    for _ in range(steps):
        t0 = time.perf_counter()
        p.set_collocation(*host_lhs(rng, n_f))
        p.adam_step(LR, sync=False)
        p.sync()
        c.append((time.perf_counter() - t0) * 1e3)
    p.close()
    walks = []
    for dim in (0, 1):
        ld.permute(np.arange(n_f, dtype=np.uint64), n_f, dim, 7, draw0, walks)
    blocks = 1 + ld.FEISTEL_ROUNDS * (walks[0].mean() + walks[1].mean())
    ma, mb, mc, md = (float(np.median(v)) for v in (a, b, c, d))
    return {"n_f": n_f, "steps": steps, "a_resident_adam_ms": ma, "b_draw_plus_adam_ms": mb, "b_over_a": mb / ma,
            "c_host_lhs_upload_adam_ms": mc, "c_over_a": mc / ma, "d_draw_kernel_ms": md,
            "d_bytes_per_s": 16 * n_f / (md * 1e-3), "d_share_of_hbm": 16 * n_f / (md * 1e-3) / (HBM_TBS * 1e12),
            "d_philox_blocks_per_point": float(blocks), "d_philox_blocks_per_s": blocks * n_f / (md * 1e-3),
            "a_spread_ms": [float(np.percentile(a, 10)), float(np.percentile(a, 90))],
            "b_spread_ms": [float(np.percentile(b, 10)), float(np.percentile(b, 90))]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.steps < 200:
        raise SystemExit("--steps: at least 200")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    rows = [measure(n, args.steps, 1000 * k) for k, n in enumerate((100000, 2000000))]
    for r in rows:
        r["d_bound"] = "HBM bandwidth" if r["d_share_of_hbm"] > 0.5 else "integer arithmetic (Philox multiplies), not HBM"
    out = {"card": card[0] if card else "unknown", "net": BURGERS, "rows": rows}
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "run_resample_h100.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
