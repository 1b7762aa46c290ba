"""Residual-based adaptive resampling on the device (pinn_draw_collocation_rad, DESIGN §4.7): its cost, and what it does to the
accuracy of a Burgers training run.

Cost, on the Burgers net [2, 20 x 8, 1] at N_f = 100 000 with a pool of 100 000 and of 1 000 000 points:
  (a) resident:  the Adam step on a collocation set that stays on the device (device events around each step);
  (b) rad:       one pinn_draw_collocation_rad call, k = 1, c = 1 (device events around the call);
  (c) split:     (b) per kernel from torch.profiler (CUDA activities, in a process of its own after everything else): pool
                 draw, pool forward (the thread-per-point probe), and head + quantise + pick;
  (d) amortised: (a + b / every) / a, the cost per Adam step relative to the resident step when RAD runs every 100 and 1000 steps.
Every shape is warmed up first; (a) and (b) are medians of `--steps` (>= 200) calls, alternated in two rounds.

Accuracy, on the tests/golden/burgers_accuracy.npz inputs (N_u = 100, N_f = 10 000, the oracle's initial weights) through the
reference-style mirror, one schedule (--adam Adam epochs at --adam-lr, then --lbfgs L-BFGS iterations at 0.8, 50 corrections) with
  fixed: the script's own X_f throughout;
  lhs:   a fresh Latin-hypercube set every --every Adam epochs (hp["resample_every"]);
  rad:   a RAD set every --every Adam epochs (hp["rad_every"], pool 10 N_f, k = 1, c = 1);
and the relative L2 error of u against X_star / u_star at the end.  L-BFGS runs on the last set Adam saw.

The card's name and power limit are read in the same run.  Run from the repository root; prints one JSON object and, with
--out DIR, writes it to DIR/run_rad_h100.json."""
import argparse
import contextlib
import io
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
LR = 1e-3
N_F = 100000
T0 = time.perf_counter()
KERNELS = {"pool_draw": ("lhs", "draw_kernel"), "pool_forward": ("mlp_forward_generic",),
           "head": ("rad", "head_kernel"), "quantise": ("rad", "quantise_kernel"), "pick": ("rad", "pick_kernel")}


def handle(n_f):
    x0 = np.linspace(-1, 1, 100)[:, None]
    p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, BURGERS, LB, UB)
    p.set_pde_params([NU])
    p.set_data(np.hstack([x0, 0 * x0]), -np.sin(np.pi * x0))
    p.set_collocation(*ld.lhs_draw(3, 0, n_f, 0, n_f, LB, UB))
    p.set_weights(init_weights(BURGERS))
    return p


def log(*msg):
    print("[run_rad %.0f s]" % (time.perf_counter() - T0), *msg, file=sys.stderr, flush=True)


def device_ms(p, steps, body):
    """Per-call device times (ms) of body(i), CUDA events on the handle's stream around each call."""
    for i in range(steps):
        p.event_record(2 * i)
        body(i)
        p.event_record(2 * i + 1)
    p.sync()
    return [p.event_elapsed_ms(2 * i, 2 * i + 1) for i in range(steps)]


def kernel_split(n_pool, calls=50):
    """Mean device time (ms) per RAD call of each of its kernels, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    p = handle(N_F)
    for i in range(10):
        p.draw_collocation_rad(7, i, N_F, n_pool)
    p.sync()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(calls):
            p.draw_collocation_rad(7, 100 + i, N_F, n_pool)
        p.sync()
    p.close()
    out = {k: 0.0 for k in KERNELS}
    for e in prof.key_averages():
        total_us = getattr(e, "device_time_total", None)
        if total_us is None:
            total_us = e.cuda_time_total
        for k, parts in KERNELS.items():
            if all(s in e.key for s in parts):
                out[k] += total_us / 1e3 / calls
    out["head_quantise_pick"] = out["head"] + out["quantise"] + out["pick"]
    return out


def measure(n_pool, steps):
    p = handle(N_F)
    step = lambda i: p.adam_step(LR, sync=False)                             # noqa: E731
    rad = lambda i: p.draw_collocation_rad(7, 1000 + i, N_F, n_pool)         # noqa: E731
    for body in (step, rad):
        device_ms(p, 20, body)
    a, b = [], []
    for _ in range(2):
        a += device_ms(p, steps, step)
        b += device_ms(p, steps, rad)
    p.close()
    ma, mb = float(np.median(a)), float(np.median(b))
    return {"n_f": N_F, "n_pool": n_pool, "steps": steps, "a_resident_adam_ms": ma, "b_rad_call_ms": mb, "b_over_a": mb / ma,
            "a_spread_ms": [float(np.percentile(a, 10)), float(np.percentile(a, 90))],
            "b_spread_ms": [float(np.percentile(b, 10)), float(np.percentile(b, 90))],
            "d_amortised_per_step_over_a": {str(e): (ma + mb / e) / ma for e in (100, 1000)}}


def accuracy(adam, adam_lr, lbfgs, every):
    from logger import Logger
    from neuralnetwork import NeuralNetwork
    g = np.load(os.path.join(ROOT, "tests", "golden", "burgers_accuracy.npz"))
    X_star, u_star = g["X_star"].astype(np.float64), g["u_star"].astype(np.float64)

    class BurgersInformedNN(NeuralNetwork):                   # 1d-burgers/inf_cont_burgers.py:48-56
        def __init__(self, hp, logger, X_f, ub, lb, nu):
            super().__init__(hp, logger, ub, lb)
            self.nu = nu
            self.x_f = self.tensor(X_f[:, 0:1]); self.t_f = self.tensor(X_f[:, 1:2])

    out = {}
    for name, extra in (("fixed", {}), ("lhs", {"resample_every": every, "resample_seed": 11}),
                        ("rad", {"rad_every": every, "resample_seed": 11})):
        hp = {"N_u": 100, "N_f": 10000, "layers": BURGERS, "tf_epochs": adam, "tf_lr": adam_lr, "tf_b1": 0.9, "tf_eps": None,
              "nt_epochs": lbfgs, "nt_lr": 0.8, "nt_ncorr": 50, "log_frequency": 50}
        hp.update(extra)
        with contextlib.redirect_stdout(io.StringIO()):
            logger = Logger(hp)
            pinn = BurgersInformedNN(hp, logger, g["X_f"], g["ub"], g["lb"], nu=NU)
            pinn._w0 = g["w0"].copy()
            err = lambda: float(np.linalg.norm(u_star - pinn.predict(X_star)) / np.linalg.norm(u_star))    # noqa: E731
            logger.set_error_fn(err)
            t0 = time.perf_counter()
            pinn.fit(g["X_u"], g["u"])
            dt = time.perf_counter() - t0
        loss, _ = pinn.grad(g["X_u"], g["u"])
        out[name] = {"hp_extra": extra, "final_loss": float(loss), "rel_l2_error_u": err(), "train_seconds": dt}
        log("accuracy", name, out[name])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--adam", type=int, default=5000)
    ap.add_argument("--adam-lr", type=float, default=1e-3)
    ap.add_argument("--lbfgs", type=int, default=5000)
    ap.add_argument("--every", type=int, default=100)
    ap.add_argument("--out", default=None)
    ap.add_argument("--split", type=int, default=None, help="(internal) print the kernel split of one pool size and exit")
    args = ap.parse_args()
    if args.split:
        print(json.dumps(kernel_split(args.split)))
        return
    if args.steps < 200:
        raise SystemExit("--steps: at least 200")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    rows = []
    for n in (100000, 1000000):
        rows.append(measure(n, args.steps))
        log("cost", rows[-1])
    acc = {"schedule": {"adam_epochs": args.adam, "adam_lr": args.adam_lr, "lbfgs_iterations": args.lbfgs, "lbfgs_lr": 0.8,
                        "every": args.every, "n_f": 10000},
           "runs": accuracy(args.adam, args.adam_lr, args.lbfgs, args.every)}
    for r in rows:
        split = subprocess.run([sys.executable, os.path.abspath(__file__), "--split", str(r["n_pool"])], capture_output=True,
                               text=True, check=True)
        r["c_split_ms"] = s = json.loads(split.stdout.strip().splitlines()[-1])
        r["c_largest"] = max(("pool_draw", "pool_forward", "head_quantise_pick"), key=lambda k: s[k])
        log("split", r["n_pool"], s)
    out = {"card": card[0] if card else "unknown", "net": BURGERS, "rows": rows, "accuracy": acc}
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "run_rad_h100.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
