"""Step times of the polynomial residual head (PINN_POLY_INF with the Burgers spec u_t + u u_x - nu u_xx) against the same
problem on the hard-wired heads: BURGERS_INF on the same generic kernel (PINN_FORCE_GENERIC=1) and BURGERS_INF on its default
specialised kernel.  Net [2, 20 x 8, 1], N_f = 10 000 and 100 000, the three configurations alternated three times.  Reported
row: the continuous-time Allen-Cahn spec u_t - 1e-4 u_xx + 5 u^3 - 5 u on [2, 100 x 4, 1] at N_f = 20 000.

Per configuration: ms per Adam step (median of device-event times of 200 asynchronous steps after a warm-up), ms per L-BFGS
iteration (host clock around 200 fixed-step iterations ending in a synchronise) and the fused kernel's own time
(pinn_time_loss_grad_kernel).  The card's name, power limit and max SM clock are read in the same run.  Run from the repo
root; prints one JSON object."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.getcwd()
sys.path[:0] = [ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "utils")]
import pinn_cabi  # noqa: E402
from bench import init_weights, timed_adam_steps  # noqa: E402

BURGERS = [2] + 8 * [20] + [1]
AC = [2] + 4 * [100] + [1]
NU = 0.01 / np.pi
LB, UB = np.array([-1.0, 0.0]), np.array([1.0, 1.0])


def inputs(n_f, seed=1234):
    rng = np.random.default_rng(seed)
    x0 = np.linspace(-1, 1, 100)[:, None]
    X_u = np.hstack([x0, 0 * x0])
    return X_u, -np.sin(np.pi * x0), LB + (UB - LB) * rng.random((n_f, 2))


def handle(kind, n_f):
    X_u, u, X_f = inputs(n_f)
    if kind == "poly_burgers":
        p = pinn_cabi.Pinn(pinn_cabi.POLY_INF, BURGERS, LB, UB)
        p.set_residual([(1.0, 0, (0, 0, 1, 0)), (1.0, 0, (1, 1, 0, 0)), (-NU, 0, (0, 0, 0, 1))])
        layers = BURGERS
    elif kind == "poly_allen_cahn":
        p = pinn_cabi.Pinn(pinn_cabi.POLY_INF, AC, LB, UB)
        p.set_residual([(1.0, 0, (0, 0, 1, 0)), (-1e-4, 0, (0, 0, 0, 1)), (5.0, 0, (3, 0, 0, 0)), (-5.0, 0, (1, 0, 0, 0))])
        u = X_u[:, :1] ** 2 * np.cos(np.pi * X_u[:, :1])
        layers = AC
    else:
        os.environ["PINN_FORCE_GENERIC"] = "1" if kind == "burgers_generic" else "0"
        p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, BURGERS, LB, UB)
        os.environ.pop("PINN_FORCE_GENERIC")
        p.set_pde_params([NU])
        layers = BURGERS
    p.set_data(X_u, u)
    p.set_collocation(X_f[:, 0], X_f[:, 1])
    p.set_weights(init_weights(layers))
    return p


def lbfgs_ms_per_iter(p, w0, iters):
    p.set_weights(w0)
    p.lbfgs(3, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, sync_every=1000)      # warm-up
    p.set_weights(w0)
    p.sync()
    t0 = time.perf_counter()
    r = p.lbfgs(iters, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, sync_every=1000)
    p.sync()
    return (time.perf_counter() - t0) * 1e3 / max(r["n_iter"], 1), r["n_iter"]


def measure(kind, n_f):
    p = handle(kind, n_f)
    for _ in range(20):
        p.adam_step(1e-3, sync=False)
    p.sync()
    adam = float(np.median(timed_adam_steps(p, 200, flush=False, lr=1e-3)))
    p.time_kernel_ms(10)
    kernel = p.time_kernel_ms(100) / 100
    lb_ms, n_it = lbfgs_ms_per_iter(p, p.get_weights(), 200)
    info = p.kernel_info()
    p.close()
    return {"config": kind, "n_f": n_f, "ms_per_adam_step": adam, "kernel_ms": kernel, "ms_per_lbfgs_iter": lb_ms, "lbfgs_iters": n_it,
            "regs": info["regs"], "local_bytes": info["local_bytes"], "grid": info["grid"]}


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    rows = []
    for rnd in range(3):
        for n_f in (10000, 100000):
            for kind in ("poly_burgers", "burgers_generic", "burgers_specialised"):
                r = measure(kind, n_f)
                r["round"] = rnd
                rows.append(r)
    summary = {}
    for n_f in (10000, 100000):
        for kind in ("poly_burgers", "burgers_generic", "burgers_specialised"):
            sel = [r for r in rows if r["n_f"] == n_f and r["config"] == kind]
            summary["%s_%d" % (kind, n_f)] = {k: float(np.median([r[k] for r in sel])) for k in
                                                ("ms_per_adam_step", "kernel_ms", "ms_per_lbfgs_iter")}
        a, b = summary["poly_burgers_%d" % n_f], summary["burgers_generic_%d" % n_f]
        summary["poly_over_generic_adam_%d" % n_f] = a["ms_per_adam_step"] / b["ms_per_adam_step"]
    out = {"card": card[0] if card else "unknown", "rows": rows, "median_of_3": summary,
           "allen_cahn_100x4_nf20000": measure("poly_allen_cahn", 20000)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
