"""Step times of the discrete-time KdV identification and Allen-Cahn inference models on the generic fused kernel, at the
upstream sizes (PINNs/main discrete_time_identification (KdV)/KdV.py: N_0 = 199, N_1 = 201, [1, 50 x 4, q],
q = ceil(0.5 ln(eps) / ln(dt)) at dt = 0.6; discrete_time_inference (AC)/AC.py: N = 200, [1, 200 x 4, 101], dt = 0.8),
seeded synthetic data.  Prints ms per Adam step and per L-BFGS iteration, with the card name and power limit of the run.
L-BFGS runs in its Gram-matrix form (PINN_LBFGS=gram): AC's upstream net has ~141k parameters, more than the single-CTA
kernel takes.  Run from the repo root."""
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

os.environ.setdefault("PINN_LBFGS", "gram")
sys.path.insert(0, os.getcwd())
sys.path.insert(0, os.path.join(os.getcwd(), "pinns-tf2.0_b200", "utils"))
import pinn_cabi  # noqa: E402
from bench import init_weights, timed_adam_steps  # noqa: E402


def lbfgs_ms_per_iter(p, w0, iters):
    p.set_weights(w0)
    p.lbfgs(3, learning_rate=0.8, n_correction=50, tol_fun=0.0, tol_x=0.0, sync_every=1000)      # warm-up
    p.set_weights(w0)
    p.sync()
    t0 = time.perf_counter()
    r = p.lbfgs(iters, learning_rate=0.8, n_correction=50, tol_fun=0.0, tol_x=0.0, sync_every=1000)
    p.sync()
    return (time.perf_counter() - t0) * 1e3 / max(r["n_iter"], 1), r["n_iter"]


def timed(p, w0):
    p.set_weights(w0)
    for _ in range(5):
        p.adam_step(1e-3, sync=False)
    p.sync()
    adam = float(np.median(timed_adam_steps(p, 50, flush=False, lr=1e-3)))
    lb_ms, n_it = lbfgs_ms_per_iter(p, w0, 50)
    return {"ms_per_adam_step": adam, "ms_per_lbfgs_iter": lb_ms, "lbfgs_iters": n_it, "kernel_ms": p.time_kernel_ms(20) / 20,
            "info": p.kernel_info()}


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    rng = np.random.default_rng(7)
    out = {"card": card[0] if card else "unknown", "lbfgs": os.environ["PINN_LBFGS"]}
    dt = 0.6
    q = int(math.ceil(0.5 * math.log(np.finfo(float).eps) / math.log(dt)))
    L = [1, 50, 50, 50, 50, q]
    x_0 = rng.uniform(-1, 1, (199, 1)); x_1 = rng.uniform(-1, 1, (201, 1))
    p = pinn_cabi.Pinn(pinn_cabi.KDV_IDE_DISC, L, [-1.0], [1.0])
    p.set_pde_params([dt])
    p.set_irk(pinn_cabi.irk_ide_disc((rng.standard_normal((q, q)) / q).astype(np.float32),
                                     (rng.standard_normal((1, q)) / q).astype(np.float32)))
    p.set_snapshot(0, x_0, np.cos(np.pi * x_0)); p.set_snapshot(1, x_1, np.cos(np.pi * x_1 + 0.3))
    out["kdv"] = dict(layers=L, q=q, **timed(p, np.concatenate([init_weights(L), [0.0, -6.0]])))
    p.close()
    q = 100
    L = [1, 200, 200, 200, 200, q + 1]
    x_0 = rng.uniform(-1, 1, (200, 1))
    p = pinn_cabi.Pinn(pinn_cabi.AC_DISC, L, [-1.0], [1.0])
    p.set_pde_params([0.8, 1e-4, 5.0])
    p.set_irk(rng.standard_normal((q + 1, q)) / q)
    p.set_data(x_0, x_0 ** 2 * np.cos(np.pi * x_0))
    out["ac"] = dict(layers=L, q=q, **timed(p, init_weights(L)))
    p.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
