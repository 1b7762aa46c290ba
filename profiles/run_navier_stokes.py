"""Step times and FP64 rate of the continuous-time Navier-Stokes identification model on its fused kernel: the upstream size
(PINNs/main continuous_time_identification (Navier-Stokes)/NavierStokes.py: [3, 20 x 8, 2], N_train = 5000) and N = 50 000,
where the kernel rather than launch latency dominates; Taylor-Green training points (2d-navier-stokes/navierstokesutil.py).

Per size: ms per Adam step (device events), fused-kernel ms (pinn_time_loss_grad_kernel), ms per L-BFGS iteration, and the
achieved FP64 rate of the kernel from the algorithmic FLOP count below, against the 67 TFLOP/s data-sheet figure and the best
measured DMMA.16x8x4 rate of profiles/microbench/fp64_peak_h100.jsonl.  For context: one evaluation of the CPU nested-autograd
oracle at N = 5000, and a short identification run with its final lambda errors (a report, not a bar).  The card's name, power
limit and max SM clock are read in the same run.  Run from the repo root; prints one JSON object."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.getcwd()
sys.path[:0] = [ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "utils"), os.path.join(ROOT, "pinns-tf2.0_b200", "2d-navier-stokes")]
import pinn_cabi  # noqa: E402
from bench import init_weights, timed_adam_steps  # noqa: E402
from navierstokesutil import TG_NU, prep_data  # noqa: E402

LAYERS = [3] + 8 * [20] + [2]
DATASHEET_FP64_TFLOPS = 67.0             # H100 SXM, FP64 tensor core, dense


def flops_per_eval(layers):
    """2 FLOP per multiply-add of the three GEMM families over the 13 streams: forward 26 S, weight gradient 26 S, input adjoint
    26 (S - 3 w_1) (the first layer has no input adjoint), S = sum in x out over the Dense layers."""
    S = sum(a * b for a, b in zip(layers[:-1], layers[1:]))
    return 26 * S + 26 * S + 26 * (S - 3 * layers[1])


def dmma16_peak():
    best = 0.0
    with open(os.path.join(ROOT, "profiles", "microbench", "fp64_peak_h100.jsonl")) as f:
        for line in f:
            r = json.loads(line)
            if r.get("shape") == "m16n8k4" and "tflops" in r:
                best = max(best, r["tflops"])
    return best


def lbfgs_ms_per_iter(p, w0, iters):
    """From w0 (weights after the timed Adam steps: from the initial weights the fixed-step L-BFGS stops after a few iterations)."""
    p.set_weights(w0)
    p.lbfgs(3, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, sync_every=1000)      # warm-up
    p.set_weights(w0)
    p.sync()
    t0 = time.perf_counter()
    r = p.lbfgs(iters, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, sync_every=1000)
    p.sync()
    return (time.perf_counter() - t0) * 1e3 / max(r["n_iter"], 1), r["n_iter"], r["reason_str"]


def timed(n, peak16):
    X, uv, lb, ub, _ = prep_data(None, N_train=n, seed=1234)
    p = pinn_cabi.Pinn(pinn_cabi.NS_IDE, LAYERS, lb, ub)
    p.set_data(X, uv)
    w0 = np.concatenate([init_weights(LAYERS), [0.0, 0.0]])
    p.set_weights(w0)
    for _ in range(10):
        p.adam_step(1e-3, sync=False)
    p.sync()
    adam = float(np.median(timed_adam_steps(p, 100, flush=False, lr=1e-3)))
    p.time_kernel_ms(10)
    kernel = p.time_kernel_ms(100) / 100
    lb_ms, n_it, why = lbfgs_ms_per_iter(p, p.get_weights(), 200)
    tflops = flops_per_eval(LAYERS) * n / (kernel * 1e-3) / 1e12
    out = {"n": n, "ms_per_adam_step": adam, "kernel_ms": kernel, "ms_per_lbfgs_iter": lb_ms, "lbfgs_iters": n_it, "lbfgs_stop": why,
           "flop_per_eval": flops_per_eval(LAYERS) * n, "kernel_tflops": tflops,
           "share_of_datasheet_67": tflops / DATASHEET_FP64_TFLOPS, "share_of_measured_dmma16x8x4": tflops / peak16,
           "info": p.kernel_info()}
    p.close()
    return out


def oracle_eval_s(n):
    from oracle import reference_port as rp, reference_port_ns as rn
    X, uv, lb, ub, _ = prep_data(None, N_train=n, seed=1234)
    pb = rn.NavierStokesIdentification(LAYERS, lb, ub, X, uv)
    w0 = np.concatenate([init_weights(LAYERS), [0.0, 0.0]])
    t0 = time.perf_counter()
    rp.loss_and_flat_grad(pb, w0)
    return time.perf_counter() - t0


def identification(adam_steps, lbfgs_iters):
    X, uv, lb, ub, _ = prep_data(None, N_train=5000, seed=1234)
    p = pinn_cabi.Pinn(pinn_cabi.NS_IDE, LAYERS, lb, ub)
    p.set_data(X, uv)
    p.set_weights(np.concatenate([init_weights(LAYERS), [0.0, 0.0]]))
    t0 = time.perf_counter()
    p.adam_steps(adam_steps, 1e-3)
    r = p.lbfgs(lbfgs_iters, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, sync_every=100)
    p.sync()
    l1, l2 = p.get_params()
    loss, _, _ = p.loss_grad()
    out = {"adam_steps": adam_steps, "lbfgs_iters": r["n_iter"], "lbfgs_reason": r["reason_str"], "seconds": time.perf_counter() - t0,
           "loss": loss, "lambda_1": l1, "lambda_2": l2, "err_lambda_1_pct": abs(l1 - 1.0) * 100,
           "err_lambda_2_pct": abs(l2 - TG_NU) / TG_NU * 100}
    p.close()
    return out


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    peak16 = dmma16_peak()
    out = {"card": card[0] if card else "unknown", "layers": LAYERS, "measured_dmma16x8x4_tflops": peak16,
           "sizes": [timed(n, peak16) for n in (5000, 50000)], "cpu_oracle_eval_s_n5000": oracle_eval_s(5000),
           "identification": identification(int(os.environ.get("NS_ADAM", "2000")), int(os.environ.get("NS_LBFGS", "5000")))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
