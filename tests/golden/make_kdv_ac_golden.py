"""Generate tests/golden/kdv_ide_disc.npz and tests/golden/ac_disc.npz (and no other file):
    PYTHONPATH=. python tests/golden/make_kdv_ac_golden.py

Seeded synthetic data: no upstream KdV.mat / AC.mat is read, and no upstream run exists to pin these fp64 models to (the
upstream scripts are TF1 float32).  The values come from ``oracle.reference_port_kdv_ac`` (nested autograd, the upstream
formulation) and are written only when ``oracle.taylor_kdv_ac`` (third-order Taylor streams) agrees to 1e-12 at every weight
point.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import reference_port as rp, reference_port_kdv_ac as rk, taylor_kdv_ac as tk  # noqa: E402

OUT = os.environ.get("PINN_GOLDEN_OUT", os.path.dirname(os.path.abspath(__file__)))


def check(name, f, g, f2, g2):
    rel_f = abs(f - f2) / abs(f)
    rel_g = np.linalg.norm(g - g2) / np.linalg.norm(g)
    print(f"{name}: loss {f:.15e} cross-check rel {rel_f:.2e}, grad rel {rel_g:.2e}")
    if not (rel_f < 1e-12 and rel_g < 1e-12):
        raise SystemExit(f"{name}: the two oracles disagree; nothing written")


def optimiser_runs(pb, out):
    wa, la, _ = rp.adam_train(pb, out["w2"], 3, lr=1e-3)
    out["adam_losses"], out["adam_w"] = la, wa
    tr = rp.lbfgs_fixed_step(lambda z: rp.loss_and_flat_grad(pb, z), out["w2"], max_iter=4, learning_rate=0.8, n_correction=50,
                             tol_fun=np.finfo(float).eps)
    out["lbfgs_x_eval"], out["lbfgs_f"], out["lbfgs_x_final"] = np.array(tr.x_eval), np.array(tr.f_hist), tr.x_final


def make_kdv():
    rng = np.random.default_rng(2023)
    q, dt = 12, 0.6
    layers = [1, 30, 30, 30, q]
    lb, ub = np.array([-1.0]), np.array([1.0])
    x_0 = rng.uniform(-1, 1, (41, 1)); u_0 = np.cos(np.pi * x_0)
    x_1 = rng.uniform(-1, 1, (39, 1)); u_1 = 0.9 * np.cos(np.pi * x_1 + 0.2)
    alpha = (rng.standard_normal((q, q)) / q).astype(np.float32)
    beta = (rng.standard_normal((1, q)) / q).astype(np.float32)
    out = dict(layers=layers, lb=lb, ub=ub, dt=dt, q=q, x_0=x_0, u_0=u_0, x_1=x_1, u_1=u_1, IRK_alpha=alpha, IRK_beta=beta,
               x_star=np.linspace(-1, 1, 33)[:, None])
    wn = rp.glorot_normal_flat(layers, rng) + 0.02 * rng.standard_normal(rp.num_params(layers))
    pb = rk.KdVDiscreteIdentification(layers, lb, ub, dt, x_0, u_0, x_1, u_1, alpha, beta)
    for tag, lam in (("", [0.0, -6.0]), ("2", [0.7, -2.5])):
        w = np.concatenate([wn, lam])
        f, g = rp.loss_and_flat_grad(pb, w)
        f2, g2, parts = tk.kdv_ide_disc_loss_grad(w, layers, lb, ub, x_0, u_0, x_1, u_1, dt, alpha, beta)
        check("kdv_ide_disc" + tag, f, g, f2, g2)
        out["w" + tag], out["loss" + tag], out["grad" + tag], out["parts" + tag] = w, f, g, np.array(parts)
    optimiser_runs(pb, out)
    return out


def make_ac():
    rng = np.random.default_rng(2024)
    q, dt = 16, 0.8
    layers = [1, 40, 40, q + 1]
    lb, ub = np.array([-1.0]), np.array([1.0])
    x_0 = rng.uniform(-1, 1, (51, 1)); u_0 = x_0 ** 2 * np.cos(np.pi * x_0)
    irk = rng.standard_normal((q + 1, q)) / q
    out = dict(layers=layers, lb=lb, ub=ub, dt=dt, q=q, d=1e-4, k=5.0, x_0=x_0, u_0=u_0, IRK=irk)
    pb = rk.AllenCahnDiscreteInference(layers, lb, ub, dt, x_0, u_0, irk, d=1e-4, k=5.0)
    w1 = rp.glorot_normal_flat(layers, rng)
    for tag, w in (("", w1), ("2", w1 + 0.05 * rng.standard_normal(w1.size))):
        f, g = rp.loss_and_flat_grad(pb, w)
        f2, g2, parts = tk.ac_disc_loss_grad(w, layers, lb, ub, x_0, u_0, dt, irk, d=1e-4, k=5.0)
        check("ac_disc" + tag, f, g, f2, g2)
        out["w" + tag], out["loss" + tag], out["grad" + tag], out["parts" + tag] = w, f, g, np.array(parts)
    optimiser_runs(pb, out)
    return out


if __name__ == "__main__":
    outs = {"kdv_ide_disc": make_kdv(), "ac_disc": make_ac()}     # both verified before either file is written
    for name, out in outs.items():
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print(name + ".npz", os.path.getsize(path) // 1024, "KiB, P =", out["w"].size)
