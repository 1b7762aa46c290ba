"""Generate tests/golden/ns_ide.npz (and no other file):
    PYTHONPATH=. python tests/golden/make_ns_golden.py

Seeded synthetic data (the Taylor-Green vortex of 2d-navier-stokes/navierstokesutil.py): no upstream cylinder_nektar_wake.mat is
read, and no upstream run exists to pin this fp64 model to (the upstream script is TF1 float32).  The values come from
``oracle.reference_port_ns`` (nested autograd, the upstream formulation) and are written only when ``oracle.taylor_ns`` (13 Taylor
streams) agrees to 1e-12 at every weight point.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "2d-navier-stokes")]
from oracle import reference_port as rp, reference_port_ns as rn, taylor_ns as tn  # noqa: E402
from navierstokesutil import prep_data  # noqa: E402

OUT = os.environ.get("PINN_GOLDEN_OUT", os.path.dirname(os.path.abspath(__file__)))


def check(name, f, g, f2, g2):
    rel_f = abs(f - f2) / abs(f)
    rel_g = np.linalg.norm(g - g2) / np.linalg.norm(g)
    print(f"{name}: loss {f:.15e} cross-check rel {rel_f:.2e}, grad rel {rel_g:.2e}")
    if not (rel_f < 1e-12 and rel_g < 1e-12):
        raise SystemExit(f"{name}: the two oracles disagree; nothing written")


def make():
    rng = np.random.default_rng(2025)
    layers = [3] + 8 * [20] + [2]
    X, uv, lb, ub, _ = prep_data(None, N_train=300, noise=0.0, seed=7)
    out = dict(layers=layers, lb=lb, ub=ub, X=X, uv=uv, X_probe=X[:64] + 0.01)
    pb = rn.NavierStokesIdentification(layers, lb, ub, X, uv)
    wn = rp.glorot_normal_flat(layers, rng) + 0.02 * rng.standard_normal(rp.num_params(layers))
    for tag, lam in (("", [0.0, 0.0]), ("2", [0.8, 0.02])):
        w = np.concatenate([wn, lam])
        f, g = rp.loss_and_flat_grad(pb, w)
        f2, g2, parts = tn.ns_ide_loss_grad(w, layers, lb, ub, X, uv)
        check("ns_ide" + tag, f, g, f2, g2)
        out["w" + tag], out["loss" + tag], out["grad" + tag], out["parts" + tag] = w, f, g, np.array(parts)
    # 13-stream probes and residuals at w2
    O, _ = tn.forward_ns(out["w2"][:-2], layers, lb, ub, out["X_probe"])
    out["probe"] = np.stack(O, 1)                                          # (64, 13, 2)
    _, fuv = pb.predict(out["w2"], X)
    out["residual"] = np.hstack(fuv)                                       # (N, 2) = (f_u, f_v)
    wa, la, _ = rp.adam_train(pb, out["w2"], 3, lr=1e-3)
    out["adam_losses"], out["adam_w"] = la, wa
    tr = rp.lbfgs_fixed_step(lambda z: rp.loss_and_flat_grad(pb, z), out["w2"], max_iter=4, learning_rate=0.8, n_correction=50,
                             tol_fun=np.finfo(float).eps)
    out["lbfgs_x_eval"], out["lbfgs_f"], out["lbfgs_x_final"] = np.array(tr.x_eval), np.array(tr.f_hist), tr.x_final
    return out


if __name__ == "__main__":
    out = make()
    path = os.path.join(OUT, "ns_ide.npz")
    np.savez_compressed(path, **out)
    print("ns_ide.npz", os.path.getsize(path) // 1024, "KiB, P =", out["w"].size)
