"""Generate tests/golden/poly.npz (and no other file):
    PYTHONPATH=. python tests/golden/make_poly_golden.py

Four user-defined residuals (PINN_POLY_INF / PINN_POLY_IDE) on seeded synthetic data.  The values come from
``oracle.reference_port_poly`` (nested autograd) and are written only when ``oracle.taylor_poly`` (Taylor streams and the
analytic seed formula) agrees to 1e-12 at every weight point.  Keys are prefixed with the case name.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT]
from oracle import reference_port as rp, reference_port_poly as rpp, taylor as ty, taylor_poly as tpo  # noqa: E402

OUT = os.environ.get("PINN_GOLDEN_OUT", os.path.dirname(os.path.abspath(__file__)))

HEAT_K = 0.25


def heat_source(x, t, k=HEAT_K):
    """s = u*_t - k u*_xx for the manufactured solution u* = e^-t sin(pi x)."""
    return (k * np.pi ** 2 - 1.0) * np.exp(-t) * np.sin(np.pi * x)


def stress_terms(rng):
    """Every stream at exponents up to 3, cross products, every kappa kind, random coefficients (12 terms)."""
    exps = [(1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1), (3, 0, 0, 0), (0, 3, 0, 0), (0, 0, 3, 0), (0, 0, 0, 3),
            (1, 2, 0, 1), (2, 1, 1, 0), (1, 1, 1, 1), (3, 3, 3, 3)]
    kinds = [0, 1, 2, 3, 4, 0, 1, 2, 3, 4, 0, 1]
    return [(float(c), k, e) for c, k, e in zip(rng.uniform(-1.5, 1.5, len(exps)), kinds, exps)]


def cases():
    """name -> dict(layers, lb, ub, terms, identification, X_u, u, X_f, source, w, X_probe)."""
    out = {}
    # continuous-time Allen-Cahn inference: u_t - 1e-4 u_xx + 5 u^3 - 5 u, initial condition x^2 cos(pi x)
    rng = np.random.default_rng(11)
    layers = [2] + 4 * [20] + [1]
    lb, ub = np.array([-1.0, 0.0]), np.array([1.0, 1.0])
    x0 = np.linspace(-1, 1, 64)[:, None]
    out["ac"] = dict(layers=layers, lb=lb, ub=ub, identification=False,
                     terms=[(1.0, 0, (0, 0, 1, 0)), (-1e-4, 0, (0, 0, 0, 1)), (5.0, 0, (3, 0, 0, 0)), (-5.0, 0, (1, 0, 0, 0))],
                     X_u=np.hstack([x0, 0 * x0]), u=x0 ** 2 * np.cos(np.pi * x0), X_f=lb + (ub - lb) * rng.random((400, 2)),
                     source=None, w=rp.glorot_normal_flat(layers, rng) + 0.02 * rng.standard_normal(rp.num_params(layers)))
    # heat with a manufactured source on x in [0, 2], t in [0, 1]: u_t - k u_xx = s, u* = e^-t sin(pi x)
    rng = np.random.default_rng(12)
    layers = [2, 16, 16, 1]
    lb, ub = np.array([0.0, 0.0]), np.array([2.0, 1.0])
    Xb = np.vstack([np.hstack([np.linspace(0, 2, 40)[:, None], np.zeros((40, 1))]),
                    np.hstack([np.zeros((20, 1)), np.linspace(0, 1, 20)[:, None]]),
                    np.hstack([2 * np.ones((20, 1)), np.linspace(0, 1, 20)[:, None]])])
    X_f = lb + (ub - lb) * rng.random((300, 2))
    out["heat"] = dict(layers=layers, lb=lb, ub=ub, identification=False,
                       terms=[(1.0, 0, (0, 0, 1, 0)), (-HEAT_K, 0, (0, 0, 0, 1))],
                       X_u=Xb, u=np.exp(-Xb[:, 1:2]) * np.sin(np.pi * Xb[:, 0:1]), X_f=X_f,
                       source=heat_source(X_f[:, 0:1], X_f[:, 1:2]),
                       w=rp.glorot_normal_flat(layers, rng) + 0.02 * rng.standard_normal(rp.num_params(layers)))
    # Fisher-KPP identification: u_t - e^l2 u_xx - l1 u + l1 u^2, data from a logistic travelling front
    rng = np.random.default_rng(13)
    layers = [2, 20, 20, 20, 1]
    lb, ub = np.array([-5.0, 0.0]), np.array([5.0, 2.0])
    X = lb + (ub - lb) * rng.random((250, 2))
    out["fisher"] = dict(layers=layers, lb=lb, ub=ub, identification=True,
                         terms=[(1.0, 0, (0, 0, 1, 0)), (-1.0, 4, (0, 0, 0, 1)), (-1.0, 1, (1, 0, 0, 0)), (1.0, 1, (2, 0, 0, 0))],
                         X_u=X, u=1.0 / (1.0 + np.exp(X[:, 0:1] - 1.5 * X[:, 1:2])), X_f=None, source=None,
                         w=np.concatenate([rp.glorot_normal_flat(layers, rng) + 0.02 * rng.standard_normal(rp.num_params(layers)),
                                           [0.7, -1.5]]))
    # stress: every stream up to exponent 3, every kappa kind, an odd net, a box far from [-1, 1]
    rng = np.random.default_rng(14)
    layers = [2, 7, 33, 1]
    lb, ub = np.array([0.5, -2.0]), np.array([3.0, 5.0])
    X = lb + (ub - lb) * rng.random((150, 2))
    out["stress"] = dict(layers=layers, lb=lb, ub=ub, identification=True, terms=stress_terms(rng),
                         X_u=X, u=np.sin(X[:, 0:1]) * np.cos(0.3 * X[:, 1:2]), X_f=None, source=0.1 * rng.standard_normal((150, 1)),
                         w=np.concatenate([rp.glorot_normal_flat(layers, rng) + 0.02 * rng.standard_normal(rp.num_params(layers)),
                                           [0.3, -0.4]]))
    for c in out.values():
        c["X_probe"] = c["lb"] + (c["ub"] - c["lb"]) * np.random.default_rng(99).random((32, 2))
    return out


def problem(c):
    return rpp.PolyProblem(c["layers"], c["lb"], c["ub"], c["terms"], c["X_u"], c["u"], X_f=c["X_f"], source=c["source"],
                           identification=c["identification"])


def taylor(c, w, **kw):
    return tpo.poly_loss_grad(w, c["layers"], c["lb"], c["ub"], c["terms"], c["X_u"], c["u"], X_f=c["X_f"], source=c["source"],
                              identification=c["identification"], **kw)


def make():
    out = {}
    for name, c in cases().items():
        pb = problem(c)
        f, g = rp.loss_and_flat_grad(pb, c["w"])
        f2, g2, parts = taylor(c, c["w"])
        rel_f, rel_g = abs(f - f2) / abs(f), np.linalg.norm(g - g2) / np.linalg.norm(g)
        print(f"{name}: P = {g.size}, loss {f:.15e}, cross-check rel {rel_f:.2e}, grad rel {rel_g:.2e}")
        if not (rel_f < 1e-12 and rel_g < 1e-12):
            raise SystemExit(f"{name}: the two oracles disagree; nothing written")
        wn = c["w"][:-2] if c["identification"] else c["w"]
        O, _ = ty.forward(wn, c["layers"], c["lb"], c["ub"], c["X_probe"])
        wa, la, _ = rp.adam_train(pb, c["w"], 5, lr=1e-3)
        tr = rp.lbfgs_fixed_step(lambda z: rp.loss_and_flat_grad(pb, z), c["w"], max_iter=6, learning_rate=0.8, n_correction=50,
                                 tol_fun=np.finfo(float).eps)
        for k, v in dict(layers=c["layers"], lb=c["lb"], ub=c["ub"], X_u=c["X_u"], u=c["u"], w=c["w"], X_probe=c["X_probe"],
                         coef=[t[0] for t in c["terms"]], kind=[t[1] for t in c["terms"]], exps=[t[2] for t in c["terms"]],
                         identification=c["identification"], loss=f, grad=g, parts=np.array(parts),
                         probe=np.stack([o[:, 0] for o in O], 1), residual=pb.f_model(c["w"]), adam_losses=la, adam_w=wa,
                         lbfgs_x_eval=np.array(tr.x_eval), lbfgs_f=np.array(tr.f_hist), lbfgs_x_final=tr.x_final).items():
            out[name + "_" + k] = np.asarray(v)
        if c["X_f"] is not None:
            out[name + "_X_f"] = c["X_f"]
        if c["source"] is not None:
            out[name + "_source"] = c["source"]
    return out


if __name__ == "__main__":
    out = make()
    path = os.path.join(OUT, "poly.npz")
    np.savez_compressed(path, **out)
    print("poly.npz", os.path.getsize(path) // 1024, "KiB")
