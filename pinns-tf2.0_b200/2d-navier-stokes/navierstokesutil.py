"""Data preparation for the continuous-time Navier-Stokes identification (the data block of PINNs/main/continuous_time_identification
(Navier-Stokes)/NavierStokes.py, restated): the upstream .mat layout X_star (N,2), t (T,1), U_star (N,2,T), p_star (N,T) is tiled
and flattened to N*T rows (x, y, t, u, v, p), N_train rows are drawn without replacement and noise * std * randn is added to u
and v.

The upstream file (cylinder_nektar_wake.mat) is not shipped.  Without a path, prep_data uses the TG vortex (the classical
decaying array of vortices), an exact Navier-Stokes solution with lambda_1 = 1 and lambda_2 = nu, generated from a seed in the
same layout, so that one code path serves both."""
import sys

import numpy as np
import scipy.io

sys.path.append("utils")

TG_K, TG_NU = 1.0, 0.01


def tg_vortex(n_space=1000, n_t=50, k=TG_K, nu=TG_NU, seed=0, x_range=(1.0, 8.0), y_range=(-2.0, 2.0), t_range=(0.0, 19.9)):
    """TG vortex in the upstream .mat layout: n_space random positions (seeded), n_t equidistant times;
        u = sin kx cos ky F,  v = -cos kx sin ky F,  p = (cos 2kx + cos 2ky) F^2 / 4,  F = exp(-2 nu k^2 t),
    stream function psi = sin kx sin ky F / k (u = psi_y, v = -psi_x)."""
    rng = np.random.default_rng(seed)
    X_star = np.stack([rng.uniform(*x_range, n_space), rng.uniform(*y_range, n_space)], 1)
    t = np.linspace(t_range[0], t_range[1], n_t)[:, None]
    x, y = X_star[:, 0:1], X_star[:, 1:2]
    F = np.exp(-2.0 * nu * k * k * t.T)                                   # (1, T)
    u = np.sin(k * x) * np.cos(k * y) * F
    v = -np.cos(k * x) * np.sin(k * y) * F
    p = 0.25 * (np.cos(2 * k * x) + np.cos(2 * k * y)) * F * F
    return {"X_star": X_star, "t": t, "U_star": np.stack([u, v], 1), "p_star": p}


def write_tg_vortex_mat(path, **kw):
    scipy.io.savemat(path, tg_vortex(**kw))
    return path


def prep_data(path=None, N_train=5000, noise=0.0, seed=1234):
    """-> X_train (N_train,3) = (x, y, t), uv_train (N_train,2), lb, ub (column min / max of the training points), and the full
    set (X_star (N*T,3), u_star, v_star, p_star, each (N*T,1)) for the error report."""
    data = scipy.io.loadmat(path) if path is not None else tg_vortex()
    U_star, P_star = data["U_star"], data["p_star"]                      # N x 2 x T, N x T
    t_star, X_star = data["t"], data["X_star"]                           # T x 1, N x 2
    N, T = X_star.shape[0], t_star.shape[0]
    XX = np.tile(X_star[:, 0:1], (1, T))
    YY = np.tile(X_star[:, 1:2], (1, T))
    TT = np.tile(t_star, (1, N)).T
    UU, VV, PP = U_star[:, 0, :], U_star[:, 1, :], P_star
    x, y, t = XX.flatten()[:, None], YY.flatten()[:, None], TT.flatten()[:, None]
    u, v, p = UU.flatten()[:, None], VV.flatten()[:, None], PP.flatten()[:, None]
    rs = np.random.RandomState(seed)
    idx = rs.choice(N * T, N_train, replace=False)
    X_train = np.hstack([x[idx], y[idx], t[idx]])
    u_train, v_train = u[idx], v[idx]
    if noise:
        u_train = u_train + noise * np.std(u_train) * rs.randn(*u_train.shape)
        v_train = v_train + noise * np.std(v_train) * rs.randn(*v_train.shape)
    lb, ub = X_train.min(0), X_train.max(0)
    return X_train, np.hstack([u_train, v_train]), lb, ub, (np.hstack([x, y, t]), u, v, p)
