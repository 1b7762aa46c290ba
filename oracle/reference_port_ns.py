"""Restated upstream model: the continuous-time Navier-Stokes identification of the PINNs repository (PINNs/main, TF1 float32)
as fp64 torch CPU autograd, in the formulation of ``oracle.reference_port``: nested reverse-mode sweeps for the derivatives of
the velocities and an outer sweep for the parameter gradient.

TEST INFRASTRUCTURE (see oracle/__init__.py).  No upstream checkout of this script is pinned, and no TF2.0 port of it exists:
the upstream constants quoted in the docstrings are from memory of NavierStokes.py.  The independent check is
``oracle.taylor_ns`` (13 forward Taylor streams and a hand-derived reverse), which shares no derivation with this module.
``reference_port.loss_and_flat_grad``, ``predict``, ``adam_train`` and ``lbfgs_fixed_step`` work on this problem unchanged.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Sequence

import numpy as np
import torch

from oracle.reference_port import _grad, mlp, num_params


@dataclass
class NavierStokesIdentification:
    """PINNs/main/continuous_time_identification (Navier-Stokes)/NavierStokes.py:113-137 (net_NS and the loss; upstream TF1
    float32, restated in fp64).  Flat vector = [net params, lambda_1, lambda_2], both raw (no exp).  The net [3, ..., 2] maps
    (x, y, t) to (psi, p); u = psi_y, v = -psi_x;
        f_u = u_t + l1 (u u_x + v u_y) + p_x - l2 (u_xx + u_yy)
        f_v = v_t + l1 (u v_x + v v_y) + p_y - l2 (v_xx + v_yy)
        loss = sum (u - u_d)^2 + sum (v - v_d)^2 + sum f_u^2 + sum f_v^2   (reduce_sum, every point carries both terms).
    Upstream values quoted from memory of the script, not read from it: lambda_1 = lambda_2 = 0.0 initially, N_train = 5000,
    layers [3, 20, 20, 20, 20, 20, 20, 20, 20, 2], data cylinder_nektar_wake.mat."""
    layers: Sequence[int]
    lb: np.ndarray
    ub: np.ndarray
    X: np.ndarray              # (N, 3) = (x, y, t)
    uv: np.ndarray             # (N, 2) = (u, v)

    def __post_init__(self):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
        self._lb, self._ub = t(self.lb).reshape(-1), t(self.ub).reshape(-1)
        self._X, self._uv = t(self.X), t(self.uv)
        self.P = num_params(self.layers) + 2

    def net_NS(self, w: torch.Tensor, X=None):
        """(u, v, p, f_u, f_v) on X (default: the training points)."""
        X = self._X if X is None else X
        x, y, t = (X[:, c:c + 1].clone().requires_grad_(True) for c in range(3))
        psi_and_p = mlp(w, torch.cat([x, y, t], 1), self.layers, self._lb, self._ub)
        psi, p = psi_and_p[:, 0:1], psi_and_p[:, 1:2]
        u = _grad(psi, y)
        v = -_grad(psi, x)
        u_t, u_x, u_y = _grad(u, t), _grad(u, x), _grad(u, y)
        u_xx, u_yy = _grad(u_x, x), _grad(u_y, y)
        v_t, v_x, v_y = _grad(v, t), _grad(v, x), _grad(v, y)
        v_xx, v_yy = _grad(v_x, x), _grad(v_y, y)
        p_x, p_y = _grad(p, x), _grad(p, y)
        l1, l2 = w[-2], w[-1]
        f_u = u_t + l1 * (u * u_x + v * u_y) + p_x - l2 * (u_xx + u_yy)
        f_v = v_t + l1 * (u * v_x + v * v_y) + p_y - l2 * (v_xx + v_yy)
        return u, v, p, f_u, f_v

    def loss_parts(self, w: torch.Tensor):
        u, v, _, f_u, f_v = self.net_NS(w)
        return (torch.sum(torch.square(self._uv[:, 0:1] - u)) + torch.sum(torch.square(self._uv[:, 1:2] - v)),
                torch.sum(torch.square(f_u)) + torch.sum(torch.square(f_v)))

    def loss(self, w: torch.Tensor) -> torch.Tensor:
        a, b = self.loss_parts(w)
        return a + b

    def predict(self, w, X_star):
        """predict of the upstream class: (u, v, p) and (f_u, f_v) on X_star, each (N, 1)."""
        wt = torch.as_tensor(np.asarray(w, dtype=np.float64))
        u, v, p, f_u, f_v = self.net_NS(wt, torch.as_tensor(np.asarray(X_star, dtype=np.float64)))
        return tuple(a.detach().numpy() for a in (u, v, p)), tuple(a.detach().numpy() for a in (f_u, f_v))
