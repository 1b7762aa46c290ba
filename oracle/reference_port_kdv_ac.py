"""Restated upstream models: the discrete-time KdV identification and Allen-Cahn inference of the PINNs repository
(PINNs/main, TF1 float32) as fp64 torch CPU autograd, in the formulation of ``oracle.reference_port``: nested reverse-mode
sweeps (the dummy-gradient trick for the x-derivatives of all outputs) and an outer sweep for the parameter gradient.

TEST INFRASTRUCTURE (see oracle/__init__.py).  No upstream checkout of these scripts is pinned: the upstream constants quoted in
the docstrings are from memory of the scripts.  The independent check is ``oracle.taylor_kdv_ac`` (forward Taylor streams with
a third-order mode), which shares no derivation with this module.  ``reference_port.loss_and_flat_grad`` and
``reference_port.predict`` work on these problems unchanged.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Sequence

import numpy as np
import torch

from oracle.reference_port import DT, mlp, num_params


def _dummy_dx(U: torch.Tensor, x: torch.Tensor, q: int) -> torch.Tensor:
    """d/dx of every output column by the dummy-gradient trick: g = vjp(U, x; dummy), U_x = d g / d dummy."""
    dummy = torch.ones(x.shape[0], q, dtype=DT, requires_grad=True)
    g = torch.autograd.grad(U, x, grad_outputs=dummy, create_graph=True)[0]
    return torch.autograd.grad(g, dummy, grad_outputs=torch.ones_like(g), create_graph=True)[0]


@dataclass
class KdVDiscreteIdentification:
    """PINNs/main/discrete_time_identification (KdV)/KdV.py (upstream TF1 float32; restated in fp64, no upstream checkout
    pinned).  Same two-snapshot IRK identification as BurgersDiscreteIdentification with
        u_t + l1 u u_x + e^{l2} u_xxx = 0,   F = -l1 U U_x - e^{l2} U_xxx,
        U_0 = U - dt F alpha^T on x_0,  U_1 = U + dt F (beta - alpha)^T on x_1,  loss = sum((U_0-u_0)^2) + sum((U_1-u_1)^2).
    U_x, U_xx, U_xxx by the dummy-gradient trick applied three times.  Upstream values quoted from memory of the script, not
    read from it: lambda_1 init 0.0, lambda_2 init -6.0, N_0 = 199, N_1 = 201, layers [1, 50, 50, 50, 50, q] with
    q = ceil(0.5 log(eps) / log(dt)), dt = 0.6."""
    layers: Sequence[int]
    lb: np.ndarray
    ub: np.ndarray
    dt: float
    x_0: np.ndarray            # (N_0, 1)
    u_0: np.ndarray            # (N_0, 1)
    x_1: np.ndarray            # (N_1, 1)
    u_1: np.ndarray            # (N_1, 1)
    IRK_alpha: np.ndarray      # (q, q)
    IRK_beta: np.ndarray       # (1, q)

    def __post_init__(self):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
        self._lb, self._ub = t(self.lb).reshape(-1), t(self.ub).reshape(-1)
        self._x0, self._u0, self._x1, self._u1 = t(self.x_0), t(self.u_0), t(self.x_1), t(self.u_1)
        self._alpha = t(self.IRK_alpha)
        self._beta_minus_alpha = t(np.asarray(self.IRK_beta) - np.asarray(self.IRK_alpha))   # in the tables' own dtype
        self.q = int(self.IRK_alpha.shape[1])
        self.P = num_params(self.layers) + 2

    def autograd(self, wn: torch.Tensor, x0: torch.Tensor):
        x = x0.clone().requires_grad_(True)
        U = mlp(wn, x, self.layers, self._lb, self._ub)
        U_x = _dummy_dx(U, x, self.q)
        U_xx = _dummy_dx(U_x, x, self.q)
        U_xxx = _dummy_dx(U_xx, x, self.q)
        return U, U_x, U_xx, U_xxx

    def F(self, w: torch.Tensor, x: torch.Tensor):
        U, U_x, _, U_xxx = self.autograd(w[:-2], x)
        l1, l2 = w[-2], torch.exp(w[-1])
        return U, -l1 * U * U_x - l2 * U_xxx

    def U_0_model(self, w: torch.Tensor, x=None):
        U, F = self.F(w, self._x0 if x is None else x)
        return U - self.dt * (F @ self._alpha.T)

    def U_1_model(self, w: torch.Tensor, x=None):
        U, F = self.F(w, self._x1 if x is None else x)
        return U + self.dt * (F @ self._beta_minus_alpha.T)

    def loss_parts(self, w: torch.Tensor):
        return (torch.sum(torch.square(self.U_0_model(w) - self._u0)),
                torch.sum(torch.square(self.U_1_model(w) - self._u1)))

    def loss(self, w: torch.Tensor) -> torch.Tensor:
        a, b = self.loss_parts(w)
        return a + b


@dataclass
class AllenCahnDiscreteInference:
    """PINNs/main/discrete_time_inference (AC)/AC.py (upstream TF1 float32; restated in fp64, no upstream checkout pinned).
    u_t - d u_xx + k u^3 - k u = 0 on x in [lb, ub].  Net [1, ..., q+1]; U1 = net(x), U = U1[:, :q];
        F = k U - k U^3 + d U_xx,  U_0 = U1 - dt F IRK^T on x_0,  x_1 = [lb; ub],
        loss = sum((U_0 - u_0)^2) + sum_j (U1_j(lb) - U1_j(ub))^2 + sum_j (d/dx U1_j(lb) - d/dx U1_j(ub))^2
    (boundary sums over all q+1 outputs).  Upstream values quoted from memory of the script, not read from it: d = 1e-4,
    k = 5, N = 200, dt = 0.8, layers [1, 200, 200, 200, 200, q+1]."""
    layers: Sequence[int]
    lb: np.ndarray
    ub: np.ndarray
    dt: float
    x_0: np.ndarray            # (N, 1)
    u_0: np.ndarray            # (N, 1)
    IRK_weights: np.ndarray    # (q+1, q)
    d: float = 1e-4
    k: float = 5.0

    def __post_init__(self):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
        self._lb, self._ub = t(self.lb).reshape(-1), t(self.ub).reshape(-1)
        self._x0, self._u0 = t(self.x_0), t(self.u_0)
        self._x1 = torch.stack([self._lb[:1], self._ub[:1]])
        self._irk = t(self.IRK_weights)
        self.q = int(self.IRK_weights.shape[1])
        self.P = num_params(self.layers)

    def U_0_model(self, w: torch.Tensor):
        x = self._x0.clone().requires_grad_(True)
        U1 = mlp(w, x, self.layers, self._lb, self._ub)
        U = U1[:, :-1]
        U_x = _dummy_dx(U, x, self.q)
        U_xx = _dummy_dx(U_x, x, self.q)
        F = self.k * U - self.k * U ** 3 + self.d * U_xx
        return U1 - self.dt * (F @ self._irk.T)

    def U_1_model(self, w: torch.Tensor):
        x = self._x1.clone().requires_grad_(True)
        U1 = mlp(w, x, self.layers, self._lb, self._ub)
        return U1, _dummy_dx(U1, x, self.q + 1)

    def loss_parts(self, w: torch.Tensor):
        U1, U1_x = self.U_1_model(w)
        return (torch.sum(torch.square(self.U_0_model(w) - self._u0)),
                torch.sum(torch.square(U1[0] - U1[1])) + torch.sum(torch.square(U1_x[0] - U1_x[1])))

    def loss(self, w: torch.Tensor) -> torch.Tensor:
        a, b = self.loss_parts(w)
        return a + b
