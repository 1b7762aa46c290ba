"""User-defined polynomial residuals (PINN_POLY_INF / PINN_POLY_IDE) as fp64 torch CPU autograd, in the formulation of
``oracle.reference_port``: nested reverse-mode sweeps (``create_graph=True``) for u_x, u_t, u_xx, then the term list, then an
outer sweep for the parameter gradient.

TEST INFRASTRUCTURE (see oracle/__init__.py).  The independent check is ``oracle.taylor_poly`` (forward Taylor streams and the
analytic seed formula), which shares no derivation with this module.  With the Burgers terms this class computes what
``reference_port.BurgersInference`` / ``BurgersIdentification`` compute, which ties it to the pinned reference run.
``reference_port.loss_and_flat_grad``, ``predict``, ``adam_train`` and ``lbfgs_fixed_step`` work on this problem unchanged.

A term is (coef, kind, (e_u, e_ux, e_ut, e_uxx)) with kind 0..4 selecting kappa = 1, l1, l2, exp(l1), exp(l2) (raw lambdas,
the last two entries of the flat vector of the identification model).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np
import torch

from oracle.reference_port import _grad, mlp, num_params


def terms_value(terms, streams, l1=0.0, l2=0.0):
    """sum_k c_k kappa_k prod_j streams[j]^e_kj (torch or numpy operands)."""
    exp = torch.exp if isinstance(l1, torch.Tensor) else np.exp
    kv = (1.0, l1, l2, exp(l1) if any(k == 3 for _, k, _ in terms) else None,
          exp(l2) if any(k == 4 for _, k, _ in terms) else None)
    f = 0.0
    for c, k, e in terms:
        m = c
        for v, p in zip(streams, e):
            for _ in range(p):
                m = m * v
        f = f + (m if k == 0 else kv[k] * m)
    return f


@dataclass
class PolyProblem:
    """f = sum_k c_k kappa_k u^a u_x^b u_t^c u_xx^d - s on the residual points.
    Inference (identification=False): loss = data_weight mean (u - u_d)^2 over X_u + sum f^2 / n_f_global over X_f (the
    BURGERS_INF structure).  Identification: the residual points are X_u, loss = mean (u - u_d)^2 + mean f^2, flat vector
    [net, l1, l2] (the BURGERS_IDE structure).  source: s at the residual points, or None (0)."""
    layers: Sequence[int]
    lb: np.ndarray
    ub: np.ndarray
    terms: Sequence
    X_u: np.ndarray
    u: np.ndarray
    X_f: Optional[np.ndarray] = None
    source: Optional[np.ndarray] = None
    identification: bool = False
    n_f_global: Optional[int] = None
    data_weight: float = 1.0

    def __post_init__(self):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
        self._lb, self._ub = t(self.lb), t(self.ub)
        self._X_u, self._u = t(self.X_u), t(self.u).reshape(-1, 1)
        self._X_f = self._X_u if self.identification else t(self.X_f)
        self._s = None if self.source is None else t(self.source).reshape(-1, 1)
        self.P = num_params(self.layers) + (2 if self.identification else 0)

    def streams(self, w: torch.Tensor, X=None):
        X = self._X_f if X is None else X
        x = X[:, 0:1].clone().requires_grad_(True)
        t = X[:, 1:2].clone().requires_grad_(True)
        u = mlp(w, torch.cat([x, t], 1), self.layers, self._lb, self._ub)
        u_x = _grad(u, x)
        u_xx = _grad(u_x, x)
        u_t = _grad(u, t)
        return u, u_x, u_t, u_xx

    def residual(self, w: torch.Tensor, X=None, source=None):
        l1, l2 = (w[-2], w[-1]) if self.identification else (0.0, 0.0)
        f = terms_value(self.terms, self.streams(w, X), l1, l2)
        s = self._s if X is None else source
        return f if s is None else f - s

    def loss_parts(self, w: torch.Tensor):
        f = self.residual(w)
        u_pred = mlp(w, self._X_u, self.layers, self._lb, self._ub)
        if self.identification:
            return torch.mean(torch.square(self._u - u_pred)), torch.mean(torch.square(f))
        n_f = self.n_f_global or f.shape[0]
        return torch.mean(torch.square(self._u - u_pred)) * self.data_weight, torch.sum(torch.square(f)) / n_f

    def loss(self, w: torch.Tensor) -> torch.Tensor:
        a, b = self.loss_parts(w)
        return a + b

    def f_model(self, w, X=None, source=None):
        """f on the residual points (or on X, minus the given source there), as numpy (N, 1)."""
        wt = torch.as_tensor(np.asarray(w, dtype=np.float64))
        Xt = None if X is None else torch.as_tensor(np.asarray(X, dtype=np.float64))
        st = None if source is None else torch.as_tensor(np.asarray(source, dtype=np.float64)).reshape(-1, 1)
        return self.residual(wt, Xt, st).detach().numpy()
