"""Restated reference: TF-free fp64 port of the PINNs-TF2.0 training hot path (torch CPU autograd).

TEST INFRASTRUCTURE (see oracle/__init__.py).  The reference has no tests of its own (parity against TensorFlow's kernels is
UNPINNED); this port is pinned to the reference's own Python executed on an emulated TensorFlow (tests/test_reference_pin.py).

The reference computes u_x, u_t, u_xx with nested ``tf.GradientTape``s and d(loss)/d(params) with an
outer tape.  This port keeps that *algorithmic structure* -- nested reverse-mode sweeps with
``create_graph=True`` -- so that (a) it is an honest "reference CPU path" to time and (b) it shares no
derivation with the forward Taylor-mode maths used by the CUDA kernels and by ``oracle.taylor``.

Every function cites the reference file:line (relative to the upstream PINNs-TF2.0 checkout) it restates.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch

DT = torch.float64
TF_KERAS_EPSILON = 1e-7  # tf.keras.backend.epsilon(); used when hp["tf_eps"] is None


# ----------------------------------------------------------------------------------------------
# Parameter layout  (utils/neuralnetwork.py:40-45 sizes_w/sizes_b, :68-89 get/set_weights)
# ----------------------------------------------------------------------------------------------
def layer_shapes(layers: Sequence[int]) -> List[Tuple[int, int]]:
    """(in, out) of every Dense layer: hidden tanh layers then the linear head (neuralnetwork.py:31-37)."""
    return [(int(layers[i]), int(layers[i + 1])) for i in range(len(layers) - 1)]


def num_params(layers: Sequence[int]) -> int:
    return sum(i * o + o for i, o in layer_shapes(layers))


def param_offsets(layers: Sequence[int]) -> List[Tuple[int, int]]:
    """Offsets (w_off, b_off) into the flat vector: per layer W.flatten() row-major [in,out], then b.

    Same order as ``get_weights`` (neuralnetwork.py:68-78) and the flat gradient (:97-100)."""
    offs, o = [], 0
    for fan_in, fan_out in layer_shapes(layers):
        offs.append((o, o + fan_in * fan_out))
        o += fan_in * fan_out + fan_out
    return offs


def glorot_normal_flat(layers: Sequence[int], rng: np.random.Generator) -> np.ndarray:
    """Keras ``glorot_normal`` look-alike (neuralnetwork.py:33,37): truncated N(0, s) at 2 s with
    s = sqrt(2/(fan_in+fan_out))/0.87962566103423978, zero biases.  TF's RNG stream cannot be
    reproduced, so parity runs always LOAD the same flat vector into both sides."""
    from scipy.stats import truncnorm

    out = []
    for fan_in, fan_out in layer_shapes(layers):
        std = math.sqrt(2.0 / (fan_in + fan_out)) / 0.87962566103423978
        W = truncnorm.rvs(-2.0, 2.0, scale=std, size=(fan_in, fan_out), random_state=rng)
        out.append(W.reshape(-1))
        out.append(np.zeros(fan_out))
    return np.concatenate(out).astype(np.float64)


# ----------------------------------------------------------------------------------------------
# Model forward  (utils/neuralnetwork.py:27-37)
# ----------------------------------------------------------------------------------------------
def mlp(w: torch.Tensor, X: torch.Tensor, layers: Sequence[int], lb: torch.Tensor, ub: torch.Tensor) -> torch.Tensor:
    """Lambda normalisation 2(X-lb)/(ub-lb)-1 (:29-30, broadcasting over the last axis exactly like the
    numpy closure does -- which is what produces quirk Q1 for a (N,1) input), tanh Dense stack, linear head."""
    H = 2.0 * (X - lb) / (ub - lb) - 1.0
    shapes = layer_shapes(layers)
    for li, ((fi, fo), (wo, bo)) in enumerate(zip(shapes, param_offsets(layers))):
        W = w[wo:wo + fi * fo].view(fi, fo)
        b = w[bo:bo + fo]
        H = H @ W + b
        if li != len(shapes) - 1:
            H = torch.tanh(H)
    return H


def _grad(y: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """``tape.gradient(y, x)`` for non-scalar y == vector-Jacobian product with ones (TF semantics)."""
    return torch.autograd.grad(y, x, torch.ones_like(y), create_graph=True)[0]


# ----------------------------------------------------------------------------------------------
# Problems
# ----------------------------------------------------------------------------------------------
@dataclass
class BurgersInference:
    """1d-burgers/inf_cont_burgers.py:48-98 (BurgersInformedNN).

    ``wf_scale`` supports data-parallel sharding (SURVEY 8(e)): MSE_f is sum(f^2)/n_f_global."""
    layers: Sequence[int]
    lb: np.ndarray
    ub: np.ndarray
    nu: float
    X_f: np.ndarray            # (N_f, 2)
    X_u: np.ndarray            # (N_u, 2)
    u: np.ndarray              # (N_u, 1)
    n_f_global: Optional[int] = None
    data_weight: float = 1.0   # 1 on the rank that owns the data term, 0 elsewhere

    def __post_init__(self):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
        self._lb, self._ub = t(self.lb), t(self.ub)
        self._x_f = t(self.X_f[:, 0:1])   # :55
        self._t_f = t(self.X_f[:, 1:2])   # :56
        self._X_u, self._u = t(self.X_u), t(self.u)
        self.P = num_params(self.layers)

    def residual(self, w: torch.Tensor):
        """f_model (:65-90): persistent tape, u_x inside the tape, u_xx and u_t after it."""
        x = self._x_f.clone().requires_grad_(True)
        t = self._t_f.clone().requires_grad_(True)
        X = torch.stack([x[:, 0], t[:, 0]], dim=1)          # :73
        u = mlp(w, X, self.layers, self._lb, self._ub)      # :76
        u_x = _grad(u, x)                                   # :78
        u_xx = _grad(u_x, x)                                # :81
        u_t = _grad(u, t)                                   # :82
        return u_t + u * u_x - self.nu * u_xx, (u, u_x, u_t, u_xx)   # :90

    def loss_parts(self, w: torch.Tensor):
        """loss (:59-62): mean((u-u_pred)^2) + mean(f^2)."""
        f, _ = self.residual(w)
        u_pred = mlp(w, self._X_u, self.layers, self._lb, self._ub)
        mse_u = torch.mean(torch.square(self._u - u_pred)) * self.data_weight
        n_f = self.n_f_global or f.shape[0]
        mse_f = torch.sum(torch.square(f)) / n_f
        return mse_u, mse_f

    def loss(self, w: torch.Tensor) -> torch.Tensor:
        a, b = self.loss_parts(w)
        return a + b


@dataclass
class BurgersIdentification:
    """1d-burgers/ide_cont_burgers.py:47-118 (file does not parse as shipped; semantics followed).

    Flat vector = [net params, lambda_1, lambda_2] (:98-107).  Residual on the DATA points (:88-91):
    f = u_t + l1*u*u_x - exp(l2)*u_xx  (:56-85, get_params :109-114)."""
    layers: Sequence[int]
    lb: np.ndarray
    ub: np.ndarray
    X_u: np.ndarray
    u: np.ndarray

    def __post_init__(self):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
        self._lb, self._ub = t(self.lb), t(self.ub)
        self._X_u, self._u = t(self.X_u), t(self.u)
        self.P = num_params(self.layers) + 2

    def residual(self, w: torch.Tensor):
        l1, l2 = w[-2], torch.exp(w[-1])
        x = self._X_u[:, 0:1].clone().requires_grad_(True)
        t = self._X_u[:, 1:2].clone().requires_grad_(True)
        X = torch.stack([x[:, 0], t[:, 0]], dim=1)
        u = mlp(w, X, self.layers, self._lb, self._ub)
        u_x = _grad(u, x)
        u_xx = _grad(u_x, x)
        u_t = _grad(u, t)
        return u_t + l1 * u * u_x - l2 * u_xx, (u, u_x, u_t, u_xx)

    def loss_parts(self, w: torch.Tensor):
        f, _ = self.residual(w)
        u_pred = mlp(w, self._X_u, self.layers, self._lb, self._ub)
        return torch.mean(torch.square(self._u - u_pred)), torch.mean(torch.square(f))

    def loss(self, w: torch.Tensor) -> torch.Tensor:
        a, b = self.loss_parts(w)
        return a + b


@dataclass
class SchrodingerInference:
    """1dcomplex-schrodinger/inf_cont_schrodinger.py:46-135 (SchrodingerInformedNN).

    ``X0`` is whatever the script hands to ``fit`` as X_u: the shipped script passes x0 of shape (N_0,1)
    (:164), which the normalising Lambda broadcasts to (N_0,2) -- quirk Q1, the IC term is evaluated at
    (x, t:=x).  Passing the intended (x0, 0) array of shape (N_0,2) gives the intended behaviour."""
    layers: Sequence[int]
    lb: np.ndarray
    ub: np.ndarray
    X_f: np.ndarray
    tb: np.ndarray             # (N_b, 1)
    X0: np.ndarray             # (N_0, 1) [quirk Q1] or (N_0, 2)
    uv0: np.ndarray            # (N_0, 2)
    n_f_global: Optional[int] = None
    aux_weight: float = 1.0    # weight of the IC + BC terms on this rank (1 on the owner, else 0)

    def __post_init__(self):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
        self._lb, self._ub = t(self.lb), t(self.ub)
        tb = np.asarray(self.tb, dtype=np.float64)
        self._X_lb = t(np.concatenate((0 * tb + self.lb[0], tb), 1))   # :50
        self._X_ub = t(np.concatenate((0 * tb + self.ub[0], tb), 1))   # :51
        self._x_f = t(self.X_f[:, 0:1])
        self._t_f = t(self.X_f[:, 1:2])
        self._X0, self._uv0 = t(self.X0), t(self.uv0)
        self.P = num_params(self.layers)

    def uvx(self, w: torch.Tensor, x: torch.Tensor, t: torch.Tensor):
        """uvx_model (:60-76): u, v and their x-derivatives (one reverse sweep per output)."""
        X = torch.cat([x, t], dim=1)
        h = mlp(w, X, self.layers, self._lb, self._ub)
        u, v = h[:, 0:1], h[:, 1:2]
        return u, v, _grad(u, x), _grad(v, x)

    def residual(self, w: torch.Tensor):
        """f_model (:79-105)."""
        x = self._x_f.clone().requires_grad_(True)
        t = self._t_f.clone().requires_grad_(True)
        u, v, u_x, v_x = self.uvx(w, x, t)
        u_xx, v_xx = _grad(u_x, x), _grad(v_x, x)
        u_t, v_t = _grad(u, t), _grad(v, t)
        h2 = u ** 2 + v ** 2
        f_u = u_t + 0.5 * v_xx + h2 * v       # :101
        f_v = v_t - 0.5 * u_xx - h2 * u       # :102
        return f_u, f_v, (u, v, u_x, v_x, u_t, v_t, u_xx, v_xx)

    def loss_parts(self, w: torch.Tensor):
        """loss (:107-129): mse_0 + mse_b + mse_f, eight separate means."""
        uv_pred = mlp(w, self._X0, self.layers, self._lb, self._ub)
        u0, v0 = self._uv0[:, 0:1], self._uv0[:, 1:2]
        msq = lambda a: torch.mean(torch.square(a))
        mse_0 = msq(u0 - uv_pred[:, 0:1]) + msq(v0 - uv_pred[:, 1:2])
        xl = self._X_lb[:, 0:1].clone().requires_grad_(True)
        tl = self._X_lb[:, 1:2].clone().requires_grad_(True)
        xu = self._X_ub[:, 0:1].clone().requires_grad_(True)
        tu = self._X_ub[:, 1:2].clone().requires_grad_(True)
        ul, vl, uxl, vxl = self.uvx(w, xl, tl)
        uu, vu, uxu, vxu = self.uvx(w, xu, tu)
        mse_b = msq(ul - uu) + msq(vl - vu) + msq(uxl - uxu) + msq(vxl - vxu)
        f_u, f_v, _ = self.residual(w)
        n_f = self.n_f_global or f_u.shape[0]
        mse_f = (torch.sum(torch.square(f_u)) + torch.sum(torch.square(f_v))) / n_f
        return mse_0 * self.aux_weight, mse_b * self.aux_weight, mse_f

    def loss(self, w: torch.Tensor) -> torch.Tensor:
        a, b, c = self.loss_parts(w)
        return a + b + c


@dataclass
class BurgersDiscreteInference:
    """1d-burgers/inf_disc_burgers.py:49-127.  Net [1, ..., q+1] on x only; the x-derivatives of the q stage outputs are
    obtained with the reference's two-step "dummy gradient" trick (:61-88): g = vjp(U, x; dummy), U_x = d g / d dummy --
    a reverse-over-reverse evaluation of the forward-mode derivative -- applied twice for U_xx."""
    layers: Sequence[int]
    lb: np.ndarray
    ub: np.ndarray
    nu: float
    dt: float
    x_0: np.ndarray            # (N, 1)
    u_0: np.ndarray            # (N, 1)
    x_1: np.ndarray            # (2, 1) boundary positions
    IRK_weights: np.ndarray    # (q+1, q)

    def __post_init__(self):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64))
        self._lb, self._ub = t(self.lb).reshape(-1), t(self.ub).reshape(-1)
        self._x0, self._u0, self._x1 = t(self.x_0), t(self.u_0), t(self.x_1)
        self._irk = t(self.IRK_weights)
        self.q = int(self.IRK_weights.shape[1])
        self.P = num_params(self.layers)

    def U_0_model(self, w: torch.Tensor):
        x = self._x0.clone().requires_grad_(True)
        dummy = torch.ones(x.shape[0], self.q, dtype=DT, requires_grad=True)          # :119
        U_1 = mlp(w, x, self.layers, self._lb, self._ub)                              # :68
        U = U_1[:, :-1]                                                               # :69
        g_U = torch.autograd.grad(U, x, grad_outputs=dummy, create_graph=True)[0]     # :72
        U_x = torch.autograd.grad(g_U, dummy, grad_outputs=torch.ones_like(g_U), create_graph=True)[0]      # :73
        g_U_x = torch.autograd.grad(U_x, x, grad_outputs=dummy, create_graph=True)[0]                       # :74
        U_xx = torch.autograd.grad(g_U_x, dummy, grad_outputs=torch.ones_like(g_U_x), create_graph=True)[0]  # :78
        N = U * U_x - self.nu * U_xx                                                  # :85
        return U_1 + self.dt * (N @ self._irk.T), (U_1, U_x, U_xx)                    # :86

    def loss_parts(self, w: torch.Tensor):
        U0, _ = self.U_0_model(w)
        u1 = mlp(w, self._x1, self.layers, self._lb, self._ub)                        # :99
        return torch.sum(torch.square(U0 - self._u0)), torch.sum(torch.square(u1))    # :100-101

    def loss(self, w: torch.Tensor) -> torch.Tensor:
        a, b = self.loss_parts(w)
        return a + b


@dataclass
class BurgersDiscreteIdentification:
    """1d-burgers/ide_disc_burgers.py:48-203 (discrete-time identification; SURVEY section 2 #11 -- the SCRIPT is broken as
    shipped (`Logger(frequency=10)` :225, `np.asscalar` in its prep_data branch) but the class is well defined).
    Net [1, ..., q] on x only, two snapshots: (x_0, u_0) at t_0 and (x_1, u_1) at t_1 = t_0 + dt.  Flat parameters
    w = [net, lambda_1, lambda_2].  U, U_x, U_xx of ALL q outputs by the dummy-gradient trick (:57-79);
        N    = l1 U U_x - e^{l2} U_xx                       U_0 = U + dt N alpha^T                 (:81-92)
        N'   = -l1 U U_x + e^{l2} U_xx                      U_1 = U + dt N' (beta - alpha)^T        (:94-108)
        loss = sum((U_0 - u_0)^2) + sum((U_1 - u_1)^2)      (sums over points AND stages, :111-115)."""
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
        # (self.IRK_beta - self.IRK_alpha) is NUMPY arithmetic in the reference (:107), i.e. it is rounded in the tables' own
        # dtype -- float32, burgersutil.py:92 -- before TensorFlow ever sees it
        self._beta_minus_alpha = t(np.asarray(self.IRK_beta) - np.asarray(self.IRK_alpha))
        self.q = int(self.IRK_alpha.shape[1])
        self.P = num_params(self.layers) + 2

    def autograd(self, wn: torch.Tensor, x0: torch.Tensor):
        x = x0.clone().requires_grad_(True)
        dummy = torch.ones(x.shape[0], self.q, dtype=DT, requires_grad=True)          # createDummy, :143-144
        U = mlp(wn, x, self.layers, self._lb, self._ub)                               # :66
        g_U = torch.autograd.grad(U, x, grad_outputs=dummy, create_graph=True)[0]     # :69
        U_x = torch.autograd.grad(g_U, dummy, grad_outputs=torch.ones_like(g_U), create_graph=True)[0]       # :70
        g_U_x = torch.autograd.grad(U_x, x, grad_outputs=dummy, create_graph=True)[0]                        # :71
        U_xx = torch.autograd.grad(g_U_x, dummy, grad_outputs=torch.ones_like(g_U_x), create_graph=True)[0]  # :75
        return U, U_x, U_xx

    def U_0_model(self, w: torch.Tensor, x=None):
        U, U_x, U_xx = self.autograd(w[:-2], self._x0 if x is None else x)
        l1, l2 = w[-2], torch.exp(w[-1])                                              # :88-89
        N = l1 * U * U_x - l2 * U_xx                                                  # :90
        return U + self.dt * (N @ self._alpha.T)                                      # :91

    def U_1_model(self, w: torch.Tensor, x=None):
        U, U_x, U_xx = self.autograd(w[:-2], self._x1 if x is None else x)
        l1, l2 = w[-2], torch.exp(w[-1])                                              # :104-105
        N = -l1 * U * U_x + l2 * U_xx                                                 # :106
        return U + self.dt * (N @ self._beta_minus_alpha.T)                           # :107

    def loss_parts(self, w: torch.Tensor):
        return (torch.sum(torch.square(self.U_0_model(w) - self._u0)),                # :111-115
                torch.sum(torch.square(self.U_1_model(w) - self._u1)))

    def loss(self, w: torch.Tensor) -> torch.Tensor:
        a, b = self.loss_parts(w)
        return a + b

    def predict(self, w, x_star):
        """predict (:197-202): both models on x_star with a fresh dummy."""
        wt = torch.as_tensor(np.asarray(w, dtype=np.float64))
        xs = torch.as_tensor(np.asarray(x_star, dtype=np.float64))
        return self.U_0_model(wt, xs).detach().numpy(), self.U_1_model(wt, xs).detach().numpy()


def loss_and_flat_grad(problem, w) -> Tuple[float, np.ndarray]:
    """get_loss_and_flat_grad closure (neuralnetwork.py:91-103): loss value + flat gradient in the
    trainable_variables order (== flat weight layout; identification appends d/dl1, d/dl2)."""
    wt = torch.as_tensor(np.asarray(w, dtype=np.float64)).clone().requires_grad_(True)
    loss = problem.loss(wt)
    (g,) = torch.autograd.grad(loss, wt)
    return float(loss.detach()), g.detach().numpy().copy()


def predict(problem, w, X_star) -> np.ndarray:
    """NeuralNetwork.predict (neuralnetwork.py:151-153): forward only."""
    with torch.no_grad():
        wt = torch.as_tensor(np.asarray(w, dtype=np.float64))
        return mlp(wt, torch.as_tensor(np.asarray(X_star, dtype=np.float64)), problem.layers, problem._lb, problem._ub).numpy()


# ----------------------------------------------------------------------------------------------
# Adam  (utils/neuralnetwork.py:19-22, 112-116; TF-2.0 OptimizerV2 Adam semantics, SURVEY a5)
# ----------------------------------------------------------------------------------------------
@dataclass
class AdamState:
    m: np.ndarray
    v: np.ndarray
    t: int = 0


def adam_init(P: int) -> AdamState:
    return AdamState(np.zeros(P), np.zeros(P), 0)


def adam_update(w: np.ndarray, g: np.ndarray, st: AdamState, lr: float, b1: float = 0.9, b2: float = 0.999,
                eps: Optional[float] = None, dtype=np.float64) -> np.ndarray:
    """ResourceApplyAdam: alpha_t = lr*sqrt(1-b2^t)/(1-b1^t); m += (g-m)(1-b1); v += (g^2-v)(1-b2);
    w -= alpha_t*m/(sqrt(v)+eps)   (eps outside the bias correction; eps None -> 1e-7).

    dtype=np.longdouble carries m, v, the bias correction and the update in that type (m and v are converted on first use);
    the float64 path is the reference's arithmetic, unchanged."""
    eps = TF_KERAS_EPSILON if eps is None else eps
    st.t += 1
    if dtype is np.float64:
        alpha = lr * math.sqrt(1.0 - b2 ** st.t) / (1.0 - b1 ** st.t)
        c1, c2 = 1.0 - b1, 1.0 - b2
    else:
        one, b1, b2, eps = dtype(1), dtype(b1), dtype(b2), dtype(eps)
        alpha = dtype(lr) * np.sqrt(one - b2 ** st.t) / (one - b1 ** st.t)
        c1, c2 = one - b1, one - b2
        st.m, st.v, g = st.m.astype(dtype, copy=False), st.v.astype(dtype, copy=False), np.asarray(g, dtype=dtype)
    st.m += (g - st.m) * c1
    st.v += (g * g - st.v) * c2
    return w - (st.m * alpha) / (np.sqrt(st.v) + eps)


def adam_train(problem, w0, steps, lr, b1=0.9, b2=0.999, eps=None):
    """tf_optimization (neuralnetwork.py:105-116): returns final weights, per-step losses (loss is the one
    evaluated BEFORE the step's update, as in the reference) and per-step weights."""
    w = np.array(w0, dtype=np.float64)
    st = adam_init(w.size)
    losses, ws = [], []
    for _ in range(steps):
        f, g = loss_and_flat_grad(problem, w)
        w = adam_update(w, g, st, lr, b1, b2, eps)
        losses.append(f)
        ws.append(w.copy())
    return w, np.array(losses), np.array(ws)


# ----------------------------------------------------------------------------------------------
# L-BFGS  (utils/custom_lbfgs.py:39-236)
# ----------------------------------------------------------------------------------------------
class LuaStruct(object):
    """custom_lbfgs.py:239-246: attribute bag whose missing keys read as 0."""

    def __getattr__(self, key):
        return 0


@dataclass
class LbfgsTrace:
    """Everything a parity test wants from one run (not part of the reference API)."""
    x_eval: List[np.ndarray] = field(default_factory=list)   # every x handed to opfunc (model weights)
    f_hist: List[float] = field(default_factory=list)
    d: List[np.ndarray] = field(default_factory=list)
    t: List[float] = field(default_factory=list)
    hist_len: List[int] = field(default_factory=list)
    curv: List[Tuple[float, float]] = field(default_factory=list)   # (y.s, sum |y*s|) of the pair formed at iterations >= 2
    logged: List[Tuple[int, float]] = field(default_factory=list)
    stop_reason: str = ""
    n_iter: int = 0
    n_eval: int = 0
    x_final: Optional[np.ndarray] = None


def _gram_direction(g: np.ndarray, S: List[np.ndarray], Y: List[np.ndarray], h_diag: float) -> Tuple[np.ndarray, float]:
    """d and g.d of the Gram-matrix formulation of the two-loop recursion (csrc/optim_kernels.cuh lbfgs_solve / lbfgs_apply),
    in float64 and in the kernels' association: the recurrences run in coefficient space over SY[a][b] = s_a.y_b and
    YY[a][b] = y_a.y_b (ages, 0 = oldest), then d = c_g g + sum_m (ca_m s_m + cb_m y_m) and g.d from the same coefficients.
    Mathematically the loop of lbfgs_fixed_step; the rounding differs, most where the stored pairs are nearly dependent."""
    k = len(S)
    Sm, Ym = np.array(S).reshape(k, g.size), np.array(Y).reshape(k, g.size)
    SY, YY, sg, yg = Sm @ Ym.T, Ym @ Ym.T, Sm @ g, Ym @ g
    ro = 1.0 / np.diag(SY)
    al, acc = np.zeros(k), -sg                                     # first loop, newest to oldest
    for j in range(k - 1, -1, -1):
        al[j] = acc[j] * ro[j]
        acc[:j] = acc[:j] - al[j] * SY[:j, j]
    yq = -yg                                                       # y_i.q, q = -g - sum_m al_m y_m
    for m in range(k):
        yq = yq - al[m] * YY[:, m]
    dl, acc = np.zeros(k), h_diag * yq                             # second loop, oldest to newest: dl_m = al_m - be_m
    for m in range(k):
        dl[m] = al[m] - acc[m] * ro[m]
        acc[m + 1:] = acc[m + 1:] + dl[m] * SY[m, m + 1:]
    cb = -h_diag * al
    d = -h_diag * g
    gtd = -h_diag * float(g @ g)
    for m in range(k):
        d = d + dl[m] * S[m]
        d = d + cb[m] * Y[m]
    for m in range(k):
        gtd = gtd + cb[m] * yg[m]
    for m in range(k):
        gtd = gtd + dl[m] * sg[m]
    return d, float(gtd)


class ScriptedOpfunc(object):
    """opfunc that returns recorded (f_k, g_k) in call order and ignores x: replays an optimiser on exactly the evaluations
    another implementation saw.  Calling it more often than there are records is an error; ``assert_consumed`` checks the
    replay asked for every record."""

    def __init__(self, fs: Sequence[float], gs: Sequence[np.ndarray]):
        assert len(fs) == len(gs)
        self.fs, self.gs, self.calls = list(fs), list(gs), 0

    def __call__(self, x):
        assert self.calls < len(self.fs), "replay asked for evaluation %d of %d recorded" % (self.calls + 1, len(self.fs))
        self.calls += 1
        return self.fs[self.calls - 1], self.gs[self.calls - 1]

    def assert_consumed(self):
        assert self.calls == len(self.fs), "replay used %d of %d recorded evaluations" % (self.calls, len(self.fs))


def lbfgs_fixed_step(opfunc: Callable[[np.ndarray], Tuple[float, np.ndarray]], x0: np.ndarray, max_iter: int,
                     learning_rate: float = 1.0, n_correction: int = 100, tol_fun: float = 1e-5,
                     tol_x: float = 1e-19, max_eval: Optional[float] = None, dtype=np.float64,
                     direction: str = "literal") -> Optional[LbfgsTrace]:
    """Control flow of ``lbfgs`` with ``lineSearch`` unset (the only reachable configuration; the branch at
    custom_lbfgs.py:168-171 is dead).  Quirks kept: first step t=min(1,1/|g|_1) (:159-161); fixed step
    afterwards (:163); history only pushed when y.s > 1e-10 (:103) but the two-loop always runs (:116-141);
    `ro` recomputed from history each iteration (:121-123); no opfunc call after the last update (:176-182);
    log after the stop tests (:217-221); returns None when maxIter == 0 (:43-44).

    dtype=np.longdouble computes every vector, dot product and scalar in that type (the gradients are converted exactly).
    direction="gram" (float64 only) replaces the two-loop recursion by its Gram-matrix formulation (_gram_direction)."""
    assert direction in ("literal", "gram") and (direction == "literal" or dtype is np.float64)
    if max_iter == 0:
        return None
    sc = float if dtype is np.float64 else dtype                   # scalars: Python floats on the reference's own path
    max_eval = max_eval or max_iter * 1.25                         # :49
    tr = LbfgsTrace()
    x = np.array(x0, dtype=dtype)
    f, g = opfunc(x)                                               # :65
    if dtype is not np.float64:
        g = np.asarray(g, dtype=dtype)
    tr.x_eval.append(x.copy()); tr.f_hist.append(f)
    n_eval = 1
    if np.sum(np.abs(g)) <= tol_fun:                               # :73-76
        tr.stop_reason = "initial optimality"; tr.n_eval = n_eval; tr.x_final = x
        return tr
    S: List[np.ndarray] = []   # old_dirs (holds s = d*t)
    Y: List[np.ndarray] = []   # old_stps (holds y = g - g_old)
    h_diag = sc(1.0)
    d = t = g_old = f_old = None
    n_iter = 0
    while n_iter < max_iter:                                       # :81
        n_iter += 1
        gtd = None
        if n_iter == 1:                                            # :91-95
            d = -g
        else:
            y = g - g_old                                          # :98
            s = d * t                                              # :99
            ys = sc(np.sum(y * s))                                 # :100
            tr.curv.append((ys, sc(np.sum(np.abs(y * s)))))
            if ys > 1e-10:                                         # :102-114
                if len(S) == n_correction:
                    S.pop(0); Y.pop(0)
                S.append(s); Y.append(y)
                h_diag = ys / sc(np.sum(y * y))
            k = len(S)
            if direction == "gram":
                d, gtd = _gram_direction(g, S, Y, h_diag)
            else:
                ro = [1.0 / sc(np.sum(Y[i] * S[i])) for i in range(k)]     # :121-123
                al = [0.0] * k
                q = -g                                             # :130
                for i in range(k - 1, -1, -1):                     # :131-133
                    al[i] = sc(np.sum(S[i] * q)) * ro[i]
                    q = q - al[i] * Y[i]
                r = q * h_diag                                     # :136
                for i in range(k):                                 # :137-139
                    be = sc(np.sum(Y[i] * r)) * ro[i]
                    r = r + (al[i] - be) * S[i]
                d = r
        g_old, f_old = g, f                                        # :144-145
        if gtd is None:
            gtd = sc(np.sum(g * d))                                # :151
        if gtd > -tol_x:                                           # :154-156
            tr.stop_reason = "no progress along direction"
            break
        t = min(1.0, 1.0 / sc(np.sum(np.abs(g)))) if n_iter == 1 else learning_rate    # :159-163
        x = x + t * d                                              # :174
        tr.d.append(d.copy()); tr.t.append(t); tr.hist_len.append(len(S))
        if n_iter != max_iter:                                     # :176-182
            f, g = opfunc(x)
            if dtype is not np.float64:
                g = np.asarray(g, dtype=dtype)
            n_eval += 1
            tr.x_eval.append(x.copy()); tr.f_hist.append(f)
        if n_iter == max_iter:                                     # :192
            tr.stop_reason = "max iterations"
            break
        if n_eval >= max_eval:                                     # :195
            tr.stop_reason = "max evaluations"
            break
        if np.sum(np.abs(g)) <= tol_fun:                           # :200-204
            tr.stop_reason = "optimality"
            break
        if np.sum(np.abs(d * t)) <= tol_x:                         # :206-210
            tr.stop_reason = "step below tolX"
            break
        if abs(f - f_old) < tol_x:                                 # :212-215
            tr.stop_reason = "f change below tolX"
            break
        tr.logged.append((n_iter, f))                              # :217-218
    tr.n_iter, tr.n_eval, tr.x_final = n_iter, n_eval, x
    return tr
