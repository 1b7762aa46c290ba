"""L-BFGS entry point with the reference's surface (utils/custom_lbfgs.py), backed by the device-resident
two-loop kernel (pinn_lbfgs in include/pinn_b200.h).

``lbfgs(opfunc, x, config, state, do_verbose, log_fn)`` keeps the reference signature and return values
(custom_lbfgs.py:39-44,76,236).  When ``opfunc`` is the closure returned by ``NeuralNetwork.get_loss_and_flat_grad`` the
whole iteration (evaluation, history update, two-loop recursion, fixed step, stop tests) runs on the GPU with one status
read-back per ``sync_every`` iterations instead of the reference's >= 6 host syncs per iteration.  Any OTHER closure is
called once per iteration, as in the reference, while the optimiser state stays on the device (``_run_foreign``).
There is deliberately no host (CPU) implementation of the optimiser arithmetic.
"""
import time

import numpy as np

import pinn_cabi

# ---- wall-time bookkeeping (custom_lbfgs.py:8-28)
global_time_list = []
global_last_time = 0


def reset_time():
    global global_time_list, global_last_time
    global_time_list = []
    global_last_time = time.perf_counter()


def record_time():
    global global_last_time, global_time_list
    new_time = time.perf_counter()
    global_time_list.append(new_time - global_last_time)
    global_last_time = time.perf_counter()


def last_time():
    """Last recorded interval in milliseconds."""
    return 1000 * global_time_list[-1] if global_time_list else 0


def dot(a, b):
    """custom_lbfgs.py:30-32 (host arrays; the training path computes its dot products on the device)."""
    return np.sum(np.asarray(a) * np.asarray(b))


final_loss = None
times = []


class dummy(object):
    pass


class Struct(dummy):
    """Lua-like struct: missing attributes read as 0 (custom_lbfgs.py:239-246)."""

    def __getattribute__(self, key):
        if key == "__dict__":
            return super(dummy, self).__getattribute__("__dict__")
        return self.__dict__.get(key, 0)


def _run_coupled(net, x, config, max_iter, opts, on_logged):
    """The closure of NeuralNetwork.get_loss_and_flat_grad: evaluations and iterations both run on the device, with one
    status read-back per ``sync_every`` iterations."""
    sync_every = int(config.syncEvery or getattr(getattr(net, "logger", None), "frequency", 1) or 1)
    net.set_weights(x)
    logged = []

    def _cb(it, f):
        logged.append((it, f))
        on_logged(it, f)

    res = net._native().lbfgs(max_iter, sync_every=max(1, sync_every), log_fn=_cb, want_x_final=True, **opts)
    f_hist = res.get("f_hist", [f for _, f in logged])
    return net._as_tensor(res["x_final"]), f_hist, res["n_iter"], res["n_eval"], res["reason"]


def _run_foreign(opfunc, x, config, max_iter, opts, on_logged):
    """Any closure x -> (f, g) (custom_lbfgs.py:39): the objective is evaluated by the caller's code, one call per iteration
    exactly where the reference calls it (:65, :178), while the iterate, the (s, y) history and the two-loop recursion stay
    on the device (pinn_lbfgs_create / pinn_lbfgs_feed -- the same kernels as the coupled path).  x is handed to opfunc
    as a float64 array with .numpy(); f and g may be anything np.asarray() understands."""
    from neuralnetwork import _t
    x0 = np.asarray(x.numpy() if hasattr(x, "numpy") else x, dtype=np.float64).reshape(-1)
    opt = pinn_cabi.Lbfgs(x0, max_iter, max_eval=float(config.maxEval or 0.0), **opts)
    try:
        xk = x0
        while True:
            f, g = opfunc(_t(xk))
            f = float(np.asarray(f.numpy() if hasattr(f, "numpy") else f).reshape(-1)[0])
            g = np.asarray(g.numpy() if hasattr(g, "numpy") else g, dtype=np.float64).reshape(-1)
            xk, status, n_iter, n_eval, logged_it, logged_f = opt.feed(f, g)
            if logged_it is not None:
                on_logged(logged_it, logged_f)
            if status != 0:
                break
        f_hist = opt.f_hist()
    finally:
        opt.close()
    return _t(xk), f_hist, n_iter, n_eval, status


def lbfgs(opfunc, x, config, state, do_verbose, log_fn):
    """Device-resident port of the reference control flow.  Returns None when maxIter == 0, ``(x, f_hist)`` when
    the initial point is already optimal, else ``(x, f_hist, currentFuncEval)``."""
    global times
    if config.maxIter == 0:
        return
    if config.lineSearch:
        raise NotImplementedError("lineSearch is dead code in the reference (custom_lbfgs.py:168-171) and is not provided")
    max_iter = int(config.maxIter)
    opts = dict(learning_rate=float(config.learningRate or 1), n_correction=int(config.nCorrection or 100),
                tol_fun=float(config.tolFun or 1e-5), tol_x=float(config.tolX or 1e-19))
    times = []

    def on_logged(it, f):
        global final_loss
        if do_verbose:
            log_fn(it, np.float64(f), True)
            record_time()
            times.append(last_time())
        if it == max_iter - 1:
            final_loss = np.float64(f)

    net = getattr(opfunc, "_pinn_net", None)
    if net is not None:
        x_out, f_hist, n_iter, n_eval, reason = _run_coupled(net, x, config, max_iter, opts, on_logged)
    else:
        x_out, f_hist, n_iter, n_eval, reason = _run_foreign(opfunc, x, config, max_iter, opts, on_logged)
    state.funcEval = state.funcEval + n_eval
    state.nIter = state.nIter + n_iter
    state.stop_reason = pinn_cabi.LBFGS_REASONS.get(reason, "?")
    if reason == 7:             # initial optimality (custom_lbfgs.py:73-76)
        return x_out, f_hist
    return x_out, f_hist, n_eval
