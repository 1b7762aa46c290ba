"""ctypes binding of libpinn_b200.so (include/pinn_b200.h).

This is the only way the Python surface (neuralnetwork.py / custom_lbfgs.py) reaches the GPU.  There is
no CPU fallback: loading fails loudly when the library is missing, and ``pinn_create`` fails loudly when
there is no sm_90 (H100) device.
"""
import ctypes as C
import os

import numpy as np

from sharding import shard_rows

_HERE = os.path.dirname(os.path.realpath(__file__))
# PINN_LIB: load another build of the same library (kernel experiments: profiles/kernel_variants.py)
LIB_PATH = os.environ.get("PINN_LIB") or os.path.join(_HERE, "..", "lib", "libpinn_b200.so")

BURGERS_INF, BURGERS_IDE, NLS_INF, BURGERS_DISC, BURGERS_IDE_DISC, KDV_IDE_DISC, AC_DISC, NS_IDE = 0, 1, 2, 3, 4, 5, 6, 7
# user-defined polynomial residual (Pinn.set_residual) with the loss structure of BURGERS_INF / BURGERS_IDE
POLY_INF, POLY_IDE = 8, 9
# kappa_k of a polynomial residual term, in the order of pinn_set_residual's kind
POLY_KINDS = ("1", "l1", "l2", "exp(l1)", "exp(l2)")
# X_k and T_k of a source-table term, in the order of pinn_set_source_terms' kinds
SOURCE_KINDS = ("1", "sin", "cos")
SOURCE_MAXT = 16
# Navier-Stokes derivative streams, in the order of pinn_derivatives' blocks
NS_STREAMS = ("u", "x", "y", "t", "xx", "xy", "yy", "xt", "yt", "xxx", "xxy", "xyy", "yyy")
LBFGS_REASONS = {0: "running", 1: "max iterations", 2: "max evaluations", 3: "optimality", 4: "step below tolX",
                 5: "f change below tolX", 6: "no progress along direction", 7: "initial optimality"}

_dp = C.POINTER(C.c_double)
LOG_CB = C.CFUNCTYPE(None, C.c_int, C.c_double, C.c_void_p)

# every symbol include/pinn_b200.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "pinn_last_error": (C.c_char_p, []),
    "pinn_version": (C.c_char_p, []),
    "pinn_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(C.c_int), _dp, _dp, C.c_int, C.c_int,
                              C.c_int, C.c_void_p]),
    "pinn_destroy": (C.c_int, [C.c_void_p]),
    "pinn_nccl_unique_id": (C.c_int, [C.c_void_p]),
    "pinn_p2p_export": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pinn_p2p_connect": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "pinn_p2p_enable": (C.c_int, [C.c_void_p, C.c_int]),
    "pinn_num_params": (C.c_int64, [C.c_void_p]),
    "pinn_set_pde_params": (C.c_int, [C.c_void_p, _dp, C.c_int]),
    "pinn_get_params": (C.c_int, [C.c_void_p, _dp, C.c_int]),
    "pinn_set_irk": (C.c_int, [C.c_void_p, _dp, C.c_int]),
    "pinn_set_collocation": (C.c_int, [C.c_void_p, _dp, _dp, C.c_int64, C.c_int64]),
    "pinn_set_collocation_mapped": (C.c_int, [C.c_void_p, _dp, _dp, C.c_int64, C.c_int64]),
    "pinn_draw_collocation": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_int64, C.c_int64, C.c_int64]),
    "pinn_draw_collocation_rad": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_int64, C.c_int64, C.c_int, C.c_double]),
    "pinn_get_collocation": (C.c_int, [C.c_void_p, _dp, _dp, C.c_int64]),
    "pinn_set_data": (C.c_int, [C.c_void_p, _dp, C.c_int64, C.c_int, _dp, C.c_int, C.c_double]),
    "pinn_set_snapshot": (C.c_int, [C.c_void_p, C.c_int, _dp, C.c_int64, _dp]),
    "pinn_set_boundary": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pinn_set_residual": (C.c_int, [C.c_void_p, C.c_int, _dp, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "pinn_set_source": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pinn_set_source_terms": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), _dp]),
    "pinn_get_source": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pinn_set_weights": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pinn_get_weights": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pinn_loss_grad": (C.c_int, [C.c_void_p, _dp, _dp, _dp, _dp]),
    "pinn_adam_step": (C.c_int, [C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_double, _dp]),
    "pinn_adam_steps": (C.c_int, [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double]),
    "pinn_adam_reset": (C.c_int, [C.c_void_p]),
    "pinn_last_loss": (C.c_int, [C.c_void_p, _dp]),
    "pinn_lbfgs": (C.c_int, [C.c_void_p, C.c_int, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int, LOG_CB, C.c_void_p,
                             C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), _dp]),
    "pinn_lbfgs_history": (C.c_int, [C.c_void_p, _dp, C.c_int, C.POINTER(C.c_int)]),
    "pinn_lbfgs_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_int64, _dp, C.c_int, C.c_double, C.c_int, C.c_double, C.c_double,
                                    C.c_double]),
    "pinn_lbfgs_feed": (C.c_int, [C.c_void_p, C.c_double, _dp, _dp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                  C.POINTER(C.c_int), _dp]),
    "pinn_lbfgs_f_hist": (C.c_int, [C.c_void_p, _dp, C.c_int, C.POINTER(C.c_int)]),
    "pinn_lbfgs_destroy": (C.c_int, [C.c_void_p]),
    "pinn_predict": (C.c_int, [C.c_void_p, _dp, C.c_int64, C.c_int, _dp]),
    "pinn_num_residual_points": (C.c_int64, [C.c_void_p]),
    "pinn_residual": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pinn_derivatives": (C.c_int, [C.c_void_p, _dp, C.c_int64, _dp]),
    "pinn_sync": (C.c_int, [C.c_void_p]),
    "pinn_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_int64]),
    "pinn_host_free": (C.c_int, [C.c_void_p]),
    "pinn_time_loss_grad_kernel": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_float)]),
    "pinn_launch_count": (C.c_int64, [C.c_void_p]),
    "pinn_event_record": (C.c_int, [C.c_void_p, C.c_int]),
    "pinn_event_elapsed_ms": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float)]),
    "pinn_flush_l2": (C.c_int, [C.c_void_p]),
    "pinn_test_tanh": (C.c_int, [_dp, C.c_int, _dp]),
    "pinn_kernel_info": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
}

_lib = None


class PinnError(RuntimeError):
    pass


def load():
    """Load the shared library (once).  No fallback: a missing library is a hard error."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.path.abspath(LIB_PATH)
    if not os.path.exists(path):
        raise PinnError(f"{path} not found: build it with `python pinns-tf2.0_b200/build.py` "
                        "(there is no CPU fallback for the PINN training core)")
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)       # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def _arr(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64))


def _p(a):
    return a.ctypes.data_as(_dp)


class Pinn(object):
    """Thin object wrapper over a ``pinn_t*`` handle."""

    def __init__(self, pde, layers, lb, ub, device=0, rank=0, world=1, nccl_uid=None):
        self.lib = load()
        self.h = C.c_void_p()
        L = (C.c_int * len(layers))(*[int(v) for v in layers])
        self._lb, self._ub = _arr(lb).reshape(-1), _arr(ub).reshape(-1)
        if self._lb.size == 1:               # 1-D models (discrete time): the ABI takes lb[2], ub[2]
            self._lb, self._ub = np.array([self._lb[0], 0.0]), np.array([self._ub[0], 1.0])
        uid = None
        if nccl_uid is not None:
            self._uid = C.create_string_buffer(bytes(nccl_uid), 128)
            uid = C.cast(self._uid, C.c_void_p)
        self._ck(self.lib.pinn_create(C.byref(self.h), int(pde), len(layers), L, _p(self._lb), _p(self._ub), int(device),
                                      int(rank), int(world), uid))
        self.pde = int(pde)
        self.layers = [int(v) for v in layers]
        self.P = int(self.lib.pinn_num_params(self.h))
        self.out_dim = self.layers[-1]
        self._keep = []

    def _ck(self, rc):
        if rc != 0:
            raise PinnError(self.lib.pinn_last_error().decode())

    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            self.lib.pinn_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- fused NVLink P2P exchange (multi-GPU)
    def p2p_export(self):
        buf = C.create_string_buffer(64)
        self._ck(self.lib.pinn_p2p_export(self.h, C.cast(buf, C.c_void_p)))
        return buf.raw

    def p2p_connect(self, handles):
        blob = b"".join(handles)
        buf = C.create_string_buffer(blob, len(blob))
        self._ck(self.lib.pinn_p2p_connect(self.h, C.cast(buf, C.c_void_p), len(handles)))

    def p2p_enable(self, on):
        self._ck(self.lib.pinn_p2p_enable(self.h, 1 if on else 0))

    # ---- problem definition
    def set_pde_params(self, params):
        a = _arr(params).reshape(-1)
        self._ck(self.lib.pinn_set_pde_params(self.h, _p(a), a.size))

    def get_params(self):
        n = {BURGERS_INF: 1, BURGERS_IDE: 2, NLS_INF: 0, BURGERS_DISC: 2, BURGERS_IDE_DISC: 2, KDV_IDE_DISC: 2, AC_DISC: 3,
             NS_IDE: 2, POLY_INF: 0, POLY_IDE: 2}[self.pde]
        out = np.zeros(max(n, 1))
        self._ck(self.lib.pinn_get_params(self.h, _p(out), n))
        return out[:n]

    def set_irk(self, irk):
        """BURGERS_DISC, AC_DISC: (q+1, q) stage matrix.  BURGERS_IDE_DISC, KDV_IDE_DISC: (2q, q) = [alpha ; -(beta - alpha)]
        (see irk_ide_disc)."""
        irk = _arr(irk)
        assert irk.ndim == 2 and irk.shape[0] in (irk.shape[1] + 1, 2 * irk.shape[1])
        self._ck(self.lib.pinn_set_irk(self.h, _p(irk), irk.shape[1]))

    def set_snapshot(self, which, x, u):
        x, u = _arr(x).reshape(-1), _arr(u).reshape(-1)
        assert x.size == u.size
        self._ck(self.lib.pinn_set_snapshot(self.h, int(which), _p(x), x.size, _p(u)))

    def set_collocation(self, x, t, n_global=None):
        x, t = _arr(x).reshape(-1), _arr(t).reshape(-1)
        assert x.size == t.size
        self._ck(self.lib.pinn_set_collocation(self.h, _p(x), _p(t), x.size, int(n_global or x.size)))

    def set_collocation_ptr(self, x_ptr, t_ptr, n, n_global=None):
        """Raw-pointer variant (pinned host buffers from host_alloc)."""
        self._ck(self.lib.pinn_set_collocation(self.h, x_ptr, t_ptr, int(n), int(n_global or n)))

    def set_collocation_mapped(self, x_ptr, t_ptr, n, n_global=None):
        """Zero-copy: the fused kernel reads the (pinned) host buffers directly; keep them alive and unchanged."""
        self._ck(self.lib.pinn_set_collocation_mapped(self.h, x_ptr, t_ptr, int(n), int(n_global or n)))

    def draw_collocation(self, seed, draw, n_global, rank=0, world=1):
        """Replace the collocation set by this rank's rows (sharding.shard_rows) of Latin-hypercube draw `draw` of `seed`, with
        n_global strata per dimension over [lb, ub] (pinn_draw_collocation).  Enqueued on the device; nothing is synchronised."""
        for name, v in (("seed", seed), ("draw", draw)):
            if not 0 <= int(v) < 1 << 64:
                raise PinnError(f"draw_collocation: {name} = {int(v)} is not an unsigned 64-bit integer")
        first, hi = shard_rows(int(n_global), int(rank), int(world))
        self._ck(self.lib.pinn_draw_collocation(self.h, int(seed), int(draw), first, hi - first, int(n_global)))

    def draw_collocation_rad(self, seed, draw, n, n_pool, k=1, c=1.0):
        """Replace the collocation set by n points drawn with replacement from Latin-hypercube draw `draw` of `seed` with n_pool
        points, with probability ~ |f|^k / mean |f|^k + c at the current weights (residual-based adaptive resampling,
        pinn_draw_collocation_rad).  Enqueued on the device; nothing is synchronised."""
        for name, v in (("seed", seed), ("draw", draw)):
            if not 0 <= int(v) < 1 << 64:
                raise PinnError(f"draw_collocation_rad: {name} = {int(v)} is not an unsigned 64-bit integer")
        self._ck(self.lib.pinn_draw_collocation_rad(self.h, int(seed), int(draw), int(n_pool), int(n), int(k), float(c)))

    def get_collocation(self):
        """(x, t) of the stored collocation set, however it got there (upload, mapped batch, draw)."""
        n = int(self.lib.pinn_num_residual_points(self.h))
        x, t = np.empty(n), np.empty(n)
        self._ck(self.lib.pinn_get_collocation(self.h, _p(x), _p(t), n))
        return x, t

    def set_data(self, X, u, weight=1.0):
        X, u = _arr(X), _arr(u)
        if X.ndim == 1:
            X = X[:, None]
        if u.ndim == 1:
            u = u[:, None]
        self._ck(self.lib.pinn_set_data(self.h, _p(X), X.shape[0], X.shape[1], _p(u), u.shape[1], float(weight)))

    def set_boundary(self, tb):
        tb = _arr(tb).reshape(-1)
        self._ck(self.lib.pinn_set_boundary(self.h, _p(tb), tb.size))

    def set_residual(self, terms):
        """POLY_INF / POLY_IDE: terms = [(coef, kind, (e_u, e_ux, e_ut, e_uxx)), ...], 1 to 16 of them; kind 0..4 selects
        kappa = 1, l1, l2, exp(l1), exp(l2) (POLY_KINDS)."""
        terms = list(terms)
        n = len(terms)
        coef = _arr([float(c) for c, _, _ in terms] or [0.0])
        kind = (C.c_int * max(n, 1))(*[int(k) for _, k, _ in terms])
        exps = (C.c_int * max(4 * n, 1))(*[int(e) for _, _, es in terms for e in es])
        if any(len(es) != 4 for _, _, es in terms):
            raise PinnError("set_residual: each term needs four exponents (u, u_x, u_t, u_xx)")
        self._ck(self.lib.pinn_set_residual(self.h, n, _p(coef), kind, exps))

    def set_source(self, s):
        """POLY_INF / POLY_IDE: the source s at the stored residual points (reset to 0 whenever new residual points are set)."""
        s = _arr(s).reshape(-1)
        self._ck(self.lib.pinn_set_source(self.h, _p(s), s.size))

    def set_source_terms(self, terms):
        """POLY_INF / POLY_IDE: the source as a table the device evaluates at every new set of residual points (see
        pack_source_terms); an empty table removes the source."""
        form, par = pack_source_terms(terms)
        fp = form.ctypes.data_as(C.POINTER(C.c_int))
        self._ck(self.lib.pinn_set_source_terms(self.h, len(form), fp, _p(par)))

    def get_source(self):
        """The stored source at the residual points, however it was formed (array, table, or zeros without a source)."""
        s = np.empty(int(self.lib.pinn_num_residual_points(self.h)))
        self._ck(self.lib.pinn_get_source(self.h, _p(s), s.size))
        return s

    # ---- parameters
    def set_weights(self, w):
        w = _arr(w).reshape(-1)
        self._ck(self.lib.pinn_set_weights(self.h, _p(w), w.size))

    def get_weights(self):
        w = np.empty(self.P)
        self._ck(self.lib.pinn_get_weights(self.h, _p(w), w.size))
        return w

    # ---- hot path
    def loss_grad(self, w=None, want_grad=True):
        loss = C.c_double()
        g = np.empty(self.P) if want_grad else None
        parts = np.empty(3)
        wa = _arr(w).reshape(-1) if w is not None else None
        if wa is not None and wa.size != self.P:
            raise PinnError(f"expected {self.P} weights, got {wa.size}")
        self._ck(self.lib.pinn_loss_grad(self.h, _p(wa) if wa is not None else None, C.byref(loss),
                                         _p(g) if g is not None else None, _p(parts)))
        return loss.value, g, parts

    def adam_step(self, lr, b1=0.9, b2=0.999, eps=1e-7, sync=True):
        if sync:
            loss = C.c_double()
            self._ck(self.lib.pinn_adam_step(self.h, lr, b1, b2, eps, C.byref(loss)))
            return loss.value
        self._ck(self.lib.pinn_adam_step(self.h, lr, b1, b2, eps, None))
        return None

    def adam_steps(self, n, lr, b1=0.9, b2=0.999, eps=1e-7):
        """n asynchronous Adam steps enqueued by one native call (no per-step binding overhead)."""
        self._ck(self.lib.pinn_adam_steps(self.h, int(n), lr, b1, b2, eps))

    def adam_reset(self):
        self._ck(self.lib.pinn_adam_reset(self.h))

    def last_loss(self):
        loss = C.c_double()
        self._ck(self.lib.pinn_last_loss(self.h, C.byref(loss)))
        return loss.value

    def lbfgs(self, max_iter, learning_rate=1.0, n_correction=100, tol_fun=1e-5, tol_x=1e-19, sync_every=1, log_fn=None,
              want_x_final=False):
        n_it, n_ev, reason = C.c_int(), C.c_int(), C.c_int()
        xf = np.empty(self.P) if want_x_final else None
        cb = LOG_CB((lambda it, f, ud: log_fn(it, f)) if log_fn else (lambda it, f, ud: None))
        self._ck(self.lib.pinn_lbfgs(self.h, int(max_iter), float(learning_rate), int(n_correction), float(tol_fun),
                                     float(tol_x), int(sync_every), cb, None, C.byref(n_it), C.byref(n_ev), C.byref(reason),
                                     _p(xf) if xf is not None else None))
        nh = C.c_int()
        self._ck(self.lib.pinn_lbfgs_history(self.h, None, 0, C.byref(nh)))
        fh = np.empty(max(nh.value, 1))
        self._ck(self.lib.pinn_lbfgs_history(self.h, _p(fh), fh.size, C.byref(nh)))
        return {"n_iter": n_it.value, "n_eval": n_ev.value, "reason": reason.value,
                "reason_str": LBFGS_REASONS.get(reason.value, "?"), "x_final": xf, "f_hist": [float(v) for v in fh[:nh.value]]}

    # ---- off-path
    def predict(self, X):
        X = _arr(X)
        if X.ndim == 1:
            X = X[:, None]
        out = np.empty((X.shape[0], self.out_dim))
        self._ck(self.lib.pinn_predict(self.h, _p(X), X.shape[0], X.shape[1], _p(out)))
        return out

    def derivatives(self, X):
        """(u, u_x, u_t, u_xx), each (n, out_dim).  NS_IDE: one (n, 13, 2) array, the streams of NS_STREAMS, each (psi, p)."""
        X = _arr(X)
        if X.ndim == 1:
            X = X[:, None]
        if X.shape[1] == 1 and self.layers[0] == 2:
            X = np.concatenate([X, X], axis=1)      # quirk Q1, as predict: an (n, 1) input is (x, t := x)
        if X.shape[1] != self.layers[0]:
            raise PinnError(f"derivatives: X has {X.shape[1]} columns, the net takes {self.layers[0]}")
        X = np.ascontiguousarray(X)
        if self.pde == NS_IDE:
            out = np.empty((X.shape[0], len(NS_STREAMS), 2))
            self._ck(self.lib.pinn_derivatives(self.h, _p(X), X.shape[0], _p(out)))
            return out
        out = np.empty((X.shape[0], 4, self.out_dim))
        self._ck(self.lib.pinn_derivatives(self.h, _p(X), X.shape[0], _p(out)))
        return out[:, 0], out[:, 1], out[:, 2], out[:, 3]

    def residual(self, n=None):
        """f_model on the stored residual points.  The buffer is sized from the count the handle holds; a caller-supplied
        `n` is only checked against it."""
        nres = 2 if self.pde in (NLS_INF, NS_IDE) else 1
        stored = int(self.lib.pinn_num_residual_points(self.h))
        if n is not None and int(n) != stored:
            raise PinnError(f"residual: {stored} residual points are stored, caller expected {int(n)}")
        out = np.empty((stored, nres))
        self._ck(self.lib.pinn_residual(self.h, _p(out), stored))
        return out

    def sync(self):
        self._ck(self.lib.pinn_sync(self.h))

    # ---- measurement
    def time_kernel_ms(self, iters):
        ms = C.c_float()
        self._ck(self.lib.pinn_time_loss_grad_kernel(self.h, int(iters), C.byref(ms)))
        return ms.value

    def event_record(self, idx):
        self._ck(self.lib.pinn_event_record(self.h, int(idx)))

    def event_elapsed_ms(self, i, j):
        ms = C.c_float()
        self._ck(self.lib.pinn_event_elapsed_ms(self.h, int(i), int(j), C.byref(ms)))
        return ms.value

    def flush_l2(self):
        self._ck(self.lib.pinn_flush_l2(self.h))

    def launch_count(self):
        return int(self.lib.pinn_launch_count(self.h))

    def kernel_info(self):
        import json
        buf = C.create_string_buffer(512)
        self._ck(self.lib.pinn_kernel_info(self.h, buf, 512))
        return json.loads(buf.value.decode())


class Lbfgs(object):
    """Stand-alone device-resident L-BFGS (pinn_lbfgs_create / _feed): any objective, evaluated by the caller."""

    def __init__(self, x0, max_iter, learning_rate=1.0, n_correction=100, tol_fun=1e-5, tol_x=1e-19, max_eval=0.0, device=0):
        self.lib = load()
        self.h = C.c_void_p()
        x0 = _arr(x0).reshape(-1)
        self.n = x0.size
        if self.lib.pinn_lbfgs_create(C.byref(self.h), int(device), self.n, _p(x0), int(max_iter), float(learning_rate),
                                      int(n_correction), float(tol_fun), float(tol_x), float(max_eval)) != 0:
            raise PinnError(self.lib.pinn_last_error().decode())

    def feed(self, f, g):
        """-> (x_next, status, n_iter, n_eval, logged_iter or None, logged_f)."""
        g = _arr(g).reshape(-1)
        if g.size != self.n:
            raise PinnError(f"lbfgs: gradient has {g.size} entries, x has {self.n}")
        x = np.empty(self.n)
        st, it, ev, li = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        lf = C.c_double()
        if self.lib.pinn_lbfgs_feed(self.h, float(f), _p(g), _p(x), C.byref(st), C.byref(it), C.byref(ev), C.byref(li),
                                    C.byref(lf)) != 0:
            raise PinnError(self.lib.pinn_last_error().decode())
        return x, st.value, it.value, ev.value, (li.value if li.value >= 0 else None), lf.value

    def f_hist(self):
        n = C.c_int()
        if self.lib.pinn_lbfgs_f_hist(self.h, None, 0, C.byref(n)) != 0:
            raise PinnError(self.lib.pinn_last_error().decode())
        out = np.empty(max(n.value, 1))
        if self.lib.pinn_lbfgs_f_hist(self.h, _p(out), out.size, C.byref(n)) != 0:
            raise PinnError(self.lib.pinn_last_error().decode())
        return [float(v) for v in out[:n.value]]

    def close(self):
        if getattr(self, "h", None):
            self.lib.pinn_lbfgs_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def pack_source_terms(terms):
    """Source-table terms (a, p, q, xkind, omega, phi, tkind, nu, psi, alpha, gamma, beta, delta) -> (form, par) of
    pinn_set_source_terms, with its checks: at most 16 terms, p and q in 0..3, kinds in 0..2 (SOURCE_KINDS), every parameter
    finite."""
    terms = [tuple(t) for t in terms]
    if len(terms) > SOURCE_MAXT:
        raise PinnError(f"set_source_terms: {len(terms)} terms; at most {SOURCE_MAXT} are supported")
    form = np.zeros(max(len(terms), 1), dtype=np.intc)
    par = np.zeros((max(len(terms), 1), 9))
    for k, t in enumerate(terms):
        if len(t) != 13:
            raise PinnError(f"set_source_terms: term {k} has {len(t)} entries, expected 13 "
                            "(a, p, q, xkind, omega, phi, tkind, nu, psi, alpha, gamma, beta, delta)")
        a, p, q, xk, om, ph, tk, nu, ps, al, ga, be, de = t
        for name, v, hi in (("p", p, 3), ("q", q, 3), ("xkind", xk, 2), ("tkind", tk, 2)):
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or not 0 <= v <= hi:
                raise PinnError(f"set_source_terms: term {k}: {name} = {v!r} is outside 0..{hi}")
        for name, v in zip(("a", "omega", "phi", "nu", "psi", "alpha", "gamma", "beta", "delta"), (a, om, ph, nu, ps, al, ga, be, de)):
            if not np.isfinite(float(v)):
                raise PinnError(f"set_source_terms: term {k}: parameter {name} is not finite")
        form[k] = int(p) | int(q) << 2 | int(xk) << 4 | int(tk) << 6
        par[k] = (a, om, ph, nu, ps, al, ga, be, de)
    return form[:len(terms)], par[:len(terms)]


def irk_ide_disc(IRK_alpha, IRK_beta):
    """Stage matrices of the discrete-time identification model for pinn_set_irk: [alpha ; -(beta - alpha)].  The difference is
    formed in the arrays' OWN dtype (float32 tables in the reference, 1d-burgers/burgersutil.py:92, ide_disc_burgers.py:107)
    before the conversion to float64 -- a float64 difference differs at the 1e-10 level."""
    a, b = np.asarray(IRK_alpha), np.asarray(IRK_beta)
    return np.concatenate([a.astype(np.float64), -(b - a).astype(np.float64)], 0)


def device_tanh(x):
    lib = load()
    x = _arr(x).reshape(-1)
    y = np.empty_like(x)
    if lib.pinn_test_tanh(_p(x), x.size, _p(y)) != 0:
        raise PinnError(lib.pinn_last_error().decode())
    return y


def nccl_unique_id():
    lib = load()
    buf = C.create_string_buffer(128)
    if lib.pinn_nccl_unique_id(C.cast(buf, C.c_void_p)) != 0:
        raise PinnError(lib.pinn_last_error().decode())
    return buf.raw


def host_alloc(n_doubles):
    """Pinned host array of n float64 (cudaHostAlloc).  Returns (ndarray view, raw pointer)."""
    lib = load()
    p = C.c_void_p()
    if lib.pinn_host_alloc(C.byref(p), int(n_doubles) * 8) != 0:
        raise PinnError(lib.pinn_last_error().decode())
    arr = np.ctypeslib.as_array(C.cast(p, _dp), shape=(int(n_doubles),))
    return arr, p
