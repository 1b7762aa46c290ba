"""``NeuralNetwork`` with the reference's Python surface (utils/neuralnetwork.py:7-159) on the H100-native core.

The reference expresses each PDE as ``tf.GradientTape`` code in ``loss``/``f_model`` overrides; here the PDE is
*recognised* (class attribute ``pde`` or the attributes the reference subclasses set: ``lambda_1`` ->
identification, ``X_lb`` -> Schrodinger, ``x_f``+``nu`` -> Burgers inference) and evaluated by ONE fused sm_90a
kernel through the C ABI (include/pinn_b200.h).  Subclass ``loss``/``f_model``/``uvx_model`` bodies written against
TensorFlow are replaced at class-creation time by native equivalents, so the reference scripts' class
definitions load unchanged.  Everything is float64, as in the reference (:24-26).  No CPU fallback exists.
"""
import numpy as np

import pinn_cabi
import poly_spec
from custom_lbfgs import Struct, lbfgs


class Tensor(np.ndarray):
    """Host fp64 array with the few EagerTensor affordances the scripts use (``.numpy()``, slicing)."""

    def numpy(self):
        return np.asarray(self)


def _t(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(Tensor)


class LazyLoss(object):
    """Loss of one asynchronous Adam step; fetched from the device only when formatted/converted.  The device keeps the loss of
    the LATEST step only, so the value must be taken (float(), format, .numpy()) before the next step is enqueued -- which is
    what the reference's loop does (it logs each epoch's loss before the next epoch).  Asking later is an error, not a silently
    wrong number."""

    def __init__(self, native, owner=None):
        self._n, self._v, self._owner = native, None, owner
        self._serial = getattr(owner, "_adam_serial", 0)

    def numpy(self):
        if self._v is None:
            if self._owner is not None and self._owner._adam_serial != self._serial:
                raise RuntimeError("this loss belongs to an earlier asynchronous training step and was never read; convert it "
                                   "(float(loss)) before calling tf_optimization_step again")
            self._v = np.float64(self._n.last_loss())
        return self._v

    def __float__(self):
        return float(self.numpy())

    def __format__(self, spec):
        return format(float(self), spec)

    def __repr__(self):
        return repr(float(self))


class _Model(object):
    """Stand-in for the Keras ``Sequential`` (neuralnetwork.py:27-37): callable on (N,in) arrays."""

    def __init__(self, net):
        self._net = net

    def __call__(self, X):
        return _t(self._net._native().predict(np.asarray(X, dtype=np.float64)))

    def summary(self):
        L = self._net.layers
        lines = ["Lambda 2(X-lb)/(ub-lb)-1"] + [f"Dense {L[i]}->{L[i+1]} {'tanh' if i < len(L) - 2 else 'linear'}"
                                                for i in range(len(L) - 1)]
        return "\n".join(lines) + f"\nTotal params: {self._net._n_net_params()}"

    @property
    def trainable_variables(self):
        return self._net._unflatten(self._net._native().get_weights()[: self._net._n_net_params()])


def _glorot_normal(layers, rng):
    """Keras glorot_normal look-alike (neuralnetwork.py:33,37): truncated N(0, s) at 2s, s = sqrt(2/(fi+fo))/.8796."""
    out = []
    for fi, fo in zip(layers[:-1], layers[1:]):
        std = np.sqrt(2.0 / (fi + fo)) / 0.87962566103423978
        W = rng.standard_normal((fi, fo))
        bad = np.abs(W) > 2.0
        while bad.any():
            W[bad] = rng.standard_normal(int(bad.sum()))
            bad = np.abs(W) > 2.0
        out += [(W * std).reshape(-1), np.zeros(fo)]
    return np.concatenate(out)


_NATIVE_OVERRIDES = {}


class NeuralNetwork(object):
    pde = None           # optional explicit PDE id: "burgers_inf" | "burgers_ide" | "nls_inf" | "burgers_disc" | "burgers_ide_disc"
    #                      | "kdv_ide_disc" | "ac_disc" | "ns_ide" | "poly" (the last four are never guessed from attributes)
    residual = None      # pde = "poly": the residual as a string, e.g. "u_t + u*u_x - nu*u_xx" (utils/poly_spec.py); a spec that
    #                      mentions l1 / l2 is identification (fit(X_u, u), residual on the data points), otherwise inference
    #                      (collocation x_f, t_f).  An optional source gives s in f = ... - s: a string such as
    #                      "(k*pi**2 - 1)*sin(pi*x)*exp(-t)" (poly_spec.parse_source), which the device evaluates at every new set of
    #                      points, or a method source(x, t), evaluated on the host whenever the points change.
    weight_seed = 1234   # stands in for tf.random.set_seed(1234) (inf_cont_burgers.py:10)

    def __init_subclass__(cls, **kw):
        super().__init_subclass__(**kw)
        # TensorFlow tape bodies in the reference subclasses are replaced by the fused-kernel equivalents
        for name in ("loss", "f_model", "uvx_model", "U_0_model", "U_1_model", "autograd", "grad", "get_loss_and_flat_grad", "get_params",
                     "wrap_training_variables", "get_weights", "set_weights"):
            if name in cls.__dict__ and name in _NATIVE_OVERRIDES and not getattr(cls.__dict__[name], "_keep", False):
                setattr(cls, "_script_" + name, cls.__dict__[name])
                setattr(cls, name, _NATIVE_OVERRIDES[name])
        # ide_disc_burgers.py writes its own training loop (fit(x_0,u_0,x_1,u_1) :149-194, predict :197-202) around tape code:
        # four-argument fit / predict of a two-snapshot model go to the native loop, everything else stays the script's
        for name in ("fit", "predict"):
            if name in cls.__dict__ and not getattr(cls.__dict__[name], "_keep", False):
                script_fn = cls.__dict__[name]
                setattr(cls, "_script_" + name, script_fn)
                setattr(cls, name, _two_snapshot_dispatch(name, script_fn))

    def __init__(self, hp, logger, ub, lb):
        layers = hp["layers"]
        self.layers = [int(v) for v in layers]
        # optimiser hyper-parameters (neuralnetwork.py:12-22)
        self.nt_config = Struct()
        self.nt_config.learningRate = hp["nt_lr"]
        self.nt_config.maxIter = hp["nt_epochs"]
        self.nt_config.nCorrection = hp["nt_ncorr"]
        self.nt_config.tolFun = 1.0 * np.finfo(float).eps
        self.tf_epochs = hp["tf_epochs"]
        self.tf_lr = hp["tf_lr"]
        self.tf_b1 = hp["tf_b1"]
        self.tf_b2 = 0.999
        self.tf_eps = 1e-7 if hp["tf_eps"] is None else hp["tf_eps"]      # Keras epsilon=None -> backend epsilon
        self.dtype = "float64"
        self.ub = np.asarray(ub, dtype=np.float64)
        self.lb = np.asarray(lb, dtype=np.float64)
        self.model = _Model(self)
        # sizes for the flat decomposition (neuralnetwork.py:40-45; uniform hidden width assumed there too)
        self.sizes_w, self.sizes_b = [], []
        for i, width in enumerate(layers):
            if i != 1:
                self.sizes_w.append(int(width * layers[1]))
                self.sizes_b.append(int(width if i != 0 else layers[1]))
        self.logger = logger
        # optional per-step resampling of the collocation set on the device (not in the reference): before Adam epoch e > 0
        # with e % resample_every == 0 the set is replaced by Latin-hypercube draw e // resample_every of resample_seed
        self.resample_every = _hp_int(hp, "resample_every", 0, 0)
        self.resample_seed = _hp_int(hp, "resample_seed", 0, 0, 1 << 64)
        # optional residual-based adaptive resampling (not in the reference): before Adam epoch e > 0 with e % rad_every == 0 the
        # set is replaced by RAD draw e // rad_every of resample_seed, N_f points from a pool of rad_pool (default 10 N_f) drawn
        # with probability ~ |f|^rad_k / mean |f|^rad_k + rad_c at the current weights (pinn_draw_collocation_rad)
        self.rad_every = _hp_int(hp, "rad_every", 0, 0)
        self.rad_pool = None if _hp_get(hp, "rad_pool") is None else _hp_int(hp, "rad_pool", 1, 1, (1 << 29) + 1)
        self.rad_k = _hp_int(hp, "rad_k", 1, 0, 5)
        self.rad_c = _hp_real(hp, "rad_c", 1.0, 0.0, 1024.0)
        if self.resample_every and self.rad_every:
            raise pinn_cabi.PinnError('hp["resample_every"] and hp["rad_every"] both redraw the collocation set: set one of them')
        self._tf_epoch = 0
        self._h = None
        self._w0 = _glorot_normal(self.layers, np.random.default_rng(self.weight_seed))
        self._bound = None
        self._bound_refs = None

    # ------------------------------------------------------------------ native handle
    def _n_net_params(self):
        return sum(a * b + b for a, b in zip(self.layers[:-1], self.layers[1:]))

    def _pde_id(self):
        tag = self.pde
        if tag is None:
            if hasattr(self, "IRK_alpha"):
                tag = "burgers_ide_disc"
            elif hasattr(self, "IRK_weights"):
                tag = "burgers_disc"
            elif hasattr(self, "lambda_1"):
                tag = "burgers_ide"
            elif hasattr(self, "X_lb"):
                tag = "nls_inf"
            elif hasattr(self, "x_f"):
                tag = "burgers_inf"
            else:
                raise pinn_cabi.PinnError("cannot recognise the PDE of %s: set the class attribute `pde`" % type(self).__name__)
        if tag == "poly":
            return pinn_cabi.POLY_IDE if self._poly_spec().identification else pinn_cabi.POLY_INF
        return {"burgers_inf": pinn_cabi.BURGERS_INF, "burgers_ide": pinn_cabi.BURGERS_IDE, "nls_inf": pinn_cabi.NLS_INF,
                "burgers_disc": pinn_cabi.BURGERS_DISC, "burgers_ide_disc": pinn_cabi.BURGERS_IDE_DISC,
                "kdv_ide_disc": pinn_cabi.KDV_IDE_DISC, "ac_disc": pinn_cabi.AC_DISC, "ns_ide": pinn_cabi.NS_IDE}[tag]

    def _resolve_name(self, name):
        """The number a free name of a residual or source string stands for: a numeric attribute of the instance, else None."""
        v = getattr(self, name, None)
        if isinstance(v, (bool, np.bool_, str, bytes)) or v is None or callable(v):
            return None
        try:
            a = np.asarray(v, dtype=np.float64)
        except (TypeError, ValueError):
            return None
        return float(a.reshape(-1)[0]) if a.size == 1 else None

    def _poly_spec(self):
        """The parsed `residual` string (pde = "poly"); free names resolve to numeric attributes of the instance."""
        if getattr(self, "_poly_cache", None) is None:
            try:
                self._poly_cache = poly_spec.parse(self.residual, self._resolve_name)
            except poly_spec.SpecError as e:
                raise pinn_cabi.PinnError("%s.residual: %s" % (type(self).__name__, e))
        return self._poly_cache

    def _source_table(self):
        """The parsed `source` string (pde = "poly"); free names resolve as in the residual.  A table whose exp factor overflows
        on the box [lb, ub] is refused."""
        if getattr(self, "_source_cache", None) is None:
            try:
                terms = poly_spec.parse_source(self.source, self._resolve_name)
                poly_spec.check_source_range(terms, self.lb, self.ub)
                self._source_cache = terms
            except poly_spec.SpecError as e:
                raise pinn_cabi.PinnError("%s.source: %s" % (type(self).__name__, e))
        return self._source_cache

    def _upload_source(self, X, h=None):
        """pde = "poly": source(x, t) on the residual points X (N, 2) just bound, when the subclass defines it."""
        fn = getattr(self, "source", None)
        if callable(fn):
            X = np.asarray(X, dtype=np.float64)
            s = np.asarray(fn(X[:, 0:1], X[:, 1:2]), dtype=np.float64)
            (h or self._native()).set_source(np.broadcast_to(s.reshape(-1) if s.size == X.shape[0] else s, (X.shape[0],)))

    def _two_snapshots(self):
        return self._pde_id() in _TWO_SNAPSHOT

    def _native(self):
        if self._h is None:
            pde = self._pde_id()
            if self.resample_every and pde not in _COLLOCATION:
                raise pinn_cabi.PinnError('hp["resample_every"]: %s has no collocation set to resample' % type(self).__name__)
            rad_ok = pde in _RAD or (pde == pinn_cabi.POLY_INF and isinstance(getattr(self, "source", None), str))
            if self.rad_every and (not rad_ok or getattr(self, "world", 1) > 1):
                raise pinn_cabi.PinnError('hp["rad_every"]: residual-based resampling runs for the Burgers and Schrodinger '
                                          'inference models and for poly inference with a string source (use "0" for none) on '
                                          'one GPU, not for %s' % type(self).__name__)
            h = pinn_cabi.Pinn(pde, self.layers, self.lb, self.ub, device=getattr(self, "device", 0),
                               rank=getattr(self, "rank", 0), world=getattr(self, "world", 1),
                               nccl_uid=getattr(self, "nccl_uid", None))
            w = self._w0
            if pde == pinn_cabi.BURGERS_INF:
                h.set_pde_params([float(self.nu)])
                h.set_collocation(np.asarray(self.x_f)[:, 0], np.asarray(self.t_f)[:, 0], getattr(self, "n_f_global", None))
            elif pde == pinn_cabi.BURGERS_DISC:                      # inf_disc_burgers.py:50-59
                h.set_pde_params([float(self.nu), float(np.asarray(self.dt).reshape(-1)[0])])
                h.set_irk(np.asarray(self.IRK_weights, dtype=np.float64))
                h.set_boundary(np.asarray(self.x_1, dtype=np.float64).reshape(-1))
            elif pde in _TWO_SNAPSHOT:                               # ide_disc_burgers.py:49-55, :151-152 (KdV.py alike)
                h.set_pde_params([float(np.asarray(self.dt).reshape(-1)[0])])
                h.set_irk(pinn_cabi.irk_ide_disc(self.IRK_alpha, self.IRK_beta))
                w = np.concatenate([w, [0.0, -6.0]])
            elif pde == pinn_cabi.AC_DISC:                           # AC.py: d = 1e-4, k = 5 unless the class sets d / k
                h.set_pde_params([float(np.asarray(self.dt).reshape(-1)[0]), float(getattr(self, "d", 1e-4)),
                                  float(getattr(self, "k", 5.0))])
                h.set_irk(np.asarray(self.IRK_weights, dtype=np.float64))
            elif pde == pinn_cabi.NS_IDE:                            # NavierStokes.py: raw lambdas, both 0.0 unless the class sets them
                w = np.concatenate([w, [_scalar(getattr(self, "lambda_1", 0.0)), _scalar(getattr(self, "lambda_2", 0.0))]])
            elif pde in _POLY:                                       # utils/poly_spec.py
                h.set_residual(self._poly_spec().terms)
                if isinstance(getattr(self, "source", None), str):   # a table: it follows every new set of residual points
                    h.set_source_terms(self._source_table())
                if pde == pinn_cabi.POLY_IDE:                        # raw lambdas, 0.0 unless the class sets them
                    w = np.concatenate([w, [_scalar(getattr(self, "lambda_1", 0.0)), _scalar(getattr(self, "lambda_2", 0.0))]])
                else:
                    X_f = np.hstack([np.asarray(self.x_f, dtype=np.float64).reshape(-1, 1),
                                     np.asarray(self.t_f, dtype=np.float64).reshape(-1, 1)])
                    h.set_collocation(X_f[:, 0], X_f[:, 1], getattr(self, "n_f_global", None))
                    self._upload_source(X_f, h)
            elif pde == pinn_cabi.BURGERS_IDE:
                l1 = float(np.asarray(self.lambda_1.numpy() if hasattr(self.lambda_1, "numpy") else self.lambda_1).reshape(-1)[0])
                l2 = float(np.asarray(self.lambda_2.numpy() if hasattr(self.lambda_2, "numpy") else self.lambda_2).reshape(-1)[0])
                w = np.concatenate([w, [l1, l2]])
            else:
                h.set_collocation(np.asarray(self.x_f)[:, 0], np.asarray(self.t_f)[:, 0], getattr(self, "n_f_global", None))
                h.set_boundary(np.asarray(self.X_lb)[:, 1])
            h.set_weights(w)
            self._h = h
        return self._h

    @staticmethod
    def _data_key(*arrays):
        """Identity AND content of the bound arrays: an array mutated in place between calls is uploaded again.  The key holds
        the object identity, the shape and a checksum of the bytes (whole array up to 1 MiB -- the data terms are at most a few
        thousand rows -- else its first and last 64 KiB)."""
        import zlib
        key = []
        for a in arrays:
            b = np.ascontiguousarray(np.asarray(a, dtype=np.float64))
            raw = b.reshape(-1).view(np.uint8)
            crc = zlib.crc32(raw.tobytes()) if raw.size <= (1 << 20) else zlib.crc32(raw[:65536].tobytes() + raw[-65536:].tobytes())
            key.append((id(a), b.shape, crc))
        return tuple(key)

    def _bind(self, X, u):
        """Upload the data term when (X,u) changes -- by identity or by content."""
        key = self._data_key(X, u)
        if self._bound != key:
            Xa, ua = np.asarray(X, dtype=np.float64), np.asarray(u, dtype=np.float64)
            self._native().set_data(Xa, ua, getattr(self, "data_weight", 1.0))
            if self._pde_id() == pinn_cabi.POLY_IDE:         # the data points are the residual points
                self._upload_source(Xa)
            self._bound = key
            self._bound_refs = (X, u)

    def _bind_snapshots(self, x_0, u_0, x_1, u_1):
        key = self._data_key(x_0, u_0, x_1, u_1)
        if self._bound != key:
            n = self._native()
            n.set_snapshot(0, np.asarray(x_0, dtype=np.float64), np.asarray(u_0, dtype=np.float64))
            n.set_snapshot(1, np.asarray(x_1, dtype=np.float64), np.asarray(u_1, dtype=np.float64))
            self._bound = key
            self._bound_refs = (x_0, u_0, x_1, u_1)

    def _as_tensor(self, a):
        return _t(a)

    def _unflatten(self, w):
        out, o = [], 0
        for fi, fo in zip(self.layers[:-1], self.layers[1:]):
            out.append(_t(w[o:o + fi * fo].reshape(fi, fo))); o += fi * fo
            out.append(_t(w[o:o + fo])); o += fo
        return out

    # ------------------------------------------------------------------ reference surface
    def loss(self, u, u_pred):
        """Base-class loss (neuralnetwork.py:51-52): plain MSE on host arrays (the PDE subclasses never reach this
        on the training path -- their composite loss is evaluated inside the fused kernel)."""
        return np.mean(np.square(np.asarray(u) - np.asarray(u_pred)))

    def grad(self, X, u):
        """(loss, per-variable gradients) (neuralnetwork.py:55-59), one fused kernel launch."""
        self._bind(X, u)
        loss, g, _ = self._native().loss_grad()
        grads = self._unflatten(g[: self._n_net_params()])
        if g.size > self._n_net_params():
            grads += [_t(g[-2:-1]), _t(g[-1:])]
        return np.float64(loss), grads

    def wrap_training_variables(self):
        var = self.model.trainable_variables
        if self._pde_id() in _LAMBDAS:                                                # ide_cont_burgers.py:93-96
            w = self._native().get_weights()
            var = var + [_t(w[-2:-1]), _t(w[-1:])]
        return var

    def get_params(self, numpy=False):
        """Base class: no PDE parameters (neuralnetwork.py:64-65); the identification models return (lambda_1, exp(lambda_2)),
        Navier-Stokes the raw (lambda_1, lambda_2)."""
        try:
            if self._pde_id() in _LAMBDAS:
                return _native_get_params(self, numpy)
        except pinn_cabi.PinnError:
            pass
        return []

    def get_weights(self, convert_to_tensor=True):
        """Flat vector: per layer W.flatten() then b (neuralnetwork.py:68-78); identification appends l1, l2."""
        w = self._native().get_weights()
        return _t(w) if convert_to_tensor else list(w)

    def set_weights(self, w):
        self._native().set_weights(np.asarray(w, dtype=np.float64))

    def get_loss_and_flat_grad(self, X, u):
        if X is not None:
            self._bind(X, u)

        def loss_and_flat_grad(w):
            loss, g, _ = self._native().loss_grad(w=np.asarray(w, dtype=np.float64))
            return np.float64(loss), _t(g)

        loss_and_flat_grad._pinn_net = self
        return loss_and_flat_grad

    def tf_optimization(self, X_u, u):
        """Adam epochs.  With hp["resample_every"] = k (or hp["rad_every"] = k) the collocation set is redrawn on the device
        before every epoch e > 0 with e % k == 0 (tf_optimization_step); epochs [0, k) train on the script's own X_f, and the
        L-BFGS phase that follows runs on the last drawn set."""
        self.logger.log_train_opt("Adam")
        self._tf_epoch = 0
        for epoch in range(self.tf_epochs):
            loss_value = self.tf_optimization_step(X_u, u)
            self.logger.log_train_epoch(epoch, loss_value)

    def tf_optimization_step(self, X_u, u):
        """One fused loss/grad evaluation + on-device Adam update, enqueued without a host sync.  With hp["resample_every"] = k,
        epoch e > 0 with e % k == 0 first replaces the collocation set by Latin-hypercube draw e // k of hp["resample_seed"] over
        the script's N_f points (n_f_global when sharded), this rank's rows of it (pinn_draw_collocation).  With
        hp["rad_every"] = k the set becomes RAD draw e // k of hp["resample_seed"] instead (pinn_draw_collocation_rad)."""
        self._bind(X_u, u)
        n = self._native()
        e, k, kr = self._tf_epoch, self.resample_every, self.rad_every
        if k and e > 0 and e % k == 0:
            self._resample(n, e // k)
        if kr and e > 0 and e % kr == 0:
            n_f = int(np.asarray(self.x_f).shape[0])
            n.draw_collocation_rad(self.resample_seed, e // kr, n_f, self.rad_pool or 10 * n_f, self.rad_k, self.rad_c)
        self._tf_epoch = e + 1
        n.adam_step(self.tf_lr, self.tf_b1, self.tf_b2, self.tf_eps, sync=False)
        self._adam_serial = getattr(self, "_adam_serial", 0) + 1
        return LazyLoss(n, self)

    def _resample(self, n, draw):
        n_global = getattr(self, "n_f_global", None) or int(np.asarray(self.x_f).shape[0])
        n.draw_collocation(self.resample_seed, draw, n_global, rank=getattr(self, "rank", 0), world=getattr(self, "world", 1))
        if n.pde == pinn_cabi.POLY_INF and callable(getattr(self, "source", None)):
            x, t = n.get_collocation()                       # the one host round trip a callable source needs
            self._upload_source(np.stack([x, t], 1), n)

    def nt_optimization(self, X_u, u):
        self.logger.log_train_opt("LBFGS")
        loss_and_flat_grad = self.get_loss_and_flat_grad(X_u, u)
        self.nt_optimization_steps(loss_and_flat_grad)

    def nt_optimization_steps(self, loss_and_flat_grad):
        lbfgs(loss_and_flat_grad, self.get_weights(), self.nt_config, Struct(), True,
              lambda epoch, loss, is_iter: self.logger.log_train_epoch(epoch, loss, "", is_iter))

    def fit(self, X_u, u):
        self.logger.log_train_start(self)
        X_u = self.tensor(X_u)
        u = self.tensor(u)
        self.tf_optimization(X_u, u)
        self.nt_optimization(X_u, u)
        self.logger.log_train_end(self.tf_epochs + self.nt_config.maxIter)

    def predict(self, X_star):
        if self._is_ns():
            return _ns_fields(self, X_star)[:3]
        return self.model(X_star).numpy()

    def f_model(self, X=None):
        """Residuals on the stored residual points (Navier-Stokes: (f_u, f_v), or on the points X when given)."""
        return _native_f_model(self, *(() if X is None else (X,)))

    def _is_ns(self):
        try:
            return self._pde_id() == pinn_cabi.NS_IDE
        except pinn_cabi.PinnError:
            return False

    def summary(self):
        return self.model.summary()

    def tensor(self, X):
        return _t(X)


# two-snapshot discrete-time identification models: fit(x_0, u_0, x_1, u_1), predict -> (U_0, U_1), flat vector ends with l1, l2
_TWO_SNAPSHOT = (pinn_cabi.BURGERS_IDE_DISC, pinn_cabi.KDV_IDE_DISC)
# every model whose flat vector ends with [lambda_1, lambda_2]
_LAMBDAS = (pinn_cabi.BURGERS_IDE, pinn_cabi.NS_IDE, pinn_cabi.POLY_IDE) + _TWO_SNAPSHOT
# user-defined polynomial residuals (pde = "poly")
_POLY = (pinn_cabi.POLY_INF, pinn_cabi.POLY_IDE)
# models with a collocation set (pinn_set_collocation, pinn_draw_collocation)
_COLLOCATION = (pinn_cabi.BURGERS_INF, pinn_cabi.NLS_INF, pinn_cabi.POLY_INF)
# models whose residual the device forms on a pool it has just drawn (pinn_draw_collocation_rad)
_RAD = (pinn_cabi.BURGERS_INF, pinn_cabi.NLS_INF)


def _hp_get(hp, key, default=None):
    return hp.get(key, default) if hasattr(hp, "get") else default


def _hp_int(hp, key, default, lo, hi=None):
    """An optional integer hyper-parameter in [lo, hi)."""
    v = _hp_get(hp, key, default)
    v = default if v is None else v
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or v < lo or (hi is not None and v >= hi):
        raise pinn_cabi.PinnError('hp["%s"] = %r: expected an integer >= %d%s' % (key, v, lo, "" if hi is None else " below %d" % hi))
    return int(v)


def _hp_real(hp, key, default, lo, hi):
    """An optional finite real hyper-parameter in [lo, hi]."""
    v = _hp_get(hp, key, default)
    v = default if v is None else v
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)) or not lo <= float(v) <= hi:
        raise pinn_cabi.PinnError('hp["%s"] = %r: expected a real number in [%g, %g]' % (key, v, lo, hi))
    return float(v)


def _scalar(v):
    return float(np.asarray(v.numpy() if hasattr(v, "numpy") else v, dtype=np.float64).reshape(-1)[0])


def _ns_fields(self, X):
    """Navier-Stokes (u, v, p, f_u, f_v) on the points X (N,3), each (N,1), from the 13 device streams of (psi, p):
    u = psi_y, v = -psi_x (NavierStokes.py net_NS)."""
    n = self._native()
    D = n.derivatives(np.asarray(X, dtype=np.float64))
    l1, l2 = n.get_weights()[-2:]
    P, Q = D[:, :, 0], D[:, :, 1]
    px, py, pxx, pxy, pyy = P[:, 1], P[:, 2], P[:, 4], P[:, 5], P[:, 6]
    f_u = P[:, 8] + l1 * (py * pxy - px * pyy) + Q[:, 1] - l2 * (P[:, 10] + P[:, 12])
    f_v = -P[:, 7] + l1 * (px * pxy - py * pxx) + Q[:, 2] + l2 * (P[:, 9] + P[:, 11])
    return tuple(_t(a[:, None]) for a in (py, -px, Q[:, 0], f_u, f_v))


# ---------------------------------------------------------------------- native replacements for subclass overrides
def _native_loss(self, *args):
    """Composite PDE loss of the recognised problem on the bound data (value only)."""
    if len(args) == 4:                                   # ide_disc_burgers.py:111-115 loss(x_0, u_0, x_1, u_1)
        self._bind_snapshots(*args)
    loss, _, _ = self._native().loss_grad(want_grad=False)
    return np.float64(loss)


def _native_f_model(self, *args):
    """f_model (inf_cont_burgers.py:65-90 / ide_cont_burgers.py:56-85 / inf_cont_schrodinger.py:79-105): on the stored
    residual points, or -- identification, where the reference passes the points explicitly -- on the given points."""
    n = self._native()
    if self._pde_id() in _POLY:
        if args:                                          # on the given points: streams from the device, the spec on the host
            X = np.asarray(args[0], dtype=np.float64)
            U, Ux, Ut, Uxx = n.derivatives(X)
            lam = n.get_weights()[-2:] if n.pde == pinn_cabi.POLY_IDE else (0.0, 0.0)
            f = poly_spec.evaluate(self._poly_spec().terms, (U, Ux, Ut, Uxx), *lam)
            fn = getattr(self, "source", None)
            if isinstance(fn, str):
                f = f - poly_spec.evaluate_source(self._source_table(), X[:, 0:1], X[:, 1:2]).reshape(f.shape)
            elif callable(fn):
                f = f - np.asarray(fn(X[:, 0:1], X[:, 1:2]), dtype=np.float64).reshape(f.shape)
            return _t(f)
        if n.pde == pinn_cabi.POLY_IDE and self._bound is None:
            raise pinn_cabi.PinnError("f_model(): no data points are bound yet -- call fit()/grad() first, or pass the points")
        return _t(n.residual())
    if self._pde_id() == pinn_cabi.NS_IDE and args:
        return _ns_fields(self, args[0])[3:]
    if self._pde_id() == pinn_cabi.BURGERS_IDE:
        if args:
            U, Ux, Ut, Uxx = n.derivatives(np.asarray(args[0], dtype=np.float64))
            w = n.get_weights()
            return _t(Ut + w[-2] * U * Ux - np.exp(w[-1]) * Uxx)
        if self._bound is None:
            raise pinn_cabi.PinnError("f_model(): no data points are bound yet -- call fit()/grad() first, or pass the points")
        return _t(n.residual())
    f = n.residual()
    if f.shape[1] == 2:
        return _t(f[:, 0:1]), _t(f[:, 1:2])
    return _t(f)


def _ide_disc_models(self, x):
    """U_0 = U + dt N alpha^T and U_1 = U - dt N (beta - alpha)^T on arbitrary points (ide_disc_burgers.py:81-108, predict
    :197-202): network value and x-derivatives from the device, the two small q x q products on the host (off the step path).
    Burgers: N = l1 U U_x - e^{l2} U_xx;  KdV: N = l1 U U_x + e^{l2} U_xxx (u_xxx comes in the u_t column block)."""
    n = self._native()
    U, Ux, Uxxx, Uxx = n.derivatives(np.asarray(x, dtype=np.float64).reshape(-1, 1))
    w = n.get_weights()
    if n.pde == pinn_cabi.KDV_IDE_DISC:
        N = w[-2] * U * Ux + np.exp(w[-1]) * Uxxx
    else:
        N = w[-2] * U * Ux - np.exp(w[-1]) * Uxx
    M = pinn_cabi.irk_ide_disc(self.IRK_alpha, self.IRK_beta)
    q = M.shape[1]
    dt = float(np.asarray(self.dt).reshape(-1)[0])
    return _t(U + dt * N @ M[:q].T), _t(U + dt * N @ M[q:].T)


def _native_U_0_model(self, x, customDummy=None):
    if self._two_snapshots():
        return _ide_disc_models(self, x)[0]
    raise pinn_cabi.PinnError("U_0_model is evaluated inside the fused kernel; use grad()/fit()/predict()")


def _native_U_1_model(self, x, customDummy=None):
    if self._two_snapshots():
        return _ide_disc_models(self, x)[1]
    raise pinn_cabi.PinnError("U_1_model belongs to the discrete-time identification model")


def _native_autograd(self, *args):
    raise pinn_cabi.PinnError("autograd (the dummy-gradient tape trick) is replaced by the fused kernel's forward derivative streams")


def _native_fit_two_snapshots(self, x_0, u_0, x_1, u_1):
    """fit(x_0, u_0, x_1, u_1) of ide_disc_burgers.py:149-194 on the device: lambda_1 = 0, lambda_2 = -6, tf_epochs Adam steps
    (loss logged with the current lambdas), then the fixed-step L-BFGS, then the closing line."""
    self.logger.log_train_start(self)
    x_0, u_0, x_1, u_1 = (self.tensor(a) for a in (x_0, u_0, x_1, u_1))
    self._bind_snapshots(x_0, u_0, x_1, u_1)
    n = self._native()
    w = n.get_weights()
    w[-2:] = [0.0, -6.0]                                  # :151-152
    n.set_weights(w)

    def custom():
        l1, l2 = self.get_params(numpy=True)
        return f"l1 = {l1:5f}  l2 = {l2:8f}"

    def log_train_epoch(epoch, loss, is_iter):
        printed = epoch % self.logger.frequency == 0       # the lambdas are read back only for the lines that are printed
        self.logger.log_train_epoch(epoch, loss, custom() if printed else "", is_iter)

    self.logger.log_train_opt("Adam")
    for epoch in range(self.tf_epochs):
        n.adam_step(self.tf_lr, self.tf_b1, self.tf_b2, self.tf_eps, sync=False)
        self._adam_serial = getattr(self, "_adam_serial", 0) + 1
        # the reference logs (loss before the update, lambdas after it): :172-176
        log_train_epoch(epoch, LazyLoss(n, self), False)
    self.logger.log_train_opt("LBFGS")
    closure = self.get_loss_and_flat_grad(None, None)
    lbfgs(closure, self.get_weights(), self.nt_config, Struct(), True, log_train_epoch)
    self.logger.log_train_end(self.tf_epochs, custom())


def _two_snapshot_dispatch(name, script_fn):
    def fit(self, *args):
        if len(args) == 4 and self._two_snapshots():
            return _native_fit_two_snapshots(self, *args)
        return script_fn(self, *args)

    def predict(self, x_star, *rest):
        try:
            two = self._two_snapshots()
        except pinn_cabi.PinnError:
            two = False
        if two:
            return _ide_disc_models(self, x_star)
        if self._is_ns():
            return _ns_fields(self, x_star)[:3]
        return script_fn(self, x_star, *rest)

    fn = fit if name == "fit" else predict
    fn.__name__ = name
    return fn


def _native_grad(self, *args):
    if len(args) == 4:                                   # ide_disc_burgers.py:117-120 grad(x_0, u_0, x_1, u_1)
        self._bind_snapshots(*args)
        loss, g, _ = self._native().loss_grad()
        return np.float64(loss), self._unflatten(g[: self._n_net_params()]) + [_t(g[-2:-1]), _t(g[-1:])]
    return NeuralNetwork.grad(self, *args)


def _native_get_loss_and_flat_grad(self, X, u):
    return NeuralNetwork.get_loss_and_flat_grad(self, X, u)


def _native_uvx_model(self, X):
    U, Ux, _, _ = self._native().derivatives(np.asarray(X, dtype=np.float64))
    return _t(U[:, 0:1]), _t(U[:, 1:2]), _t(Ux[:, 0:1]), _t(Ux[:, 1:2])


def _native_get_params(self, numpy=False):
    pde = self._pde_id()
    if pde == pinn_cabi.BURGERS_INF:
        return self.nu
    if pde in (pinn_cabi.NS_IDE, pinn_cabi.POLY_IDE):
        l1, l2 = self._native().get_weights()[-2:]     # raw lambdas (NavierStokes.py; the poly residual's l1, l2)
        return (l1, l2) if numpy else (_t([l1]), _t([l2]))
    if pde in (pinn_cabi.BURGERS_IDE,) + _TWO_SNAPSHOT:
        w = self._native().get_weights()
        l1, l2 = w[-2], np.exp(w[-1])            # ide_cont_burgers.py:109-114, ide_disc_burgers.py:138-143
        return (l1, l2) if numpy else (_t([l1]), _t([l2]))
    return []


def _native_wrap_training_variables(self):
    return NeuralNetwork.wrap_training_variables(self)


def _native_get_weights(self, convert_to_tensor=True):
    return NeuralNetwork.get_weights(self, convert_to_tensor)


def _native_set_weights(self, w):
    return NeuralNetwork.set_weights(self, w)


_NATIVE_OVERRIDES.update(U_0_model=_native_U_0_model, U_1_model=_native_U_1_model, autograd=_native_autograd, grad=_native_grad,
                         get_loss_and_flat_grad=_native_get_loss_and_flat_grad)
_NATIVE_OVERRIDES.update(loss=_native_loss, f_model=_native_f_model, uvx_model=_native_uvx_model,
                         get_params=_native_get_params, wrap_training_variables=_native_wrap_training_variables,
                         get_weights=_native_get_weights, set_weights=_native_set_weights)
