"""Label MLP training on the H100: ``DeviceMLPClassifier``, sklearn's ``MLPClassifier`` with ``fit`` on the GPU.

``DeviceMLPClassifier`` overrides ``fit`` only.  The host driver below makes every decision sklearn 1.9's
``MLPClassifier._fit_stochastic`` makes, with the same random draws in the same order: the initial parameters
(sklearn's own ``_initialize``), the early-stopping split, one ``shuffle`` per epoch, the batch sizes, the learning rate
of every Adam step, the stopping rule, the best-parameter snapshot and the ``ConvergenceWarning``.  The steps themselves
-- forward, loss, backward, Adam -- run on the device behind ``ie_mlp_train_*`` (include/issue_emb_b200.h): split-bf16
wgmma products, a float64 loss, and an Adam step bit-exact to sklearn's ``AdamOptimizer`` on float32 arrays.  One epoch
is one library call with no host synchronisation between its steps.

After ``fit`` the estimator holds only numpy attributes (``coefs_`` and ``intercepts_`` float32, ``loss_curve_``,
``validation_scores_``, ...), so it pickles with dill, ``MLPHead.from_sklearn`` runs it on the GPU, and a pickled model
predicts through the inherited sklearn code on a machine without one.

Supported: ``solver='adam'``, ``activation='relu'``, a 0/1 multilabel indicator or binary y (logistic outputs).  Refused
with ``ValueError`` before anything is launched: other solvers and activations, multiclass y (softmax),
``sample_weight``, ``warm_start`` and ``partial_fit``.  There is no CPU fallback: without a GPU ``fit`` raises
``RuntimeError``.  ``learning_rate``, ``momentum``, ``power_t`` and ``nesterovs_momentum`` are accepted and ignored, as
sklearn ignores them for adam.  Search it with ``GridSearchCV(..., n_jobs=1)``: the fits share one GPU, and a process
pool gains nothing on it.
"""
from __future__ import annotations

import ctypes as C
import warnings

import numpy as np
from sklearn.exceptions import ConvergenceWarning
from sklearn.metrics import accuracy_score
from sklearn.model_selection import train_test_split
from sklearn.neural_network import MLPClassifier
from sklearn.utils import check_random_state, gen_batches, shuffle

from . import _lib
from ._lib import check


class DeviceSteps:
    """The steps of an Adam fit on the device (one ``ie_mlp_train`` handle); the driver's step backend."""

    dtype = np.float32   # parameters and data are float32 on the device, whatever X's dtype

    def __init__(self, layer_units, device: int = 0):
        self._lib = _lib.load()
        self.units = [int(u) for u in layer_units]
        dims = (C.c_int32 * len(self.units))(*self.units)
        h = C.c_void_p()
        check(self._lib.ie_mlp_train_create(len(self.units) - 1, dims, device, C.byref(h)))
        self._h = h
        self.n_val = 0

    def set_params(self, coefs, intercepts):
        """Parameters in sklearn's layout; restarts Adam at t = 0."""
        for l, (w, b) in enumerate(zip(coefs, intercepts)):
            w = np.ascontiguousarray(w, dtype=np.float32)
            b = np.ascontiguousarray(b, dtype=np.float32)
            check(self._lib.ie_mlp_train_set_layer(self._h, l, w.ctypes.data, b.ctypes.data))

    def params(self, best: bool = False):
        coefs, intercepts = [], []
        for l in range(len(self.units) - 1):
            w = np.empty((self.units[l], self.units[l + 1]), dtype=np.float32)
            b = np.empty(self.units[l + 1], dtype=np.float32)
            check(self._lib.ie_mlp_train_get_layer(self._h, l, int(best), w.ctypes.data, b.ctypes.data))
            coefs.append(w)
            intercepts.append(b)
        return coefs, intercepts

    def set_data(self, X, Y, X_val=None):
        X = np.ascontiguousarray(X, dtype=np.float32)
        Y = np.ascontiguousarray(Y, dtype=np.uint8)
        check(self._lib.ie_mlp_train_set_data(self._h, 0, X.ctypes.data, Y.ctypes.data, X.shape[0]))
        if X_val is not None:
            X_val = np.ascontiguousarray(X_val, dtype=np.float32)
            check(self._lib.ie_mlp_train_set_data(self._h, 1, X_val.ctypes.data, None, X_val.shape[0]))
            self.n_val = X_val.shape[0]

    def epoch(self, order, batch_size, lrs, alpha, beta_1, beta_2, epsilon) -> np.ndarray:
        """Steps on rows order[k*batch_size ...] with learning rates lrs[k] -> each step's batch loss (float64)."""
        order = np.ascontiguousarray(order, dtype=np.int32)
        lrs = np.ascontiguousarray(lrs, dtype=np.float64)
        if len(lrs) != -(-len(order) // batch_size):
            raise ValueError(f"{len(lrs)} learning rates for {len(order)} rows in batches of {batch_size}")
        losses = np.empty(len(lrs), dtype=np.float64)
        check(self._lib.ie_mlp_train_epoch(self._h, order.ctypes.data, len(order), int(batch_size), lrs.ctypes.data,
                                           float(alpha), float(beta_1), float(beta_2), float(epsilon),
                                           losses.ctypes.data))
        return losses

    def val_proba(self) -> np.ndarray:
        probs = np.empty((self.n_val, self.units[-1]), dtype=np.float32)
        check(self._lib.ie_mlp_train_validation_proba(self._h, probs.ctypes.data))
        return probs

    def snapshot(self):
        check(self._lib.ie_mlp_train_snapshot(self._h, 0))

    @property
    def launches(self) -> int:
        return int(self._lib.ie_mlp_train_launch_count(self._h))

    def last_epoch_ms(self) -> float:
        ms = C.c_float()
        check(self._lib.ie_mlp_train_last_epoch_ms(self._h, C.byref(ms)))
        return ms.value

    def debug_step(self, rows, alpha: float) -> dict:
        """Test hook ``ie_debug_mlp_train_step`` mode 0: one forward + backward pass on training rows `rows`, parameters
        unchanged -> {'acts': hidden activations, 'p', 'deltas', 'coef_grads', 'intercept_grads', 'loss'}."""
        rows = np.ascontiguousarray(rows, dtype=np.int32)
        b, u = len(rows), self.units
        widths = u[1:-1] + [u[-1]] + u[1:]
        n_packed = sum(u[l] * u[l + 1] + u[l + 1] for l in range(len(u) - 1))
        out = np.empty(b * sum(widths) + n_packed, dtype=np.float32)
        loss = C.c_double()
        consts = np.array([alpha], dtype=np.float64)
        check(self._lib.ie_debug_mlp_train_step(self._h, 0, rows.ctypes.data, b, consts.ctypes.data, None,
                                                out.ctypes.data, out.size, C.byref(loss)))
        mats, o = [], 0
        for w in widths:
            mats.append(out[o:o + b * w].reshape(b, w))
            o += b * w
        nh = len(u) - 2
        cg, ig = _unpack(out[o:], u)
        return {"acts": mats[:nh], "p": mats[nh], "deltas": mats[nh + 1:], "coef_grads": cg, "intercept_grads": ig,
                "loss": loss.value}

    def debug_adam(self, coef_grads, intercept_grads, lr_t, beta_1, beta_2, epsilon):
        """Test hook ``ie_debug_mlp_train_step`` mode 1: one Adam step with the given gradients -> (params, m, v), each
        a list in sklearn's order (every coef, then every intercept)."""
        g = np.concatenate([np.ravel(x).astype(np.float32) for x in list(coef_grads) + list(intercept_grads)])
        out = np.empty(3 * g.size, dtype=np.float32)
        consts = np.array([lr_t, beta_1, beta_2, epsilon], dtype=np.float64)
        check(self._lib.ie_debug_mlp_train_step(self._h, 1, None, 0, consts.ctypes.data, g.ctypes.data,
                                                out.ctypes.data, out.size, None))
        res = []
        for i in range(3):
            cs, bs = _unpack(out[i * g.size:(i + 1) * g.size], self.units)
            res.append(cs + bs)
        return tuple(res)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.ie_mlp_train_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _unpack(flat, units):
    """sklearn's packing (every coef, then every intercept) -> (coefs, intercepts) copies."""
    coefs, intercepts, o = [], [], 0
    for l in range(len(units) - 1):
        n = units[l] * units[l + 1]
        coefs.append(np.array(flat[o:o + n]).reshape(units[l], units[l + 1]))
        o += n
    for l in range(len(units) - 1):
        intercepts.append(np.array(flat[o:o + units[l + 1]]))
        o += units[l + 1]
    return coefs, intercepts


class DeviceMLPClassifier(MLPClassifier):
    """sklearn ``MLPClassifier`` whose ``fit`` runs on the H100 (module docstring).  Every constructor parameter,
    ``predict``, ``predict_proba``, ``score``, ``get_params`` / ``set_params`` and pickling are sklearn's own."""

    device = 0   # CUDA device the fits run on (a class attribute, so that get_params / clone are unchanged)

    def fit(self, X, y, sample_weight=None):
        return self._fit_with(X, y, DeviceSteps, sample_weight)

    def partial_fit(self, X, y, sample_weight=None, classes=None):
        raise ValueError("partial_fit is not supported by DeviceMLPClassifier (only whole fits run on the device)")

    def _refuse(self, sample_weight):
        if self.solver != "adam":
            raise ValueError(f"solver={self.solver!r} is not supported: DeviceMLPClassifier trains with solver='adam'")
        if self.activation != "relu":
            raise ValueError(f"activation={self.activation!r} is not supported: the device trains relu hidden layers")
        if sample_weight is not None:
            raise ValueError("sample_weight is not supported by DeviceMLPClassifier")
        if self.warm_start:
            raise ValueError("warm_start=True is not supported by DeviceMLPClassifier")

    def _fit_with(self, X, y, steps_cls, sample_weight=None):
        """The driver: sklearn 1.9's _fit + _fit_stochastic decision for decision, the steps on `steps_cls` (DeviceSteps;
        the CPU tests substitute oracle.mlp_train_ref.NumpySteps)."""
        self._validate_params()
        self._refuse(sample_weight)
        hidden = self.hidden_layer_sizes
        if not hasattr(hidden, "__iter__"):
            hidden = [hidden]
        hidden = list(hidden)
        if np.any(np.array(hidden) <= 0):
            raise ValueError("hidden_layer_sizes must be > 0, got %s." % hidden)
        X, y = self._validate_input(X, y, incremental=False, reset=True)
        if self._label_binarizer.y_type_ == "multiclass":
            raise ValueError("y is multiclass (softmax output): DeviceMLPClassifier trains logistic outputs only -- a 0/1 "
                             "multilabel indicator or a binary y")
        if hasattr(X, "toarray"):
            X = X.toarray()
        dtype = steps_cls.dtype or X.dtype
        X = np.asarray(X, dtype=dtype)
        if not np.isfinite(X).all():
            raise ValueError(f"X contains values that are not finite in {np.dtype(dtype).name}")
        if y.ndim == 1:
            y = y.reshape((-1, 1))
        self.n_outputs_ = y.shape[1]
        layer_units = [X.shape[1]] + hidden + [self.n_outputs_]
        self._random_state = check_random_state(self.random_state)
        self._initialize(y, layer_units, dtype)

        early_stopping = self.early_stopping
        if early_stopping:
            stratify = y if self.n_outputs_ == 1 else None   # not stratified for multilabel
            X_train, X_val, y_train, y_val = train_test_split(X, y, random_state=self._random_state,
                                                              test_size=self.validation_fraction, stratify=stratify)
            if X_val.shape[0] < 2:
                raise ValueError("The validation set is too small. Increase 'validation_fraction' or the size of your "
                                 "dataset.")
            y_val = self._label_binarizer.inverse_transform(y_val)
        else:
            X_train, y_train, X_val, y_val = X, y, None, None
        n_samples = X_train.shape[0]
        sample_idx = np.arange(n_samples, dtype=int)
        if self.batch_size == "auto":
            batch_size = min(200, n_samples)
        else:
            if self.batch_size > n_samples:
                warnings.warn("Got `batch_size` less than 1 or larger than sample size. It is going to be clipped")
            batch_size = np.clip(self.batch_size, 1, n_samples)
        batch_size = int(batch_size)
        slices = list(gen_batches(n_samples, batch_size))

        steps = steps_cls(layer_units, self.device)
        try:
            steps.set_params(self.coefs_, self.intercepts_)
            steps.set_data(X_train, y_train, X_val)
            if early_stopping:
                steps.snapshot()          # sklearn's _best_coefs start as the initial parameters
            t = 0
            self.n_iter_ = 0
            for _ in range(self.max_iter):
                if self.shuffle:
                    sample_idx = shuffle(sample_idx, random_state=self._random_state)
                lrs = np.empty(len(slices))
                for k in range(len(slices)):   # AdamOptimizer._get_updates, step by step
                    t += 1
                    lrs[k] = self.learning_rate_init * np.sqrt(1 - self.beta_2 ** t) / (1 - self.beta_1 ** t)
                losses = steps.epoch(sample_idx, batch_size, lrs, self.alpha, self.beta_1, self.beta_2, self.epsilon)
                accumulated_loss = 0.0
                for batch_loss, sl in zip(losses, slices):
                    accumulated_loss += batch_loss * (sl.stop - sl.start)
                self.n_iter_ += 1
                self.loss_ = accumulated_loss / X_train.shape[0]
                self.t_ += n_samples
                self.loss_curve_.append(self.loss_)
                if self.verbose:
                    print("Iteration %d, loss = %.8f" % (self.n_iter_, self.loss_))
                if early_stopping:
                    p = steps.val_proba()
                    y_pred = self._label_binarizer.inverse_transform(p.ravel() if self.n_outputs_ == 1 else p)
                    val_score = accuracy_score(y_val, y_pred)
                    self.validation_scores_.append(val_score)
                    if self.verbose:
                        print("Validation score: %f" % val_score)
                    if val_score < self.best_validation_score_ + self.tol:
                        self._no_improvement_count += 1
                    else:
                        self._no_improvement_count = 0
                    if val_score > self.best_validation_score_:
                        self.best_validation_score_ = val_score
                        steps.snapshot()
                else:
                    if self.loss_curve_[-1] > self.best_loss_ - self.tol:
                        self._no_improvement_count += 1
                    else:
                        self._no_improvement_count = 0
                    if self.loss_curve_[-1] < self.best_loss_:
                        self.best_loss_ = self.loss_curve_[-1]
                if self._no_improvement_count > self.n_iter_no_change:
                    if self.verbose:
                        what = "Validation score" if early_stopping else "Training loss"
                        print("%s did not improve more than tol=%f for %d consecutive epochs. Stopping."
                              % (what, self.tol, self.n_iter_no_change))
                    break   # AdamOptimizer.trigger_stopping always stops
                if self.n_iter_ == self.max_iter:
                    warnings.warn("Stochastic Optimizer: Maximum iterations (%d) reached and the optimization hasn't "
                                  "converged yet." % self.max_iter, ConvergenceWarning)
            self.coefs_, self.intercepts_ = steps.params(best=early_stopping)
        finally:
            steps.close()
        if early_stopping:
            self._best_coefs = [c.copy() for c in self.coefs_]
            self._best_intercepts = [b.copy() for b in self.intercepts_]
        if not all(np.isfinite(w).all() for w in self.coefs_ + self.intercepts_):
            raise ValueError("Solver produced non-finite parameter weights. The input data may contain large values and "
                             "need to be preprocessed.")
        return self
