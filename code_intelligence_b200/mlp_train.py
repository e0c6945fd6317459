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
sklearn ignores them for adam.  Search it with ``DeviceGridSearchCV``: its fits train together in lockstep groups on one
``ie_mlp_group`` handle per architecture and batch size, each bit-identical to its own ``fit``.
"""
from __future__ import annotations

import ctypes as C
import threading
import time
import warnings

import numpy as np
from sklearn.exceptions import ConvergenceWarning
from sklearn.metrics import accuracy_score
from sklearn.base import clone
from sklearn.model_selection import GridSearchCV, ParameterGrid, train_test_split
from sklearn.neural_network import MLPClassifier
from sklearn.utils import _safe_indexing, check_random_state, gen_batches, shuffle

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
        """The driver: sklearn 1.9's _fit + _fit_stochastic decision for decision (``_Fit``), the steps on `steps_cls`
        (DeviceSteps; the CPU tests substitute oracle.mlp_train_ref.NumpySteps).  Inside ``DeviceGridSearchCV`` the fit
        was already trained with its group and is installed instead."""
        replay = getattr(_REPLAY, "queue", None)
        if replay is not None:
            return _replay_fit(self, X, y, replay, sample_weight)
        fit = _Fit(self, X, y, steps_cls.dtype, sample_weight)
        steps = steps_cls(fit.layer_units, self.device)
        try:
            steps.set_params(self.coefs_, self.intercepts_)
            tr = fit.train_rows
            steps.set_data(fit.X[tr], fit.y[tr], fit.X[fit.val_rows] if fit.early_stopping else None)
            if fit.early_stopping:
                steps.snapshot()          # sklearn's _best_coefs start as the initial parameters
            while True:
                order, lrs = fit.epoch_inputs()
                losses = steps.epoch(order, fit.batch_size, lrs, self.alpha, self.beta_1, self.beta_2, self.epsilon)
                snap, done = fit.after_epoch(losses, steps.val_proba() if fit.early_stopping else None)
                if snap:
                    steps.snapshot()
                if done:
                    break
            coefs, intercepts = steps.params(best=fit.early_stopping)
        finally:
            steps.close()
        fit.finish(coefs, intercepts)
        return self


class _Fit:
    """One fit's host state, sklearn 1.9's ``_fit`` / ``_fit_stochastic`` cut at the epoch boundary, so that one driver
    runs a single fit (``DeviceMLPClassifier._fit_with``) and many in lockstep (``_train_groups``).

    begin (the constructor): validation, refusals, ``_initialize``, the early-stopping split as row maps into X and the
    batch size; ``epoch_inputs``: the shuffle and the learning rates; ``after_epoch``: the loss, the validation score,
    the stopping rule and the snapshot decision; ``finish``: parameters, best copies and the non-finite error."""

    def __init__(self, est, X, y, dtype=None, sample_weight=None):
        self.est = est
        est._validate_params()
        est._refuse(sample_weight)
        hidden = est.hidden_layer_sizes
        if not hasattr(hidden, "__iter__"):
            hidden = [hidden]
        hidden = list(hidden)
        if np.any(np.array(hidden) <= 0):
            raise ValueError("hidden_layer_sizes must be > 0, got %s." % hidden)
        X, y = est._validate_input(X, y, incremental=False, reset=True)
        if est._label_binarizer.y_type_ == "multiclass":
            raise ValueError("y is multiclass (softmax output): DeviceMLPClassifier trains logistic outputs only -- a 0/1 "
                             "multilabel indicator or a binary y")
        if hasattr(X, "toarray"):
            X = X.toarray()
        dtype = dtype or X.dtype
        X = np.asarray(X, dtype=dtype)
        if not np.isfinite(X).all():
            raise ValueError(f"X contains values that are not finite in {np.dtype(dtype).name}")
        if y.ndim == 1:
            y = y.reshape((-1, 1))
        est.n_outputs_ = y.shape[1]
        self.layer_units = [X.shape[1]] + hidden + [est.n_outputs_]
        est._random_state = check_random_state(est.random_state)
        est._initialize(y, self.layer_units, dtype)
        self.X, self.y = X, y
        self.early_stopping = est.early_stopping
        if self.early_stopping:
            # the split of an index array: the partition train_test_split(X, y, ...) makes, as row maps
            stratify = y if est.n_outputs_ == 1 else None   # not stratified for multilabel
            self.train_rows, self.val_rows = _split_rows(X.shape[0], est._random_state, est.validation_fraction,
                                                         stratify)
            if self.val_rows.shape[0] < 2:
                raise ValueError("The validation set is too small. Increase 'validation_fraction' or the size of your "
                                 "dataset.")
            self.y_val = est._label_binarizer.inverse_transform(y[self.val_rows])
        else:
            self.train_rows, self.val_rows = np.arange(X.shape[0]), None
        n_samples = self.train_rows.shape[0]
        self.n_samples = n_samples
        self.sample_idx = np.arange(n_samples, dtype=int)
        if est.batch_size == "auto":
            batch_size = min(200, n_samples)
        else:
            if est.batch_size > n_samples:
                warnings.warn("Got `batch_size` less than 1 or larger than sample size. It is going to be clipped")
            batch_size = np.clip(est.batch_size, 1, n_samples)
        self.batch_size = int(batch_size)
        self.slices = list(gen_batches(n_samples, self.batch_size))
        self.t = 0
        est.n_iter_ = 0

    def epoch_inputs(self):
        """-> (row order of this epoch into the training rows, learning rate of every step)."""
        est = self.est
        if est.shuffle:
            self.sample_idx = shuffle(self.sample_idx, random_state=est._random_state)
        lrs = np.empty(len(self.slices))
        for k in range(len(self.slices)):   # AdamOptimizer._get_updates, step by step
            self.t += 1
            lrs[k] = est.learning_rate_init * np.sqrt(1 - est.beta_2 ** self.t) / (1 - est.beta_1 ** self.t)
        return self.sample_idx, lrs

    def after_epoch(self, losses, val_proba=None):
        """The epoch's batch losses (and validation probabilities) -> (snapshot now, stop)."""
        est = self.est
        accumulated_loss = 0.0
        for batch_loss, sl in zip(losses, self.slices):
            accumulated_loss += batch_loss * (sl.stop - sl.start)
        est.n_iter_ += 1
        est.loss_ = accumulated_loss / self.n_samples
        est.t_ += self.n_samples
        est.loss_curve_.append(est.loss_)
        if est.verbose:
            print("Iteration %d, loss = %.8f" % (est.n_iter_, est.loss_))
        snap = False
        if self.early_stopping:
            p = val_proba
            y_pred = est._label_binarizer.inverse_transform(p.ravel() if est.n_outputs_ == 1 else p)
            val_score = accuracy_score(self.y_val, y_pred)
            est.validation_scores_.append(val_score)
            if est.verbose:
                print("Validation score: %f" % val_score)
            if val_score < est.best_validation_score_ + est.tol:
                est._no_improvement_count += 1
            else:
                est._no_improvement_count = 0
            if val_score > est.best_validation_score_:
                est.best_validation_score_ = val_score
                snap = True
        else:
            if est.loss_curve_[-1] > est.best_loss_ - est.tol:
                est._no_improvement_count += 1
            else:
                est._no_improvement_count = 0
            if est.loss_curve_[-1] < est.best_loss_:
                est.best_loss_ = est.loss_curve_[-1]
        if est._no_improvement_count > est.n_iter_no_change:
            if est.verbose:
                what = "Validation score" if self.early_stopping else "Training loss"
                print("%s did not improve more than tol=%f for %d consecutive epochs. Stopping."
                      % (what, est.tol, est.n_iter_no_change))
            return snap, True   # AdamOptimizer.trigger_stopping always stops
        if est.n_iter_ == est.max_iter:
            warnings.warn("Stochastic Optimizer: Maximum iterations (%d) reached and the optimization hasn't "
                          "converged yet." % est.max_iter, ConvergenceWarning)
            return snap, True
        return snap, False

    def finish(self, coefs, intercepts):
        est = self.est
        est.coefs_, est.intercepts_ = coefs, intercepts
        if self.early_stopping:
            est._best_coefs = [c.copy() for c in est.coefs_]
            est._best_intercepts = [b.copy() for b in est.intercepts_]
        if not all(np.isfinite(w).all() for w in est.coefs_ + est.intercepts_):
            raise ValueError("Solver produced non-finite parameter weights. The input data may contain large values and "
                             "need to be preprocessed.")


def _split_rows(n, random_state, validation_fraction, stratify=None):
    """sklearn's early-stopping ``train_test_split`` run on row indices -> (training rows, validation rows); the same
    partition, in the same order, as splitting X and y themselves."""
    return train_test_split(np.arange(n), random_state=random_state, test_size=validation_fraction, stratify=stratify)


# ---------------------------------------------------------------------------------------------------------------------
# Many fits at once: the group handle and the lockstep runner behind DeviceGridSearchCV
# ---------------------------------------------------------------------------------------------------------------------
class DeviceGroupSteps:
    """The steps of many Adam fits of one architecture and batch size on the device (one ``ie_mlp_group`` handle); the
    group runner's step backend.  Model j trains on rows of the shared X / Y that the runner names each epoch."""

    dtype = np.float32

    def __init__(self, layer_units, n_models: int, batch_size: int, device: int = 0):
        self._lib = _lib.load()
        self.units = [int(u) for u in layer_units]
        dims = (C.c_int32 * len(self.units))(*self.units)
        h = C.c_void_p()
        check(self._lib.ie_mlp_group_create(len(self.units) - 1, dims, int(n_models), int(batch_size), device,
                                            C.byref(h)))
        self._h = h
        self.n_val = {}

    @staticmethod
    def capacity(layer_units, batch_size: int, device: int = 0) -> int:
        """Models of this shape that fit in 80 % of the device's free memory."""
        lib = _lib.load()
        units = [int(u) for u in layer_units]
        dims = (C.c_int32 * len(units))(*units)
        per, n = C.c_int64(), C.c_int32()
        check(lib.ie_mlp_group_capacity(len(units) - 1, dims, int(batch_size), device, 0.8, C.byref(per), C.byref(n)))
        return int(n.value)

    def set_data(self, X, Y):
        X = np.ascontiguousarray(X, dtype=np.float32)
        Y = np.ascontiguousarray(Y, dtype=np.uint8)
        check(self._lib.ie_mlp_group_set_data(self._h, X.ctypes.data, Y.ctypes.data, X.shape[0]))

    def set_model(self, j, coefs, intercepts, alpha, beta_1, beta_2, epsilon, val_rows=None):
        for l, (w, b) in enumerate(zip(coefs, intercepts)):
            w = np.ascontiguousarray(w, dtype=np.float32)
            b = np.ascontiguousarray(b, dtype=np.float32)
            check(self._lib.ie_mlp_group_set_layer(self._h, j, l, w.ctypes.data, b.ctypes.data))
        check(self._lib.ie_mlp_group_set_hyper(self._h, j, float(alpha), float(beta_1), float(beta_2), float(epsilon)))
        if val_rows is not None:
            rows = np.ascontiguousarray(val_rows, dtype=np.int32)
            check(self._lib.ie_mlp_group_set_validation(self._h, j, rows.ctypes.data, len(rows)))
            self.n_val[j] = len(rows)

    def epoch(self, models, rows, lrs):
        """models[i] steps on X rows rows[i] with learning rates lrs[i] -> each model's batch losses."""
        ids = np.ascontiguousarray(models, dtype=np.int32)
        n_rows = np.array([len(r) for r in rows], dtype=np.int64)
        flat = np.ascontiguousarray(np.concatenate(rows), dtype=np.int32)
        lr = np.ascontiguousarray(np.concatenate(lrs), dtype=np.float64)
        out = np.empty(lr.size, dtype=np.float64)
        check(self._lib.ie_mlp_group_epoch(self._h, len(ids), ids.ctypes.data, n_rows.ctypes.data, flat.ctypes.data,
                                           lr.ctypes.data, out.ctypes.data))
        return np.split(out, np.cumsum([len(x) for x in lrs])[:-1])

    def val_proba(self, j):
        probs = np.empty((self.n_val[j], self.units[-1]), dtype=np.float32)
        check(self._lib.ie_mlp_group_validation_proba(self._h, j, probs.ctypes.data))
        return probs

    def snapshot(self, j):
        check(self._lib.ie_mlp_group_snapshot(self._h, j, 0))

    def params(self, j, best: bool = False):
        coefs, intercepts = [], []
        for l in range(len(self.units) - 1):
            w = np.empty((self.units[l], self.units[l + 1]), dtype=np.float32)
            b = np.empty(self.units[l + 1], dtype=np.float32)
            check(self._lib.ie_mlp_group_get_layer(self._h, j, l, int(best), w.ctypes.data, b.ctypes.data))
            coefs.append(w)
            intercepts.append(b)
        return coefs, intercepts

    @property
    def launches(self) -> int:
        return int(self._lib.ie_mlp_group_launch_count(self._h))

    def last_epoch_ms(self) -> float:
        ms = C.c_float()
        check(self._lib.ie_mlp_group_last_epoch_ms(self._h, C.byref(ms)))
        return ms.value

    def close(self):
        if getattr(self, "_h", None):
            self._lib.ie_mlp_group_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_GROUP_CAP = None   # tests only: an upper bound on the models of one group (None: free device memory decides)


class _Trained:
    """The outcome of one fit trained by ``_train_groups``: the fitted estimator or the exception its fit raised, the
    warnings it emitted and its share of the training time."""

    def __init__(self, est):
        self.est, self.error, self.warnings, self.seconds = est, None, [], 0.0


def _captured(rec, fn, *args):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            return fn(*args)
        finally:
            rec.warnings.extend(w)


def _train_groups(jobs, X, y, group_steps_cls=DeviceGroupSteps, device=0, stats=None):
    """Train every fit of `jobs` -- (estimator, row indices of X / y it is fitted on) -- in lockstep groups of one
    architecture and batch size, each fit deciding exactly as ``_fit_with`` would -> one ``_Trained`` per job."""
    out = [_Trained(est) for est, _ in jobs]
    fits = {}
    for i, (est, rows) in enumerate(jobs):
        t0 = time.perf_counter()
        try:
            fits[i] = _captured(out[i], _Fit, est, _safe_indexing(X, rows), _safe_indexing(y, rows),
                                group_steps_cls.dtype)
            fits[i].X = fits[i].y = None   # the group reads the shared X / Y through row maps: keep no copy per fit
        except Exception as e:   # refused: replayed as this fit's own exception
            out[i].error = e
        out[i].seconds += time.perf_counter() - t0
    # shared data: X once in the backend's dtype; Y as each fit's label binarizer encodes the whole y (one group per
    # encoding, in practice one)
    Xs = _as_dense(X, group_steps_cls.dtype)
    yd = np.asarray(y)
    encodings, groups = {}, {}
    for i, f in fits.items():
        lb = f.est._label_binarizer   # its encoding of y depends only on the target type and the classes
        enc = (lb.y_type_, tuple(np.asarray(lb.classes_).tolist()))
        if enc not in encodings:
            encodings[enc] = (len(encodings), lb.transform(yd).reshape(len(yd), -1).astype(np.uint8))
        key = (tuple(f.layer_units), f.batch_size, encodings[enc][0])
        groups.setdefault(key, (encodings[enc][1], []))[1].append(i)
    for (units, bs, _), (Y, members) in groups.items():
        cap = group_steps_cls.capacity(units, bs, device) if hasattr(group_steps_cls, "capacity") else len(members)
        if _GROUP_CAP is not None:
            cap = min(cap, _GROUP_CAP)
        if cap < 1:
            raise MemoryError(f"one model of shape {list(units)} at batch size {bs} does not fit in free device memory")
        for g0 in range(0, len(members), cap):
            _train_one_group([(i, fits[i], jobs[i][1]) for i in members[g0:g0 + cap]], Xs, Y, units, bs, out,
                             group_steps_cls, device, stats)
    return out


def _as_dense(X, dtype):
    if hasattr(X, "toarray"):
        X = X.toarray()
    X = np.asarray(X)
    return np.asarray(X, dtype=dtype or (X.dtype if X.dtype in (np.float32, np.float64) else np.float64))


def _train_one_group(members, X, Y, units, bs, out, group_steps_cls, device, stats):
    t0 = time.perf_counter()
    steps = group_steps_cls(units, len(members), bs, device)
    try:
        steps.set_data(X, Y)
        for j, (i, f, rows) in enumerate(members):
            est = f.est
            val = rows[f.val_rows] if f.early_stopping else None
            steps.set_model(j, est.coefs_, est.intercepts_, est.alpha, est.beta_1, est.beta_2, est.epsilon, val)
            if f.early_stopping:
                steps.snapshot(j)
        active = list(range(len(members)))
        while active:
            orders, lrs = [], []
            for j in active:
                i, f, rows = members[j]
                order, lr = _captured(out[i], f.epoch_inputs)
                orders.append(rows[f.train_rows[order]])   # the fit's k-th training row is X row rows[train_rows[k]]
                lrs.append(lr)
            losses = steps.epoch(active, orders, lrs)
            if stats is not None:
                stats.append((len(active), max(len(x) for x in lrs), steps.last_epoch_ms(), steps.launches))
            still = []
            for j, loss in zip(active, losses):
                i, f, _ = members[j]
                p = steps.val_proba(j) if f.early_stopping else None
                snap, done = _captured(out[i], f.after_epoch, loss, p)
                if snap:
                    steps.snapshot(j)
                if not done:
                    still.append(j)
            active = still
        for j, (i, f, _) in enumerate(members):
            coefs, intercepts = steps.params(j, best=f.early_stopping)
            try:
                _captured(out[i], f.finish, coefs, intercepts)
            except Exception as e:
                out[i].error = e
    finally:
        steps.close()
    share = (time.perf_counter() - t0) / len(members)
    for i, _, _ in members:
        out[i].seconds += share


_REPLAY = threading.local()


def _replay_fit(est, X, y, queue, sample_weight=None):
    """Install the next pre-trained fit of a ``DeviceGridSearchCV`` into `est` (the search's own fit call); the
    refusals of the call itself (``sample_weight``) are made first, as the serial fit makes them."""
    if not queue:
        raise RuntimeError("DeviceGridSearchCV: more fits requested than were trained")
    want_params, Xd, yd, rows, rec = queue.pop(0)
    got = est.get_params(deep=False)
    same = got.keys() == want_params.keys() and all(_same_param(got[k], want_params[k]) for k in got)
    Xa = X.toarray() if hasattr(X, "toarray") else np.asarray(X)
    # the fit's data are the rows it was trained on: every label, and the first and last row of X
    if (not same or Xa.shape != (len(rows),) + Xd.shape[1:] or not np.array_equal(np.asarray(y), yd[rows])
            or not np.array_equal(Xa[[0, -1]], Xd[rows[[0, -1]]])):
        raise RuntimeError("DeviceGridSearchCV: the search asked for a fit in a different order or on different data "
                           "than the one trained for it")
    est._validate_params()
    est._refuse(sample_weight)
    for w in rec.warnings:
        warnings.warn(w.message, w.category)
    if rec.error is not None:
        raise rec.error
    est.__dict__.update(rec.est.__dict__)
    return est


def _same_param(a, b):
    if isinstance(a, np.random.RandomState) and isinstance(b, np.random.RandomState):
        return True   # each clone holds its own copy of the same generator
    try:
        return bool(a == b)
    except Exception:
        return a is b


class _FixedSplits:
    """A splitter that yields splits computed before (sklearn's ``cv`` protocol)."""

    def __init__(self, splits):
        self.splits = splits

    def split(self, X=None, y=None, groups=None, **kw):
        yield from self.splits

    def get_n_splits(self, X=None, y=None, groups=None, **kw):
        return len(self.splits)


class DeviceGridSearchCV(GridSearchCV):
    """sklearn's ``GridSearchCV`` whose (candidate, split) fits train together on the H100.

    The estimator must be a ``DeviceMLPClassifier``.  Every fit of the search is first trained by the lockstep group
    runner: fits of one architecture and batch size share one ``ie_mlp_group`` handle and every step is one launch per
    stage for all of them, each fit bit-identical to its own ``DeviceMLPClassifier.fit``.  Then sklearn's own search
    runs -- candidates, splits, scoring on the host, ``error_score``, ``cv_results_``, ``best_*`` and the refit -- and
    each fit it asks for is installed from what was trained; a fit asked for in another order or on other data raises.
    A candidate the estimator refuses fails as it fails in a serial search, and so does a search given
    ``sample_weight``.  The splits are drawn once, so a shuffling splitter without a seed trains and scores the same
    splits.  X may be anything sklearn's search indexes (an array, a list of rows, a DataFrame, a sparse matrix).

    ``n_jobs`` is accepted and ignored (the fits share one GPU).  ``cv_results_``'s ``mean_fit_time`` and
    ``std_fit_time`` are each fit's share of its group's training time plus its own host work.  With an int or a
    ``RandomState`` as the estimator's ``random_state`` the search reproduces the serial search bit for bit; with
    ``None`` the fits draw from NumPy's global generator in lockstep order -- a valid search, but not the draws a serial
    one (itself not reproducible) would make."""

    _group_steps_cls = DeviceGroupSteps

    def fit(self, X, y=None, **params):
        if not isinstance(self.estimator, DeviceMLPClassifier):
            raise ValueError(f"DeviceGridSearchCV searches a DeviceMLPClassifier, not {type(self.estimator).__name__} "
                             "(use sklearn's GridSearchCV on the host)")
        n_jobs = self.n_jobs
        self._search_args = (X, y, params)
        self.n_jobs = None
        try:
            super().fit(X, y, **params)
        finally:
            self.n_jobs = n_jobs
            del self._search_args
            _REPLAY.queue = None
        return self

    def _run_search(self, evaluate_candidates):
        X, y, params = self._search_args
        candidates = list(ParameterGrid(self.param_grid))
        splits = [(np.asarray(tr), np.asarray(te)) for tr, te in self._checked_cv_orig.split(X, y, params.get("groups"))]
        base = clone(self.estimator)
        jobs = []
        for cand in candidates:
            for train, _ in splits:
                est = clone(base).set_params(**clone(cand, safe=False))
                jobs.append((est, np.asarray(train)))
        yarr = np.asarray(y)
        trained = _train_groups(jobs, X, y, self._group_steps_cls, self.estimator.device)
        Xd = X.toarray() if hasattr(X, "toarray") else np.asarray(X)
        queue = [(est.get_params(deep=False), Xd, yarr, rows, rec) for (est, rows), rec in zip(jobs, trained)]
        # fit times: each fit's share of its group (the replayed fit itself takes no time)
        self._fit_seconds = np.array([r.seconds for r in trained]).reshape(len(candidates), len(splits))
        del jobs, trained   # each trained fit is released once the search has scored it
        _REPLAY.queue = queue
        try:
            # the splits the fits were trained on, not a second draw of a splitter that may shuffle
            evaluate_candidates(candidates, cv=_FixedSplits(splits))
        finally:
            _REPLAY.queue = None
            del self._fit_seconds
        if queue:
            raise RuntimeError(f"DeviceGridSearchCV: {len(queue)} trained fits were never asked for")

    def _format_results(self, candidate_params, n_splits, out, more_results=None):
        results = super()._format_results(candidate_params, n_splits, out, more_results)
        secs = getattr(self, "_fit_seconds", None)
        if secs is not None and secs.shape == (len(candidate_params), n_splits):
            mean = np.average(secs, axis=1)
            results["mean_fit_time"] = mean
            results["std_fit_time"] = np.sqrt(np.average((secs - mean[:, None]) ** 2, axis=1))
        return results
