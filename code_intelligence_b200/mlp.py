"""Label_Microservice MLP head on the H100.

``MLPWrapper`` keeps the reference's interface (py/label_microservice/mlp.py:14-138) -- the constructor, ``fit``,
``predict_probabilities``, ``find_probability_thresholds``, ``grid_search``, ``save_model`` / ``load_model`` -- but
``predict_probabilities`` (mlp.py:56-63, sklearn ``MLPClassifier.predict_proba``) runs the fitted network's forward
pass relu(relu(X W0 + b0) W1 + b1) ... -> sigmoid through the wgmma GEMM kernel behind ``ie_mlp_*``
(include/issue_emb_b200.h).  ``fit`` and ``grid_search`` train whatever estimator the wrapper holds: a plain sklearn
``MLPClassifier`` fits on the host, ``mlp_train.DeviceMLPClassifier`` fits on the GPU (search it with ``n_jobs=1``).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import check


PR_MAX_SAMPLES = 16384   # ie::kPrMaxSamples


def pr_thresholds_host(scores, truth, precision_threshold, recall_threshold):
    """The reference's per-label loop (mlp.py:81-98) on sklearn's precision_recall_curve -> (thr, prec, rec) lists."""
    from sklearn.metrics import precision_recall_curve
    import warnings
    thr_o, prec_o, rec_o = [], [], []
    for label in range(truth.shape[1]):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")              # "No positive class found": recall is set to one, as on the GPU
            prec, rec, thr = precision_recall_curve(truth[:, label], scores[:, label])
        prec, rec = prec[:-1], rec[:-1]                  # the curve's last point has no threshold
        ok = (prec >= precision_threshold) & (rec >= recall_threshold) & (prec > 0.0)
        if ok.any():
            k = int(np.argmax(np.where(ok, prec, -1.0)))  # first index of the best qualifying precision
            thr_o.append(float(thr[k])); prec_o.append(float(prec[k])); rec_o.append(float(rec[k]))
        else:
            thr_o.append(None); prec_o.append(0.0); rec_o.append(0.0)
    return thr_o, prec_o, rec_o


def pr_thresholds(scores, truth, precision_threshold, recall_threshold, device: int = 0):
    """Same on the GPU (``ie_pr_thresholds``, csrc/pr_curve.cu): scores (n, L) float32, truth (n, L) 0/1, n <= 16384.
    Raises ValueError on NaN or infinite scores, as sklearn's precision_recall_curve does."""
    scores = np.ascontiguousarray(scores, dtype=np.float32)
    if not np.isfinite(scores).all():
        raise ValueError("scores contain NaN or infinity")
    lib = _lib.load()
    truth = np.ascontiguousarray(np.asarray(truth) != 0, dtype=np.uint8)
    n, L = scores.shape
    assert truth.shape == (n, L)
    thr = np.empty(L, dtype=np.float32)
    prec = np.empty(L, dtype=np.float64)
    rec = np.empty(L, dtype=np.float64)
    check(lib.ie_pr_thresholds(scores.ctypes.data, truth.ctypes.data, n, L, float(precision_threshold),
                               float(recall_threshold), thr.ctypes.data, prec.ctypes.data, rec.ctypes.data, device, 0, None))
    return [None if np.isnan(t) else float(t) for t in thr], [float(p) for p in prec], [float(r) for r in rec]


class MLPHead:
    """Owner of an ``ie_mlp`` handle: weights in sklearn layout (coefs_[l] is [fan_in, fan_out])."""

    def __init__(self, coefs: Sequence[np.ndarray], intercepts: Sequence[np.ndarray], device: int = 0):
        self._lib = _lib.load()
        if len(coefs) != len(intercepts) or len(coefs) < 1:
            raise ValueError("coefs / intercepts mismatch")
        dims = [int(coefs[0].shape[0])] + [int(w.shape[1]) for w in coefs]
        for l, (w, b) in enumerate(zip(coefs, intercepts)):
            if w.shape != (dims[l], dims[l + 1]) or b.shape != (dims[l + 1],):
                raise ValueError(f"layer {l}: coef {w.shape} intercept {b.shape} do not chain from {dims[l]}")
        self.dims = dims
        arr = (C.c_int32 * len(dims))(*dims)
        h = C.c_void_p()
        check(self._lib.ie_mlp_create(len(coefs), arr, device, C.byref(h)))
        self._h = h
        for l, (w, b) in enumerate(zip(coefs, intercepts)):
            w = np.ascontiguousarray(w, dtype=np.float32)
            b = np.ascontiguousarray(b, dtype=np.float32)
            check(self._lib.ie_mlp_load_layer(self._h, l, w.ctypes.data, b.ctypes.data))

    @classmethod
    def from_sklearn(cls, clf, device: int = 0) -> "MLPHead":
        est = getattr(clf, "best_estimator_", clf)  # GridSearchCV delegates (mlp.py:114)
        if getattr(est, "out_activation_", "logistic") != "logistic" or getattr(est, "activation", "relu") != "relu":
            raise ValueError("only relu hidden layers with a logistic (multilabel) output are supported")
        return cls(est.coefs_, est.intercepts_, device)

    def predict_proba(self, X) -> np.ndarray:
        X = np.ascontiguousarray(np.asarray(X), dtype=np.float32)
        if X.ndim != 2 or X.shape[1] != self.dims[0]:
            raise ValueError(f"X must be (n, {self.dims[0]}), got {X.shape}")
        probs = np.empty((X.shape[0], self.dims[-1]), dtype=np.float32)
        if X.shape[0]:
            check(self._lib.ie_mlp_predict_proba(self._h, X.ctypes.data, X.shape[0], probs.ctypes.data, 0, None))
        return probs

    def predict_proba_device(self, X, out=None, stream=None):
        """Asynchronous device-resident variant: X cuda float32 (n, D_in) -> cuda float32 (n, n_labels) on `stream`
        (default: torch's current stream)."""
        import torch
        assert X.is_cuda and X.dtype == torch.float32 and X.dim() == 2 and X.shape[1] == self.dims[0]
        X = X.contiguous()
        if out is None:
            out = torch.empty((X.shape[0], self.dims[-1]), dtype=torch.float32, device=X.device)
        s = stream if stream is not None else torch.cuda.current_stream(X.device)
        if X.shape[0]:
            check(self._lib.ie_mlp_predict_proba(self._h, X.data_ptr(), X.shape[0], out.data_ptr(),
                                                 _lib.IE_FLAG_DEVICE_PTRS, C.c_void_p(s.cuda_stream)))
        return out

    def close(self):
        if getattr(self, "_h", None):
            self._lib.ie_mlp_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MLPWrapper:
    """Wrapper for Multi-Layer Perceptron classifier (mirror of py/label_microservice/mlp.py:14)."""

    def __init__(self, clf, model_file="model.dpkl", precision_threshold=0.7, recall_threshold=0.5,
                 load_from_model=False, device: int = 0):
        self._device = device
        self._head: Optional[MLPHead] = None
        if clf:
            self.clf = clf
        elif load_from_model:
            self.load_model(model_file=model_file)
        else:
            raise Exception("You need to pass a MLPClassifier object to the wrapper")
        self.model_file = model_file
        self.precision_threshold = precision_threshold
        self.recall_threshold = recall_threshold
        self.precisions = None
        self.probability_thresholds = None
        self.recalls = None
        self.total_labels_count = None

    def fit(self, X, y):
        """Train the classifier: on the host for sklearn's MLPClassifier, on the GPU for mlp_train.DeviceMLPClassifier."""
        self.clf.fit(X, y)
        self._head = None

    def predict_probabilities(self, X):
        """Predict probabilities of all labels for data -> (n_samples, n_classes); on the H100.  Like sklearn's
        predict_proba, a network with one output unit (one label column, or a 1-D y) gives (n, 2) = [1 - p, p]."""
        if self._head is None:
            self._head = MLPHead.from_sklearn(self.clf, self._device)
        p = self._head.predict_proba(X)
        if p.shape[1] == 1:
            return np.hstack([1.0 - p, p])
        return p

    def find_probability_thresholds(self, X, y, test_size=0.3):
        """mlp.py:65-98: hold out ``test_size`` of the data (random_state 1234), fit on the rest, and for every label keep
        the probability threshold with the highest precision among the points of its precision-recall curve that meet
        both ``precision_threshold`` and ``recall_threshold`` (first such point on ties; ``None`` when no point
        qualifies, which makes the label unpredictable, repo_specific_model.py:138-141).  ``fit`` trains the wrapped
        estimator (on the GPU for mlp_train.DeviceMLPClassifier); the
        hold-out ``predict_proba`` and the per-label curve search run on the GPU (``ie_pr_thresholds``: sort + prefix sum +
        argmax per label in one kernel); hold-out sets above 16384 rows use sklearn's curve on the host."""
        from sklearn.model_selection import train_test_split
        X_train, X_test, y_train, y_test = train_test_split(X, y, test_size=test_size, random_state=1234)
        self.fit(X_train, y_train)
        truth = np.asarray(y_test)
        self.total_labels_count = truth.shape[1]
        # label l is scored by column l, as the reference indexes y_pred[:, label]: with one label column that is the
        # [1 - p, p] head's column 0
        scores = self.predict_probabilities(X_test)[:, :self.total_labels_count]
        if truth.shape[0] <= PR_MAX_SAMPLES:
            thr, prec, rec = pr_thresholds(scores, truth, self.precision_threshold, self.recall_threshold, self._device)
        else:
            thr, prec, rec = pr_thresholds_host(scores, truth, self.precision_threshold, self.recall_threshold)
        self.probability_thresholds = {l: thr[l] for l in range(self.total_labels_count)}
        self.precisions = {l: prec[l] for l in range(self.total_labels_count)}
        self.recalls = {l: rec[l] for l in range(self.total_labels_count)}

    def grid_search(self, params=None, cv=5, n_jobs=-1):
        from sklearn.model_selection import GridSearchCV
        if not params:
            params = {'hidden_layer_sizes': [(100,), (200,), (400,), (50, 50), (100, 100), (200, 200)],
                      'alpha': [.001, .01, .1, 1, 10],
                      'learning_rate': ['constant', 'adaptive'],
                      'learning_rate_init': [.001, .01, .1]}
        from .mlp_train import DeviceGridSearchCV, DeviceMLPClassifier
        # a device estimator's fits train together on the GPU (DeviceGridSearchCV ignores n_jobs)
        search = DeviceGridSearchCV if isinstance(self.clf, DeviceMLPClassifier) else GridSearchCV
        self.clf = search(self.clf, params, cv=cv, n_jobs=n_jobs)
        self._head = None

    def save_model(self, model_file=None):
        import dill as dpickle
        if model_file:
            self.model_file = model_file
        with open(self.model_file, 'wb') as f:
            dpickle.dump(self.clf, f)

    def load_model(self, model_file=None):
        import dill as dpickle
        if model_file:
            self.model_file = model_file
        if not os.path.exists(self.model_file):
            raise Exception(f"Model path {self.model_file} does not exist")
        with open(self.model_file, 'rb') as f:
            self.clf = dpickle.load(f)
        self._head = None


def filter_predictions(label_names: Sequence[str], probabilities: Sequence[float],
                       label_thresholds: Dict[str, Optional[float]]) -> Dict[str, float]:
    """The end-to-end "labels" definition of RepoSpecificLabelModel.predict_issue_labels
    (py/label_microservice/repo_specific_model.py:126-146): zip names with probabilities, drop a label when its
    threshold is falsy (None / 0) or the probability is below it."""
    predictions = dict(zip(label_names, probabilities))
    labels_to_remove = []
    for label, probability in predictions.items():
        if not label_thresholds[label]:
            labels_to_remove.append(label)
            continue
        if probability < label_thresholds[label]:
            labels_to_remove.append(label)
    for l in labels_to_remove:
        del predictions[l]
    return predictions


def calculate_auc(predictions, y_holdout, label_columns):
    """Per-label ROC AUC and positive counts (py/label_microservice/mlp.py:140-160; evaluation helper of the training
    notebooks, host-side sklearn).  Returns the DataFrame the reference ``display()``s."""
    import pandas as pd
    from sklearn.metrics import roc_auc_score
    predictions, y_holdout = np.asarray(predictions), np.asarray(y_holdout)
    auc_scores = [roc_auc_score(y_true=y_holdout[:, i], y_score=predictions[:, i]) for i, _ in enumerate(label_columns)]
    counts = y_holdout.sum(axis=0)
    return pd.DataFrame({'label': list(label_columns), 'auc': auc_scores, 'count': counts})
