"""ORACLE (test infrastructure, NOT product code): sklearn 1.9's Adam fit of MLPClassifier restated in numpy.

``NumpySteps`` is a step backend for the host driver of code_intelligence_b200/mlp_train.py (``DeviceMLPClassifier.
_fit_with``): the same interface as the device's ``DeviceSteps``, with every step computed by the numpy expressions of
sklearn's ``_backprop`` / ``_forward_pass_fast`` / ``AdamOptimizer`` in the data's own dtype.  Run on float64 data, the
driver with this backend reproduces ``MLPClassifier.fit`` bit for bit, which is what proves that the driver makes
sklearn's random draws and decisions.

``adam_f32`` is the float32 Adam step the device implements (csrc/mlp_train.cu adam_kernel), written with explicit
roundings instead of NumPy's promotion rules: each f32 product and sum rounded on its own, the learning rate and the
update in float64, the parameter rounded once from f64(p) + update.
"""
from __future__ import annotations

import numpy as np
from scipy.special import expit, xlogy
from sklearn.utils import gen_batches


def binary_log_loss(y_true, y_prob):
    """sklearn.neural_network._base.binary_log_loss (no sample weights)."""
    eps = np.finfo(y_prob.dtype).eps
    y_prob = np.clip(y_prob, eps, 1 - eps)
    return -np.average(xlogy(y_true, y_prob) + xlogy(1 - y_true, 1 - y_prob), axis=0).sum()


def forward(X, coefs, intercepts):
    """sklearn _forward_pass: [X, relu hidden activations..., logistic output]."""
    acts = [X]
    for i, (w, b) in enumerate(zip(coefs, intercepts)):
        a = acts[i] @ w
        a += b
        if i != len(coefs) - 1:
            np.maximum(a, 0, out=a)
        acts.append(a)
    expit(acts[-1], out=acts[-1])
    return acts


def backprop(X, y, coefs, intercepts, alpha):
    """sklearn _backprop without sample weights -> (loss, coef_grads, intercept_grads, activations, deltas)."""
    n = X.shape[0]
    acts = forward(X, coefs, intercepts)
    loss = binary_log_loss(y, acts[-1])
    values = 0
    for s in coefs:
        s = s.ravel()
        values += np.dot(s, s)
    loss += (0.5 * alpha) * values / n
    last = len(coefs) - 1
    deltas = [None] * len(coefs)
    cg, ig = [None] * len(coefs), [None] * len(coefs)

    def grad(layer):
        cg[layer] = acts[layer].T @ deltas[layer]
        cg[layer] += alpha * coefs[layer]
        cg[layer] /= n
        ig[layer] = np.sum(deltas[layer], axis=0) / n

    deltas[last] = acts[-1] - y
    grad(last)
    for i in range(last, 0, -1):
        deltas[i - 1] = deltas[i] @ coefs[i].T
        deltas[i - 1][acts[i] == 0] = 0
        grad(i - 1)
    return loss, cg, ig, acts, deltas


class NumpySteps:
    """Step backend in numpy, in the dtype of the data it is given (the driver passes X's own dtype)."""

    dtype = None

    def __init__(self, layer_units, device: int = 0):
        self.units = list(layer_units)
        self.t = 0

    def set_params(self, coefs, intercepts):
        self.coefs = [np.array(c) for c in coefs]
        self.intercepts = [np.array(b) for b in intercepts]
        self.ms = [np.zeros_like(p) for p in self.coefs + self.intercepts]
        self.vs = [np.zeros_like(p) for p in self.coefs + self.intercepts]
        self.best = self.params()

    def params(self, best: bool = False):
        if best:
            return [c.copy() for c in self.best[0]], [b.copy() for b in self.best[1]]
        return [c.copy() for c in self.coefs], [b.copy() for b in self.intercepts]

    def set_data(self, X, Y, X_val=None):
        self.X, self.Y, self.X_val = X, Y, X_val

    def epoch(self, order, batch_size, lrs, alpha, beta_1, beta_2, epsilon):
        losses = []
        for k, sl in enumerate(gen_batches(len(order), batch_size)):
            idx = order[sl]
            loss, cg, ig, _, _ = backprop(self.X[idx], self.Y[idx], self.coefs, self.intercepts, alpha)
            losses.append(loss)
            grads = cg + ig
            # sklearn AdamOptimizer._get_updates + update_params
            self.ms = [beta_1 * m + (1 - beta_1) * g for m, g in zip(self.ms, grads)]
            self.vs = [beta_2 * v + (1 - beta_2) * (g ** 2) for v, g in zip(self.vs, grads)]
            lr = lrs[k]
            for p, m, v in zip(self.coefs + self.intercepts, self.ms, self.vs):
                p += -lr * m / (np.sqrt(v) + epsilon)
        return np.array(losses, dtype=np.float64)

    def val_proba(self):
        return forward(self.X_val, self.coefs, self.intercepts)[-1]

    def snapshot(self):
        self.best = self.params()

    def close(self):
        pass


def adam_f32(params, grads, ms, vs, lr_t, beta_1=0.9, beta_2=0.999, epsilon=1e-8):
    """One float32 Adam step with explicit roundings -> (params, ms, vs), new arrays.  lr_t is the float64 learning rate
    learning_rate_init * sqrt(1 - beta_2^t) / (1 - beta_1^t)."""
    f32, f64 = np.float32, np.float64
    b1, omb1, b2, omb2, e = f32(beta_1), f32(1 - beta_1), f32(beta_2), f32(1 - beta_2), f32(epsilon)
    out_p, out_m, out_v = [], [], []
    for p, g, m, v in zip(params, grads, ms, vs):
        p, g, m, v = (np.asarray(a, dtype=f32) for a in (p, g, m, v))
        m = (b1 * m).astype(f32) + (omb1 * g).astype(f32)
        v = (b2 * v).astype(f32) + (omb2 * (g * g).astype(f32)).astype(f32)
        den = (np.sqrt(v).astype(f32) + e).astype(f32)
        upd = (-f64(lr_t) * m.astype(f64)) / den.astype(f64)
        out_p.append((p.astype(f64) + upd).astype(f32))
        out_m.append(m.astype(f32))
        out_v.append(v.astype(f32))
    return out_p, out_m, out_v
