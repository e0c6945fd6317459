"""ORACLE (test infrastructure, NOT product code): sklearn 1.9's Adam fit of MLPClassifier restated in numpy.

``NumpySteps`` is a step backend for the host driver of code_intelligence_b200/mlp_train.py (``DeviceMLPClassifier.
_fit_with``): the same interface as the device's ``DeviceSteps``, with every step computed by the numpy expressions of
sklearn's ``_backprop`` / ``_forward_pass_fast`` / ``AdamOptimizer`` in the data's own dtype.  Run on float64 data, the
driver with this backend reproduces ``MLPClassifier.fit`` bit for bit, which is what proves that the driver makes
sklearn's random draws and decisions.

``adam_f32`` is the float32 Adam step the device implements (csrc/mlp_train.cu adam_kernel), written with explicit
roundings instead of NumPy's promotion rules: each f32 product and sum rounded on its own, the learning rate and the
update in float64, the parameter rounded once from f64(p) + update.

``check_step`` checks one training step of the device (``DeviceSteps.debug_step``) stage by stage, each stage fed the
device's own f32 inputs, against the bounds of DESIGN.md section 2 "Bounds of the training step".
"""
from __future__ import annotations

import numpy as np
import torch
from scipy.special import expit, xlogy
from sklearn.utils import gen_batches

from . import device_numerics as DN


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


def _check_in(name, dev, lo, hi, ref, stats):
    """dev inside [lo, hi] elementwise; stats[name] = max |dev - ref| / eps with eps the wider side of the interval."""
    dev = torch.as_tensor(np.asarray(dev, dtype=np.float64), device=lo.device)
    ok = (dev >= lo) & (dev <= hi)
    eps = torch.maximum(hi - ref, ref - lo).clamp_min(1e-30)
    stats[name] = float(((dev - ref).abs() / eps).max())
    assert bool(ok.all()), (name, int((~ok).sum()), stats[name])


def check_step(out, X, Y, rows, coefs, intercepts, alpha, device=None) -> dict:
    """Every stage of one device step on rows `rows` of (X, Y) at parameters (coefs, intercepts), fed the device's own
    f32 inputs from `out` (``DeviceSteps.debug_step``), inside its bound: hidden activations and p (``gemm_interval``,
    segs 3), the output delta p - y exactly, the masked deltas (exactly 0 where the device's activation is 0), the coef
    gradients through the monotone f32 add and divide, the intercept gradients and the f64 loss.  An AssertionError
    whose first item names the stage on the first one outside; otherwise {stage: max |dev - ref| / eps}.  `device` is
    where the float64 references are computed (None: the CPU)."""
    f32 = np.float32
    rows = np.asarray(rows)
    b = len(rows)
    stats = {}
    x = np.asarray(X[rows], dtype=f32)
    nl = len(coefs)
    ins = [x] + list(out["acts"])
    for l in range(nl - 1):
        lo, hi, ref = DN.gemm_interval(ins[l], coefs[l].T, intercepts[l], 1, "f32", 3, device)
        _check_in(f"a{l + 1}", out["acts"][l], lo, hi, ref, stats)
    lo, hi, ref = DN.gemm_interval(ins[-1], coefs[-1].T, intercepts[-1], 2, "f32", 3, device)
    _check_in("p", out["p"], lo, hi, ref, stats)
    y = np.asarray(Y[rows]).astype(f32)
    assert np.array_equal(out["deltas"][-1], (out["p"] - y).astype(f32)), (f"delta{nl - 1}",)
    for l in range(nl - 1, 0, -1):
        lo, hi, ref = DN.gemm_interval(out["deltas"][l], coefs[l], None, 0, "f32", 3, device)
        mask = torch.as_tensor(out["acts"][l - 1] != 0, device=lo.device)
        zero = torch.zeros_like(lo)
        lo, hi, ref = torch.where(mask, lo, zero), torch.where(mask, hi, zero), torch.where(mask, ref, zero)
        _check_in(f"delta{l - 1}", out["deltas"][l - 1], lo, hi, ref, stats)
    for l in range(nl):
        lo, hi, ref = DN.gemm_interval(ins[l].T, out["deltas"][l].T, None, 0, "f32", 3, device)
        aw = (f32(alpha) * coefs[l]).astype(f32)
        fin = [torch.as_tensor((((t.cpu().numpy().astype(f32) + aw).astype(f32)) / f32(b)).astype(f32)
                               .astype(np.float64), device=lo.device) for t in (lo, hi)]
        _check_in(f"coef_grad{l}", out["coef_grads"][l], fin[0], fin[1],
                  (ref + torch.as_tensor(aw.astype(np.float64), device=lo.device)) / b, stats)
        dl = out["deltas"][l].astype(np.float64)
        ref_b = dl.sum(0) / b
        eps_b = 2.0 ** -24 * np.abs(ref_b) + b * 2.0 ** -53 * np.abs(dl).sum(0) / b + DN.TINY
        err = np.abs(out["intercept_grads"][l] - ref_b)
        stats[f"intercept_grad{l}"] = float((err / eps_b).max())
        assert (err <= eps_b).all(), (f"intercept_grad{l}", stats)
    pc = np.clip(out["p"].astype(np.float64), 2.0 ** -23, 1 - 2.0 ** -23)
    terms = np.where(np.asarray(Y[rows]) != 0, np.log(pc), np.log1p(-pc))
    reg = 0.5 * alpha * sum(float((c.astype(np.float64) ** 2).sum()) for c in coefs) / b
    ref_loss = -terms.sum() / b + reg
    eps_loss = 1e-13 * (np.abs(terms).sum() / b + reg)
    stats["loss"] = abs(out["loss"] - ref_loss) / eps_loss
    assert abs(out["loss"] - ref_loss) <= eps_loss, ("loss", stats)
    return stats
