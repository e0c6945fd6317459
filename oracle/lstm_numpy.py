"""CPU ORACLE (test infrastructure, NOT product code): explicit-loop numpy restatement of the encoder.

Independent of torch.nn.LSTM -- writes out SURVEY.md Appendix A line by line so that the torch-module
oracle (oracle/awd_lstm_ref.py) is cross-checked by a second implementation:

    x^0_t = Emb[ids[:, t]]                                        (F.embedding; padding_idx affects grads only)
    z     = x_t W_ih^T + b_ih + h_{t-1} W_hh^T + b_hh             rows ordered i | f | g | o  (torch.nn.LSTM)
    i,f,o = sigmoid(z_i), sigmoid(z_f), sigmoid(z_o); g = tanh(z_g)
    c_t   = f*c_{t-1} + i*g ; h_t = o*tanh(c_t)                   h_{-1}=c_{-1}=0 (inference.py:56,66 reset())
    out[b] = [mean_{t<len} y | max_{t<len} y | y[len-1]]          (inference.py:239)

Use only for small cases (pure numpy, float64 or float32 accumulations selectable).
"""
from __future__ import annotations

import numpy as np


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def lstm_layer(x, w_ih, w_hh, b_ih, b_hh, dtype=np.float64):
    """x (B,T,in) -> (B,T,out)."""
    x = x.astype(dtype)
    w_ih, w_hh, b_ih, b_hh = (a.astype(dtype) for a in (w_ih, w_hh, b_ih, b_hh))
    B, T, _ = x.shape
    H = w_hh.shape[1]
    h = np.zeros((B, H), dtype)
    c = np.zeros((B, H), dtype)
    ys = np.empty((B, T, H), dtype)
    for t in range(T):
        z = x[:, t] @ w_ih.T + b_ih + h @ w_hh.T + b_hh
        i, f, g, o = z[:, :H], z[:, H:2 * H], z[:, 2 * H:3 * H], z[:, 3 * H:]
        c = _sigmoid(f) * c + _sigmoid(i) * np.tanh(g)
        h = _sigmoid(o) * np.tanh(c)
        ys[:, t] = h
    return ys


def encode(emb, layers, ids, lengths, dtype=np.float64):
    """emb (V,E); layers list of dict(w_ih,w_hh,b_ih,b_hh); ids (B,T) right padded -> (B,3E)."""
    x = emb[np.asarray(ids)]
    for L in layers:
        x = lstm_layer(x, L['w_ih'], L['w_hh'], L['b_ih'], L['b_hh'], dtype)
    out = []
    for b, n in enumerate(lengths):
        e = x[b, :n]
        out.append(np.concatenate([e.mean(0), e.max(0), e[-1]]))
    return np.stack(out), x


def mlp_forward(X, coefs, intercepts, dtype=np.float64):
    """sklearn MLPClassifier._forward_pass_fast for relu hidden + logistic output
    (py/label_microservice/mlp.py:63 -> predict_proba; multilabel => out_activation_ 'logistic').
    coefs[i] is stored [fan_in, fan_out]."""
    a = np.asarray(X, dtype)
    n = len(coefs)
    for i, (W, b) in enumerate(zip(coefs, intercepts)):
        a = a @ np.asarray(W, dtype) + np.asarray(b, dtype)
        if i != n - 1:
            a = np.maximum(a, 0)
    return 1.0 / (1.0 + np.exp(-a))


def seeded_mlp(seed, dims, n_rows):
    """Seeded MLP head parameters (Glorot-uniform, as sklearn initialises them) and N(0, 0.1^2) inputs: the
    production-shape fixture (tests/golden/mlp_ref_prod.npz) stores only these arguments and the reference's outputs.
    numpy's PCG64 stream is the same on every machine."""
    rng = np.random.default_rng(seed)
    coefs, intercepts = [], []
    for fan_in, fan_out in zip(dims[:-1], dims[1:]):
        bound = np.sqrt(6.0 / (fan_in + fan_out))
        coefs.append(rng.uniform(-bound, bound, (fan_in, fan_out)).astype(np.float32))
        intercepts.append(rng.uniform(-bound, bound, fan_out).astype(np.float32))
    # output biases of a head trained on labels with ~20 % base rates (what sklearn's fit gives in a few steps)
    intercepts[-1] = rng.uniform(-1.75, -1.15, dims[-1]).astype(np.float32)
    X = (rng.standard_normal((n_rows, dims[0])) * 0.1).astype(np.float32)
    return coefs, intercepts, X


def load_mlp_fixture(path):
    """(coefs, intercepts, X, reference probabilities) of a tests/golden/mlp_ref_*.npz fixture: stored arrays, or the
    arguments of seeded_mlp."""
    z = np.load(path)
    if "seed" in z.files:
        coefs, intercepts, X = seeded_mlp(int(z["seed"]), [int(v) for v in z["dims"]], int(z["n_rows"]))
    else:
        n = int(z["n_layers"])
        coefs, intercepts, X = [z[f"coef{i}"] for i in range(n)], [z[f"intercept{i}"] for i in range(n)], z["X"]
    return coefs, intercepts, X, z["probs"]


def filter_labels(label_names, probs, thresholds):
    """py/label_microservice/repo_specific_model.py:126-146 -- keep label iff its threshold is truthy
    and prob >= threshold."""
    out = {}
    for name, p in zip(label_names, probs):
        thr = thresholds[name]
        if not thr:
            continue
        if p < thr:
            continue
        out[name] = p
    return out
