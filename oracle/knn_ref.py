"""Float64 brute-force k-nearest neighbours: the oracle of the similar-issue index (code_intelligence_b200/knn.py).

Distances follow sklearn's ``kneighbors``: cosine 1 - cos, computed as |q/|q| - x/|x||^2 / 2 (a zero vector has
distance 1 to everything), euclidean |q - x|.  Results ascend by distance, ties to the lower index.  The candidate set
comes from the f64 expanded form (error ~1e-13 of the scale, far below any gap the tests plant); the best rows are then
recomputed from the differences themselves, so a query equal to a stored row is at distance exactly 0.

Also the exact stage-1 scores of the device's shortlist and their error bound eps (DESIGN.md section 2), and the
neighbour vote of sklearn's KNeighborsClassifier.
"""
from __future__ import annotations

import numpy as np

U24 = 2.0 ** -24
SPLIT_PRODUCT = 3.1 * 2.0 ** -18   # split-bf16 (hi*hi + lo*hi + hi*lo) vs the exact product, relative to |q~ x~|
PASSES = 3                         # split-bf16 K loop: hi*hi, lo*hi, hi*lo into one f32 accumulator
# f32 accumulation: one rounding of at most 2^-23 of the running sum (|.| <= sum |q~ x~|) per k16 MMA step, K_pad / 16
# steps per pass.  The per-pass 8 * 2^-24 of the encoder's checks assumes sums far below sum |q~ x~|; centred
# clustered data keeps the partial sums of a query's own cluster near sum |q~ x~|, where that is exceeded.
ACC_STEP = 2.0 ** -23


def _exact(Q, X, cand, metric):
    q = Q[:, None, :]
    x = X[cand]
    if metric == "euclidean":
        return np.sqrt(((q - x) ** 2).sum(-1))
    qn = np.sqrt((Q * Q).sum(-1))[:, None, None]
    xn = np.sqrt((x * x).sum(-1))[..., None]
    with np.errstate(invalid="ignore", divide="ignore"):
        d = 0.5 * ((q / qn - x / xn) ** 2).sum(-1)
    zero = (qn[..., 0] == 0) | (xn[..., 0] == 0)
    return np.where(zero, 1.0, d)


def brute(X, Q, k, metric="cosine", extra=64, chunk=256):
    """-> (dist (nq, k) float64, idx (nq, k) int64)."""
    X = np.asarray(X, dtype=np.float64)
    Q = np.asarray(Q, dtype=np.float64)
    n = X.shape[0]
    m = min(n, k + extra)
    out_d = np.empty((Q.shape[0], k))
    out_i = np.empty((Q.shape[0], k), dtype=np.int64)
    if metric == "euclidean":
        xn2 = (X * X).sum(1)
    else:
        xn = np.sqrt((X * X).sum(1))
        Xh = X / np.where(xn == 0, 1.0, xn)[:, None]
    for r0 in range(0, Q.shape[0], chunk):
        q = Q[r0:r0 + chunk]
        if metric == "euclidean":
            approx = xn2[None, :] - 2.0 * q @ X.T
        else:
            qn = np.sqrt((q * q).sum(1))
            qh = q / np.where(qn == 0, 1.0, qn)[:, None]
            approx = -(qh @ Xh.T)
            approx[:, xn == 0] = 0.0
            approx[qn == 0, :] = 0.0
        for j in range(q.shape[0]):
            row = approx[j]
            # every row within rounding of the m-th smallest approximate distance: ties (zero vectors, duplicates) all
            # reach the exact pass, which breaks them by index
            t = np.partition(row, m - 1)[m - 1]
            cand = np.nonzero(row <= t + 1e-9 * np.abs(row).max())[0]
            d = _exact(q[j:j + 1], X, cand[None, :], metric)[0]
            order = np.lexsort((cand, d))[:k]
            out_d[r0 + j] = d[order]
            out_i[r0 + j] = cand[order]
    return out_d, out_i


def center(X_first):
    """The index's centre: the f64 mean of the first add's rows, rounded to f32."""
    return np.asarray(X_first, dtype=np.float64).mean(0).astype(np.float32)


def stage1_scores(X, Q, c, metric):
    """Exact stage-1 scores (larger is nearer), (nq, n) f64, and their per-element error bound eps of the device's
    split-bf16 tensor-core pass and f32 affine epilogue."""
    X = np.asarray(X, dtype=np.float64)
    Q = np.asarray(Q, dtype=np.float64)
    c = np.asarray(c, dtype=np.float64)
    Xt, Qt = X - c, Q - c
    dot_t = Qt @ Xt.T
    abs_t = np.abs(Qt) @ np.abs(Xt).T
    k_pad = -(-X.shape[1] // 64) * 64
    e_acc = (SPLIT_PRODUCT + PASSES * (k_pad // 16) * ACC_STEP) * abs_t
    if metric == "euclidean":
        h = 0.5 * (Xt * Xt).sum(1)[None, :]
        s = dot_t - h
        eps = e_acc + U24 * (abs_t + 2.0 * h)
    else:
        a = (Qt @ c + c @ c)[:, None]
        b = (Xt @ c)[None, :]
        xn = np.sqrt((X * X).sum(1))
        rn = np.where(xn == 0, 0.0, 1.0 / np.where(xn == 0, 1.0, xn))[None, :]
        t = dot_t + a + b
        s = t * rn
        eps = rn * (e_acc + U24 * (3 * np.abs(a) + 3 * np.abs(b) + 2 * abs_t + 2 * np.abs(t)))
    return s, 1.01 * eps + 1e-300


def exactness_holds(s_row, eps_row, k, extra=32):
    """The condition under which the device's answer is exact brute force: at most `extra` rows outside the exact top k
    (by stage-1 score, ties to the lower index) score within 2 eps of the exact k-th score."""
    order = np.lexsort((np.arange(s_row.size), -s_row))
    sk = s_row[order[k - 1]]
    rest = order[k:]
    e_top = np.max(eps_row[order[:k]])
    return int((s_row[rest] >= sk - eps_row[rest] - e_top).sum()) <= extra


def vote(neigh_ind, dist, Y, weights):
    """sklearn KNeighborsClassifier.predict_proba per 0/1 label, column of class 1, stacked -> (n, L)."""
    dist = np.asarray(dist, dtype=np.float64)
    if weights == "uniform":
        w = np.ones_like(dist)
    else:
        with np.errstate(divide="ignore"):
            w = 1.0 / dist
        inf = np.isinf(w)
        rows = inf.any(1)
        w[rows] = inf[rows]
    Y = (np.asarray(Y) != 0).astype(np.float64)
    if Y.ndim == 1:
        Y = Y[:, None]
    num = np.einsum("nk,nkl->nl", w, Y[neigh_ind])
    den = w.sum(1, keepdims=True)
    den[den == 0] = 1.0
    return num / den
