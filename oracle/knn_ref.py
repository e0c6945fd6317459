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
# f32 accumulation (oracle/tc_accum.py MODEL, measured on the H100): each k16 MMA step loses less than
# 17 * 2^-25 of its largest term (C or a product) to alignment and 2^-23 of its result to the truncation to f32; every
# such value is at most the sum of |split products|, <= (1 + 2^-6) sum |q~ x~|.  K_pad / 16 steps per pass.  (Centred
# clustered data keeps the partial sums of a query's own cluster near sum |q~ x~|, so no per-pass constant holds.)
ACC_STEP = 17 * 2.0 ** -25 + 2.0 ** -23


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
    e_acc = (SPLIT_PRODUCT + PASSES * (k_pad // 16) * ACC_STEP * (1 + 2.0 ** -6)) * abs_t
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


# ---- lattice data: the whole device computation is exact, so the device can be checked bit for bit ----------------
# Entries are small integers (|x_i| <= 3, D <= 8192 with |x_i| <= 1): bf16 holds them exactly (lo = 0), every dot
# product and |x|^2 / 2 is an integer below 2^24, exact in f32 in any summation order.  The first add is a block and
# its negation, so the f64 mean (the centre) is exactly 0, and so are a_q and b_x.  Cosine rows are +-1 on a
# power-of-4 count of coordinates, so |x| is a power of two: r_x = 1/|x| is exact, and so are q/|q| - x/|x| and the f64
# re-rank sum in any order.  Exact stage-1 scores mean that exact ties are real ties, which stage 1 must break by index.

def lattice_rows(rng, n, D, metric, lo=-3, hi=3, nnz=None):
    """(n, D) float32 lattice rows: euclidean entries uniform in [lo, hi]; cosine +-1 on `nnz` (a power of 4 <= D,
    default the largest) random coordinates."""
    if metric == "euclidean":
        return rng.integers(lo, hi + 1, (n, D)).astype(np.float32)
    if nnz is None:
        nnz = 4 ** int(np.floor(np.log(D) / np.log(4)))
    assert nnz <= D and 4 ** round(np.log(nnz) / np.log(4)) == nnz, nnz
    X = np.zeros((n, D), np.float32)
    cols = np.argsort(rng.random((n, D)), axis=1)[:, :nnz]
    np.put_along_axis(X, cols, rng.choice(np.float32([-1, 1]), (n, nnz)), axis=1)
    return X


def with_zero_centre(B):
    """The first add of a lattice index: B and -B, whose f64 mean is exactly 0."""
    return np.vstack([B, -B])


def lattice_scores(X, Q, metric, dot=None):
    """Stage-1 scores (nq, n) float64 exactly as the device forms them on lattice data with centre 0: euclidean
    acc - f32(|x|^2 / 2), cosine f32(acc * f32(1 / sqrt(|x|^2))) with the square root in f64 and r = 0 for a zero row,
    acc = q.x (exact).  `dot` may pass a precomputed exact Q @ X.T.  Zeros are +0 (the device keys -0 as +0)."""
    X = np.asarray(X, dtype=np.float64)
    acc = np.asarray(Q, dtype=np.float64) @ X.T if dot is None else np.asarray(dot, dtype=np.float64)
    x2 = (X * X).sum(1)
    if metric == "euclidean":
        s = acc - (0.5 * x2)[None, :]
    else:
        with np.errstate(divide="ignore"):
            r = np.where(x2 > 0, 1.0 / np.sqrt(x2), 0.0).astype(np.float32)
        s = (acc.astype(np.float32) * r[None, :]).astype(np.float64)
    return s + 0.0


def topk_exact(s, kp):
    """The best kp of each row of scores s (nq, n) by (score descending, index ascending) -> (score (nq, kp) float32,
    idx (nq, kp) int64), -inf / -1 past n (the device shortlist's convention)."""
    nq, n = s.shape
    order = np.lexsort((np.broadcast_to(np.arange(n), s.shape), -s), axis=1)[:, :kp]
    score = np.full((nq, kp), -np.inf, np.float32)
    idx = np.full((nq, kp), -1, np.int64)
    m = min(n, kp)
    score[:, :m] = np.take_along_axis(s, order, 1)[:, :m]
    idx[:, :m] = order[:, :m]
    return score, idx


def lattice_distances(X, Q, metric, dot=None):
    """Exact f64 distances (nq, n) on lattice data (sklearn convention, as `brute`): every value is the correctly
    rounded f64 of the exact distance, so equal distances are exact ties."""
    X = np.asarray(X, dtype=np.float64)
    Q = np.asarray(Q, dtype=np.float64)
    acc = Q @ X.T if dot is None else np.asarray(dot, dtype=np.float64)
    x2 = (X * X).sum(1)[None, :]
    q2 = (Q * Q).sum(1)[:, None]
    if metric == "euclidean":
        return np.sqrt(q2 - 2.0 * acc + x2)
    with np.errstate(invalid="ignore", divide="ignore"):
        d = 1.0 - acc / (np.sqrt(q2) * np.sqrt(x2))   # |q|, |x| powers of two: exact
    return np.where((q2 == 0) | (x2 == 0), 1.0, d)


def lattice_brute(X, Q, k, metric, dot=None):
    """Exact k nearest on lattice data, ties to the lower index -> (dist (nq, k) float32, idx (nq, k) int64)."""
    d = lattice_distances(X, Q, metric, dot)
    idx = np.lexsort((np.broadcast_to(np.arange(d.shape[1]), d.shape), d), axis=1)[:, :k]
    return np.take_along_axis(d, idx, 1).astype(np.float32), idx


def plan(nq, n, kp, num_sms, merge_max=16384):
    """Restates ``knn_plan`` in csrc/knn.cu for one pass of nq <= 128 * num_sms queries: (S slices, nbs 256-row
    blocks per slice) -- one wave of (128-row query block, slice) items, at most merge_max / kp slices -- and the merge's
    sort size P (the power of two >= S * kp)."""
    m_blocks = -(-nq // 128)
    n_blocks = -(-n // 256)
    s = min(max(1, num_sms // m_blocks), n_blocks, merge_max // kp)
    nbs = -(-n_blocks // s)
    S = -(-n_blocks // nbs)
    P = 1
    while P < S * kp:
        P *= 2
    return S, nbs, P


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
