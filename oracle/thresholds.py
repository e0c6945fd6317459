"""Exact reference of the label head's per-label threshold search (the loop of MLPWrapper.find_probability_thresholds,
py/label_microservice/mlp.py:81-98, on sklearn's precision_recall_curve), written from the definition and not from
sklearn, vectorised over labels:

  - the curve's points are the distinct scores (-0.0 and +0.0 are one score); at score s, tp and fp count the samples
    with score >= s, exactly, in integers;
  - precision = tp / (tp + fp) and recall = tp / P are each one float64 division of those integers (recall := 1 when
    the label has no positive sample), which is what sklearn and csrc/pr_curve.cu both compute;
  - the chosen point has the highest precision among points with precision >= p_thr, recall >= r_thr and
    precision > 0; on ties the lowest threshold; None (precision = recall = 0) when no point qualifies.
"""
from __future__ import annotations

import numpy as np


def pr_thresholds(scores, truth, precision_threshold, recall_threshold, stop_at_full_recall: bool = False):
    """scores (n, L) float32, truth (n, L) 0/1 -> (thresholds, precisions, recalls) lists, thresholds float or None.
    stop_at_full_recall: drop the curve points below the first one that reaches full recall, as scikit-learn releases
    before 1.1 did; the result must not change."""
    scores = np.asarray(scores, dtype=np.float32)
    truth = np.asarray(truth) != 0
    if scores.ndim != 2 or truth.shape != scores.shape:
        raise ValueError(f"scores {scores.shape} and truth {truth.shape} must be the same (n, L)")
    if not np.isfinite(scores).all():
        raise ValueError("scores contain NaN or infinity")
    n, L = scores.shape
    s = np.where(scores == 0, np.float32(0.0), scores)             # -0.0 -> +0.0
    order = np.argsort(s, axis=0, kind="stable")[::-1]              # descending; order inside a tie group is irrelevant
    ss = np.take_along_axis(s, order, 0)
    tp = np.cumsum(np.take_along_axis(truth, order, 0), axis=0, dtype=np.int64)
    count = np.arange(1, n + 1, dtype=np.int64)[:, None]            # tp + fp at each sorted position
    point = np.ones((n, L), dtype=bool)                             # a position that ends a group of equal scores
    point[:-1] = ss[:-1] != ss[1:]
    total = tp[-1]
    if stop_at_full_recall:
        full = point & (tp == total)
        first = np.argmax(full, axis=0)                             # the last position always qualifies
        point &= np.arange(n)[:, None] <= first
    prec = tp.astype(np.float64) / count.astype(np.float64)
    rec = np.where(total > 0, tp.astype(np.float64) / np.maximum(total, 1).astype(np.float64), 1.0)
    ok = point & (prec >= precision_threshold) & (rec >= recall_threshold) & (prec > 0.0)
    key = np.where(ok, prec, -1.0)
    best = key.max(axis=0)
    last = n - 1 - np.argmax((ok & (key == best))[::-1], axis=0)    # highest sorted position = lowest threshold
    thr, prec_o, rec_o = [], [], []
    for l in range(L):
        if ok[:, l].any():
            i = int(last[l])
            thr.append(float(ss[i, l])); prec_o.append(float(prec[i, l])); rec_o.append(float(rec[i, l]))
        else:
            thr.append(None); prec_o.append(0.0); rec_o.append(0.0)
    return thr, prec_o, rec_o
