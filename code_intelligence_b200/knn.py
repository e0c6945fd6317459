"""Similar-issue search on the H100: an exact k-nearest-neighbour index over issue embeddings.

The reference serves the 2400-d embedding to duplicate detection and label models through brute-force neighbour
searches on the host: the FewShot notebook's ``oneshotlabeler`` (``CosineSimilarity`` against every stored issue) and
``KNeighborsClassifier(n_neighbors=2, weights='distance', metric='cosine')``, and notebook 08's
``KNeighborsClassifier(weights='distance', n_neighbors=10)`` on the ``[:, :1600]`` features.  ``IssueIndex`` is that
search behind ``ie_knn_*`` (include/issue_emb_b200.h): a split-bf16 tensor-core shortlist over the centred data with a
fused top-k, re-ranked exactly in float64 (DESIGN.md section 2).  ``KNeighborsLabeler`` is the notebooks' label model on
top of it.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import check

KNN_MAX_K = 64
SHORTLIST_EXTRA = 32   # stage 1 keeps k + 32 rows per query (ie::kKnnExtra)
_METRICS = {"cosine": _lib.IE_KNN_COSINE, "euclidean": _lib.IE_KNN_EUCLIDEAN}


def _stream_ptr(t):
    import torch
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


class IssueIndex:
    """Rows numbered 0.. in insertion order; ``search(Q, k)`` -> (dist (nq, k) float32, idx (nq, k) int64), ascending by
    distance, ties to the lower index.  Distances follow sklearn's ``kneighbors``: cosine 1 - cos (a zero vector is at
    distance 1 from everything), euclidean |q - x|.  ``X`` and ``Q`` are float32 numpy arrays (synchronous) or CUDA
    float32 torch tensors (asynchronous on torch's current stream; results come back as CUDA tensors).

    Every row of ``X`` and ``Q`` must be finite with norm 0 or between 2^-48 and 2^48 (the range in which every
    stage-1 score is finite, DESIGN.md section 2): numpy input outside it raises ValueError; CUDA input outside it makes
    that call's answer undefined and is reported by ``check_errors``."""

    def __init__(self, dim: int, metric: str = "cosine", device: int = 0):
        if metric not in _METRICS:
            raise ValueError(f"metric must be one of {sorted(_METRICS)}, got {metric!r}")
        self._lib = _lib.load()
        self.dim, self.metric, self.device = int(dim), metric, device
        h = C.c_void_p()
        check(self._lib.ie_knn_create(self.dim, _METRICS[metric], device, C.byref(h)))
        self._h = h
        self._n = 0

    def __len__(self) -> int:
        return self._n

    def _shape_check(self, X, name):
        if X.ndim != 2 or X.shape[1] != self.dim:
            raise ValueError(f"{name} must be (n, {self.dim}), got {tuple(X.shape)}")

    def add(self, X) -> "IssueIndex":
        if _is_cuda_tensor(X):
            import torch
            if X.dtype != torch.float32:
                raise ValueError("X must be float32")
            self._shape_check(X, "X")
            X = X.contiguous()
            if X.shape[0]:
                check(self._lib.ie_knn_add(self._h, X.data_ptr(), X.shape[0], _lib.IE_FLAG_DEVICE_PTRS, _stream_ptr(X)))
        else:
            X = np.ascontiguousarray(np.asarray(X), dtype=np.float32)
            self._shape_check(X, "X")
            if X.shape[0]:
                check(self._lib.ie_knn_add(self._h, X.ctypes.data, X.shape[0], 0, None))
        self._n += int(X.shape[0])
        return self

    def search(self, Q, k: int):
        k = int(k)
        if _is_cuda_tensor(Q):
            import torch
            if Q.dtype != torch.float32:
                raise ValueError("Q must be float32")
            self._shape_check(Q, "Q")
            Q = Q.contiguous()
            dist = torch.empty((Q.shape[0], k), dtype=torch.float32, device=Q.device)
            idx = torch.empty((Q.shape[0], k), dtype=torch.int64, device=Q.device)
            if Q.shape[0]:
                check(self._lib.ie_knn_search(self._h, Q.data_ptr(), Q.shape[0], k, dist.data_ptr(), idx.data_ptr(),
                                              _lib.IE_FLAG_DEVICE_PTRS, _stream_ptr(Q)))
            return dist, idx
        Q = np.ascontiguousarray(np.asarray(Q), dtype=np.float32)
        self._shape_check(Q, "Q")
        dist = np.empty((Q.shape[0], k), dtype=np.float32)
        idx = np.empty((Q.shape[0], k), dtype=np.int64)
        if Q.shape[0]:
            check(self._lib.ie_knn_search(self._h, Q.ctypes.data, Q.shape[0], k, dist.ctypes.data, idx.ctypes.data, 0,
                                          None))
        return dist, idx

    def check_errors(self) -> None:
        """Raise ValueError if a non-finite value or a row outside the norm range reached the index through
        device-pointer input (waits for the last call); host input is checked before anything is launched."""
        check(self._lib.ie_knn_check_errors(self._h))

    def _shortlist(self, Q, k: int):
        """Test hook ``ie_debug_knn_shortlist``: stage 1's k + 32 best rows per query by the tensor-core score (larger is
        nearer) -> (score (nq, k + 32) float32, idx int64)."""
        Q = np.ascontiguousarray(np.asarray(Q), dtype=np.float32)
        self._shape_check(Q, "Q")
        kp = int(k) + SHORTLIST_EXTRA
        score = np.empty((Q.shape[0], kp), dtype=np.float32)
        idx = np.empty((Q.shape[0], kp), dtype=np.int64)
        check(self._lib.ie_debug_knn_shortlist(self._h, Q.ctypes.data, Q.shape[0], int(k), score.ctypes.data,
                                               idx.ctypes.data))
        return score, idx

    def close(self):
        if getattr(self, "_h", None):
            self._lib.ie_knn_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _is_cuda_tensor(x) -> bool:
    return type(x).__module__.startswith("torch") and getattr(x, "is_cuda", False)


def vote_weights(dist: np.ndarray, weights: str) -> np.ndarray:
    """sklearn's ``_get_weights``: uniform -> ones; distance -> 1/d, except that a row with an exact zero distance gives
    weight 1 to those neighbours and 0 to the rest."""
    if weights == "uniform":
        return np.ones_like(dist, dtype=np.float64)
    if weights != "distance":
        raise ValueError(f"weights must be 'uniform' or 'distance', got {weights!r}")
    dist = np.asarray(dist, dtype=np.float64)
    with np.errstate(divide="ignore"):
        w = 1.0 / dist
    inf = np.isinf(w)
    rows = inf.any(axis=1)
    w[rows] = inf[rows]
    return w


def vote_proba(neigh_ind: np.ndarray, dist: np.ndarray, Y: np.ndarray, weights: str) -> np.ndarray:
    """P(label = 1) per query and label from the (n, k) neighbours: sum of weights of neighbours with the label over the
    sum of all weights (sklearn ``predict_proba`` per output, its column for class 1)."""
    w = vote_weights(dist, weights)
    Y = np.asarray(Y)
    pos = (Y[neigh_ind] != 0).astype(np.float64)              # (n, k, L)
    num = np.einsum("nk,nkl->nl", w, pos)
    den = w.sum(axis=1, keepdims=True)
    den[den == 0.0] = 1.0
    return num / den


class KNeighborsLabeler:
    """Mirror of sklearn's ``KNeighborsClassifier`` on a 0/1 multilabel target, its neighbour search on the H100.
    ``predict_proba(X)`` -> (n, n_labels) P(label = 1): the notebooks' ``np.stack([x[:, 1] for x in
    knn.predict_proba(X)]).T`` (a label constant in ``Y`` gives its constant)."""

    def __init__(self, n_neighbors: int = 5, weights: str = "uniform", metric: str = "minkowski", device: int = 0):
        if weights not in ("uniform", "distance"):
            raise ValueError(f"weights must be 'uniform' or 'distance', got {weights!r}")
        m = {"minkowski": "euclidean", "euclidean": "euclidean", "cosine": "cosine"}.get(metric)
        if m is None:
            raise ValueError(f"metric must be 'minkowski', 'euclidean' or 'cosine', got {metric!r}")
        self.n_neighbors, self.weights, self.metric, self.device = int(n_neighbors), weights, metric, device
        self._metric = m
        self._index = None
        self._Y = None

    def fit(self, X, Y) -> "KNeighborsLabeler":
        X = np.ascontiguousarray(np.asarray(X), dtype=np.float32)
        Y = np.asarray(Y)
        if Y.ndim == 1:
            Y = Y[:, None]
        if Y.shape[0] != X.shape[0]:
            raise ValueError(f"X has {X.shape[0]} rows, Y {Y.shape[0]}")
        if self._index is not None:
            self._index.close()
        self._index = IssueIndex(X.shape[1], self._metric, self.device).add(X)
        self._Y = (Y != 0).astype(np.uint8)
        return self

    def kneighbors(self, X, n_neighbors=None, return_distance=True):
        if self._index is None:
            raise ValueError("this KNeighborsLabeler is not fitted yet: call fit(X, Y) first")
        k = self.n_neighbors if n_neighbors is None else int(n_neighbors)
        dist, idx = self._index.search(X, k)
        return (dist, idx) if return_distance else idx

    def predict_proba(self, X) -> np.ndarray:
        dist, idx = self.kneighbors(X)
        return vote_proba(idx, dist, self._Y, self.weights)

    def close(self):
        if self._index is not None:
            self._index.close()
            self._index = None
