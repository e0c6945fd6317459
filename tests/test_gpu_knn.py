"""GPU tests of the similar-issue index (code_intelligence_b200/knn.py, csrc/knn.cu): exact answers against the f64
brute-force oracle, the project's own near-parallel embeddings, stage 1 per element against its error bound, bit-exact
invariants, edges and sklearn parity through KNeighborsLabeler."""
import numpy as np
import pytest
import torch
from threadpoolctl import threadpool_limits

from oracle import knn_ref as K

pytestmark = pytest.mark.gpu

REL, ABS = 2.0 ** -20, 1e-7


def _knn():
    from code_intelligence_b200.knn import IssueIndex
    return IssueIndex


def _planted(n, D, seed, dup_every=0):
    """Clusters with spread, a common offset, near-duplicates and exact duplicate rows."""
    rng = np.random.default_rng(seed)
    n_c = max(1, n // 50)
    centres = rng.standard_normal((n_c, D)) * 3.0 + 5.0
    X = centres[rng.integers(0, n_c, n)] + rng.standard_normal((n, D))
    if n > 10:
        nd = max(1, n // 20)
        src = rng.integers(0, n, nd)
        dst = rng.integers(0, n, nd)
        X[dst] = X[src] + rng.standard_normal((nd, D)) * 1e-3   # near-duplicates
    if dup_every and n > dup_every:
        X[dup_every::dup_every] = X[0]                            # exact duplicates of row 0
    return X.astype(np.float32)


def _queries(X, nq, seed):
    rng = np.random.default_rng(seed + 1)
    Q = X[rng.integers(0, X.shape[0], nq)] + rng.standard_normal((nq, X.shape[1])).astype(np.float32) * 0.5
    Q[: max(1, nq // 4)] = X[rng.integers(0, X.shape[0], max(1, nq // 4))]   # some queries equal a stored row
    return Q.astype(np.float32)


def _check(dist, idx, want_d, want_i, what=""):
    assert (idx == want_i).all(), f"{what}: {(idx != want_i).sum()} indices differ"
    err = np.abs(dist.astype(np.float64) - want_d)
    assert (err <= REL * np.abs(want_d) + ABS).all(), f"{what}: max |d - ref| {err.max():.3e}"


CASES = [  # (n, D, k, nq)
    (1, 7, 1, 1), (255, 64, 5, 127), (256, 1, 1, 128), (257, 2401, 10, 129), (1000, 1600, 64, 1),
    (3000, 2400, 10, 1280), (100_000, 64, 10, 3000), (100_000, 1600, 5, 128),
]


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
@pytest.mark.parametrize("n,D,k,nq", CASES)
def test_exact_answers(metric, n, D, k, nq):
    X = _planted(n, D, seed=n + D)
    Q = _queries(X, nq, seed=n + D)
    index = _knn()(D, metric).add(X)
    dist, idx = index.search(Q, k)
    want_d, want_i = K.brute(X, Q, k, metric)
    if D == 1 and metric == "cosine":
        # every row is at cosine distance 0, 1 or 2 from a query: hundreds of exact ties, far outside the 32-row margin
        # of the exactness condition, so only the distances are determined
        np.testing.assert_allclose(dist, want_d, rtol=REL, atol=ABS)
    else:
        _check(dist, idx, want_d, want_i, f"{metric} n={n} D={D} k={k} nq={nq}")
    index.close()


@pytest.mark.parametrize("scale", [1.0, 2.0])
def test_project_embeddings_near_parallel(scale):
    from code_intelligence_b200 import IssueEncoder
    from oracle import awd_lstm_ref as R
    ref = R.make_encoder(11, scale=scale)
    emb, layers = ref.export_weights()
    enc = IssueEncoder().load_weights(emb, layers)
    B, T = 2000, 48
    docs = R.synthetic_ids(B, T, seed=12, min_len=8)
    ids = np.full((B, T), 1, dtype=np.int64)
    for i, d in enumerate(docs):
        ids[i, :len(d)] = d
    lengths = np.array([len(d) for d in docs], dtype=np.int32)
    E = enc.encode_ids(ids, lengths)[:, :1600].copy()
    enc.close()
    k = 10
    for metric in ("cosine", "euclidean"):
        index = _knn()(1600, metric).add(E)
        dist, idx = index.search(E, k)
        want_d, want_i = K.brute(E, E, k, metric)
        s, eps = K.stage1_scores(E, E, K.center(E), metric)
        held = sum(K.exactness_holds(s[r], eps[r], k) for r in range(E.shape[0]))
        print(f"scale {scale} {metric}: the sufficient exactness condition holds for {held} of {B} queries")
        _check(dist, idx, want_d, want_i, f"{metric} scale={scale}")
        assert (idx[:, 0] == np.arange(B)).all() and (dist[:, 0] == 0).all()
        index.close()


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
@pytest.mark.parametrize("n,D,k,nq", [(4000, 1600, 10, 64), (20_000, 64, 64, 200), (600, 2401, 1, 129)])
def test_stage1_per_element(metric, n, D, k, nq):
    X = _planted(n, D, seed=7 + n)
    Q = _queries(X, nq, seed=7 + n)
    index = _knn()(D, metric).add(X)
    score, sidx = index._shortlist(Q, k)
    s, eps = K.stage1_scores(X, Q, K.center(X), metric)
    kp = k + 32
    rows = np.arange(nq)[:, None]
    valid = sidx >= 0
    assert valid.sum(1).min() == min(kp, n)
    delta = np.abs(score.astype(np.float64) - s[rows, np.maximum(sidx, 0)])
    ratio = np.where(valid, delta / eps[rows, np.maximum(sidx, 0)], 0.0)
    print(f"stage 1 {metric} n={n} D={D}: max |d|/eps {ratio.max():.3f}  rms {np.sqrt((ratio[valid] ** 2).mean()):.3f}")
    assert ratio.max() <= 1.0
    last = score[:, kp - 1].astype(np.float64) if n >= kp else np.full(nq, -np.inf)
    mask = np.ones_like(s, dtype=bool)
    mask[rows.repeat(kp, 1)[valid], sidx[valid]] = False
    outside = np.where(mask, s - 2 * eps, -np.inf).max(1)
    assert (outside <= last).all()
    index.close()


def test_bit_exact_invariants():
    D, k = 1600, 10
    X = _planted(20_000, D, seed=3, dup_every=997)
    Q = _queries(X, 1280, seed=3)
    for metric in ("cosine", "euclidean"):
        index = _knn()(D, metric).add(X)
        d_all, i_all = index.search(Q, k)
        d_one, i_one = index.search(Q[5:6], k)
        assert (i_one == i_all[5:6]).all() and (d_one == d_all[5:6]).all()
        d_rep, i_rep = index.search(Q, k)
        assert (i_rep == i_all).all() and (d_rep == d_all).all()
        Qt = torch.from_numpy(Q).cuda()
        d_dev, i_dev = index.search(Qt, k)
        torch.cuda.synchronize()
        assert (i_dev.cpu().numpy() == i_all).all() and (d_dev.cpu().numpy() == d_all).all()
        index.check_errors()
        # one add after the first batch vs several (host and device pointers): the same centre, the same answer
        one = _knn()(D, metric).add(X[:5000]).add(X[5000:])
        many = _knn()(D, metric).add(X[:5000])
        many.add(torch.from_numpy(X[5000:12000]).cuda())
        torch.cuda.synchronize()
        many.add(X[12000:])
        assert len(many) == len(X)
        d_o, i_o = one.search(Q, k)
        d_m, i_m = many.search(Q, k)
        assert (i_m == i_o).all() and (d_m == d_o).all()
        assert (i_o == i_all).all()   # exact answers do not depend on the centre
        # duplicated rows come back lower index first
        d0, i0 = index.search(X[:1], 25)
        dups = [0] + list(range(997, 20_000, 997))
        assert list(i0[0, :len(dups)]) == dups[:25] and (d0[0, :len(dups)] == 0).all()
        for h in (index, many, one):
            h.close()


def test_edges():
    IssueIndex = _knn()
    rng = np.random.default_rng(0)
    X = rng.standard_normal((300, 24)).astype(np.float32)
    X[7] = 0
    index = IssueIndex(24, "cosine")
    with pytest.raises(RuntimeError, match="empty"):
        index.search(X[:2], 3)
    index.add(X)
    Q = np.vstack([np.zeros((1, 24), np.float32), X[7:8], X[:3]])
    dist, idx = index.search(Q, 5)
    assert (dist[0] == 1).all() and list(idx[0]) == [0, 1, 2, 3, 4]
    assert (dist[1] == 1).all()
    want_d, want_i = K.brute(X, Q, 5, "cosine")
    _check(dist, idx, want_d, want_i, "zero vectors")
    small = IssueIndex(24, "cosine").add(X[:3])
    with pytest.raises(ValueError, match="exceeds"):
        small.search(X[:2], 4)
    small.close()
    with pytest.raises(ValueError, match="not in"):
        index.search(X[:2], 65)
    with pytest.raises(ValueError, match="must be"):
        index.search(X[:2, :10], 3)
    bad = X[:2].copy()
    bad[1, 3] = np.nan
    with pytest.raises(ValueError, match="not finite"):
        index.search(bad, 3)
    with pytest.raises(ValueError, match="not finite"):
        index.add(bad)
    index.search(torch.from_numpy(bad).cuda(), 3)
    with pytest.raises(ValueError, match="non-finite"):
        index.check_errors()
    index.check_errors()   # cleared
    index.close()


@pytest.mark.parametrize("cfg", [dict(n_neighbors=10, weights="distance"),
                                 dict(n_neighbors=2, weights="distance", metric="cosine")])
def test_sklearn_parity(cfg):
    from sklearn.neighbors import KNeighborsClassifier
    from code_intelligence_b200.knn import KNeighborsLabeler
    rng = np.random.default_rng(5)
    n, D, L = 100_000, 64, 6
    X = (rng.standard_normal((n, D)) + 2.0).astype(np.float32)
    Y = (rng.random((n, L)) < 0.3).astype(np.int64)
    Y[:, 5] = 1
    Xq = (rng.standard_normal((300, D)) + 2.0).astype(np.float32)
    ours = KNeighborsLabeler(**cfg).fit(X, Y).predict_proba(Xq)
    with threadpool_limits(limits=1):   # no machine-wide OpenMP pool left spinning behind sklearn's search
        sk = KNeighborsClassifier(algorithm="brute", **cfg).fit(X, Y)
        want = np.stack([p[:, 1] if p.shape[1] > 1 else np.full(len(Xq), float(c[0]))
                         for p, c in zip(sk.predict_proba(Xq), sk.classes_)]).T
    assert np.abs(ours - want).max() <= 1e-5
