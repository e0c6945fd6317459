"""CPU tests of the similar-issue search's oracle (oracle/knn_ref.py), its host-side vote (code_intelligence_b200/knn.py),
the C header and the sm_90a build of csrc/knn.cu.

Every test here is single-threaded: sklearn's brute-force neighbour search and numpy's BLAS would otherwise start
thread pools as wide as the machine that stay behind (spinning) while the rest of the suite runs."""
import os
import re
import subprocess

import numpy as np
import pytest
from threadpoolctl import threadpool_limits

from oracle import knn_ref as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _one_thread():
    with threadpool_limits(limits=1):
        yield


def _gapped(n, D, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((n, D)) + 1.5).astype(np.float32)


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_oracle_matches_sklearn(metric):
    from sklearn.neighbors import NearestNeighbors
    X, Q = _gapped(4000, 48, 1), _gapped(60, 48, 2)
    d, i = K.brute(X, Q, 10, metric)
    # the same f32 values, given to sklearn as float64 so that it computes in float64 too
    sd, si = NearestNeighbors(n_neighbors=10, algorithm="brute", metric=metric).fit(X.astype(np.float64)).kneighbors(
        Q.astype(np.float64))
    assert (i == si).all()
    assert (np.abs(d - sd) <= 1e-6 * np.abs(sd) + 1e-12).all()


def test_oracle_ties_zero_vectors_and_self():
    X = _gapped(200, 16, 3)
    X[5] = 0
    X[50] = X[10]
    d, i = K.brute(X, np.vstack([np.zeros((1, 16), np.float32), X[10:11]]), 4, "cosine")
    assert list(i[0]) == [0, 1, 2, 3] and (d[0] == 1).all()
    assert list(i[1, :2]) == [10, 50] and (d[1, :2] == 0).all()
    d, i = K.brute(X, X[10:11], 2, "euclidean")
    assert list(i[0]) == [10, 50] and (d[0] == 0).all()


@pytest.mark.parametrize("cfg", [dict(n_neighbors=10, weights="distance"),
                                 dict(n_neighbors=2, weights="distance", metric="cosine"),
                                 dict(n_neighbors=5)])
def test_vote_matches_sklearn_predict_proba(cfg):
    from sklearn.neighbors import KNeighborsClassifier
    from code_intelligence_b200.knn import vote_proba
    rng = np.random.default_rng(4)
    X, Xq = _gapped(3000, 32, 5), _gapped(80, 32, 6)
    Xq[:5] = X[:5]                                     # exact zero distances
    Y = (rng.random((3000, 5)) < 0.3).astype(np.int64)
    Y[:, 3] = 0
    Y[:, 4] = 1
    sk = KNeighborsClassifier(algorithm="brute", **cfg).fit(X.astype(np.float64), Y)
    want = np.stack([p[:, 1] if p.shape[1] > 1 else np.full(len(Xq), float(c[0]))
                     for p, c in zip(sk.predict_proba(Xq.astype(np.float64)), sk.classes_)]).T
    d, i = K.brute(X, Xq, cfg["n_neighbors"], cfg.get("metric", "euclidean"))
    assert np.abs(K.vote(i, d, Y, cfg["weights"] if "weights" in cfg else "uniform") - want).max() <= 1e-6
    assert np.abs(vote_proba(i, d, Y, cfg.get("weights", "uniform")) - want).max() <= 1e-6


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_lattice_scores_are_the_exact_stage1_scores(metric):
    """On lattice data with the zero centre, the device-form restatement equals the exact f64 stage-1 score."""
    rng = np.random.default_rng(11)
    B = K.lattice_rows(rng, 40, 64, metric)
    X = np.vstack([K.with_zero_centre(B), K.lattice_rows(rng, 300, 64, metric), np.zeros((2, 64), np.float32)])
    Q = np.vstack([K.lattice_rows(rng, 30, 64, metric), -np.abs(X[:1]), np.zeros((1, 64), np.float32)])
    c = K.center(X[:80])
    assert (c == 0).all()
    s = K.lattice_scores(X, Q, metric)
    s1, _ = K.stage1_scores(X, Q, c, metric)
    assert (s == s1).all()
    assert (s.astype(np.float32).astype(np.float64) == s).all()   # every score is an f32 value
    assert not np.signbit(s[s == 0]).any()
    if metric == "cosine":   # |x| powers of two: the distances are 1 - s / |q|, exactly
        d = K.lattice_distances(X, Q[:30], metric)
        assert (d == 1.0 - s[:30] / np.sqrt((Q[:30].astype(np.float64) ** 2).sum(1))[:, None]).all()


def test_topk_exact_equals_a_naive_sort():
    rng = np.random.default_rng(12)
    s = rng.integers(-4, 4, (20, 500)).astype(np.float64)   # hundreds of ties per score
    s[3] = 0.0
    for kp in (1, 33, 96, 500, 600):
        score, idx = K.topk_exact(s, kp)
        for r in range(s.shape[0]):
            naive = sorted(range(s.shape[1]), key=lambda j: (-s[r, j], j))[:kp]
            m = len(naive)
            assert list(idx[r, :m]) == naive and (score[r, :m] == s[r, naive]).all()
            assert (idx[r, m:] == -1).all() and (score[r, m:] == -np.inf).all()
    d, i = K.lattice_brute(K.lattice_rows(rng, 700, 16, "euclidean", -1, 1), np.zeros((2, 16), np.float32), 64,
                           "euclidean")
    assert (np.diff(d, axis=1) >= 0).all()
    for r in range(2):   # within one distance, ascending index
        same = d[r, 1:] == d[r, :-1]
        assert (i[r, 1:][same] > i[r, :-1][same]).all()


def test_plan_restates_knn_plan():
    # one query block: one slice per SM (capped by the merge), P = 16384 once S * k' > 8192
    assert K.plan(128, 256 * 132 * 2, 96, 132) == (132, 2, 16384)
    assert K.plan(128, 256 * 114 * 2, 96, 114) == (114, 2, 16384)
    assert K.plan(100, 100_000, 37, 132) == (131, 3, 8192)
    # many query blocks share the SMs; at least one slice; never more slices than blocks
    assert K.plan(3000, 100_000, 42, 132) == (5, 79, 256)
    assert K.plan(128 * 132, 1000, 33, 132) == (1, 4, 64)
    assert K.plan(1, 300, 96, 132) == (2, 1, 256)


def _bf16(x):
    """Round float32 to bf16 (nearest even), returned as float64."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def test_stage1_bound_covers_the_split_representation():
    """eps dominates the error of an emulated split-bf16 product with f32 epilogue rounding (a sanity check of the
    bound's form; the device check is tests/test_gpu_knn.py)."""
    X, Q = _gapped(300, 96, 7), _gapped(20, 96, 8)
    c = K.center(X)
    for metric in ("cosine", "euclidean"):
        s, eps = K.stage1_scores(X, Q, c, metric)

        def split(a):
            t = a.astype(np.float64) - c.astype(np.float64)
            hi = _bf16(t.astype(np.float32))
            lo = _bf16((t - hi).astype(np.float32))
            return hi, lo
        qh, ql = split(Q)
        xh, xl = split(X)
        acc = (qh @ xh.T + ql @ xh.T + qh @ xl.T).astype(np.float32).astype(np.float64)
        Xt, Qt = X.astype(np.float64) - c, Q.astype(np.float64) - c
        if metric == "euclidean":
            got = acc - 0.5 * (Xt * Xt).sum(1)[None, :]
        else:
            a = Qt @ c + float(c.astype(np.float64) @ c)
            got = (acc + a[:, None] + (Xt @ c)[None, :]) / np.sqrt((X.astype(np.float64) ** 2).sum(1))[None, :]
        assert (np.abs(got - s) <= eps).all(), metric


def test_header_compiles_as_c99(tmp_path):
    src = tmp_path / "knn_decl.c"
    src.write_text('#include "issue_emb_b200.h"\n'
                   'int main(void) { ie_knn* h = 0; (void)h; return IE_KNN_COSINE + IE_KNN_EUCLIDEAN - 1; }\n')
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                    "-c", str(src), "-o", str(tmp_path / "knn_decl.o")], check=True)


def test_knn_cu_built_for_sm_90a_reports_registers_and_spills():
    """The library build compiles csrc/knn.cu for sm_90a with `-Xptxas -v` (csrc/Makefile); its log holds every kernel's
    registers and spills (read here rather than compiling the file a second time)."""
    from code_intelligence_b200 import _lib
    _lib.load()                                            # builds the library if needed
    log = os.path.join(ROOT, "code_intelligence_b200", "csrc", "build", "knn.ptxas.log")
    text = open(log).read()
    assert "sm_90a" in text
    entries = re.findall(r"Compiling entry function '([^']+)'", text)
    assert any("KnnEpi" in e for e in entries) and any("knn_merge_rerank" in e for e in entries), entries
    regs = [int(r) for r in re.findall(r"Used (\d+) registers", text)]
    print("knn.cu ptxas:", [l.strip() for l in text.splitlines() if "registers" in l or "spill" in l])
    assert regs and max(regs) <= 168


def test_index_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("checks the no-GPU failure mode")
    from code_intelligence_b200.knn import IssueIndex
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        IssueIndex(16, "cosine")
