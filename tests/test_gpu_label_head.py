"""GPU tests of the Label_Microservice head: the per-label threshold search (csrc/pr_curve.cu) against the exact
reference oracle/thresholds.py, and the MLP head per element (oracle/device_numerics.mlp_head) at the shapes the
reference's grid search trains, which are the shapes that exercise the padding of ie_mlp_create / ie_mlp_predict_proba
and both paths of launch_convert_rows.

Padding the MLP cases reach (GEMM tile width bn, columns a layer writes n_pad, columns the next layer reads k_pad):
  width 100: bn 112, n_pad 112, next k_pad 128 (112..127 never written by this layer)
  width 200: bn 208, n_pad 208, next k_pad 256
  width 400: bn 256, n_pad 512, next k_pad 448
  n_labels 240 / 256: n_pad = n_labels, stored straight into the caller's array in device-pointer mode
  n_labels 272: bn 256, n_pad 512, staged store
"""
import ctypes as C
import itertools
import warnings

import numpy as np
import pytest
import torch

from oracle import lstm_numpy as N
from oracle import thresholds as T
from test_gpu_numerics import _mlp_check
from test_thresholds_reference import EXACT_CASES, NS, SCORE_PATTERNS, THRESHOLDS, TRUTH_PATTERNS, _flat, assert_same, \
    case_matrix

pytestmark = pytest.mark.gpu

N_PATTERNS = len(SCORE_PATTERNS) * len(TRUTH_PATTERNS)


def _cuda():
    return torch.device("cuda", 0)


# ------------------------------------------------------------------------------------------------ threshold search
def _device_mode(scores, truth, p_thr, r_thr, n=None, n_labels=None):
    """ie_pr_thresholds with device pointers (torch tensors) on a non-default stream -> (rc, thr, prec, rec) numpy.
    The outputs start as 7.0 so that an entry the kernel did not write shows."""
    from code_intelligence_b200 import _lib
    dev = _cuda()
    s = torch.from_numpy(np.ascontiguousarray(scores, dtype=np.float32)).to(dev)
    t = torch.from_numpy(np.ascontiguousarray(np.asarray(truth) != 0, dtype=np.uint8)).to(dev)
    n = s.shape[0] if n is None else n
    n_labels = s.shape[1] if n_labels is None else n_labels
    width = max(s.shape[1], 1)
    thr = torch.full((width,), 7.0, dtype=torch.float32, device=dev)
    prec = torch.full((width,), 7.0, dtype=torch.float64, device=dev)
    rec = torch.full((width,), 7.0, dtype=torch.float64, device=dev)
    stream = torch.cuda.Stream(dev)
    stream.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(stream):
        rc = _lib.load().ie_pr_thresholds(s.data_ptr(), t.data_ptr(), n, n_labels, float(p_thr), float(r_thr),
                                          thr.data_ptr(), prec.data_ptr(), rec.data_ptr(), 0, _lib.IE_FLAG_DEVICE_PTRS,
                                          C.c_void_p(stream.cuda_stream))
    stream.synchronize()
    return rc, thr.cpu().numpy(), prec.cpu().numpy(), rec.cpu().numpy()


def _as_lists(thr, prec, rec):
    return [None if np.isnan(t) else float(t) for t in thr], [float(p) for p in prec], [float(r) for r in rec]


def _bits(x, dtype):
    return np.asarray(x, dtype=dtype).view(np.int32 if dtype == np.float32 else np.int64)


def _check_both_modes(scores, truth, p_thr, r_thr, tag):
    """Host mode equals the reference (thresholds by value, ratios bit for bit); device mode equals host mode bit for
    bit, NaN thresholds included."""
    from code_intelligence_b200.mlp import pr_thresholds
    want = T.pr_thresholds(scores, truth, p_thr, r_thr)
    got = pr_thresholds(scores, truth, p_thr, r_thr)
    assert_same(got, want, tag)
    rc, thr, prec, rec = _device_mode(scores, truth, p_thr, r_thr)
    assert rc == 0, tag
    host_thr = np.array([np.nan if t is None else t for t in got[0]], np.float32)
    np.testing.assert_array_equal(_bits(thr, np.float32), _bits(host_thr, np.float32), err_msg=str(tag))
    np.testing.assert_array_equal(_bits(prec, np.float64), _bits(got[1], np.float64), err_msg=str(tag))
    np.testing.assert_array_equal(_bits(rec, np.float64), _bits(got[2], np.float64), err_msg=str(tag))
    return want


@pytest.mark.parametrize("n", NS)
def test_threshold_search_matches_reference(n):
    """Every score pattern x truth pattern as one 60-label call, at every (p_thr, r_thr), in host and device-pointer
    mode; and single-label calls (column stride 1) of a few of the columns."""
    scores, truth = case_matrix(n, N_PATTERNS)
    for p_thr, r_thr in THRESHOLDS:
        want = _check_both_modes(scores, truth, p_thr, r_thr, (n, p_thr, r_thr))
        if (p_thr, r_thr) in ((0.0, 0.0), (0.75, 0.5)):
            for k in (52, 47, 18):             # straddle / random truth, signed zero / alternating, huge / all positive
                one = _check_both_modes(scores[:, k:k + 1], truth[:, k:k + 1], p_thr, r_thr, (n, p_thr, k))
                assert_same(one, ([want[0][k]], [want[1][k]], [want[2][k]]), (n, p_thr, k))


@pytest.mark.parametrize("n", (1025, 4097, 16384))
def test_threshold_search_600_labels(n):
    """The production label count: 600 columns, each pattern pair ten times with fresh draws."""
    scores, truth = case_matrix(n, 600, seed=3)
    for p_thr, r_thr in THRESHOLDS:
        _check_both_modes(scores, truth, p_thr, r_thr, (n, 600, p_thr, r_thr))


@pytest.mark.parametrize("name,scores,truth,p_thr,r_thr,expected", EXACT_CASES, ids=[c[0] for c in EXACT_CASES])
def test_threshold_search_exact_cases(name, scores, truth, p_thr, r_thr, expected):
    """Hand-checked answers: a tie group of -0.0 and +0.0, precision and recall attaining the thresholds exactly,
    precision ties, a label without positives, one tie group."""
    scores, truth = _flat(scores, truth)
    want = ([None if expected[0] is None else float(expected[0])], [expected[1]], [expected[2]])
    assert_same(_check_both_modes(scores, truth, p_thr, r_thr, name), want, name)


@pytest.mark.parametrize("n,n_labels", [(0, 3), (16385, 3), (37, 0)])
def test_threshold_search_rejects_bad_sizes(n, n_labels):
    from code_intelligence_b200 import _lib
    from code_intelligence_b200.mlp import pr_thresholds
    scores, truth = case_matrix(max(n, 1), max(n_labels, 1))
    with pytest.raises(ValueError):
        pr_thresholds(scores[:n, :n_labels], truth[:n, :n_labels], 0.5, 0.5)
    rc, thr, _, _ = _device_mode(scores, truth, 0.5, 0.5, n=n, n_labels=n_labels)
    assert rc == _lib.IE_ERR_INVALID
    assert (thr == 7.0).all()


NON_FINITE = {"nan": np.float32(np.nan), "-nan all ones": np.uint32(0xFFFFFFFF).view(np.float32),
              "inf": np.float32(np.inf), "-inf": np.float32(-np.inf)}


@pytest.mark.parametrize("bad", list(NON_FINITE))
def test_threshold_search_host_mode_rejects_non_finite(bad):
    """sklearn raises on NaN / inf; the host-pointer entry point refuses them before launching anything."""
    from code_intelligence_b200 import _lib
    from code_intelligence_b200.mlp import pr_thresholds
    scores, truth = case_matrix(1025, 5)
    scores[1000, 3] = NON_FINITE[bad]
    thr = np.full(5, 7.0, np.float32)
    prec, rec = np.full(5, 7.0), np.full(5, 7.0)
    rc = _lib.load().ie_pr_thresholds(scores.ctypes.data, truth.ctypes.data, 1025, 5, 0.5, 0.5, thr.ctypes.data,
                                      prec.ctypes.data, rec.ctypes.data, 0, 0, None)
    assert rc == _lib.IE_ERR_INVALID
    assert (thr == 7.0).all() and (prec == 7.0).all()
    with pytest.raises(ValueError):
        pr_thresholds(scores, truth, 0.5, 0.5)


@pytest.mark.parametrize("n", (3, 2049))
def test_threshold_search_device_mode_marks_non_finite_labels(n):
    """A device-pointer call cannot fail on data: a label with a NaN or infinite score gets NaN threshold, precision
    and recall (an excluded label is NaN / 0 / 0); the other labels are unaffected."""
    scores, truth = case_matrix(n, N_PATTERNS, seed=4)
    bad_cols = {}
    for j, (name, v) in zip((2, 21, 33, 59), NON_FINITE.items()):
        scores[n // 2, j] = v
        bad_cols[j] = name
    good = [j for j in range(N_PATTERNS) if j not in bad_cols]
    for p_thr, r_thr in ((0.0, 0.0), (0.75, 0.5), (1.01, 0.0)):
        rc, thr, prec, rec = _device_mode(scores, truth, p_thr, r_thr)
        assert rc == 0
        for j, name in bad_cols.items():
            assert np.isnan(thr[j]) and np.isnan(prec[j]) and np.isnan(rec[j]), (n, name, thr[j], prec[j], rec[j])
        assert_same(_as_lists(thr[good], prec[good], rec[good]),
                    T.pr_thresholds(scores[:, good], truth[:, good], p_thr, r_thr), (n, p_thr))


# ------------------------------------------------------------------------------------------------ MLP head
GRID_HIDDEN = [(100,), (200,), (400,), (50, 50), (100, 100), (200, 200)]   # MLPWrapper.grid_search defaults
LABEL_COUNTS = (1, 17, 240, 256, 272)
GRID_CASES = [(d_in, hidden, LABEL_COUNTS[i % len(LABEL_COUNTS)])
              for i, (d_in, hidden) in enumerate(itertools.product((2400, 1600), GRID_HIDDEN))]


def _head(dims, seed):
    from code_intelligence_b200.mlp import MLPHead
    coefs, intercepts, _ = N.seeded_mlp(seed, dims, 1)
    return MLPHead(coefs, intercepts), coefs, intercepts


def _host_and_device(head, X, coefs, intercepts, tag):
    """Host mode inside the per-element interval; device-pointer mode identical to it bit for bit."""
    host = head.predict_proba(X)
    _mlp_check(host, X, coefs, intercepts, tag)
    dev = head.predict_proba_device(torch.from_numpy(X).to(_cuda()))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(dev.cpu().numpy(), host, err_msg=tag)
    return host


@pytest.mark.parametrize("d_in,hidden,n_labels", GRID_CASES)
def test_mlp_head_grid_search_shapes(d_in, hidden, n_labels):
    dims = [d_in, *hidden, n_labels]
    head, coefs, intercepts = _head(dims, sum(dims))
    rng = np.random.default_rng(len(dims) + n_labels)
    for n in (1, 129, 300):
        X = (rng.standard_normal((n, d_in)) * 0.5).astype(np.float32)
        _host_and_device(head, X, coefs, intercepts, f"{dims} n={n}")
    head.close()


@pytest.mark.parametrize("d_in,n_labels", [(2, 3), (5, 5)])
def test_mlp_head_reference_test_shapes(d_in, n_labels):
    """The reference's own unit-test shapes: D_in not a multiple of 4 takes the scalar convert_rows_kernel."""
    dims = [d_in, 100, n_labels]
    head, coefs, intercepts = _head(dims, 11 + d_in)
    rng = np.random.default_rng(d_in)
    for n in (1, 20, 129):
        X = rng.random((n, d_in)).astype(np.float32)
        _host_and_device(head, X, coefs, intercepts, f"{dims} n={n}")
    head.close()


def test_mlp_head_stale_activation_columns():
    """(400, 100, 100): layer 0 writes 512 columns of one activation buffer, layer 2 writes 112 of the same buffer and
    layer 3 reads 128, so columns 112..127 still hold layer 0's values; they must meet zero weight columns."""
    dims = [1600, 400, 100, 100, 17]
    head, coefs, intercepts = _head(dims, 21)
    X = (np.random.default_rng(5).standard_normal((300, 1600)) * 0.5).astype(np.float32)
    _host_and_device(head, X, coefs, intercepts, f"{dims}")
    head.close()


def test_mlp_head_host_multi_pass():
    """Host pointers are staged through a 65536-row buffer: 65536 + 129 rows take two passes; every row is checked."""
    dims = [256, 100, 17]
    head, coefs, intercepts = _head(dims, 31)
    X = (np.random.default_rng(6).standard_normal((65536 + 129, 256)) * 0.5).astype(np.float32)
    _mlp_check(head.predict_proba(X), X, coefs, intercepts, "host multi-pass")
    head.close()


def test_mlp_head_misaligned_device_input():
    """A device X 4 bytes off 16-byte alignment cannot take the 128-bit loads: launch_convert_rows sends it to the
    scalar kernel, which must give the aligned call's bits."""
    dims = [1600, 200, 17]
    head, coefs, intercepts = _head(dims, 41)
    X = (np.random.default_rng(7).standard_normal((129, 1600)) * 0.5).astype(np.float32)
    aligned = torch.from_numpy(X).to(_cuda())
    buf = torch.zeros(X.size + 4, dtype=torch.float32, device=_cuda())
    shifted = buf[1:1 + X.size].view(X.shape)
    shifted.copy_(aligned)
    assert aligned.data_ptr() % 16 == 0 and shifted.data_ptr() % 16 == 4
    a = head.predict_proba_device(aligned)
    b = head.predict_proba_device(shifted)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(b.cpu().numpy(), a.cpu().numpy())
    _mlp_check(b.cpu().numpy(), X, coefs, intercepts, "misaligned device X")
    head.close()


def test_mlp_head_saturated_logits():
    """Inputs scaled until output logits pass both +90 and -90: every probability finite, in [0, 1] and inside its
    interval (a saturated head returns exactly 0 and 1, which the threshold search sees as ties)."""
    dims = [64, 100, 17]
    head, coefs, intercepts = _head(dims, 51)
    X = np.random.default_rng(8).standard_normal((300, 64)).astype(np.float32)

    def logits(x):
        a = x.astype(np.float64)
        for l, (w, b) in enumerate(zip(coefs, intercepts)):
            a = a @ w.astype(np.float64) + b
            a = np.maximum(a, 0) if l < len(coefs) - 1 else a
        return a

    while not ((logits(X) > 90).any() and (logits(X) < -90).any()):
        X = X * np.float32(2)
    probs = head.predict_proba(X)
    assert np.isfinite(probs).all() and (probs >= 0).all() and (probs <= 1).all()
    assert (probs == 0).any() and (probs == 1).any()
    _mlp_check(probs, X, coefs, intercepts, "saturated")
    head.close()


# ------------------------------------------------------------------------------------------------ wrapper
def _fit_quietly(est, X, y):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        est.fit(X, y)


@pytest.mark.parametrize("y_shape", ["(n, 1)", "(n,)"])
def test_wrapper_single_output_matches_sklearn_shape(y_shape):
    """One label column, or a 1-D y, gives sklearn a single output unit, and predict_proba returns (n, 2) = [1 - p, p];
    the wrapper must return the same."""
    from sklearn.neural_network import MLPClassifier
    from code_intelligence_b200.mlp import MLPWrapper
    rng = np.random.default_rng(9)
    X = rng.random((80, 12)).astype(np.float32)
    y = (X[:, 0] + 0.3 * rng.random(80) > 0.6).astype(int)
    y = y[:, None] if y_shape == "(n, 1)" else y
    clf = MLPClassifier(random_state=1234, max_iter=50)
    w = MLPWrapper(clf=clf)
    _fit_quietly(w, X, y)
    assert clf.n_outputs_ == 1
    Xt = rng.random((300, 12)).astype(np.float32)
    got, want = w.predict_probabilities(Xt), clf.predict_proba(Xt)
    assert got.shape == want.shape == (300, 2)
    np.testing.assert_allclose(got, want, atol=5e-3)


def test_wrapper_single_label_thresholds_score_column_zero():
    """find_probability_thresholds on y (n, 1) scores label 0 by column 0 of predict_probabilities, as the reference's
    y_pred[:, label] does."""
    from sklearn.model_selection import train_test_split
    from sklearn.neural_network import MLPClassifier
    from code_intelligence_b200.mlp import MLPWrapper, pr_thresholds_host
    rng = np.random.default_rng(10)
    X = rng.random((200, 12)).astype(np.float32)
    y = (X[:, :1] + 0.3 * rng.random((200, 1)) > 0.6).astype(int)
    w = MLPWrapper(clf=MLPClassifier(random_state=1234, max_iter=50), precision_threshold=0.0, recall_threshold=0.0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        w.find_probability_thresholds(X, y)
    _, X_test, _, y_test = train_test_split(X, y, test_size=0.3, random_state=1234)
    scores = w.predict_probabilities(X_test)
    np.testing.assert_allclose(scores, w.clf.predict_proba(X_test), atol=5e-3)    # column 0 is 1 - p
    thr, prec, rec = pr_thresholds_host(scores[:, :1], y_test, 0.0, 0.0)
    assert w.total_labels_count == 1
    assert w.probability_thresholds == {0: thr[0]} and w.precisions == {0: prec[0]} and w.recalls == {0: rec[0]}


def test_wrapper_grid_search_estimator():
    """A fitted GridSearchCV goes through MLPHead.from_sklearn via best_estimator_."""
    from sklearn.neural_network import MLPClassifier
    from code_intelligence_b200.mlp import MLPWrapper
    rng = np.random.default_rng(11)
    X = rng.random((80, 12)).astype(np.float32)
    y = rng.choice([0, 1], size=(80, 4))
    w = MLPWrapper(clf=MLPClassifier(random_state=1234, max_iter=30))
    w.grid_search(params={"hidden_layer_sizes": [(100,), (50, 50)]}, cv=2, n_jobs=1)
    _fit_quietly(w, X, y)
    Xt = rng.random((300, 12)).astype(np.float32)
    np.testing.assert_allclose(w.predict_probabilities(Xt), w.clf.predict_proba(Xt), atol=5e-3)
    assert w._head.dims == [12, *w.clf.best_estimator_.hidden_layer_sizes, 4]
