"""CPU tests of oracle/thresholds.py, the exact reference the device threshold search (csrc/pr_curve.cu) is checked
against in tests/test_gpu_label_head.py, and the case generator both files share.

The cases are built around the kernel's structure: the padded sort size n_pow2 = max(1024, 2^ceil(log2 n)) steps at
1024 / 2048 / 4096 / 8192 / 16384 and each of the 1024 threads owns per = n_pow2 / 1024 consecutive sorted positions,
so tie groups are placed to straddle those runs; and around the float edges of the score encoding: adjacent floats,
subnormals, negative scores, +-0, exact 0 and 1, magnitudes near FLT_MAX."""
import numpy as np
import pytest

from oracle import thresholds as T

NS = (1, 2, 3, 1023, 1024, 1025, 2047, 2048, 2049, 4097, 8191, 8193, 16383, 16384)
# (0.75, 0.5) and (0.1, 0) are attained exactly by EXACT_CASES; fl(0.1) > 1/10, so a precision of 1/10 computed in
# float64 passes `>= 0.1` although the exact ratio is below the exact threshold
THRESHOLDS = ((0.0, 0.0), (1.0, 1.0), (0.75, 0.5), (0.1, 0.0), (1.01, 0.0))
SCORE_PATTERNS = ("equal", "two_values", "straddle", "adjacent", "subnormal", "negative", "saturated", "signed_zero",
                  "huge", "sigmoid_q")
TRUTH_PATTERNS = ("none", "all", "top", "bottom", "alternating", "random")
F32_MAX = np.finfo(np.float32).max


def per_thread(n):
    """Sorted positions each thread of pr_threshold_kernel owns."""
    n_pow2 = 1024
    while n_pow2 < n:
        n_pow2 *= 2
    return n_pow2 // 1024


def score_pattern(name, n, rng):
    f = np.float32
    if name == "equal":
        return np.full(n, 0.5, f)
    if name == "two_values":
        return rng.choice(np.array([0.25, 0.75], f), n)
    if name == "straddle":
        # tie groups in sorted order whose sizes cycle around the thread run length, rows shuffled
        per = per_thread(n)
        sizes = np.resize(np.array([per + 1, 1, 2 * per + 1, per, max(per - 1, 1), 3 * per + 2]), n)
        group = np.repeat(np.arange(n), sizes)[:n]
        values = np.linspace(1.0, 0.0, group[-1] + 1).astype(f)
        return values[group][rng.permutation(n)]
    if name == "adjacent":
        chain = [f(1.0)]
        for _ in range(63):
            chain.append(np.nextafter(chain[-1], f(0.0)))
        return np.array(chain, f)[rng.integers(0, 64, n)]
    if name == "subnormal":
        bits = rng.integers(0, 0x00800001, n, dtype=np.uint32)        # +0 .. the smallest normal
        bits[: min(n, 4)] = [1, 2, 0x007FFFFF, 0x00800000][: min(n, 4)]
        bits |= np.where(rng.random(n) < 0.5, np.uint32(0x80000000), np.uint32(0))
        return bits.view(f)
    if name == "negative":
        return (-np.round(rng.exponential(1.0, n) * 64) / 64).astype(f)
    if name == "saturated":                                            # what a head whose logits pass +-90 returns
        mid = (1 / (1 + np.exp(-rng.standard_normal(n) * 4))).astype(f)
        return np.where(rng.random(n) < 0.4, f(0.0), np.where(rng.random(n) < 0.67, f(1.0), mid)).astype(f)
    if name == "signed_zero":
        return rng.choice(np.array([-0.0, 0.0, 0.25, -0.25], f), n, p=[0.4, 0.4, 0.1, 0.1])
    if name == "huge":
        fixed = np.array([F32_MAX, -F32_MAX, 1e38, -1e38, np.nextafter(f(1e38), f(0)), 3e38], f)
        out = rng.choice(fixed, n)
        wide = rng.random(n) < 0.3
        out[wide] = (rng.uniform(-3.4, 3.4, int(wide.sum())) * 1e38).astype(f)
        return out
    if name == "sigmoid_q":
        return (np.round(256 / (1 + np.exp(-3 * rng.standard_normal(n)))) / 256).astype(f)
    raise KeyError(name)


def truth_pattern(name, scores, rng):
    n = len(scores)
    t = np.zeros(n, np.uint8)
    rank = np.argsort(-scores.astype(np.float64), kind="stable")      # rank[0] holds the highest score
    if name == "all":
        t[:] = 1
    elif name == "top":
        t[rank[0]] = 1
    elif name == "bottom":
        t[rank[-1]] = 1
    elif name == "alternating":
        t[rank[::2]] = 1
    elif name == "random":
        t[:] = rng.random(n) < 0.3
    elif name != "none":
        raise KeyError(name)
    return t


def case_matrix(n, n_labels, seed=0):
    """(scores, truth), each (n, n_labels): column j has score pattern j % 10 and truth pattern (j // 10) % 6, so 60
    labels cover every pair and wider matrices repeat them with fresh draws."""
    scores = np.empty((n, n_labels), np.float32)
    truth = np.empty((n, n_labels), np.uint8)
    for j in range(n_labels):
        rng = np.random.default_rng([seed, n, j])
        s = score_pattern(SCORE_PATTERNS[j % len(SCORE_PATTERNS)], n, rng)
        scores[:, j] = s
        truth[:, j] = truth_pattern(TRUTH_PATTERNS[(j // len(SCORE_PATTERNS)) % len(TRUTH_PATTERNS)], s, rng)
    return scores, truth


def _column(scores_sorted_desc, truth_sorted_desc, n_rows_perm_seed):
    s = np.asarray(scores_sorted_desc, np.float32)
    t = np.asarray(truth_sorted_desc, np.uint8)
    p = np.random.default_rng(n_rows_perm_seed).permutation(len(s))
    return s[p][:, None], t[p][:, None]


# Small cases whose answer is known by hand: (name, scores, truth, p_thr, r_thr, (threshold, precision, recall)).
EXACT_CASES = [
    # sklearn's loop: one tie group {-0, 0, 0, -0} at threshold 0 -> precision 3/5, recall 1.  Ordering -0 below +0
    # would give the point "+0 and above" (precision 2/3, recall 2/3) instead.
    ("signed_zero", np.array([0, -0.0, 0.5, 0, -0.0], np.float32), np.array([1, 0, 1, 0, 1], np.uint8), 0.6, 0.6,
     (0.0, 0.6, 1.0)),
    # precision exactly 3/4 at recall exactly 1/2 (3 of 6 positives in the top 4); every other point fails a threshold
    ("attained_0.75_0.5", *_column(np.arange(10, 0, -1) / 16, [1, 1, 0, 1, 0, 0, 0, 1, 1, 1], 1), 0.75, 0.5,
     (7 / 16, 0.75, 0.5)),
    # the only positive is the lowest of 10 distinct scores: precision 1/10 == fl(0.1) qualifies for p_thr = 0.1
    ("attained_0.1", *_column(np.arange(10, 0, -1) / 16, [0] * 9 + [1], 2), 0.1, 0.0, (1 / 16, 0.1, 1.0)),
    # all positive: every point has precision 1, the lowest threshold wins
    ("ties_lowest_threshold", *_column([0.875, 0.75, 0.75, 0.25], [1, 1, 1, 1], 3), 0.0, 0.0, (0.25, 1.0, 1.0)),
    # no positive: precision 0 everywhere, never selected even at p_thr = 0
    ("no_positive", *_column([0.875, 0.5, 0.125], [0, 0, 0], 4), 0.0, 0.0, (None, 0.0, 0.0)),
    # one tie group, alternating truth: the only point is the whole group (precision 1/2); a point inside the group
    # would reach precision 1
    ("one_group", *_column([0.5] * 6, [1, 0, 1, 0, 1, 0], 5), 0.0, 0.0, (0.5, 0.5, 1.0)),
]


def _flat(scores, truth):
    return np.asarray(scores, np.float32).reshape(len(scores), -1), np.asarray(truth, np.uint8).reshape(len(truth), -1)


def assert_same(got, want, tag=""):
    """Thresholds by value (-0.0 == +0.0), precisions and recalls bit for bit."""
    assert [t is None for t in got[0]] == [t is None for t in want[0]], tag
    assert [t for t in got[0] if t is not None] == [t for t in want[0] if t is not None], tag
    for g, w in ((got[1], want[1]), (got[2], want[2])):
        np.testing.assert_array_equal(np.array(g, np.float64).view(np.int64), np.array(w, np.float64).view(np.int64),
                                      err_msg=str(tag))


@pytest.mark.parametrize("name,scores,truth,p_thr,r_thr,expected", EXACT_CASES, ids=[c[0] for c in EXACT_CASES])
def test_exact_cases_by_hand(name, scores, truth, p_thr, r_thr, expected):
    from code_intelligence_b200.mlp import pr_thresholds_host
    scores, truth = _flat(scores, truth)
    want = ([None if expected[0] is None else float(expected[0])], [expected[1]], [expected[2]])
    assert_same(T.pr_thresholds(scores, truth, p_thr, r_thr), want, name)
    assert_same(pr_thresholds_host(scores, truth, p_thr, r_thr), want, name)


@pytest.mark.parametrize("n", NS)
def test_reference_equals_sklearn_loop(n):
    """Every score pattern x truth pattern x (p_thr, r_thr), at every n the kernel's structure distinguishes: the
    reference equals the reference's own loop on sklearn's curve, exactly."""
    from code_intelligence_b200.mlp import pr_thresholds_host
    scores, truth = case_matrix(n, len(SCORE_PATTERNS) * len(TRUTH_PATTERNS))
    for p_thr, r_thr in THRESHOLDS:
        assert_same(T.pr_thresholds(scores, truth, p_thr, r_thr), pr_thresholds_host(scores, truth, p_thr, r_thr),
                    (n, p_thr, r_thr))


@pytest.mark.parametrize("n", (3, 1025, 16384))
def test_stopping_the_curve_at_full_recall_changes_nothing(n):
    """scikit-learn before 1.1 ends the curve at the first point of full recall; every later point has the same tp and
    more fp, hence a strictly lower precision, so it is never chosen and the result does not depend on the release."""
    scores, truth = case_matrix(n, len(SCORE_PATTERNS) * len(TRUTH_PATTERNS), seed=1)
    for p_thr, r_thr in THRESHOLDS:
        assert_same(T.pr_thresholds(scores, truth, p_thr, r_thr, stop_at_full_recall=True),
                    T.pr_thresholds(scores, truth, p_thr, r_thr), (n, p_thr, r_thr))
    for name, s, t, p_thr, r_thr, _ in EXACT_CASES:
        s, t = _flat(s, t)
        assert_same(T.pr_thresholds(s, t, p_thr, r_thr, stop_at_full_recall=True), T.pr_thresholds(s, t, p_thr, r_thr),
                    name)


def test_reference_is_fast_at_the_largest_shape():
    """600 labels x 16384 rows, the widest call the device path takes, in seconds."""
    import time
    scores, truth = case_matrix(16384, 600, seed=2)
    t0 = time.perf_counter()
    T.pr_thresholds(scores, truth, 0.7, 0.5)
    assert time.perf_counter() - t0 < 20.0


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf, np.uint32(0xFFFFFFFF).view(np.float32)])
def test_non_finite_scores_are_rejected_before_the_library(bad, monkeypatch):
    """sklearn's curve raises ValueError on NaN / inf; pr_thresholds() does the same before it loads the library (so
    this runs without one), and so does the reference."""
    from code_intelligence_b200 import _lib, mlp
    def no_library():
        raise AssertionError("the library must not be reached")
    monkeypatch.setattr(_lib, "load", no_library)
    scores, truth = case_matrix(37, 3)
    scores[5, 1] = bad
    with pytest.raises(ValueError):
        mlp.pr_thresholds(scores, truth, 0.5, 0.5)
    with pytest.raises(ValueError):
        T.pr_thresholds(scores, truth, 0.5, 0.5)
    with pytest.raises(ValueError):
        mlp.pr_thresholds_host(scores, truth, 0.5, 0.5)
