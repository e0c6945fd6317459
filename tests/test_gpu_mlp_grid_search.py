"""GPU tests of the grid search on the device (code_intelligence_b200/mlp_train.py DeviceGridSearchCV, csrc/mlp_group.cu):
every fit trained in a group equals its own DeviceMLPClassifier.fit bit for bit, the default grid equals the serial
search, launches per step do not grow with the group, group size does not change bits, a diverging fit stays in its
slot, and the MLPWrapper path works end to end."""
import warnings

import numpy as np
import pytest

from code_intelligence_b200 import mlp_train as MT
from code_intelligence_b200.mlp_train import DeviceGridSearchCV, DeviceGroupSteps, DeviceMLPClassifier, DeviceSteps

pytestmark = pytest.mark.gpu


def _data(n, D, L, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, D)).astype(np.float32)
    Y = (X @ rng.standard_normal((D, L)) + 0.5 * rng.standard_normal((n, L)) > 0).astype(int)
    return X, Y


def _standalone(params, X, y):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return DeviceMLPClassifier(**params).fit(X, y)


def _assert_same_fit(a, b):
    for u, v in zip(a.coefs_ + a.intercepts_, b.coefs_ + b.intercepts_):
        assert u.dtype == v.dtype == np.float32 and np.array_equal(u.view(np.uint32), v.view(np.uint32))
    assert a.loss_curve_ == b.loss_curve_ and a.n_iter_ == b.n_iter_ and a.t_ == b.t_
    assert getattr(a, "validation_scores_", None) == getattr(b, "validation_scores_", None)
    assert a.best_loss_ == b.best_loss_ or (a.best_loss_ is None and b.best_loss_ is None)
    assert getattr(a, "best_validation_score_", None) == getattr(b, "best_validation_score_", None)


def _group_vs_standalone(X, y, jobs, cap=None):
    """jobs: (params, rows) -> every group-trained fit == its standalone fit on X[rows], y[rows]."""
    ests = [(DeviceMLPClassifier(**p), np.asarray(rows)) for p, rows in jobs]
    old, MT._GROUP_CAP = MT._GROUP_CAP, cap
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            trained = MT._train_groups(ests, X, np.asarray(y))
    finally:
        MT._GROUP_CAP = old
    for (p, rows), rec in zip(jobs, trained):
        try:
            want = _standalone(p, X[rows], np.asarray(y)[rows])
        except ValueError as e:
            assert rec.error is not None and str(rec.error) == str(e), (p, rec.error, e)
            continue
        assert rec.error is None, (p, rec.error)
        _assert_same_fit(rec.est, want)
    return trained


def test_production_width_fits_equal_standalone():
    X, Y = _data(420, 1600, 60)
    folds = [np.arange(0, 336), np.arange(84, 420), np.r_[0:84, 168:420]]
    jobs = [(dict(hidden_layer_sizes=(600, 600), alpha=a, learning_rate_init=lr, random_state=s, max_iter=3), f)
            for a, lr, s in [(1e-4, 1e-3, 0), (1.0, 1e-2, 1), (10.0, 1e-1, 2)] for f in folds]
    _group_vs_standalone(X, Y, jobs)


def test_default_grid_hidden_sizes_and_edges_equal_standalone():
    X, Y = _data(240, 48, 6)
    rows_a, rows_b = np.arange(0, 192), np.arange(47, 240)   # 192 / 193 rows: short last batches of 3 / 4 rows at b = 7
    jobs = []
    for h in [(100,), (200,), (400,), (50, 50), (100, 100), (200, 200)]:
        jobs.append((dict(hidden_layer_sizes=h, random_state=3, max_iter=3), rows_a))
        jobs.append((dict(hidden_layer_sizes=h, random_state=4, max_iter=3, batch_size=7), rows_b))
    jobs += [
        (dict(hidden_layer_sizes=(50,), random_state=1, max_iter=2, batch_size=1), np.arange(0, 40)),
        (dict(hidden_layer_sizes=(50,), random_state=1, max_iter=2, batch_size=1), np.arange(5, 45)),
        (dict(hidden_layer_sizes=(50,), random_state=2, max_iter=4, batch_size=1000), rows_a),
        (dict(hidden_layer_sizes=(50,), random_state=2, max_iter=4, batch_size=200), rows_b),
        (dict(hidden_layer_sizes=(50,), random_state=2, max_iter=4, batch_size=25), np.arange(0, 200)),
        (dict(hidden_layer_sizes=(50,), random_state=2, max_iter=4, batch_size=25), np.arange(0, 201)),   # 8 vs 9 steps
        (dict(hidden_layer_sizes=(50,), random_state=5, max_iter=4, shuffle=False, batch_size=30), rows_a),
        # early stopping: fits stopping at different epochs, some at max_iter
        (dict(hidden_layer_sizes=(30, 20), random_state=6, max_iter=25, early_stopping=True, n_iter_no_change=1,
              learning_rate_init=0.05), rows_a),
        (dict(hidden_layer_sizes=(30, 20), random_state=7, max_iter=25, early_stopping=True, n_iter_no_change=3), rows_b),
        (dict(hidden_layer_sizes=(30, 20), random_state=8, max_iter=6, tol=1e-6, batch_size=40), rows_a),
        (dict(hidden_layer_sizes=(30, 20), random_state=9, max_iter=60, tol=5e-2, n_iter_no_change=1,
              batch_size=40), rows_b),
    ]
    trained = _group_vs_standalone(X, Y, jobs)
    iters = {rec.est.n_iter_ for rec in trained[-4:]}
    assert len(iters) >= 3, iters
    # binary y
    _group_vs_standalone(X, Y[:, 0], [(dict(hidden_layer_sizes=(64,), random_state=s, max_iter=4,
                                            early_stopping=bool(s % 2)), rows) for s in range(4)
                                      for rows in (rows_a, rows_b)])


def test_launches_per_epoch_do_not_grow_with_the_group():
    X, Y = _data(400, 64, 6)
    units, bs = [64, 100, 100, 6], 200
    single = DeviceSteps(units)
    rng = np.random.default_rng(0)
    coefs = [rng.standard_normal((units[l], units[l + 1])).astype(np.float32) * 0.1 for l in range(3)]
    ints = [np.zeros(units[l + 1], np.float32) for l in range(3)]
    single.set_params(coefs, ints)
    single.set_data(X, Y)
    order = rng.permutation(400)
    lrs = np.full(2, 1e-3)
    n0 = single.launches
    single.epoch(order, bs, lrs, 1e-4, 0.9, 0.999, 1e-8)
    want = single.launches - n0
    single.close()
    counts = []
    for G in (1, 64):
        g = DeviceGroupSteps(units, G, bs)
        g.set_data(X, Y)
        for j in range(G):
            g.set_model(j, coefs, ints, 1e-4, 0.9, 0.999, 1e-8)
        n0 = g.launches
        g.epoch(list(range(G)), [order] * G, [lrs] * G)
        counts.append(g.launches - n0)
        g.close()
    assert counts == [want, want], (counts, want)
    assert want == 2 * 23


def _small_grid_search(cap, X, Y):
    old, MT._GROUP_CAP = MT._GROUP_CAP, cap
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return DeviceGridSearchCV(DeviceMLPClassifier(random_state=0, max_iter=3),
                                      {"hidden_layer_sizes": [(20,), (10, 10)], "alpha": [1e-3, 1.0],
                                       "learning_rate_init": [1e-3, 1e-2]}, cv=3).fit(X, Y)
    finally:
        MT._GROUP_CAP = old


def test_group_size_does_not_change_bits():
    X, Y = _data(150, 32, 5)
    runs = [_small_grid_search(cap, X, Y) for cap in (1, 7, None)]
    for r in runs[1:]:
        for k in runs[0].cv_results_:
            if not k.endswith("_time"):
                assert np.array_equal(np.asarray(runs[0].cv_results_[k], dtype=object),
                                      np.asarray(r.cv_results_[k], dtype=object)), k
        _assert_same_fit(runs[0].best_estimator_, r.best_estimator_)


def test_diverging_fit_stays_in_its_slot():
    X, Y = _data(200, 40, 4)
    X[:, 0] *= 1e3
    rows = np.arange(200)
    jobs = [(dict(hidden_layer_sizes=(32,), random_state=s, max_iter=5, learning_rate_init=lr), rows)
            for s, lr in [(0, 1e-3), (1, 1e38), (2, 1e-2), (3, 1e12)]]
    trained = _group_vs_standalone(X, Y, jobs)   # each fit, the diverging one included, equals its standalone fit
    bad = trained[1]
    assert bad.error is not None or not np.isfinite(bad.est.loss_curve_).all() or max(bad.est.loss_curve_) > 1e6
    for i in (0, 2):
        assert trained[i].error is None and np.isfinite(trained[i].est.loss_curve_).all()


def test_default_grid_equals_serial_search_and_wrapper():
    """The reference's default grid (180 candidates x 5 folds) at 300 x 64 with 6 labels: cv_results_ equal to the serial
    GridSearchCV(DeviceMLPClassifier, n_jobs=1) except times, the best estimator bit-identical, and MLPWrapper.grid_search
    returns the same search.  Device memory returns to its level before the search."""
    import torch
    from sklearn.model_selection import GridSearchCV

    from code_intelligence_b200.mlp import MLPWrapper
    X, Y = _data(300, 64, 6, seed=3)
    free0 = torch.cuda.mem_get_info()[0]
    base = dict(random_state=1, max_iter=2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        w = MLPWrapper(DeviceMLPClassifier(**base), model_file="unused")
        w.grid_search()
        got = w.clf.fit(X, Y)
        want = GridSearchCV(DeviceMLPClassifier(**base), w.clf.param_grid, cv=5, n_jobs=1).fit(X, Y)
    assert type(got) is DeviceGridSearchCV and len(got.cv_results_["params"]) == 180
    for k in want.cv_results_:
        if not k.endswith("_time"):
            assert np.array_equal(np.asarray(want.cv_results_[k], dtype=object),
                                  np.asarray(got.cv_results_[k], dtype=object)), k
    assert want.best_index_ == got.best_index_ and want.best_score_ == got.best_score_
    _assert_same_fit(want.best_estimator_, got.best_estimator_)
    assert (np.asarray(got.cv_results_["mean_fit_time"]) > 0).all()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 64 << 20


def test_wrapper_search_thresholds_predict_and_dill(tmp_path):
    from code_intelligence_b200.mlp import MLPWrapper
    X, Y = _data(400, 48, 4, seed=5)
    w = MLPWrapper(DeviceMLPClassifier(random_state=0, max_iter=20), model_file=str(tmp_path / "m.dpkl"),
                   precision_threshold=0.5, recall_threshold=0.3)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        w.grid_search({"hidden_layer_sizes": [(32,), (16, 16)], "alpha": [1e-4, 1e-2]}, cv=3)
        w.find_probability_thresholds(X, Y)
    assert isinstance(w.clf, DeviceGridSearchCV) and len(w.probability_thresholds) == 4
    p = w.predict_probabilities(X[:10])
    assert p.shape == (10, 4)
    ref = w.clf.best_estimator_.predict_proba(X[:10])
    assert np.abs(p - ref).max() < 5e-3
    w.save_model()
    w2 = MLPWrapper(None, model_file=str(tmp_path / "m.dpkl"), load_from_model=True)
    assert np.abs(w2.predict_probabilities(X[:10]) - p).max() == 0
