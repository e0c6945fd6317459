"""CPU tests of the grid search's host side (code_intelligence_b200/mlp_train.py DeviceGridSearchCV): the lockstep group
runner on a numpy step backend -- G oracle.mlp_train_ref.NumpySteps stepping together -- against sklearn's own
GridSearchCV(MLPClassifier), the index-based early-stopping split, the no-fallback rule, the C header and the sm_90a
build of csrc/mlp_group.cu.

Single-threaded BLAS: bit-for-bit comparisons with sklearn need the same summation order in both searches."""
import os
import re
import subprocess
import warnings

import numpy as np
import pytest
from sklearn.model_selection import GridSearchCV, train_test_split
from sklearn.neural_network import MLPClassifier
from threadpoolctl import threadpool_limits

from code_intelligence_b200 import mlp_train as MT
from code_intelligence_b200.mlp_train import DeviceGridSearchCV, DeviceMLPClassifier
from oracle import mlp_train_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _one_thread():
    with threadpool_limits(limits=1):
        yield


class NumpyGroupSteps:
    """Group backend of G NumpySteps in lockstep, each on rows of the shared X / Y the runner names."""

    dtype = None

    def __init__(self, layer_units, n_models, batch_size, device=0):
        self.steps = [R.NumpySteps(layer_units) for _ in range(n_models)]
        self.bs = batch_size
        self.consts = [None] * n_models

    def set_data(self, X, Y):
        self.X, self.Y = X, Y

    def set_model(self, j, coefs, intercepts, alpha, beta_1, beta_2, epsilon, val_rows=None):
        self.steps[j].set_params(coefs, intercepts)
        self.steps[j].set_data(self.X, self.Y, None if val_rows is None else self.X[val_rows])
        self.consts[j] = (alpha, beta_1, beta_2, epsilon)

    def epoch(self, models, rows, lrs):
        return [self.steps[j].epoch(r, self.bs, lr, *self.consts[j]) for j, r, lr in zip(models, rows, lrs)]

    def val_proba(self, j):
        return self.steps[j].val_proba()

    def snapshot(self, j):
        self.steps[j].snapshot()

    def params(self, j, best=False):
        return self.steps[j].params(best)

    def close(self):
        pass


class NumpyMLP(DeviceMLPClassifier):
    """DeviceMLPClassifier whose single fits (the refit) run on the numpy steps."""

    def fit(self, X, y, sample_weight=None):
        return self._fit_with(X, y, R.NumpySteps, sample_weight)


class NumpyGridSearch(DeviceGridSearchCV):
    _group_steps_cls = NumpyGroupSteps


def _data(n=157, D=13, L=4, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, D))
    Y = (X @ rng.standard_normal((D, L)) + 0.3 * rng.standard_normal((n, L)) > 0).astype(int)
    return X, Y


def _assert_same_search(want, got):
    keys = [k for k in want.cv_results_ if not k.endswith("_time")]
    assert sorted(keys) == sorted(k for k in got.cv_results_ if not k.endswith("_time"))
    for k in keys:
        a, b = want.cv_results_[k], got.cv_results_[k]
        if isinstance(a, np.ma.MaskedArray):
            assert list(a) == list(b), k
        else:
            a, b = np.asarray(a), np.asarray(b)
            assert a.shape == b.shape and (np.array_equal(a, b, equal_nan=a.dtype.kind == "f")), (k, a, b)
    assert want.best_index_ == got.best_index_ and want.best_params_ == got.best_params_
    assert want.best_score_ == got.best_score_ or (np.isnan(want.best_score_) and np.isnan(got.best_score_))
    for a, b in zip(want.best_estimator_.coefs_ + want.best_estimator_.intercepts_,
                    got.best_estimator_.coefs_ + got.best_estimator_.intercepts_):
        assert a.dtype == b.dtype and (a == b).all()
    assert want.best_estimator_.loss_curve_ == got.best_estimator_.loss_curve_


def _both(X, y, base, grid, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = GridSearchCV(MLPClassifier(**base), grid, n_jobs=1, **kw).fit(X, y)
        got = NumpyGridSearch(NumpyMLP(**base), grid, n_jobs=-1, **kw).fit(X, y)
    return want, got


SEARCHES = {
    # mixed hidden sizes and batch sizes; 157 rows in 5 folds: training sets of 125 and 126 rows, so with batch 25 the
    # folds' step counts differ by one
    "mixed": (dict(random_state=3, max_iter=8),
              {"hidden_layer_sizes": [(9,), (6, 5)], "batch_size": [25, "auto"], "alpha": [1e-4, 1.0]}),
    "early_stopping": (dict(random_state=1, max_iter=15, early_stopping=True, n_iter_no_change=2),
                       {"hidden_layer_sizes": [(7,), (8, 4)], "learning_rate_init": [0.001, 0.05]}),
    "stop_by_loss": (dict(random_state=2, max_iter=60, tol=1e-2, n_iter_no_change=2, batch_size=40),
                     {"learning_rate_init": [0.01, 0.1], "learning_rate": ["constant", "adaptive"]}),
}


@pytest.mark.parametrize("ydim", [2, 1], ids=["multilabel", "binary"])
@pytest.mark.parametrize("case", sorted(SEARCHES))
def test_group_runner_reproduces_sklearn_search_bit_for_bit(case, ydim):
    """Group runner + float64 numpy steps in lockstep == GridSearchCV(MLPClassifier) on float64 inputs: every
    cv_results_ key except the times, best_index_, best_params_, best_score_ and the refit's parameters."""
    X, Y = _data()
    y = Y if ydim == 2 else Y[:, 0]
    base, grid = SEARCHES[case]
    want, got = _both(X, y, base, grid, cv=5, return_train_score=True)
    _assert_same_search(want, got)


def test_folds_with_different_step_counts_are_covered():
    X, _ = _data()
    from sklearn.model_selection import KFold
    sizes = {len(tr) for tr, _ in KFold(5).split(X)}
    assert {-(-s // 25) for s in sizes} == {5, 6}


@pytest.mark.parametrize("ydim", [2, 1], ids=["multilabel", "binary"])
def test_refused_candidate_fails_as_in_the_serial_search(ydim):
    X, Y = _data(80)
    y = Y if ydim == 2 else Y[:, 0]
    base = dict(random_state=0, max_iter=4, hidden_layer_sizes=(5,))
    grid = {"activation": ["relu", "tanh"], "alpha": [1e-4, 1e-2]}
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        got = NumpyGridSearch(NumpyMLP(**base), grid, cv=3, error_score=np.nan).fit(X, y)
    assert any(type(x.message).__name__ == "FitFailedWarning" for x in w)
    refused = [i for i, p in enumerate(got.cv_results_["params"]) if p["activation"] == "tanh"]
    assert refused and all(np.isnan(got.cv_results_["mean_test_score"][i]) for i in refused)
    assert got.best_params_["activation"] == "relu"
    # the same candidates that sklearn's search accepts score exactly as there
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = GridSearchCV(MLPClassifier(**base), {"alpha": [1e-4, 1e-2]}, cv=3).fit(X, y)
    ok = [i for i, p in enumerate(got.cv_results_["params"]) if p["activation"] == "relu"]
    assert list(got.cv_results_["mean_test_score"][ok]) == list(want.cv_results_["mean_test_score"])
    with pytest.raises(ValueError, match="activation"):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            NumpyGridSearch(NumpyMLP(**base), grid, cv=3, error_score="raise").fit(X, y)
    with pytest.raises(ValueError, match="solver"):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            NumpyGridSearch(NumpyMLP(**base), {"solver": ["sgd"]}, cv=3, error_score="raise").fit(X, y)


def test_random_state_instance_reproduces_the_serial_search():
    X, Y = _data(90)
    base = dict(random_state=np.random.RandomState(5), max_iter=5, hidden_layer_sizes=(6,))
    want, got = _both(X, Y, base, {"alpha": [1e-4, 0.1]}, cv=3)
    _assert_same_search(want, got)


@pytest.mark.parametrize("ydim", [2, 1], ids=["multilabel", "binary"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_index_split_equals_the_copy_split(ydim, seed):
    """The early-stopping split of an index array (stratified by y for binary y) is the partition train_test_split
    makes of X and y themselves."""
    X, Y = _data(101, seed=seed)
    y = Y if ydim == 2 else Y[:, :1]
    stratify = y if ydim == 1 else None
    Xt, Xv, yt, yv = train_test_split(X, y, random_state=np.random.RandomState(seed), test_size=0.2, stratify=stratify)
    tr, va = MT._split_rows(len(X), np.random.RandomState(seed), 0.2, stratify)
    assert (X[tr] == Xt).all() and (X[va] == Xv).all() and (y[tr] == yt).all() and (y[va] == yv).all()


def test_other_estimators_are_refused():
    X, Y = _data(40)
    with pytest.raises(ValueError, match="DeviceMLPClassifier"):
        DeviceGridSearchCV(MLPClassifier(), {"alpha": [1e-4]}).fit(X, Y)


def test_search_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("checks the no-GPU failure mode")
    X, Y = _data(40, 5, 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        DeviceGridSearchCV(DeviceMLPClassifier(hidden_layer_sizes=(4,), max_iter=2), {"alpha": [1e-4, 1e-3]},
                           cv=2).fit(X, Y)


def test_wrapper_builds_the_device_search_for_the_device_estimator():
    from code_intelligence_b200.mlp import MLPWrapper
    w = MLPWrapper(DeviceMLPClassifier(), model_file="unused")
    w.grid_search({"alpha": [1e-4]}, cv=2)
    assert type(w.clf) is DeviceGridSearchCV
    w = MLPWrapper(MLPClassifier(), model_file="unused")
    w.grid_search({"alpha": [1e-4]}, cv=2)
    assert type(w.clf) is GridSearchCV


def test_header_declares_the_group_abi(tmp_path):
    src = tmp_path / "group_decl.c"
    src.write_text('#include "issue_emb_b200.h"\n'
                   'int main(void) { ie_mlp_group* h = 0; (void)h; (void)&ie_mlp_group_create; (void)&ie_mlp_group_epoch;'
                   ' (void)&ie_mlp_group_capacity; (void)&ie_mlp_group_validation_proba; (void)&ie_mlp_group_snapshot;'
                   ' return 0; }\n')
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                    "-c", str(src), "-o", str(tmp_path / "group_decl.o")], check=True)


def test_mlp_group_cu_built_for_sm_90a_without_spills():
    """csrc/mlp_group.cu is compiled for sm_90a with `-Xptxas -v`: every group kernel and the GEMM's group instantiation
    are there, none spills."""
    from code_intelligence_b200 import _lib
    _lib.load()
    text = open(os.path.join(ROOT, "code_intelligence_b200", "csrc", "build", "mlp_group.ptxas.log")).read()
    assert "sm_90a" in text
    entries = re.findall(r"Compiling entry function '([^']+)'", text)
    for k in ("group_split_store_kernel", "group_output_kernel", "group_grad_kernel", "group_loss_kernel",
              "group_adam_kernel", "GroupEpi"):
        assert any(k in e for e in entries), (k, entries)
    print("mlp_group.cu ptxas:", [l.strip() for l in text.splitlines() if "registers" in l or "spill" in l])
    spills = [int(s) for s in re.findall(r"(\d+) bytes spill stores", text)]
    assert len(entries) == 6 and not any(spills)
