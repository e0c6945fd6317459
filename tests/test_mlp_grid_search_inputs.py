"""CPU tests of DeviceGridSearchCV's handling of what sklearn's search passes to each fit: `sample_weight` is refused
as the serial search refuses it, an unseeded shuffling splitter is drawn once, and list or DataFrame X search as the
array does.  The numpy group backend and helpers are those of test_mlp_grid_search_reference.py."""
import os
import sys
import warnings

import numpy as np
import pytest
from sklearn.model_selection import GridSearchCV
from sklearn.neural_network import MLPClassifier
from threadpoolctl import threadpool_limits

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_mlp_grid_search_reference import NumpyGridSearch, NumpyMLP, _assert_same_search, _data  # noqa: E402


@pytest.fixture(autouse=True)
def _one_thread():
    with threadpool_limits(limits=1):
        yield


@pytest.mark.parametrize("refit", [False, True])
def test_sample_weight_is_refused_as_in_the_serial_search(refit):
    """sklearn's search hands `sample_weight` to every fit; DeviceMLPClassifier refuses it, so every fit fails as it
    does in GridSearchCV(DeviceMLPClassifier) -- no fit trained without the weights is reported."""
    X, Y = _data(60)
    w = np.ones(len(X))
    base = dict(random_state=0, max_iter=2, hidden_layer_sizes=(4,))
    errors = []
    for search in (GridSearchCV(NumpyMLP(**base), {"alpha": [1e-4, 1e-2]}, cv=2, refit=refit),
                   NumpyGridSearch(NumpyMLP(**base), {"alpha": [1e-4, 1e-2]}, cv=2, refit=refit)):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            with pytest.raises(ValueError) as e:
                search.fit(X, Y, sample_weight=w)
        errors.append(str(e.value))
    for e in errors:   # the same failure; the messages differ only in the line numbers of their tracebacks
        assert "sample_weight is not supported by DeviceMLPClassifier" in e
    assert ("All the" in errors[0]) == ("All the" in errors[1])


def test_unseeded_shuffling_splitter_scores_the_splits_it_trained():
    """A splitter that draws new splits on every call (KFold(shuffle=True) without a seed) is drawn once: the search
    scores each fit on the split it was trained on, as a serial search given those splits does."""
    from sklearn.model_selection import KFold
    X, Y = _data(90)
    base = dict(random_state=0, max_iter=3, hidden_layer_sizes=(5,))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = NumpyGridSearch(NumpyMLP(**base), {"alpha": [1e-4, 1e-1]}, cv=KFold(3, shuffle=True)).fit(X, Y)
    assert np.isfinite(got.cv_results_["mean_test_score"]).all()
    assert got.n_splits_ == 3 and len(got.cv_results_["params"]) == 2


def test_list_and_dataframe_inputs_search_as_arrays():
    import pandas as pd
    X, Y = _data(80)
    base = dict(random_state=0, max_iter=3, hidden_layer_sizes=(5,))
    grid = {"alpha": [1e-4, 1e-1]}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = GridSearchCV(MLPClassifier(**base), grid, cv=3).fit(X, Y)
        for Xin in (X.tolist(), pd.DataFrame(X)):
            got = NumpyGridSearch(NumpyMLP(**base), grid, cv=3).fit(Xin, Y)
            _assert_same_search(want, got)
