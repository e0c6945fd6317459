"""GPU tests of the label-MLP trainer (csrc/mlp_train.cu + the split-bf16 GEMM, driven by code_intelligence_b200/
mlp_train.py): the Adam step bit for bit, one training step teacher-forced stage by stage within the bounds of
oracle/device_numerics (DESIGN.md section 9), the driver's decisions against a real sklearn fit, determinism, the
outcome at the RepoMLP configuration against sklearn's float64 fit, and the paths through MLPWrapper, dill and
GridSearchCV."""
import os
import warnings

import numpy as np
import pytest

from code_intelligence_b200.mlp_train import DeviceMLPClassifier, DeviceSteps
from oracle import mlp_train_ref as R

pytestmark = pytest.mark.gpu


def _init(units, seed):
    rng = np.random.RandomState(seed)
    coefs, ints = [], []
    for a, b in zip(units[:-1], units[1:]):
        bound = np.sqrt(6.0 / (a + b))
        coefs.append(rng.uniform(-bound, bound, (a, b)).astype(np.float32))
        ints.append(rng.uniform(-bound, bound, b).astype(np.float32))
    return coefs, ints


# ------------------------------------------------------------------------------------------------ Adam
def test_adam_step_bit_exact():
    """Given gradients in, the device's parameters and moments equal oracle.mlp_train_ref.adam_f32 bit for bit over
    several steps, with zero, subnormal and huge gradients among them."""
    units = [37, 70, 5, 3]
    coefs, ints = _init(units, 1)
    steps = DeviceSteps(units)
    steps.set_params(coefs, ints)
    rng = np.random.default_rng(2)
    p = coefs + ints
    m = [np.zeros_like(x) for x in p]
    v = [np.zeros_like(x) for x in p]
    specials = np.array([0.0, -0.0, 1e-45, 1e-40, 1e30, -1e30, 1e-20], dtype=np.float32)
    b1, b2, eps = 0.9, 0.999, 1e-8
    for t in range(1, 9):
        gs = []
        for x in p:
            g = (rng.standard_normal(x.shape) * 10.0 ** rng.integers(-6, 2)).astype(np.float32)
            flat = g.reshape(-1)
            pick = rng.random(flat.size) < 0.2
            flat[pick] = rng.choice(specials, pick.sum())
            gs.append(g)
        lr_t = 0.001 * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        p, m, v = R.adam_f32(p, gs, m, v, lr_t, b1, b2, eps)
        dp, dm, dv = steps.debug_adam(gs[:3], gs[3:], lr_t, b1, b2, eps)
        for want, got in zip(p + m + v, dp + dm + dv):
            assert np.array_equal(want.view(np.uint32), got.view(np.uint32)), t
    c, i = steps.params()
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(p, c + i))
    steps.close()


# ------------------------------------------------------------------------------------------------ one step per stage
SHAPES = {   # (D, hidden, L, b)
    "production": (1600, (600, 600), 60, 200),
    "b1": (100, (64,), 7, 1),
    "b63": (100, (64, 48), 7, 63),
    "b64": (100, (64, 48), 7, 64),
    "b65": (100, (64, 48), 7, 65),
    "b129": (100, (300,), 20, 129),
    "short_last_batch": (200, (100, 100), 12, 57),
    "D37": (37, (40,), 9, 50),
    "hidden5": (64, (5,), 6, 80),
    "three_hidden": (90, (70, 50, 30), 11, 100),
    "binary_L1": (80, (40,), 1, 90),
    "L257": (120, (260,), 257, 130),
}
# edge cases on a shape of SHAPES: alpha; the last layer's intercepts (saturated outputs: +40 gives p = 1.0f exactly,
# -40 a p far below the loss's clip, about -88 a zero from __fdividef's denominator above 2^126, -100 a zero from an
# infinite one); a dead first hidden layer (every relu output 0); constant label columns; X scaled by a power of two
EDGES = {
    "alpha0": ("b65", dict(alpha=0.0)),
    "alpha1e-4_production": ("production", dict(alpha=1e-4)),
    "alpha10": ("b65", dict(alpha=10.0)),
    "out_bias+40": ("b65", dict(out_bias=40.0)),
    "out_bias-40": ("b65", dict(out_bias=-40.0)),
    "out_bias-88": ("b65", dict(out_bias=-88.0)),
    "out_bias-100": ("b65", dict(out_bias=-100.0)),
    "dead_hidden": ("b65", dict(dead=True)),
    "constant_labels": ("short_last_batch", dict(constant_labels=True)),
    "x_scale_2^20": ("b65", dict(x_scale=2.0 ** 20)),
    "x_scale_2^-40": ("b65", dict(x_scale=2.0 ** -40)),
}


@pytest.mark.parametrize("shape", list(SHAPES) + list(EDGES))
def test_one_step_teacher_forced_per_stage(shape):
    """Each stage of one step, fed the device's own inputs, lies inside its bound (DESIGN.md section 9): activations,
    probabilities, output deltas (exact), masked deltas, coef and intercept gradients, the batch loss.  The edge shapes
    put rows and columns of padding into every product: a padding row or column that contributed would leave a bound.
    The edge cases reach the loss's clip with both label values, exact zeros through a dead layer, and inputs far from
    unit scale."""
    base, knobs = EDGES.get(shape, (shape, {}))
    D, hidden, L, b = SHAPES[base]
    units = [D, *hidden, L]
    rng = np.random.default_rng(3)
    n = max(2 * b, 300)
    X = rng.standard_normal((n, D)).astype(np.float32) * np.float32(knobs.get("x_scale", 1.0))
    Y = (rng.random((n, L)) < 0.3).astype(np.uint8)
    if knobs.get("constant_labels"):
        Y[:, 0::3] = 0
        Y[:, 1::3] = 1
    coefs, ints = _init(units, 4)
    if "out_bias" in knobs:
        ints[-1][:] = knobs["out_bias"]
    if knobs.get("dead"):
        ints[0][:] = -1e3
    alpha = knobs.get("alpha", 1e-2)
    steps = DeviceSteps(units)
    steps.set_params(coefs, ints)
    steps.set_data(X, Y)
    rows = rng.choice(n, b, replace=False).astype(np.int32)
    out = steps.debug_step(rows, alpha)
    steps.close()
    stats = R.check_step(out, X, Y, rows, coefs, ints, alpha)
    print(shape, {k: round(v, 3) for k, v in stats.items()})
    f32 = np.float32
    if "out_bias" in knobs:   # the clip is reached with both label values
        pc = np.clip(out["p"], f32(2.0 ** -23), f32(1 - 2.0 ** -23))
        clipped = pc != out["p"]
        assert (clipped & (Y[rows] == 0)).any() and (clipped & (Y[rows] == 1)).any()
        if knobs["out_bias"] == 40.0:
            assert (out["p"] == 1.0).all()
        if knobs["out_bias"] <= -88.0:
            assert (out["p"] == 0.0).any()
    if knobs.get("dead"):     # exact: a1 = 0, so delta0 = 0 and the first two coef gradients are f32(f32(alpha W) / b)
        assert (out["acts"][0] == 0).all() and (out["deltas"][0] == 0).all() and (out["intercept_grads"][0] == 0).all()
        for l in (0, 1):
            want = ((f32(alpha) * coefs[l]).astype(f32) / f32(b)).astype(f32)
            assert np.array_equal(out["coef_grads"][l].view(np.uint32), want.view(np.uint32)), l


# ------------------------------------------------------------------------------------------------ decisions
class _Recording(DeviceSteps):
    log = {}

    def set_params(self, coefs, intercepts):
        _Recording.log.setdefault("init", ([c.copy() for c in coefs], [b.copy() for b in intercepts]))
        super().set_params(coefs, intercepts)

    def set_data(self, X, Y, X_val=None):
        _Recording.log["data"] = (X.copy(), None if X_val is None else X_val.copy())
        super().set_data(X, Y, X_val)

    def epoch(self, order, *args):
        _Recording.log.setdefault("orders", []).append(np.array(order))
        return super().epoch(order, *args)


def test_same_decisions_as_sklearn(monkeypatch):
    """The initial parameters, the validation split and every epoch's row order the device receives are the ones a real
    sklearn fit of the same float32 data draws (recorded from inside sklearn)."""
    from sklearn.neural_network import MLPClassifier
    import sklearn.neural_network._multilayer_perceptron as mp
    rng = np.random.default_rng(5)
    X = rng.standard_normal((300, 21)).astype(np.float32)
    Y = (rng.random((300, 6)) < 0.4).astype(int)
    params = dict(hidden_layer_sizes=(17, 9), random_state=11, max_iter=4, early_stopping=True, batch_size=64)
    seen = {"orders": []}
    real_shuffle, real_split, real_init = mp.shuffle, mp.train_test_split, MLPClassifier._initialize

    def rec_shuffle(idx, random_state):
        out = real_shuffle(idx, random_state=random_state)
        seen["orders"].append(np.array(out))
        return out

    def rec_split(*a, **k):
        out = real_split(*a, **k)
        seen["split"] = (out[0].copy(), out[1].copy())
        return out

    def rec_init(self, y, units, dtype):
        real_init(self, y, units, dtype)
        seen["init"] = ([c.copy() for c in self.coefs_], [b.copy() for b in self.intercepts_])

    monkeypatch.setattr(mp, "shuffle", rec_shuffle)
    monkeypatch.setattr(mp, "train_test_split", rec_split)
    monkeypatch.setattr(MLPClassifier, "_initialize", rec_init)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        MLPClassifier(**params).fit(X, Y)
    monkeypatch.undo()
    _Recording.log = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        DeviceMLPClassifier(**params)._fit_with(X, Y, _Recording)
    log = _Recording.log
    for a, b in zip(seen["init"][0] + seen["init"][1], log["init"][0] + log["init"][1]):
        assert a.dtype == b.dtype == np.float32 and np.array_equal(a, b)
    assert np.array_equal(seen["split"][0], log["data"][0]) and np.array_equal(seen["split"][1], log["data"][1])
    assert len(seen["orders"]) == len(log["orders"]) == 4
    assert all(np.array_equal(a, b) for a, b in zip(seen["orders"], log["orders"]))


# ------------------------------------------------------------------------------------------------ determinism
def test_fits_are_deterministic_and_ignore_the_learning_rate_schedule():
    rng = np.random.default_rng(6)
    X = rng.standard_normal((700, 50)).astype(np.float32)
    Y = (rng.random((700, 8)) < 0.3).astype(int)
    fits = []
    for lr in ("constant", "constant", "adaptive"):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            fits.append(DeviceMLPClassifier(hidden_layer_sizes=(64, 32), random_state=2, max_iter=5, early_stopping=True,
                                            learning_rate=lr).fit(X, Y))
    a = fits[0]
    for b in fits[1:]:
        for u, v in zip(a.coefs_ + a.intercepts_, b.coefs_ + b.intercepts_):
            assert np.array_equal(u.view(np.uint32), v.view(np.uint32))
        assert a.loss_curve_ == b.loss_curve_ and a.validation_scores_ == b.validation_scores_


# ------------------------------------------------------------------------------------------------ quality
def _teacher(n, seed=0, D=1600, L=60, k=16):
    """A learnable multilabel set: 1600-d inputs carrying a 16-d latent factor under noise, labels the top 10 % of a
    fixed random linear teacher on the factor."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((k, D))
    W = rng.standard_normal((k, L))
    Z = rng.standard_normal((n, k))
    X = (Z @ A / np.sqrt(k) + 0.5 * rng.standard_normal((n, D))).astype(np.float32)
    logits = Z @ W
    return X, (logits > np.quantile(logits, 0.9, axis=0)).astype(int)


REPO_MLP = dict(solver="adam", activation="relu", hidden_layer_sizes=(600, 600), alpha=1e-4, early_stopping=True,
                validation_fraction=0.1, n_iter_no_change=5, max_iter=3000, random_state=1234,
                learning_rate="adaptive")
AUC_TOL = 0.01


def test_quality_at_the_repo_mlp_configuration():
    """Held-out micro-averaged AUC of the device fit vs sklearn's float64 fit, both at the RepoMLP hyperparameters; both
    stop before max_iter.  Also reports (without asserting) how far the device's coefs drift from float64 steps on the
    same rows after 1, 10 and 100 steps."""
    from sklearn.metrics import roc_auc_score
    from sklearn.neural_network import MLPClassifier
    X, Y = _teacher(4000)
    Xtr, Ytr, Xte, Yte = X[:3000], Y[:3000], X[3000:], Y[3000:]
    dev = DeviceMLPClassifier(**REPO_MLP).fit(Xtr, Ytr)
    sk = MLPClassifier(**REPO_MLP).fit(Xtr.astype(np.float64), Ytr)
    auc_dev = roc_auc_score(Yte, dev.predict_proba(Xte), average="micro")
    auc_sk = roc_auc_score(Yte, sk.predict_proba(Xte.astype(np.float64)), average="micro")
    print(f"AUC device {auc_dev:.5f} ({dev.n_iter_} epochs)  sklearn f64 {auc_sk:.5f} ({sk.n_iter_} epochs)  "
          f"gap {auc_dev - auc_sk:+.5f}")
    assert dev.n_iter_ < REPO_MLP["max_iter"] and sk.n_iter_ < REPO_MLP["max_iter"]
    assert auc_sk > 0.9
    assert auc_dev >= auc_sk - AUC_TOL

    units = [1600, 600, 600, 60]
    coefs, ints = _init(units, 9)
    d, h = DeviceSteps(units), R.NumpySteps(units)
    d.set_params(coefs, ints)
    h.set_params([c.astype(np.float64) for c in coefs], [b.astype(np.float64) for b in ints])
    Xs, Ys = Xtr[:200], Ytr[:200].astype(bool)     # one full batch per epoch: epoch k is step k
    d.set_data(Xs, Ys)
    h.set_data(Xs.astype(np.float64), Ys)
    order = np.arange(200)
    report = {}
    for t in range(1, 101):
        lr = np.array([0.001 * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)])
        d.epoch(order, 200, lr, 1e-4, 0.9, 0.999, 1e-8)
        h.epoch(order, 200, lr, 1e-4, 0.9, 0.999, 1e-8)
        if t in (1, 10, 100):
            cd, ch = d.params()[0], h.params()[0]
            num = sum(float(((a.astype(np.float64) - b) ** 2).sum()) for a, b in zip(cd, ch))
            report[t] = np.sqrt(num / sum(float((b ** 2).sum()) for b in ch))
    d.close()
    print("coef rel-L2 device vs float64 steps after 1 / 10 / 100 steps:", {k: f"{v:.3e}" for k, v in report.items()})


# ------------------------------------------------------------------------------------------------ integration
def _small_set(n=600, seed=8):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 40)).astype(np.float32)
    Y = (X @ rng.standard_normal((40, 5)) + 0.5 * rng.standard_normal((n, 5)) > 0.8).astype(int)
    return X, Y


def test_wrapper_thresholds_dill_round_trip_and_grid_search(tmp_path):
    """MLPWrapper(DeviceMLPClassifier) end to end: find_probability_thresholds agrees with pr_thresholds_host on the
    estimator's own hold-out probabilities; save_model / load_model (dill) round-trips, and the loaded model predicts
    through sklearn's host code too; GridSearchCV with n_jobs=1 refits the best estimator, which loads into MLPHead."""
    from sklearn.model_selection import train_test_split
    from code_intelligence_b200.mlp import MLPHead, MLPWrapper, pr_thresholds_host
    X, Y = _small_set()
    clf = DeviceMLPClassifier(hidden_layer_sizes=(32, 16), random_state=1, max_iter=40, early_stopping=True)
    w = MLPWrapper(clf, model_file=str(tmp_path / "model.dpkl"), precision_threshold=0.6, recall_threshold=0.4)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        w.find_probability_thresholds(X, Y)
    _, X_te, _, y_te = train_test_split(X, Y, test_size=0.3, random_state=1234)
    probs = w.predict_probabilities(X_te)
    thr, prec, rec = pr_thresholds_host(probs, y_te, 0.6, 0.4)
    for l in range(Y.shape[1]):
        got = w.probability_thresholds[l]
        assert (got is None) == (thr[l] is None), l
        if got is not None:
            assert got == pytest.approx(thr[l], abs=1e-7)
            assert w.precisions[l] == pytest.approx(prec[l]) and w.recalls[l] == pytest.approx(rec[l])
    assert isinstance(w.clf, DeviceMLPClassifier) and all(c.dtype == np.float32 for c in w.clf.coefs_)
    w.save_model()
    w2 = MLPWrapper(None, model_file=str(tmp_path / "model.dpkl"), load_from_model=True)
    assert np.array_equal(w2.predict_probabilities(X_te), probs)
    assert np.abs(w2.clf.predict_proba(X_te) - probs).max() < 5e-3        # sklearn's host forward pass

    g = MLPWrapper(DeviceMLPClassifier(hidden_layer_sizes=(16,), random_state=2, max_iter=20))
    g.grid_search(params={"alpha": [1e-4, 1e-1], "learning_rate": ["constant", "adaptive"]}, cv=2, n_jobs=1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        g.fit(X, Y)
    best = g.clf.best_estimator_
    assert isinstance(best, DeviceMLPClassifier)
    head = MLPHead.from_sklearn(g.clf)
    assert np.abs(head.predict_proba(X[:50]) - best.predict_proba(X[:50])).max() < 5e-3
    head.close()
