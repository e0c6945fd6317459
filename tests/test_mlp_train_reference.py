"""CPU tests of the label-MLP trainer's host side: the driver of code_intelligence_b200/mlp_train.py run on the numpy
step backend (oracle/mlp_train_ref.py) against sklearn's own MLPClassifier.fit, the float32 Adam restatement against
sklearn's AdamOptimizer, the refusals, the no-fallback rule, the C header and the sm_90a build of csrc/mlp_train.cu.

Single-threaded BLAS: bit-for-bit comparisons with sklearn need the same summation order in both fits, and no thread
pool is left spinning behind the suite."""
import os
import re
import subprocess
import warnings

import numpy as np
import pytest
from threadpoolctl import threadpool_limits

from code_intelligence_b200.mlp_train import DeviceMLPClassifier
from oracle import mlp_train_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _one_thread():
    with threadpool_limits(limits=1):
        yield


def _data(n=157, D=13, L=4, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, D))
    Y = (X @ rng.standard_normal((D, L)) + 0.3 * rng.standard_normal((n, L)) > 0).astype(int)
    return X, Y


CASES = {
    "defaults": dict(),
    "early_stopping": dict(early_stopping=True),
    "early_stopping_patience_2": dict(early_stopping=True, n_iter_no_change=2, batch_size=50),
    "no_shuffle_batch_7": dict(shuffle=False, batch_size=7),
    "no_shuffle_early": dict(shuffle=False, early_stopping=True, batch_size=40),
    "batch_1": dict(batch_size=1, max_iter=3),
    "batch_over_n": dict(batch_size=1000, max_iter=20),
    "stop_by_loss": dict(tol=1e-2, n_iter_no_change=3, max_iter=200),
    "adaptive_lr_ignored": dict(learning_rate="adaptive", momentum=0.5, power_t=0.1, nesterovs_momentum=False),
    "three_hidden": dict(hidden_layer_sizes=(7, 6, 5), alpha=1e-2),
}


@pytest.mark.parametrize("ydim", [2, 1], ids=["multilabel", "binary"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_driver_reproduces_sklearn_fit_bit_for_bit(case, ydim):
    """Driver + float64 numpy steps == MLPClassifier.fit on float64 inputs: parameters, loss curve, validation scores,
    best values, iterations and t_ bit for bit -- the driver makes sklearn's random draws and decisions."""
    from sklearn.neural_network import MLPClassifier
    X, Y = _data()
    y = Y if ydim == 2 else Y[:, 0]
    params = dict(hidden_layer_sizes=(9, 5), random_state=3, max_iter=30)
    params.update(CASES[case])
    with warnings.catch_warnings(record=True) as wa:
        warnings.simplefilter("always")
        want = MLPClassifier(**params).fit(X, y)
    with warnings.catch_warnings(record=True) as wb:
        warnings.simplefilter("always")
        got = DeviceMLPClassifier(**params)._fit_with(X, y, R.NumpySteps)
    for a, b in zip(want.coefs_ + want.intercepts_, got.coefs_ + got.intercepts_):
        assert a.dtype == b.dtype == np.float64 and (a == b).all()
    assert got.loss_curve_ == want.loss_curve_ and got.loss_ == want.loss_
    assert got.validation_scores_ == want.validation_scores_
    assert got.best_validation_score_ == want.best_validation_score_ and got.best_loss_ == want.best_loss_
    assert (got.n_iter_, got.t_, got.n_layers_, got.n_outputs_, got.out_activation_) == \
        (want.n_iter_, want.t_, want.n_layers_, want.n_outputs_, want.out_activation_)
    assert (got.classes_ == want.classes_).all()
    assert (got.predict_proba(X) == want.predict_proba(X)).all()
    conv = [type(w.message).__name__ for w in wa], [type(w.message).__name__ for w in wb]
    assert conv[0].count("ConvergenceWarning") == conv[1].count("ConvergenceWarning"), conv


def test_cases_cover_both_stopping_rules():
    from sklearn.neural_network import MLPClassifier
    X, Y = _data()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        stop = MLPClassifier(hidden_layer_sizes=(9, 5), random_state=3, **CASES["stop_by_loss"]).fit(X, Y)
        early = MLPClassifier(hidden_layer_sizes=(9, 5), random_state=3, max_iter=30, **CASES["early_stopping"]).fit(X, Y)
        full = MLPClassifier(hidden_layer_sizes=(9, 5), random_state=3, max_iter=30).fit(X, Y)
    assert stop.n_iter_ < 200 and early.n_iter_ < 30 and full.n_iter_ == 30


def _sk_adam(params, grads_seq, **kw):
    from sklearn.neural_network._stochastic_optimizers import AdamOptimizer
    params = [p.copy() for p in params]
    opt = AdamOptimizer(params, **kw)
    for g in grads_seq:
        opt.update_params(params, g)
    return params, opt.ms, opt.vs, opt.t


@pytest.mark.parametrize("kw", [dict(), dict(learning_rate_init=0.1, beta_1=0.5, beta_2=0.9, epsilon=1e-3)])
def test_f32_adam_restatement_matches_sklearn_bit_for_bit(kw):
    """adam_f32 (the device's arithmetic) == sklearn's AdamOptimizer on float32 arrays under NumPy 2's rules, over 60 steps
    with ordinary, zero, subnormal and huge (1e30: v overflows to inf) gradients."""
    rng = np.random.default_rng(7)
    shapes = [(17, 5), (5,), (3, 3)]
    params = [rng.standard_normal(s).astype(np.float32) for s in shapes]
    specials = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, 1e-38, 1e30, -1e30, 3e38, 1e-20], dtype=np.float32)
    grads_seq = []
    for t in range(60):
        gs = []
        for s in shapes:
            g = (rng.standard_normal(s) * 10.0 ** rng.integers(-8, 3)).astype(np.float32)
            flat = g.reshape(-1)
            pick = rng.random(flat.size) < 0.3
            flat[pick] = rng.choice(specials, pick.sum())
            gs.append(g)
        grads_seq.append(gs)
    want_p, want_m, want_v, t_end = _sk_adam(params, grads_seq, **kw)
    lr0, b1, b2 = kw.get("learning_rate_init", 0.001), kw.get("beta_1", 0.9), kw.get("beta_2", 0.999)
    eps = kw.get("epsilon", 1e-8)
    p, m, v = params, [np.zeros_like(x) for x in params], [np.zeros_like(x) for x in params]
    for t, gs in enumerate(grads_seq, start=1):
        lr_t = lr0 * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        p, m, v = R.adam_f32(p, gs, m, v, lr_t, b1, b2, eps)
    assert t_end == 60
    for a, b in zip(want_p + want_m + want_v, p + m + v):
        assert a.dtype == np.float32
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _refused(**kw):
    X, Y = _data(40, 5, 3)
    y = kw.pop("y", Y)
    sw = kw.pop("sample_weight", None)
    with pytest.raises(ValueError) as e:
        DeviceMLPClassifier(hidden_layer_sizes=(4,), max_iter=2, **kw).fit(X if "X" not in kw else kw.pop("X"), y,
                                                                             sample_weight=sw)
    return str(e.value)


def test_refusals_name_the_parameter():
    assert "solver" in _refused(solver="sgd")
    assert "solver" in _refused(solver="lbfgs")
    assert "activation" in _refused(activation="tanh")
    assert "sample_weight" in _refused(sample_weight=np.ones(40))
    assert "warm_start" in _refused(warm_start=True)
    assert "multiclass" in _refused(y=np.arange(40) % 3)
    X, Y = _data(40, 5, 3)
    X[3, 2] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        DeviceMLPClassifier(hidden_layer_sizes=(4,)).fit(X, Y)
    X[3, 2] = np.inf
    with pytest.raises(ValueError, match="infinity"):
        DeviceMLPClassifier(hidden_layer_sizes=(4,)).fit(X, Y)
    with pytest.raises(ValueError, match="partial_fit"):
        DeviceMLPClassifier(hidden_layer_sizes=(4,)).partial_fit(X, Y)


def test_fit_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("checks the no-GPU failure mode")
    X, Y = _data(40, 5, 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        DeviceMLPClassifier(hidden_layer_sizes=(4,), max_iter=2).fit(X, Y)


def test_estimator_is_sklearn_compatible():
    from sklearn.base import clone
    est = DeviceMLPClassifier(hidden_layer_sizes=(600, 600), alpha=1e-4, early_stopping=True, learning_rate="adaptive")
    c = clone(est)
    assert type(c) is DeviceMLPClassifier and c.get_params() == est.get_params()


def test_header_compiles_as_c99(tmp_path):
    src = tmp_path / "train_decl.c"
    src.write_text('#include "issue_emb_b200.h"\n'
                   'int main(void) { ie_mlp_train* h = 0; (void)h; return 0; }\n')
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                    "-c", str(src), "-o", str(tmp_path / "train_decl.o")], check=True)


def test_mlp_train_cu_built_for_sm_90a_reports_registers_and_spills():
    """The library build compiles csrc/mlp_train.cu for sm_90a with `-Xptxas -v` (csrc/Makefile): every kernel of the
    training step is there, without spills (DESIGN.md section 9 states the figures)."""
    from code_intelligence_b200 import _lib
    _lib.load()
    text = open(os.path.join(ROOT, "code_intelligence_b200", "csrc", "build", "mlp_train.ptxas.log")).read()
    assert "sm_90a" in text
    entries = re.findall(r"Compiling entry function '([^']+)'", text)
    for k in ("split_store_kernel", "output_kernel", "grad_kernel", "loss_kernel", "adam_kernel"):
        assert any(k in e for e in entries), (k, entries)
    print("mlp_train.cu ptxas:", [l.strip() for l in text.splitlines() if "registers" in l or "spill" in l])
    spills = [int(s) for s in re.findall(r"(\d+) bytes spill stores", text)]
    regs = [int(r) for r in re.findall(r"Used (\d+) registers", text)]
    assert len(regs) == 5 and max(regs) <= 64 and not any(spills)


def _device_like_step(X, Y, rows, coefs, ints, alpha):
    """One training step in float64 from the float32 inputs, rounded to f32 where the device rounds: every activation,
    p, every delta (the masked ones on the f32 activation), the product a^T delta, the add of f32(alpha) W and the
    division by b; the intercept gradient and the loss in f64 from those values, as DeviceSteps.debug_step returns it."""
    f32, f64 = np.float32, np.float64
    b, nl = len(rows), len(coefs)
    a = [X[rows].astype(f32)]
    for l in range(nl):
        z = a[-1].astype(f64) @ coefs[l].astype(f64) + ints[l].astype(f64)
        a.append((np.maximum(z, 0) if l < nl - 1 else 1.0 / (1.0 + np.exp(-z))).astype(f32))
    p = a[-1]
    d = [None] * nl
    d[-1] = (p - Y[rows].astype(f32)).astype(f32)
    for l in range(nl - 1, 0, -1):
        d[l - 1] = np.where(a[l] != 0, (d[l].astype(f64) @ coefs[l].T.astype(f64)).astype(f32), f32(0))
    cg = [(((a[l].T.astype(f64) @ d[l].astype(f64)).astype(f32) + (f32(alpha) * coefs[l]).astype(f32)).astype(f32)
           / f32(b)).astype(f32) for l in range(nl)]
    ig = [(d[l].astype(f64).sum(0) / b).astype(f32) for l in range(nl)]
    pc = np.clip(p.astype(f64), 2.0 ** -23, 1 - 2.0 ** -23)
    terms = np.where(Y[rows] != 0, np.log(pc), np.log1p(-pc))
    loss = -terms.sum() / b + 0.5 * alpha * sum(float((c.astype(f64) ** 2).sum()) for c in coefs) / b
    return {"acts": a[1:-1], "p": p, "deltas": d, "coef_grads": cg, "intercept_grads": ig, "loss": float(loss)}


def _stage_failing(out, X, Y, rows, coefs, ints, alpha):
    try:
        R.check_step(out, X, Y, rows, coefs, ints, alpha)
    except AssertionError as e:
        return e.args[0][0]
    return None


@pytest.mark.parametrize("layer", [0, 2])
def test_step_checker_accepts_a_device_like_step_and_rejects_stale_rows_and_unmasked_deltas(layer):
    """oracle.mlp_train_ref.check_step is sharp enough for what it is meant to catch: it accepts a step rounded where
    the device rounds, and rejects (at the right stage) the same step whose coef gradient of one layer also carries
    28 rows of another batch (workspace rows of an earlier batch left in a short batch's K padding), and one whose
    masked delta lets through a single element where the activation is 0."""
    units = [40, 24, 16, 5]
    rng = np.random.default_rng(17)
    n, b, alpha = 300, 57, 1e-2
    X = rng.standard_normal((n, units[0])).astype(np.float32)
    Y = (rng.random((n, units[-1])) < 0.3).astype(np.uint8)
    coefs, ints = [], []
    for fi, fo in zip(units[:-1], units[1:]):
        bound = np.sqrt(6.0 / (fi + fo))
        coefs.append(rng.uniform(-bound, bound, (fi, fo)).astype(np.float32))
        ints.append(rng.uniform(-bound, bound, fo).astype(np.float32))
    order = rng.permutation(n).astype(np.int32)
    rows, stale = order[:b], order[b:b + 28]
    out = _device_like_step(X, Y, rows, coefs, ints, alpha)
    stats = R.check_step(out, X, Y, rows, coefs, ints, alpha)
    assert max(stats.values()) <= 1.0, stats

    # 28 extra rows in layer `layer`'s product a^T delta, divided by the batch's own b
    both = _device_like_step(X, Y, np.concatenate([rows, stale]), coefs, ints, alpha)
    a_all = ([X[np.concatenate([rows, stale])]] + both["acts"])[layer].astype(np.float64)
    d_all = both["deltas"][layer].astype(np.float64)
    f32 = np.float32
    dw = (a_all[:b].T @ d_all[:b] + a_all[b:].T @ d_all[b:]).astype(f32)
    bad = dict(out, coef_grads=list(out["coef_grads"]))
    bad["coef_grads"][layer] = ((dw + (f32(alpha) * coefs[layer]).astype(f32)).astype(f32) / f32(b)).astype(f32)
    assert _stage_failing(bad, X, Y, rows, coefs, ints, alpha) == f"coef_grad{layer}"

    # one delta not masked: an element where the f32 activation is 0 keeps its product value
    l = 1 if layer == 0 else 0
    unmasked = (out["deltas"][l + 1].astype(np.float64) @ coefs[l + 1].T.astype(np.float64)).astype(f32)
    r, c = np.argwhere((out["acts"][l] == 0) & (unmasked != 0))[0]
    bad = dict(out, deltas=[x.copy() for x in out["deltas"]])
    bad["deltas"][l][r, c] = unmasked[r, c]
    assert _stage_failing(bad, X, Y, rows, coefs, ints, alpha) == f"delta{l}"
