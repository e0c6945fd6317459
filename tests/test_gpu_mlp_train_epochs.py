"""GPU tests of the label-MLP trainer across whole epochs (``ie_mlp_train_epoch``, ``ie_mlp_train_validation_proba``,
``ie_mlp_train_snapshot``; DESIGN.md section 9).

A fit enqueues every step of an epoch in one call: each step takes its own learning rate, its loss reads the
sum |W|^2 partials the previous Adam pass wrote, the last batch is short and runs on a workspace sized for the full
batch, and the Adam moments carry over from one call to the next.  Here an epoch handle E is pinned to a replay handle S
that runs the same steps one at a time through the debug hook, each step checked stage by stage
(``oracle.mlp_train_ref.check_step``) and each Adam pass bit for bit against ``adam_f32``.  The validation pass
(chunks of the workspace's rows), the best-parameter snapshot and its restore, and the parameters a fit returns are
tied bit for bit to fresh handles and to the recorded snapshots."""
import warnings

import numpy as np
import pytest
import torch

from code_intelligence_b200.mlp_train import DeviceMLPClassifier, DeviceSteps
from oracle import mlp_train_ref as R

pytestmark = pytest.mark.gpu

B1, B2, EPS, LR0 = 0.9, 0.999, 1e-8, 0.001
CHECK_DEVICE = "cuda"   # where check_step forms its float64 references


def _init(units, seed):
    rng = np.random.RandomState(seed)
    coefs, ints = [], []
    for a, b in zip(units[:-1], units[1:]):
        bound = np.sqrt(6.0 / (a + b))
        coefs.append(rng.uniform(-bound, bound, (a, b)).astype(np.float32))
        ints.append(rng.uniform(-bound, bound, b).astype(np.float32))
    return coefs, ints


def _lr(t):
    """The driver's (and sklearn's AdamOptimizer's) learning rate of Adam step t >= 1."""
    return LR0 * np.sqrt(1 - B2 ** t) / (1 - B1 ** t)


def _tie(name, want, got):
    """Bit-for-bit equality of two lists of float32 arrays; on failure the count of differing elements and the largest
    difference in units of the reference's last place."""
    assert len(want) == len(got), name
    for i, (a, b) in enumerate(zip(want, got)):
        a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
        assert a.shape == b.shape, (name, i, a.shape, b.shape)
        diff = a.view(np.uint32) != b.view(np.uint32)
        if diff.any():
            ulp = np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.spacing(np.abs(a)).astype(np.float64)
            raise AssertionError((name, i, int(diff.sum()), float(ulp[diff].max())))


def _tie_step(name, want, got):
    """Two debug steps equal bit for bit: activations, p, deltas, gradients and the f64 loss."""
    for k in ("acts", "deltas", "coef_grads", "intercept_grads"):
        _tie(f"{name}:{k}", want[k], got[k])
    _tie(f"{name}:p", [want["p"]], [got["p"]])
    assert np.float64(want["loss"]).view(np.uint64) == np.float64(got["loss"]).view(np.uint64), \
        (f"{name}:loss", want["loss"], got["loss"])


def _data(units, n, seed, n_val=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, units[0])).astype(np.float32)
    Y = (rng.random((n, units[-1])) < 0.3).astype(np.uint8)
    Xv = rng.standard_normal((n_val, units[0])).astype(np.float32) if n_val else None
    return X, Y, Xv


def _fresh(units, coefs, ints, X, Y, X_val=None):
    h = DeviceSteps(units)
    h.set_params(coefs, ints)
    h.set_data(X, Y, X_val)
    return h


def _flat(params):
    return list(params[0]) + list(params[1])


# ------------------------------------------------------------------------------------------------ a. epoch = its steps
# name: (layer units, n, the batch size of each epoch call, alpha, validation pass before the first epoch)
EPOCHS = {
    "production": ([1600, 600, 600, 60], 457, (200, 200, 200), 1e-4, False),   # 200/200/57: kb 64 of kb_cap 256
    "b64_last1": ([100, 64, 48, 7], 129, (64, 64, 64), 1e-2, False),             # 64/64/1
    "b65": ([100, 64, 48, 7], 130, (65, 65, 65), 1e-2, False),                   # 65/65: kb_cap 128
    "b129_last42": ([100, 64, 48, 7], 300, (129, 129, 129), 1e-2, False),        # 129/129/42: kb_cap 192
    "b1": ([37, 40, 9], 5, (1, 1, 1), 1e-2, False),                              # one row per step
    "one_step_per_call": ([100, 64, 48, 7], 150, (150, 150, 150), 1e-2, False),  # Adam state crosses calls at lr[0]
    "b1000": ([100, 300, 20], 2100, (1000, 1000, 1000), 1e-2, False),            # cap_m 1024, last batch 100
    "three_hidden": ([90, 70, 50, 30, 11], 250, (100, 100, 100), 1e-2, False),   # 100/100/50
    "binary_L1": ([80, 40, 1], 200, (90, 90, 90), 1e-2, False),                  # 90/90/20
    "L257": ([120, 260, 257], 300, (130, 130, 130), 1e-2, False),                # 130/130/40
    "val_first": ([100, 64, 48, 7], 200, (64, 64, 64), 1e-2, True),              # epochs on a 256-row workspace
    "growing_batch": ([100, 64, 48, 7], 457, (64, 200, 64), 1e-2, False),        # the workspace grows mid-fit
}


@pytest.mark.parametrize("name", list(EPOCHS))
def test_epoch_equals_its_checked_steps(name):
    """E runs whole epochs (one shuffled order and the driver's lr_t per call, t continuing across calls); S replays
    every step through the debug hook at the parameters it holds, checks it stage by stage, then applies Adam with the
    device's own gradients, bit for bit against adam_f32 on host-tracked moments.  E's batch losses and final
    parameters equal S's bit for bit, and one probe Adam pass with the same gradients ties E's moments too.  Each short
    last step also equals a fresh handle's step (workspace rows == b) bit for bit: no row of an earlier batch leaks."""
    units, n, batch_sizes, alpha, val_first = EPOCHS[name]
    X, Y, Xv = _data(units, n, seed=11, n_val=300 if val_first else 0)
    coefs, ints = _init(units, 12)
    mem0 = torch.cuda.mem_get_info()[0]
    E, S = _fresh(units, coefs, ints, X, Y, Xv), _fresh(units, coefs, ints, X, Y)
    if val_first:
        E.val_proba()
    host_m = [np.zeros_like(p) for p in coefs + ints]
    host_v = [np.zeros_like(p) for p in coefs + ints]
    rng = np.random.default_rng(13)
    t, worst, n_short = 0, {}, 0
    for bs in batch_sizes:
        order = rng.permutation(n).astype(np.int32)
        steps = -(-n // bs)
        lrs = np.array([_lr(t + k + 1) for k in range(steps)])
        losses = E.epoch(order, bs, lrs, alpha, B1, B2, EPS)
        for k in range(steps):
            rows = order[k * bs:(k + 1) * bs]
            c, i = S.params()
            out = S.debug_step(rows, alpha)
            try:
                stats = R.check_step(out, X, Y, rows, c, i, alpha, CHECK_DEVICE)
            except AssertionError as e:
                raise AssertionError((name, "step", t + k + 1, len(rows), *e.args)) from None
            for s, v in stats.items():
                worst[s] = max(worst.get(s, 0.0), v)
            assert losses[k] == out["loss"], (name, t + k + 1, losses[k], out["loss"])
            if len(rows) < bs:
                F = _fresh(units, c, i, X, Y)
                _tie_step(f"{name} fresh handle, step {t + k + 1}", F.debug_step(rows, alpha), out)
                F.close()
                n_short += 1
            grads = out["coef_grads"] + out["intercept_grads"]
            p, host_m, host_v = R.adam_f32(c + i, grads, host_m, host_v, lrs[k], B1, B2, EPS)
            dp, dm, dv = S.debug_adam(out["coef_grads"], out["intercept_grads"], lrs[k], B1, B2, EPS)
            _tie(f"{name} adam step {t + k + 1}", p + host_m + host_v, dp + dm + dv)
        t += steps
    _tie(f"{name} epoch vs replay parameters", _flat(S.params()), _flat(E.params()))
    # probe: the same gradients into both handles' moments
    p_now = _flat(S.params())
    g = [(rng.standard_normal(x.shape) * 1e-2).astype(np.float32) for x in p_now]
    nl = len(units) - 1
    want = R.adam_f32(p_now, g, host_m, host_v, _lr(t + 1), B1, B2, EPS)
    got_e = E.debug_adam(g[:nl], g[nl:], _lr(t + 1), B1, B2, EPS)
    got_s = S.debug_adam(g[:nl], g[nl:], _lr(t + 1), B1, B2, EPS)
    mem = mem0 - torch.cuda.mem_get_info()[0]
    _tie(f"{name} probe E vs S", sum(got_s, []), sum(got_e, []))
    _tie(f"{name} probe S vs adam_f32", sum(want, []), sum(got_s, []))
    E.close()
    S.close()
    assert n_short == sum(n % bs != 0 for bs in batch_sizes)
    print(name, f"{t} steps, {n_short} short; two handles {mem / 2 ** 20:.0f} MiB;",
          {k: round(v, 3) for k, v in worst.items()})


# ------------------------------------------------------------------------------------------------ b. validation
# name: (layer units, n_train, batch size, n_val); chunks of the workspace's rows: 256 after a batch of at most 256
VALIDATION = {
    "nval1": ([100, 64, 48, 7], 300, 64, 1),
    "nval2": ([100, 64, 48, 7], 300, 64, 2),
    "nval255": ([100, 64, 48, 7], 300, 64, 255),
    "nval256": ([100, 64, 48, 7], 300, 64, 256),
    "nval257": ([100, 64, 48, 7], 300, 200, 257),     # two chunks
    "nval513": ([100, 64, 48, 7], 300, 200, 513),     # three chunks, the last of one row
    "nval257_L16": ([100, 64, 16], 300, 200, 257),    # L a multiple of 16
    "nval257_production": ([1600, 600, 600, 60], 457, 200, 257),
    "nval2001_b1000": ([100, 300, 20], 2100, 1000, 2001),   # chunks of 1000, 1000, 1
}


@pytest.mark.parametrize("name", list(VALIDATION))
def test_validation_proba_equals_a_checked_forward(name):
    """After each of two epochs, val_proba equals bit for bit the p of a debug step over the same rows on a fresh handle
    at the epoch handle's parameters (the validation X as its training set, one forward over every row), and that
    step's stages pass check_step: the chunk loop neither drops, shifts nor mixes a row."""
    units, n, bs, n_val = VALIDATION[name]
    X, Y, Xv = _data(units, n, seed=21, n_val=n_val)
    Yv = (np.random.default_rng(22).random((n_val, units[-1])) < 0.3).astype(np.uint8)
    coefs, ints = _init(units, 23)
    E = _fresh(units, coefs, ints, X, Y, Xv)
    rng = np.random.default_rng(24)
    t = 0
    for _ in range(2):
        steps = -(-n // bs)
        E.epoch(rng.permutation(n).astype(np.int32), bs, [_lr(t + k + 1) for k in range(steps)], 1e-2, B1, B2, EPS)
        t += steps
        vp = E.val_proba()
        c, i = E.params()
        F = _fresh(units, c, i, Xv, Yv)
        rows = np.arange(n_val, dtype=np.int32)
        out = F.debug_step(rows, 1e-2)
        F.close()
        stats = R.check_step(out, Xv, Yv, rows, c, i, 1e-2, CHECK_DEVICE)
        _tie(f"{name} val_proba vs debug step", [out["p"]], [vp])
    E.close()
    print(name, {k: round(v, 3) for k, v in stats.items() if k in ("p", "a1")})


# ------------------------------------------------------------------------------------------------ c. snapshot
@pytest.mark.parametrize("units", [[100, 64, 48, 7], [1600, 600, 600, 60]], ids=["small", "production"])
def test_restore_refreshes_every_derived_copy(units):
    """A snapshot at P0 survives three epochs (params(best=True) == P0); after ie_mlp_train_snapshot(restore=1) the
    parameters are P0 and the validation probabilities and a whole debug step (activations, gradients, loss) equal a
    fresh handle's at P0 bit for bit: the split-bf16 weight copies and the sum |W|^2 partials were rebuilt."""
    n, bs = 457, 200
    X, Y, Xv = _data(units, n, seed=31, n_val=300)
    coefs, ints = _init(units, 32)
    E = _fresh(units, coefs, ints, X, Y, Xv)
    E.snapshot()
    rng = np.random.default_rng(33)
    t = 0
    for _ in range(3):
        E.epoch(rng.permutation(n).astype(np.int32), bs, [_lr(t + k + 1) for k in range(3)], 1e-2, B1, B2, EPS)
        t += 3
        E.val_proba()
    moved = _flat(E.params())
    assert any(not np.array_equal(a, b) for a, b in zip(moved, coefs + ints))
    _tie("best before restore", coefs + ints, _flat(E.params(best=True)))
    assert E._lib.ie_mlp_train_snapshot(E._h, 1) == 0
    _tie("params after restore", coefs + ints, _flat(E.params()))
    F = _fresh(units, coefs, ints, X, Y, Xv)
    _tie("val_proba after restore", [F.val_proba()], [E.val_proba()])
    rows = rng.permutation(n)[:bs].astype(np.int32)
    _tie_step("debug step after restore", F.debug_step(rows, 1e-2), E.debug_step(rows, 1e-2))
    F.close()
    E.close()


# ------------------------------------------------------------------------------------------------ d. the fit's result
class _Recording(DeviceSteps):
    """Records params() after every epoch and at every snapshot (with the number of epochs run before it)."""
    log = None

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        _Recording.log = {"epochs": [], "snapshots": []}

    def epoch(self, *a):
        out = super().epoch(*a)
        _Recording.log["epochs"].append(_flat(self.params()))
        return out

    def snapshot(self):
        super().snapshot()
        _Recording.log["snapshots"].append((len(_Recording.log["epochs"]), _flat(self.params())))


def _fit_set(n=900, seed=41):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 30)).astype(np.float32)
    Y = (X @ rng.standard_normal((30, 4)) + 1.5 * rng.standard_normal((n, 4)) > 0.5).astype(int)
    return X, Y


def test_fit_returns_the_last_snapshot():
    """An early-stopping fit returns, bit for bit, the parameters of its last snapshot, taken after the epoch of the
    first maximum of validation_scores_, which here comes before the last epoch; a fit without early stopping returns
    the last epoch's parameters."""
    X, Y = _fit_set()
    params = dict(hidden_layer_sizes=(32, 16), random_state=5, max_iter=60, batch_size=64, n_iter_no_change=4)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        clf = DeviceMLPClassifier(early_stopping=True, **params)._fit_with(X, Y, _Recording)
    log = _Recording.log
    scores = clf.validation_scores_
    best = int(np.argmax(scores)) + 1           # epochs are counted from 1; np.argmax takes the first maximum
    assert len(log["epochs"]) == clf.n_iter_ == len(scores)
    assert best < clf.n_iter_, (best, scores)
    last_epoch, last_params = log["snapshots"][-1]
    assert last_epoch == best, (last_epoch, best, scores)
    assert log["snapshots"][0][0] == 0 and len(log["snapshots"]) >= 2
    _tie("snapshot vs its epoch", log["epochs"][best - 1], last_params)
    _tie("coefs_ vs last snapshot", last_params, clf.coefs_ + clf.intercepts_)
    _tie("_best_coefs vs last snapshot", last_params, clf._best_coefs + clf._best_intercepts)
    assert any(not np.array_equal(a, b) for a, b in zip(log["epochs"][-1], last_params))
    print("validation scores", scores, "best epoch", best, "of", clf.n_iter_)

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        full = DeviceMLPClassifier(early_stopping=False, **{**params, "max_iter": 8})._fit_with(X, Y, _Recording)
    assert full.n_iter_ == len(_Recording.log["epochs"]) and _Recording.log["snapshots"] == []
    _tie("fit without early stopping vs last epoch", _Recording.log["epochs"][-1], full.coefs_ + full.intercepts_)
