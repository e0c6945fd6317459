"""GPU tests of the grouped label-MLP trainer slot by slot (``ie_mlp_group_*``, csrc/mlp_group.cu; DESIGN.md section 9.1).

Every test drives a ``DeviceGroupSteps`` handle directly, so it chooses each slot's rows, learning rates, position and
the order of calls.  Each active slot j has a twin: a single ``DeviceSteps`` handle with the same initial parameters,
alpha and Adam constants, whose training set is X[train_rows_j] and whose validation set is X[val_rows_j].  In an epoch
slot j steps on the shared X's rows train_rows_j[perm] and its twin on its own rows perm, with the same learning rates,
so both see the same rows in the same order.  After every epoch the two agree bit for bit: each batch loss (as float64
bit patterns), the parameters, the snapshot where one was taken and the validation probabilities.  The single handle is
pinned stage by stage to the float64 oracle (test_gpu_mlp_train.py, test_gpu_mlp_train_epochs.py), so this ties every
slot to it.  The group has no getter for the Adam moments; every test compares at least one epoch after another one on
the same moments, so moments that differ show in that epoch's losses and parameters.

Slots are placed at the first, a middle and the last position of a group with unused slots between them, and the model
list of an epoch is unordered, so no result depends on a model sitting in slot 0."""
import hashlib
import time

import numpy as np
import pytest
import torch

from code_intelligence_b200 import _lib
from code_intelligence_b200.mlp_train import DeviceGroupSteps, DeviceSteps
from oracle import mlp_train_ref as R
from test_gpu_mlp_train import SHAPES
from test_gpu_mlp_train_epochs import EPOCHS, _init, _tie

pytestmark = pytest.mark.gpu

B1, B2, EPS = 0.9, 0.999, 1e-8
CHECK_DEVICE = "cuda"   # where check_step forms its float64 references


def _lr(lr0, t):
    """sklearn AdamOptimizer's learning rate of step t >= 1."""
    return lr0 * np.sqrt(1 - B2 ** t) / (1 - B1 ** t)


def _data(units, n, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, units[0])).astype(np.float32)
    Y = (rng.random((n, units[-1])) < 0.3).astype(np.uint8)
    return X, Y


def _flat(params):
    return list(params[0]) + list(params[1])


def _tie_losses(name, want, got):
    want, got = np.asarray(want, dtype=np.float64), np.asarray(got, dtype=np.float64)
    assert want.shape == got.shape, (name, want.shape, got.shape)
    bad = np.flatnonzero(want.view(np.uint64) != got.view(np.uint64))
    assert bad.size == 0, (name, "steps", bad.tolist(), want[bad].tolist(), got[bad].tolist())


def _digest(arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _last_error(lib):
    return (lib.ie_last_error() or b"").decode()


class _Slot:
    def __init__(self, twin, train_rows, val_rows, alpha, lr0):
        self.twin, self.train_rows, self.val_rows, self.alpha, self.lr0, self.t = twin, train_rows, val_rows, alpha, lr0, 0


class _Twins:
    """A group of G slots over (X, Y) and a single twin handle for every slot it has set.  One group handle per batch
    size: ``epoch(bs=...)`` on another batch size moves every slot's current parameters into that handle's slot with
    ``set_model`` and into its twin with ``set_params``, both of which restart Adam."""

    def __init__(self, units, G, bs, X, Y):
        self.units, self.G, self.X, self.Y = list(units), G, X, Y
        self.handles, self.slots = {}, {}
        self.bs = bs
        self.g = self._handle(bs)

    def _handle(self, bs):
        if bs not in self.handles:
            g = DeviceGroupSteps(self.units, self.G, bs)
            g.set_data(self.X, self.Y)
            self.handles[bs] = g
        return self.handles[bs]

    def set_slot(self, j, params, train_rows, alpha, lr0=1e-3, val_rows=None):
        """(Re)sets slot j: parameters, constants and validation rows on the group, and a fresh twin."""
        old = self.slots.pop(j, None)
        if old is not None:
            old.twin.close()
        train_rows = np.asarray(train_rows)
        self.g.set_model(j, params[0], params[1], alpha, B1, B2, EPS, val_rows)
        tw = DeviceSteps(self.units)
        tw.set_params(*params)
        tw.set_data(self.X[train_rows], self.Y[train_rows], None if val_rows is None else self.X[val_rows])
        self.slots[j] = _Slot(tw, train_rows, val_rows, alpha, lr0)

    def _switch(self, bs):
        if bs == self.bs:
            return
        self.g, self.bs = self._handle(bs), bs
        for j, s in self.slots.items():
            c, i = s.twin.params()
            self.g.set_model(j, c, i, s.alpha, B1, B2, EPS, s.val_rows)
            s.twin.set_params(c, i)
            s.t = 0

    def epoch(self, rng, models=None, bs=None, name=""):
        """One epoch of `models` (default: every set slot, in the order they were set) on the group and on each twin;
        the losses and the parameters afterwards are tied."""
        if bs is not None:
            self._switch(bs)
        models = list(self.slots) if models is None else list(models)
        perms, lrs = [], []
        for j in models:
            s = self.slots[j]
            perms.append(rng.permutation(len(s.train_rows)).astype(np.int32))
            steps = -(-len(s.train_rows) // self.bs)
            lrs.append(np.array([_lr(s.lr0, s.t + k + 1) for k in range(steps)]))
            s.t += steps
        got = self.g.epoch(models, [self.slots[j].train_rows[p] for j, p in zip(models, perms)], lrs)
        for j, p, lr, loss in zip(models, perms, lrs, got):
            s = self.slots[j]
            want = s.twin.epoch(p, self.bs, lr, s.alpha, B1, B2, EPS)
            _tie_losses(f"{name} slot {j} losses", want, loss)
        self.tie_params(models, name=name)
        return got

    def tie_params(self, models=None, best=False, name=""):
        for j in (list(self.slots) if models is None else models):
            _tie(f"{name} slot {j} params(best={best})", _flat(self.slots[j].twin.params(best)),
                 _flat(self.g.params(j, best)))

    def tie_val(self, j, name=""):
        vp = self.g.val_proba(j)
        _tie(f"{name} slot {j} val_proba", [self.slots[j].twin.val_proba()], [vp])
        return vp

    def snapshot(self, j):
        self.g.snapshot(j)
        self.slots[j].twin.snapshot()

    def close(self):
        for s in self.slots.values():
            s.twin.close()
        for g in self.handles.values():
            g.close()


# ------------------------------------------------------------------------------------------- a. the single trainer's shapes
# Every entry of the single trainer's two shape tables runs through a group: EPOCHS of test_gpu_mlp_train_epochs.py
# (ids "epochs-<name>": its layer units, alpha and the batch size of each of its three epoch calls) and SHAPES of
# test_gpu_mlp_train.py (ids "shapes-<name>": its units and b, three epochs).  Here each entry only adds the training
# rows of three slots; an entry added to either table fails here, by name, until it has them.  The row counts differ,
# so one step runs the launch sequences of several batch sizes (full, each short last batch) and some slots have fewer
# steps than others.  growing_batch runs on two group handles over the same slots' parameters (set_model restarts Adam,
# so its twins restart it too with set_params), and its third epoch sets live slots of the first handle again.
SLOT_ROWS = {
    "epochs-production": (457, 400, 201),        # last batches 57 / - / 1
    "epochs-b64_last1": (129, 128, 100),         # 64/64/1, 64/64, 64/36
    "epochs-b65": (130, 131, 70),                # 65/65, 65/65/1, 65/5
    "epochs-b129_last42": (300, 258, 129),       # 129/129/42, 129/129, one step
    "epochs-b1": (5, 3, 1),
    "epochs-one_step_per_call": (150, 151, 200),  # b = n for one slot
    "epochs-b1000": (2100, 2000, 1001),          # last 100 / - / 1
    "epochs-three_hidden": (250, 300, 199),
    "epochs-binary_L1": (200, 180, 91),
    "epochs-L257": (300, 260, 131),
    "epochs-val_first": (200, 192, 65),          # a 300-row validation pass before the first epoch
    "epochs-growing_batch": (457, 400, 263),
    "shapes-production": (200, 400, 399),
    "shapes-b1": (3, 2, 1),
    "shapes-b63": (126, 130, 63),
    "shapes-b64": (128, 129, 64),
    "shapes-b65": (65, 130, 129),
    "shapes-b129": (129, 257, 300),              # last 128 (= m_pad) / 42
    "shapes-short_last_batch": (114, 120, 170),
    "shapes-D37": (100, 123, 50),
    "shapes-hidden5": (160, 200, 81),
    "shapes-three_hidden": (100, 250, 301),
    "shapes-binary_L1": (90, 200, 181),
    "shapes-L257": (130, 300, 261),
}
SLOTS, G_SMALL = [4, 0, 2], 5   # the last, the first and a middle slot of five, listed out of order


@pytest.mark.parametrize("name", [f"epochs-{k}" for k in EPOCHS] + [f"shapes-{k}" for k in SHAPES])
def test_slots_equal_single_handles(name):
    """Three slots of a group, each with its own rows, alpha and initial learning rate, equal their twins after each of
    three epochs (and, for val_first, in a validation pass before the first)."""
    table, key = name.split("-", 1)
    if table == "epochs":
        units, _, batch_sizes, alpha, val_first = EPOCHS[key]
    else:
        D, hidden, L, b = SHAPES[key]
        units, batch_sizes, alpha, val_first = [D, *hidden, L], (b,) * 3, 1e-4 if key == "production" else 1e-2, False
    rows = SLOT_ROWS[name]
    assert min(rows) >= max(batch_sizes), (name, rows, batch_sizes)
    n_val = 300 if val_first else 0
    nX = max(max(rows), n_val) + 37
    X, Y = _data(units, nX, seed=51)
    rng = np.random.default_rng(52)
    tw = _Twins(units, G_SMALL, batch_sizes[0], X, Y)
    try:
        for s, (j, r) in enumerate(zip(SLOTS, rows)):
            val = rng.choice(nX, n_val, replace=False) if n_val else None
            tw.set_slot(j, _init(units, 53 + s), rng.choice(nX, r, replace=False), alpha * (1, 10, 0.1)[s],
                        (1e-3, 1e-2, 3e-3)[s], val)
        if val_first:
            for j in SLOTS:
                tw.tie_val(j, name)
        for e, bs in enumerate(batch_sizes):
            tw.epoch(rng, models=SLOTS[::-1] if e % 2 else SLOTS, bs=bs, name=f"{name} epoch {e + 1}")
    finally:
        tw.close()


# ------------------------------------------------------------------------------------------------------ b. validation
# name: (layer units, batch size, n_val of each slot; chunks of max(b, 256) rows)
GROUP_VALIDATION = {
    "b200": ([100, 64, 48, 7], 200, (1, 255, 256, 257, 513)),        # one to three chunks of 256
    "b300_nval601": ([100, 64, 48, 7], 300, (601, 300, 2)),          # chunks of 300: 300/300/1
    "b1000_nval2001": ([100, 300, 20], 1000, (2001, 1000, 999)),     # chunks of 1000: 1000/1000/1
}


@pytest.mark.parametrize("name", list(GROUP_VALIDATION))
def test_validation_chunks_equal_single_handles(name):
    """Slots with validation sets of one to three chunks, plus one slot without: epoch, validation of some slots, epoch,
    validation of every slot, epoch -- training and every val_proba equal the twins.  A validation pass writes only its
    own slot's workspace, so the slots not validated still equal twins that never ran one.  The slot without validation
    rows is refused with IE_ERR_STATE, and after a second set_data so is every slot: its rows index the old data."""
    units, bs, n_vals = GROUP_VALIDATION[name]
    nX = max(max(n_vals), 3 * bs) + 101
    X, Y = _data(units, nX, seed=61)
    rng = np.random.default_rng(62)
    slots = [5, 0, 3, 6, 1][:len(n_vals)] + [2]
    G = 7
    tw = _Twins(units, G, bs, X, Y)
    lib = tw.g._lib
    try:
        for s, j in enumerate(slots):
            nv = n_vals[s] if s < len(n_vals) else 0
            tw.set_slot(j, _init(units, 63 + s), rng.choice(nX, bs + 17 * s + (bs // 3) * (s % 2), replace=False),
                        1e-2 * (s + 1), 1e-3 * (s + 1), rng.choice(nX, nv, replace=False) if nv else None)
        with_val = slots[:len(n_vals)]
        probs = np.empty((1, units[-1]), dtype=np.float32)
        assert lib.ie_mlp_group_validation_proba(tw.g._h, slots[-1], probs.ctypes.data) == _lib.IE_ERR_STATE
        assert "no validation rows" in _last_error(lib)
        tw.epoch(rng, name=f"{name} epoch 1")
        for j in with_val[::2]:
            tw.tie_val(j, f"{name} after epoch 1")
        tw.epoch(rng, models=slots[::-1], name=f"{name} epoch 2")
        for j in with_val[::-1]:
            tw.tie_val(j, f"{name} after epoch 2")
        tw.epoch(rng, name=f"{name} epoch 3")
        tw.g.set_data(X, Y)
        for j in slots:
            big = np.empty((max(n_vals), units[-1]), dtype=np.float32)
            assert lib.ie_mlp_group_validation_proba(tw.g._h, j, big.ctypes.data) == _lib.IE_ERR_STATE, j
            assert f"model {j}: no validation rows" in _last_error(lib)
    finally:
        tw.close()


def test_validation_equals_a_checked_forward_at_production_width():
    """At 1600 -> (600, 600) -> 60 with 257 validation rows (two chunks), after each of two epochs val_proba(j) equals
    the twin's, and the p of a debug step over the same rows on a fresh single handle at slot j's parameters, whose
    stages pass check_step: the group's validation is tied to the float64 oracle directly."""
    units, bs, n_val = [1600, 600, 600, 60], 200, 257
    nX = 700
    X, Y = _data(units, nX, seed=71)
    rng = np.random.default_rng(72)
    tw = _Twins(units, 3, bs, X, Y)
    try:
        for s, j in enumerate([2, 0]):
            tw.set_slot(j, _init(units, 73 + s), rng.choice(nX, 457 - 56 * s, replace=False), 1e-4, 1e-3,
                        rng.choice(nX, n_val, replace=False))
        for e in range(2):
            tw.epoch(rng, name=f"production epoch {e + 1}")
            for j, s in tw.slots.items():
                vp = tw.tie_val(j, f"production epoch {e + 1}")
                c, i = tw.g.params(j)
                Xv, Yv = X[s.val_rows], Y[s.val_rows]
                F = DeviceSteps(units)
                F.set_params(c, i)
                F.set_data(Xv, Yv)
                rows = np.arange(n_val, dtype=np.int32)
                out = F.debug_step(rows, s.alpha)
                F.close()
                stats = R.check_step(out, Xv, Yv, rows, c, i, s.alpha, CHECK_DEVICE)
                _tie(f"slot {j} val_proba vs checked debug step", [out["p"]], [vp])
        print({k: round(v, 3) for k, v in stats.items() if k in ("p", "a1")})
    finally:
        tw.close()


# ------------------------------------------------------------------------------------------------ c. snapshot and restore
@pytest.mark.parametrize("units", [[100, 64, 48, 7], [1600, 600, 600, 60]], ids=["small", "production"])
def test_restore_of_one_slot(units):
    """Every slot is snapshotted at its P0 and trains three epochs with validation between them.  ie_mlp_group_snapshot
    (j, restore=1) on one slot sets its parameters to P0 and leaves the other slots and every snapshot as they were.
    The next epoch of every slot equals twins that went through the same snapshot and restore on ie_mlp_train_snapshot:
    its first loss reads the rebuilt sum |W|^2 partials and its first forward the rebuilt split-bf16 weights."""
    bs, nX = 200, 600
    X, Y = _data(units, nX, seed=81)
    rng = np.random.default_rng(82)
    tw = _Twins(units, 4, bs, X, Y)
    slots, r = [3, 0, 2], 2
    try:
        p0 = {}
        for s, j in enumerate(slots):
            p0[j] = _init(units, 83 + s)
            tw.set_slot(j, p0[j], rng.choice(nX, (457, 400, 300)[s], replace=False), 1e-2 * 10 ** -s, 1e-3 * (s + 1),
                        rng.choice(nX, 300, replace=False))
            tw.snapshot(j)
        for e in range(3):
            tw.epoch(rng, name=f"epoch {e + 1}")
            for j in slots:
                tw.tie_val(j, f"epoch {e + 1}")
        before = {j: _flat(tw.g.params(j)) for j in slots}
        assert any(not np.array_equal(a, b) for a, b in zip(before[r], _flat(p0[r])))
        lib = tw.g._lib
        assert lib.ie_mlp_group_snapshot(tw.g._h, r, 1) == 0
        assert tw.slots[r].twin._lib.ie_mlp_train_snapshot(tw.slots[r].twin._h, 1) == 0
        for j in slots:
            _tie(f"slot {j} params after restoring slot {r}", _flat(p0[j]) if j == r else before[j], _flat(tw.g.params(j)))
            _tie(f"slot {j} snapshot after restoring slot {r}", _flat(p0[j]), _flat(tw.g.params(j, best=True)))
        tw.tie_params()
        tw.epoch(rng, name="epoch after restore")
        for j in slots:
            tw.tie_val(j, "after restore")
        tw.tie_params(best=True)
    finally:
        tw.close()


# ------------------------------------------------------------------------------------ d. reused slots, re-uploaded data
def test_reused_slots_and_reuploaded_data():
    """Two slots trained for two epochs are set again with new parameters, alpha and learning rates: they equal fresh
    twins, so set_model restarted their Adam moments, while the slot left alone still equals its running twin.  Then
    the data are uploaded again, larger (the row, learning-rate and loss buffers regrow and their pitch changes) and
    smaller, and after each upload every slot, set again, equals fresh twins, validation included."""
    units, bs = [100, 64, 48, 7], 64
    X, Y = _data(units, 300, seed=91)
    rng = np.random.default_rng(92)
    tw = _Twins(units, G_SMALL, bs, X, Y)
    try:
        for s, j in enumerate(SLOTS):
            tw.set_slot(j, _init(units, 93 + s), rng.choice(300, (300, 200, 129)[s], replace=False), 1e-2, 1e-2)
        tw.epoch(rng, name="first data, epoch 1")
        tw.epoch(rng, name="first data, epoch 2")
        for s, j in enumerate([4, 2]):
            tw.set_slot(j, _init(units, 96 + s), tw.slots[j].train_rows, 1e-3 * (s + 1), 3e-3)
        tw.epoch(rng, name="re-set slots, epoch 1")
        tw.epoch(rng, models=SLOTS[::-1], name="re-set slots, epoch 2")
        for n, seed in ((500, 100), (150, 110)):
            X, Y = _data(units, n, seed=seed)
            tw.X, tw.Y = X, Y
            tw.g.set_data(X, Y)
            for s, j in enumerate(SLOTS):
                tw.set_slot(j, _init(units, seed + s), rng.choice(n, (n, n - 61, bs + 1)[s], replace=False),
                            1e-2 / (s + 1), 1e-2, rng.choice(n, n // 2 + s, replace=False) if s != 1 else None)
            for e in range(2):
                tw.epoch(rng, models=SLOTS[::-1] if e else SLOTS, name=f"n={n}, epoch {e + 1}")
                for j in (4, 2):
                    tw.tie_val(j, f"n={n}, epoch {e + 1}")
    finally:
        tw.close()


# ------------------------------------------------------------------------------------ e. refusals leave nothing behind
def _raw_epoch(g, models, rows, bs):
    lib = g._lib
    ids = np.ascontiguousarray(models, dtype=np.int32)
    n_rows = np.array([len(r) for r in rows], dtype=np.int64)
    flat = np.ascontiguousarray(np.concatenate(rows), dtype=np.int32)
    lr = np.full(int(sum(-(-len(r) // bs) for r in rows)), 1e-3)
    out = np.full(lr.size, -1.0)
    rc = lib.ie_mlp_group_epoch(g._h, len(ids), ids.ctypes.data, n_rows.ctypes.data, flat.ctypes.data, lr.ctypes.data,
                                out.ctypes.data)
    return rc, _last_error(lib), out


def test_refused_epochs_leave_every_slot_untouched():
    """Each invalid ie_mlp_group_epoch call returns its code and message before anything is uploaded or launched: the
    launch count does not move, no slot's parameters change, and the next valid epoch still equals the twins.  A group
    of 0 or of 65536 models is refused at create (the group kernels carry the model in gridDim.y / gridDim.z)."""
    units, bs, n = [100, 64, 48, 7], 64, 300
    X, Y = _data(units, n, seed=121)
    rng = np.random.default_rng(122)
    tw = _Twins(units, G_SMALL, bs, X, Y)
    g, lib = tw.g, tw.g._lib
    try:
        for s, j in enumerate(SLOTS):
            tw.set_slot(j, _init(units, 123 + s), rng.choice(n, (300, 200, 129)[s], replace=False), 1e-2, 1e-2)
        c, i = _init(units, 127)
        for l in range(3):   # slot 1: parameters without constants
            assert lib.ie_mlp_group_set_layer(g._h, 1, l, c[l].ctypes.data, i[l].ctypes.data) == 0
        assert lib.ie_mlp_group_set_layer(g._h, 3, 0, c[0].ctypes.data, i[0].ctypes.data) == 0   # slot 3: one layer
        assert lib.ie_mlp_group_set_hyper(g._h, 3, 1e-2, B1, B2, EPS) == 0
        tw.epoch(rng, name="before the refusals")
        ok = [tw.slots[j].train_rows for j in SLOTS]
        bad_row = ok[2].copy()
        bad_row[-1] = n
        neg_row = ok[1].copy()
        neg_row[5] = -1
        cases = {
            "model listed twice": ([4, 0, 4], [ok[0], ok[1], ok[0]], _lib.IE_ERR_INVALID, "model 4 listed twice"),
            "rows below the batch size": ([4, 0, 2], [ok[0], ok[1][:bs - 1], ok[2]], _lib.IE_ERR_INVALID,
                                          f"model 0: {bs - 1} rows, not in [batch_size {bs}, {n}]"),
            "row past the end": ([4, 0, 2], [ok[0], ok[1], bad_row], _lib.IE_ERR_INVALID,
                                 f"row {len(bad_row) - 1} = {n} outside [0, {n})"),
            "negative row": ([4, 0, 2], [ok[0], neg_row, ok[2]], _lib.IE_ERR_INVALID, "row 5 = -1 outside"),
            "more models than slots": ([4, 0, 2, 1, 3, 4], [ok[0]] * 6, _lib.IE_ERR_INVALID,
                                       f"n_active=6 not in [1, {G_SMALL}]"),
            "model out of range": ([4, 5], [ok[0], ok[0]], _lib.IE_ERR_INVALID, f"model 5 not in [0, {G_SMALL})"),
            "model without constants": ([4, 0, 1], [ok[0], ok[1], ok[0]], _lib.IE_ERR_STATE,
                                        "model 1: constants not set"),
            "model without every layer": ([2, 3], [ok[2], ok[0]], _lib.IE_ERR_STATE, "model 3: parameters not set"),
        }
        params = {j: _flat(g.params(j)) for j in range(G_SMALL)}
        n0 = g.launches
        for what, (models, rows, code, msg) in cases.items():
            rc, err, out = _raw_epoch(g, models, rows, bs)
            assert rc == code and msg in err, (what, rc, err)
            assert g.launches == n0, what
            assert (out == -1.0).all(), what
        for j in range(G_SMALL):
            _tie(f"slot {j} after the refusals", params[j], _flat(g.params(j)))
        tw.epoch(rng, name="after the refusals")
        tw.epoch(rng, models=SLOTS[::-1], name="after the refusals, epoch 2")
    finally:
        tw.close()
    for G in (0, 65536):
        with pytest.raises(ValueError, match=f"n_models={G} not in \\[1, 65535\\]"):
            DeviceGroupSteps(units, G, bs)


# ------------------------------------------------------------------------------- f. full-size groups at production width
# The default grid's groups: 30 candidates (5 alphas x 2 learning-rate modes, which adam ignores, x 3 initial rates) x
# 5 folds per architecture.  n = 2001 rows in five folds: 1600 or 1601 training rows, 8 batches of 200 and a last one
# of 1 where there are 1601; early stopping validates on the fold's 400 or 401 held-out rows (chunks of 256 + 144/145).
FULL = {
    "h400": ((400,), False),
    "h200_200": ((200, 200), False),
    "h400_early_stopping": ((400,), True),
}
FULL_G, FULL_N, FULL_BS = 150, 2001, 200


@pytest.mark.parametrize("name", list(FULL))
def test_full_size_group_equals_single_handles(name):
    """A group of 150 models of 1600 -> hidden -> 60 trains two epochs; then every slot's twin, one at a time, runs the
    same two epochs and equals it bit for bit after each: losses, parameters (after the first epoch by digest) and,
    with early stopping, both validation passes."""
    hidden, early = FULL[name]
    units = [1600, *hidden, 60]
    X, Y = _data(units, FULL_N, seed=131)
    folds = np.array_split(np.arange(FULL_N), 5)
    rng = np.random.default_rng(132)
    jobs = []
    for c in range(FULL_G // 5):
        alpha, lr0 = (1e-3, 1e-2, 1e-1, 1.0, 10.0)[c % 5], (1e-3, 1e-2, 1e-1)[c // 10]
        for f in range(5):
            train = np.concatenate([folds[k] for k in range(5) if k != f])
            jobs.append(dict(params=_init(units, 1000 + len(jobs)), train=train, val=folds[f] if early else None,
                             alpha=alpha, lr0=lr0, perms=[rng.permutation(len(train)) for _ in range(2)]))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.perf_counter()
    g = DeviceGroupSteps(units, FULL_G, FULL_BS)
    try:
        g.set_data(X, Y)
        for j, job in enumerate(jobs):
            g.set_model(j, *job["params"], job["alpha"], B1, B2, EPS, job["val"])
        mem = free0 - torch.cuda.mem_get_info()[0]
        models = list(rng.permutation(FULL_G))   # the model list out of slot order
        rec = {j: {"losses": [], "lrs": [], "val": []} for j in range(FULL_G)}
        for e in range(2):
            lrs = []
            for j in models:
                steps = -(-len(jobs[j]["train"]) // FULL_BS)
                lrs.append(np.array([_lr(jobs[j]["lr0"], e * steps + k + 1) for k in range(steps)]))
            losses = g.epoch(models, [jobs[j]["train"][jobs[j]["perms"][e]] for j in models], lrs)
            for j, loss, lr in zip(models, losses, lrs):
                rec[j]["losses"].append(loss)
                rec[j]["lrs"].append(lr)
                if e == 0:
                    rec[j]["digest"] = _digest(_flat(g.params(j)))
                if early:
                    rec[j]["val"].append(g.val_proba(j))
        t_group = time.perf_counter() - t0
        for j, job in enumerate(jobs):
            tw = DeviceSteps(units)
            try:
                tw.set_params(*job["params"])
                tw.set_data(X[job["train"]], Y[job["train"]], None if job["val"] is None else X[job["val"]])
                for e in range(2):
                    want = tw.epoch(job["perms"][e], FULL_BS, rec[j]["lrs"][e], job["alpha"], B1, B2, EPS)
                    _tie_losses(f"{name} slot {j} epoch {e + 1}", want, rec[j]["losses"][e])
                    if e == 0:
                        assert _digest(_flat(tw.params())) == rec[j]["digest"], (name, "slot", j, "params after epoch 1")
                    else:
                        _tie(f"{name} slot {j} params after epoch 2", _flat(tw.params()), _flat(g.params(j)))
                    if early:
                        _tie(f"{name} slot {j} val_proba after epoch {e + 1}", [tw.val_proba()], [rec[j]["val"][e]])
            finally:
                tw.close()
    finally:
        g.close()
    print(f"{name}: G = {FULL_G}, group of {mem / 2 ** 30:.2f} GiB (free-memory drop), group {t_group:.1f} s, "
          f"all {time.perf_counter() - t0:.1f} s")
