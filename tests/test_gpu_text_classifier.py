"""The text classifier on the GPU (csrc/clas.cu behind ie_clas_*, code_intelligence_b200/text_classifier.py):

* the pool on the device's own last-layer states: last and max bit for bit, the mean within its float64 bound, at every
  window edge of fastai's chunk rule, with pads in front, inside the window, on its last step, and pad ids 0 and V-1;
* the head element by element against its float64 restatement: BatchNorm with non-trivial statistics, one to three
  stages, 1 to 60 classes, sigmoid and softmax;
* end to end against the torch restatement of fastai's model (06_FineTune's shape, a small one, long issues);
* per-item results independent of the batch, the padded-batch mode's pad-first semantics, and the interface."""

import numpy as np
import pytest
import torch

from code_intelligence_b200 import IssueEncoder
from code_intelligence_b200.text_classifier import TextClassifier
from oracle import awd_lstm_ref as R
from oracle import text_clas_ref as TR

pytestmark = pytest.mark.gpu

SMALL = dict(vocab_sz=500, emb_sz=96, n_hid=200, n_layers=3)


def _encoder(ref: TR.ClassifierRef, pad_idx=1) -> IssueEncoder:
    e = ref.enc
    emb, layers = e.export_weights()
    return IssueEncoder(e.n_layers, e.emb_sz, e.n_hid, e.vocab_sz, pad_idx, 0).load_weights(emb, layers)


def _ids(B, T, vocab, seed, pad=1):
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, vocab, size=(B, T)).astype(np.int64)
    ids[ids == pad] = (pad + 1) % vocab
    return ids


@pytest.fixture(scope="module")
def small():
    ref = TR.make_classifier(seed=11, n_class=3, scale=2.0, **SMALL)
    enc = _encoder(ref)
    clf = TextClassifier(enc, ref.stages())
    yield ref, enc, clf
    clf.close()
    enc.close()


def _check_pool(clf, enc, ids, starts, ends, pad):
    got = clf._call(ids, starts, ends, pooled=True)
    raw = enc.raw_features(ids)
    last, mx, avg, bound = TR.pool_f64(raw, ids, starts, ends, pad)
    E = enc.emb_sz
    np.testing.assert_array_equal(got[:, :E], last)
    np.testing.assert_array_equal(got[:, E:2 * E], mx)
    err = np.abs(got[:, 2 * E:] - avg)
    assert (err <= bound).all(), (err / np.maximum(bound, 1e-300)).max()
    return got


# ------------------------------------------------------------------------------------------------------------- pool
@pytest.mark.parametrize("T", [1, 69, 70, 1399, 1400, 1401, 1469, 1470, 2800, 2801])
def test_pool_at_every_window_edge(small, T):
    _, enc, clf = small
    ids = _ids(3, T, SMALL["vocab_sz"], seed=T)
    if T > 8:
        ids[0, :5] = 1                                  # front padding
        ids[1, T // 2] = 1                              # a pad inside the window
        ids[2, -1] = 1                                  # the window's last step is a pad: last is still o[:, -1]
    s = TR.window_start(T)
    got = _check_pool(clf, enc, ids, np.full(3, s, np.int32), np.full(3, T, np.int32), 1)
    np.testing.assert_array_equal(got, clf.pooled_features(ids=ids))


def test_pool_per_row_windows_and_masks(small):
    _, enc, clf = small
    T = 300
    ids = _ids(6, T, SMALL["vocab_sz"], seed=5)
    ids[:, 250:] = 1                                    # right padding beyond each row's end
    ids[1, 10:40] = 1
    ids[3, 100] = 1
    starts = np.array([0, 5, 70, 0, 140, 299], np.int32)
    ends = np.array([250, 250, 210, 101, 250, 300], np.int32)
    ids[5, 299] = 7
    _check_pool(clf, enc, ids, starts, ends, 1)


@pytest.mark.parametrize("pad", [0, SMALL["vocab_sz"] - 1])
def test_pool_with_other_pad_ids(pad):
    ref = TR.make_classifier(seed=12, n_class=2, **SMALL)
    enc = _encoder(ref, pad_idx=pad)
    clf = TextClassifier(enc, ref.stages())
    try:
        T = 160
        ids = _ids(4, T, SMALL["vocab_sz"], seed=pad + 3, pad=pad)
        ids[0, :30] = pad
        ids[1, 90:120] = pad
        ids[2, -1] = pad
        s = TR.window_start(T)
        _check_pool(clf, enc, ids, np.full(4, s, np.int32), np.full(4, T, np.int32), pad)
        with pytest.raises(ValueError, match="entirely pad"):
            clf._call(np.full((1, 10), pad, np.int64), np.zeros(1, np.int32), np.full(1, 10, np.int32), True)
    finally:
        clf.close()
        enc.close()


# ------------------------------------------------------------------------------------------------------------- head
HEADS = [([], 1, "sigmoid"), ([50], 3, "sigmoid"), ([100, 50], 60, "sigmoid"), ([], 3, "softmax"),
         ([50], 60, "softmax"), ([100, 50], 1, "softmax"), ([50], 1, "sigmoid"), ([100, 50], 3, "softmax")]


@pytest.mark.parametrize("lin_ftrs,n_class,act", HEADS)
def test_head_per_element_within_its_bound(small, lin_ftrs, n_class, act):
    _, enc, _ = small
    calib = _ids(24, 90, SMALL["vocab_sz"], seed=1)
    ref = TR.make_classifier(seed=11, n_class=n_class, lin_ftrs=lin_ftrs, calib_ids=calib, scale=2.0, **SMALL)
    clf = TextClassifier(enc, ref.stages(), activation=act)           # a second handle on the shared encoder
    try:
        ids = _ids(40, 120, SMALL["vocab_sz"], seed=n_class)
        ids[:5, :20] = 1
        pooled = clf.pooled_features(ids=ids)
        logits, p = clf.forward_padded(ids)
        z64, ez, p64, ep = TR.head_f64(pooled, ref.stages(), act)
        assert (np.abs(logits - z64) <= ez).all(), (np.abs(logits - z64) / ez).max()
        assert (np.abs(p - p64) <= ep).all(), (np.abs(p - p64) / ep).max()
        assert np.std(z64) > 0.05                                    # the BatchNorm statistics matter
        if act == "softmax":
            np.testing.assert_allclose(p.sum(1), 1, atol=1e-5)
    finally:
        clf.close()


# ------------------------------------------------------------------------------------------------------- end to end
def _parity(clf, ref, docs, act, cos_tol=1e-4):
    got_pool = clf.pooled_features(docs)
    want_pool = np.vstack([ref.pooled(np.asarray(d)[None, :]).numpy() for d in docs])
    m = R.parity_metrics(got_pool, want_pool)
    assert m["min_cosine"] >= 1 - cos_tol and m["rel_l2"] <= 1e-2, m
    got = clf.predict_proba(docs)
    want = np.vstack([ref.predict_one(d, act) for d in docs])
    assert np.abs(got - want).max() <= 2e-2, np.abs(got - want).max()
    z = clf.predict_logits(docs)
    zw = np.vstack([ref(np.asarray(d)[None, :]).numpy() for d in docs])
    assert np.linalg.norm(z - zw) <= 5e-2 * np.linalg.norm(zw), (z, zw)
    return m


def test_end_to_end_at_the_notebook_shape():
    """06_FineTune: emb_sz 800, n_hid 2400, 4 layers, lin_ftrs [50], a multi-label head, sigmoid."""
    calib = np.vstack(R.synthetic_ids(8, 48, seed=3))
    ref = TR.make_classifier(seed=21, vocab_sz=60000, emb_sz=800, n_hid=2400, n_layers=4, n_class=12, calib_ids=calib,
                             scale=2.0)
    clf = TextClassifier.from_state_dict({"model": ref.fastai_state_dict(), "opt": {}})
    try:
        docs = R.synthetic_ids(3, 160, seed=4, min_len=20)
        print("notebook shape:", _parity(clf, ref, docs, "sigmoid"))
    finally:
        clf.close()


@pytest.mark.parametrize("act", ["sigmoid", "softmax"])
def test_end_to_end_small(act):
    calib = _ids(32, 60, SMALL["vocab_sz"], seed=9)
    ref = TR.make_classifier(seed=31, n_class=5, lin_ftrs=[40], ps=[0.0], calib_ids=calib, **SMALL)
    clf = TextClassifier.from_state_dict(ref.fastai_state_dict(), activation=act)
    try:
        docs = R.synthetic_ids(12, 200, seed=5, vocab_sz=SMALL["vocab_sz"], min_len=1)
        _parity(clf, ref, docs, act)
    finally:
        clf.close()


def test_end_to_end_long_issues_across_the_window_and_the_time_chunk():
    """1469 and 1470 steps (the window moves by a chunk), and 4400 steps: past the encoder's 4096-step time chunk of a
    one-batch call, with only the last 1400-odd steps pooled."""
    calib = _ids(16, 60, SMALL["vocab_sz"], seed=19)
    ref = TR.make_classifier(seed=41, n_class=4, calib_ids=calib, **SMALL)
    clf = TextClassifier.from_state_dict(ref.fastai_state_dict())
    try:
        docs = [a for a in R.synthetic_ids(1, 4400, seed=6, vocab_sz=SMALL["vocab_sz"])]
        docs += [docs[0][:1469], docs[0][:1470], docs[0][:1401]]
        _parity(clf, ref, docs, "sigmoid")
    finally:
        clf.close()


# -------------------------------------------------------------------------------------------------------- invariants
def test_per_item_results_do_not_depend_on_the_batch(small):
    _, _, clf = small
    docs = R.synthetic_ids(50, 300, seed=7, vocab_sz=SMALL["vocab_sz"], min_len=1)
    full = clf.predict_proba(docs)
    for i in (0, 7, 23, 49):
        np.testing.assert_array_equal(clf.predict_proba([docs[i]])[0], full[i])
    perm = np.random.default_rng(0).permutation(50)
    np.testing.assert_array_equal(clf.predict_proba([docs[i] for i in perm]), full[perm])
    np.testing.assert_array_equal(clf.predict_proba(docs[10:17] + docs[:3]), np.vstack([full[10:17], full[:3]]))


def test_padded_batch_is_fastais_pad_first_forward(small):
    ref, _, clf = small
    docs = R.synthetic_ids(6, 150, seed=8, vocab_sz=SMALL["vocab_sz"], min_len=40)
    T = max(len(d) for d in docs)
    ids = np.full((6, T), 1, np.int64)
    for b, d in enumerate(docs):
        ids[b, T - len(d):] = d                         # pad_collate(pad_first=True)
    logits, p = clf.forward_padded(ids)
    want = ref(ids).numpy()
    assert np.abs(logits - want).max() <= 5e-2 * max(1.0, np.abs(want).max()), np.abs(logits - want).max()
    np.testing.assert_allclose(p, torch.sigmoid(torch.as_tensor(want)).numpy(), atol=2e-2)
    per_item = clf.predict_proba(docs)
    full = [b for b, d in enumerate(docs) if len(d) == T]
    padded = [b for b, d in enumerate(docs) if len(d) < T - 10]
    assert full and padded
    for b in full:                                      # no pads: the same rows bit for bit
        np.testing.assert_array_equal(p[b], per_item[b])
    # front pads run through the LSTM and are masked out of max / mean only: the padded rows differ from per-item
    assert min(np.abs(p[b] - per_item[b]).max() for b in padded) > 1e-5
    want_item = np.vstack([ref.predict_one(docs[b]) for b in padded])
    want_pad = torch.sigmoid(torch.as_tensor(want[padded])).numpy()
    assert np.abs(want_item - want_pad).max() > 1e-4    # fastai differs in the same way


# --------------------------------------------------------------------------------------------------------- interface
def test_predict_text_returns_the_thresholded_labels(small):
    ref, enc, _ = small
    itos = ["xxunk", "xxpad", "xxbos", "xxfld", "xxmaj", "xxup", "xxrep", "xxwrep"] + [f"w{i}" for i in range(492)]
    classes = ["bug", "feature", "question"]
    clf = TextClassifier(enc, ref.stages(), classes=classes, itos=itos)
    soft = TextClassifier(enc, ref.stages(), activation="softmax", classes=classes, itos=itos)
    try:
        text = "w5 w17 w300 the w42 crashes w7 w7 w99"
        labels, y, probs = clf.predict(text)
        np.testing.assert_array_equal(probs, clf.predict_proba([clf.numericalize(text)])[0])
        np.testing.assert_array_equal(y, (probs >= 0.5).astype(np.float32))
        assert labels == [c for c, v in zip(classes, probs) if v >= 0.5]
        want = ref.predict_one(clf.numericalize(text))
        assert np.abs(probs - want).max() <= 2e-2
        lab, k, ps = soft.predict(text)
        assert k == int(np.argmax(ps)) and lab == classes[k] and abs(float(ps.sum()) - 1) < 1e-5
    finally:
        soft.close()
        clf.close()


def test_device_pointers_on_a_side_stream(small):
    _, _, clf = small
    ids = _ids(9, 130, SMALL["vocab_sz"], seed=13)
    ids[:3, :12] = 1
    logits, p = clf.forward_padded(ids)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_ids = torch.as_tensor(ids).cuda()
        st = torch.full((9,), TR.window_start(130), dtype=torch.int32, device="cuda")
        en = torch.full((9,), 130, dtype=torch.int32, device="cuda")
        z_d, p_d = clf.forward_padded_device(d_ids, st, en, stream=s)
    s.synchronize()
    clf.check_errors()
    np.testing.assert_array_equal(z_d.cpu().numpy(), logits)
    np.testing.assert_array_equal(p_d.cpu().numpy(), p)


def test_two_handles_on_one_encoder_and_row_groups(small, monkeypatch):
    ref, enc, clf = small
    docs = R.synthetic_ids(20, 100, seed=14, vocab_sz=SMALL["vocab_sz"], min_len=10)
    want = clf.predict_proba(docs)
    # a raw-state budget of one row: every row its own group, the same bits
    monkeypatch.setenv("IE_CLAS_RAW_BUDGET", "1")
    one = TextClassifier(enc, ref.stages())
    monkeypatch.delenv("IE_CLAS_RAW_BUDGET")
    other = TextClassifier(enc, TR.make_classifier(seed=99, n_class=7, **SMALL).stages(), activation="softmax")
    try:
        n0 = one.launch_count
        np.testing.assert_array_equal(one.predict_proba(docs), want)
        assert one.launch_count - n0 == 20 * 4          # pool, two head stages, activation per row
        o1 = other.predict_proba(docs)
        np.testing.assert_array_equal(clf.predict_proba(docs), want)
        np.testing.assert_array_equal(other.predict_proba(docs), o1)
    finally:
        other.close()
        one.close()


def test_errors_leave_the_encoder_usable(small):
    _, enc, clf = small
    ids = _ids(4, 50, SMALL["vocab_sz"], seed=15)
    want = clf.forward_padded(ids)[1]
    enc_want = enc.encode_ids(ids)
    bad = ids.copy()
    bad[2, 7] = SMALL["vocab_sz"] + 3
    with pytest.raises(ValueError, match="token id"):
        clf.forward_padded(bad)
    allpad = ids.copy()
    allpad[2, 40] = 1
    with pytest.raises(ValueError, match="entirely pad"):
        clf._call(allpad, np.array([0, 0, 40, 0], np.int32), np.array([50, 50, 41, 50], np.int32), False)
    with pytest.raises(ValueError, match="outside"):
        clf._call(ids, np.zeros(4, np.int32), np.full(4, 51, np.int32), False)
    # device pointers: the window is checked on the device, the row comes back NaN, check_errors reports it
    d_ids = torch.as_tensor(ids).cuda()
    st = torch.tensor([0, 30, 0, 0], dtype=torch.int32, device="cuda")
    en = torch.tensor([50, 20, 50, 50], dtype=torch.int32, device="cuda")
    z, p = clf.forward_padded_device(d_ids, st, en)
    with pytest.raises(ValueError, match="window"):
        clf.check_errors()
    p = p.cpu().numpy()
    assert np.isnan(p[1]).all() and np.isfinite(np.delete(p, 1, 0)).all()
    clf.check_errors()                                   # cleared
    np.testing.assert_array_equal(clf.forward_padded(ids)[1], want)
    np.testing.assert_array_equal(enc.encode_ids(ids), enc_want)
    with pytest.raises(ValueError, match="inputs"):
        TextClassifier(enc, [dict(bn_weight=np.ones(10), bn_bias=np.zeros(10), bn_mean=np.zeros(10),
                                  bn_var=np.ones(10), weight=np.ones((2, 10)), bias=np.zeros(2))])
