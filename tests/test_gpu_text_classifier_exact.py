"""The text classifier's kernels bit for bit against the exact float32 restatement of oracle/text_clas_ref.py, at the
shapes that run: 06_FineTune's encoder (4 x 2400, emb 800, vocab 60000) in the default and the fp32-accurate mode.

* the pool on the device's own last-layer states, 1 to 1280 rows (one to five encoder launch batches, 1-row tails) by
  1 to 1470 steps, per-row windows with pads in front, inside the window and on its last step;
* the head's logits on the classifier's own pool: 2400 -> hidden -> n_class (the benchmark's 2400 -> 50 -> 28 among
  them), hidden widths around the Linear kernel's 128-wide k chunk, three stages, 1 to 1280 rows around its 8-row CTAs;
* the BatchNorm fold through an identity Linear;
* sigmoid and softmax on exactly known logits, against relative bounds;
* the default row-group split of a 1280 x 1400 call (921 + 359 rows), against four groups and a device-pointer call;
* the fp32-accurate mode end to end against torch, strictly closer than the default mode.

Bits are compared through uint32 views, so -0 against +0 is a difference.  Rows of a call are independent (pinned in
test_gpu_text_classifier.py), so the states of a call's rows are fetched for row subsets."""
import functools

import numpy as np
import pytest
import torch

from code_intelligence_b200 import IssueEncoder, _lib
from code_intelligence_b200.text_classifier import TextClassifier, head_stages
from oracle import awd_lstm_ref as R
from oracle import text_clas_ref as TR

pytestmark = pytest.mark.gpu

BIG = dict(vocab_sz=60000, emb_sz=800, n_hid=2400, n_layers=4)
SMALL = dict(vocab_sz=500, emb_sz=96, n_hid=200, n_layers=3)
MODES = {"bf16": 0, "fp32": _lib.IE_CFG_FP32}
PAD = 1


def _bits(x) -> np.ndarray:
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def _assert_bits_equal(got, want, what):
    g, w = _bits(got), _bits(want)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = np.argwhere(g != w)
    assert bad.size == 0, (what, f"{len(bad)} of {g.size} differ; first", bad[:5].tolist(),
                           g.view(np.float32)[tuple(bad[0])], w.view(np.float32)[tuple(bad[0])])


@functools.lru_cache(maxsize=1)
def _big_state_dict():
    """06's classifier with random weights and BatchNorm statistics: the 2400 -> 50 -> 28 head of tools/clas_bench.py."""
    ref = TR.make_classifier(seed=61, n_class=28, scale=2.0, **BIG)
    sd = ref.fastai_state_dict()
    return sd, head_stages(sd, 3 * BIG["emb_sz"])


@pytest.fixture(scope="module", params=sorted(MODES))
def big(request):
    sd, stages = _big_state_dict()
    clf = TextClassifier.from_state_dict(sd, flags=MODES[request.param])
    yield request.param, clf, stages
    clf.close()


def _rows(B, T, seed, vocab=BIG["vocab_sz"]):
    """ids (B, T) and per-row windows: rows cycle through four forms -- per-item (right-padded after the row's own
    length, window from that length), pad-first (front pads, window from T), a pad inside the window, and a pad on the
    window's last step.  Rows 0 and B - 1 run the full T."""
    rng = np.random.default_rng(seed)
    ids = rng.integers(2, vocab, size=(B, T)).astype(np.int64)
    lengths = rng.integers(1, T + 1, size=B)
    lengths[0] = lengths[-1] = T
    starts, ends = np.empty(B, np.int32), np.empty(B, np.int32)
    for b in range(B):
        n = int(lengths[b])
        ids[b, n:] = PAD
        s, e = TR.window_start(n), n
        kind = b % 4
        if kind == 1 and T > 2:                          # pad-first: the window from T, pads in front of the tokens
            ids[b] = rng.integers(2, vocab, size=T)
            f = int(rng.integers(1, T))
            ids[b, :f] = PAD
            s, e = TR.window_start(T), T
        elif kind == 2 and e - s >= 3:
            ids[b, s + (e - s) // 2] = PAD
        elif kind == 3 and e - s >= 2:
            ids[b, e - 1] = PAD
        starts[b], ends[b] = s, e
    return ids, starts, ends


def _check_pool_rows(clf, ids, starts, ends, got, sel, control=False):
    """got (B, 2400): the device's pool of the call; sel: the rows checked against pool_f32 on their own states."""
    sel = np.asarray(sel)
    raw = torch.as_tensor(clf.encoder.raw_features(ids[sel])).cuda()
    want = TR.pool_f32(raw, ids[sel], starts[sel], ends[sel], PAD)
    _assert_bits_equal(got[sel], want, "pool")
    if control:                                          # a two-accumulator sum is seen
        pw = TR.pool_f32(raw, ids[sel], starts[sel], ends[sel], PAD, pairwise=True)
        E = raw.shape[2]
        assert (_bits(got[sel][:, 2 * E:]) != _bits(pw[:, 2 * E:])).mean() > 0.05


def _check_rows(B):
    """Rows checked of a B-row call: every row up to 40, else the edges of each 256-row launch batch and the last."""
    if B <= 40:
        return list(range(B))
    sel = {0, 1, 2, 3, B - 3, B - 2, B - 1}
    for k in range(256, B, 256):
        sel |= {k - 2, k - 1, k, k + 1}
    return sorted(r for r in sel if r < B)


# ------------------------------------------------------------------------------------------------------------- pool
@pytest.mark.parametrize("T", [1, 70, 512, 1400, 1470])
@pytest.mark.parametrize("B", [1, 255, 256, 257, 1280])
def test_pool_bit_for_bit(big, B, T):
    _, clf, _ = big
    ids, starts, ends = _rows(B, T, seed=B * 7 + T)
    got = clf._call(ids, starts, ends, pooled=True)
    _check_pool_rows(clf, ids, starts, ends, got, _check_rows(B), control=T >= 512)


# ------------------------------------------------------------------------------------------------------------- head
def _calibrated(pooled: np.ndarray, dims, seed):
    """Head stages with BatchNorm statistics those of their inputs over ``pooled`` (float64 forward between stages)."""
    rng = np.random.default_rng(seed)
    a, stages = pooled.astype(np.float64), []
    for k, (K, N) in enumerate(zip(dims[:-1], dims[1:])):
        st = dict(bn_weight=(1 + 0.2 * rng.standard_normal(K)).astype(np.float32),
                  bn_bias=(0.1 * rng.standard_normal(K)).astype(np.float32),
                  bn_mean=a.mean(0).astype(np.float32), bn_var=(a.var(0) + 1e-4).astype(np.float32),
                  weight=(rng.standard_normal((N, K)) * 2 / np.sqrt(K)).astype(np.float32),
                  bias=(0.1 * rng.standard_normal(N)).astype(np.float32))
        stages.append(st)
        a = ((a - st["bn_mean"]) / np.sqrt(st["bn_var"].astype(np.float64) + 1e-5) * st["bn_weight"] + st["bn_bias"]
             ) @ st["weight"].T.astype(np.float64) + st["bias"]
        if k < len(dims) - 2:
            a = np.maximum(a, 0)
    return stages


@pytest.fixture(scope="module")
def head_inputs(big):
    """1280 short issues (per-item windows) and their pool, from the module's classifier."""
    _, clf, _ = big
    ids, starts, ends = _rows(1280, 48, seed=3)
    return ids, starts, ends, clf._call(ids, starts, ends, pooled=True)


HEADS = [([50], n) for n in (1, 12, 28, 31, 32, 33, 60)] + [([h], 28) for h in (127, 128, 129)] + [([100, 50], 28)]


@pytest.mark.parametrize("lin_ftrs,n_class", HEADS)
def test_head_logits_bit_for_bit(big, head_inputs, lin_ftrs, n_class):
    _, clf, _ = big
    ids, starts, ends, pooled = head_inputs
    act = "softmax" if n_class in (12, 31, 33) or len(lin_ftrs) > 1 else "sigmoid"
    stages = _calibrated(pooled[:256], [2400] + lin_ftrs + [n_class], seed=n_class + sum(lin_ftrs))
    want = TR.head_f32(torch.as_tensor(pooled).cuda(), stages)
    assert float(want.std()) > 0.3                                  # the calibrated statistics spread the logits
    head = TextClassifier(clf.encoder, stages, activation=act)
    try:
        for n in (1, 7, 8, 9, 1279, 1280):                          # around the Linear kernel's 8-row CTAs
            p, z = head._call(ids[:n], starts[:n], ends[:n], pooled=False)
            _assert_bits_equal(z, want[:n], f"logits, {n} rows")
            p64, bound = (TR.sigmoid_bound if act == "sigmoid" else TR.softmax_bound)(want[:n])
            err = (torch.as_tensor(p).cuda().double() - p64).abs()
            assert bool((err <= bound).all()), float((err / bound).max())
        rev = TR.head_f32(torch.as_tensor(pooled).cuda(), stages, reverse=True)
        assert (_bits(z) != _bits(rev)).mean() > 0.05                # the order is what the equality pins
    finally:
        head.close()


def test_bn_fold_on_the_device(big, head_inputs):
    """One stage with an identity Linear (N = K = 2400, zero bias): the logits are fma(x, alpha, beta) of the host's
    fold, the only rounding the chain adds being none (x * 1 + 0 products, zeros elsewhere)."""
    _, clf, _ = big
    ids, starts, ends, pooled = head_inputs
    rng = np.random.default_rng(5)
    K = 2400
    st = dict(bn_weight=(rng.standard_normal(K) * 3).astype(np.float32),
              bn_bias=rng.standard_normal(K).astype(np.float32),
              bn_mean=(pooled.mean(0) + 0.01 * rng.standard_normal(K)).astype(np.float32),
              bn_var=(10.0 ** rng.uniform(-6, 3, K)).astype(np.float32),
              weight=np.eye(K, dtype=np.float32), bias=np.zeros(K, np.float32))
    head = TextClassifier(clf.encoder, [st])
    try:
        _, z = head._call(ids, starts, ends, pooled=False)
    finally:
        head.close()
    alpha, beta = TR.bn_fold_f32(st)
    x = torch.as_tensor(pooled, dtype=torch.float64)
    want = TR.fma_f32(x, alpha[None, :], beta[None, :])
    _assert_bits_equal(z, want, "x * alpha + beta")
    unfused = TR._f32(TR._f32(x * alpha[None, :]) + beta[None, :])   # the same fold without the fma is seen
    assert (_bits(z) != _bits(unfused)).mean() > 0.01


# ------------------------------------------------------------------------------------------------------- activation
@pytest.fixture(scope="module")
def small_encoder():
    ref = TR.make_classifier(seed=13, n_class=2, **SMALL)
    e = ref.enc
    emb, layers = e.export_weights()
    enc = IssueEncoder(e.n_layers, e.emb_sz, e.n_hid, e.vocab_sz, PAD, 0).load_weights(emb, layers)
    yield enc
    enc.close()


def _logits_as_bias(enc, bias, act, rows=9):
    """A one-stage head with zero weights: acc stays +0, so each logit is f32(+0 + bias) -- the bias itself, -0 going
    to +0.  Returns (logits, p, exact logits) of ``rows`` identical rows."""
    K, N = 3 * enc.emb_sz, len(bias)
    st = dict(bn_weight=np.ones(K, np.float32), bn_bias=np.zeros(K, np.float32), bn_mean=np.zeros(K, np.float32),
              bn_var=np.ones(K, np.float32), weight=np.zeros((N, K), np.float32), bias=np.asarray(bias, np.float32))
    head = TextClassifier(enc, [st], activation=act)
    try:
        ids = np.random.default_rng(0).integers(2, SMALL["vocab_sz"], size=(rows, 20))
        p, z = head._call(ids, np.zeros(rows, np.int32), np.full(rows, 20, np.int32), pooled=False)
    finally:
        head.close()
    want = np.where(np.asarray(bias, np.float32) == 0, np.float32(0), np.asarray(bias, np.float32))
    _assert_bits_equal(z, np.broadcast_to(want, z.shape), "logits = bias")
    return z, p


def test_sigmoid_on_exact_logits(small_encoder):
    f = np.float32
    special = [0.0, -0.0, 88.72, -88.72, 88.7228, -88.7228, 87.33, -87.33, 103.9, -103.9, 110, -110, 16.6, 17.33,
               17.4, -17.33, 1e-30, -1e-30, 1e-45, -1e-45, 2.0 ** -126, 1.0, -1.0]
    sweep = np.linspace(-110, 110, 65536 - len(special)).astype(f)
    z_in = np.concatenate([np.array(special, f), sweep])
    z, p = _logits_as_bias(small_encoder, z_in, "sigmoid", rows=3)
    p64, bound = TR.sigmoid_bound(torch.as_tensor(z[0]))
    err = (torch.as_tensor(p).double() - p64[None]).abs()
    assert bool((err <= bound[None]).all()), float((err / bound).max())
    assert (p[:, :2] == f(0.5)).all() and (p <= 1).all() and (p >= 0).all()
    assert (p[:, np.flatnonzero(z_in >= 17.4)] == 1).all()             # 1 + expf(-z) rounds to 1 there
    _assert_bits_equal(p, np.broadcast_to(p[0], p.shape), "rows alike")
    tiny = (p64 > 1e-30) & (p64 < 1e-5)
    assert int(tiny.sum()) > 1000 and bool((bound[tiny] < 1e-5 * p64[tiny]).all())   # relative where it matters


@pytest.mark.parametrize("N", [1, 2, 31, 32, 33, 1000, 65536])
def test_softmax_on_exact_logits(small_encoder, N):
    rng = np.random.default_rng(N)
    z_in = rng.uniform(-120, 10, N).astype(np.float32)           # spreads past 104: terms flush to zero
    z_in[rng.integers(N)] = 12.5
    if N > 3:
        z_in[:3] = [0.0, -0.0, 12.5]                              # a tied maximum and signed zeros
    z, p = _logits_as_bias(small_encoder, z_in, "softmax")
    _assert_bits_equal(p, np.broadcast_to(p[0], p.shape), "rows alike")
    if N == 1:
        assert (p == np.float32(1)).all()
        return
    p64, bound = TR.softmax_bound(torch.as_tensor(z))
    err = (torch.as_tensor(p).double() - p64).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    if N >= 1000:
        assert (p == 0).any()                                     # flushed terms are exercised


# ------------------------------------------------------------------------------------------------------- row groups
def test_row_groups_at_the_default_budget(big, monkeypatch):
    """1280 x 1400 at emb 800: states of 1400 * 832 * 4 bytes a row, 921 rows fit 4 GB -- groups of 921 and 359."""
    mode, clf, stages = big
    B, T = 1280, 1400
    ids, starts, ends = _rows(B, T, seed=17)
    n0 = clf.launch_count
    p, z = clf._call(ids, starts, ends, pooled=False)
    assert clf.launch_count - n0 == 2 * (len(stages) + 2)
    monkeypatch.setenv("IE_CLAS_RAW_BUDGET", str(320 * T * 832 * 4))
    four = TextClassifier(clf.encoder, stages)
    monkeypatch.delenv("IE_CLAS_RAW_BUDGET")
    try:
        n0 = four.launch_count
        p4, z4 = four._call(ids, starts, ends, pooled=False)
        assert four.launch_count - n0 == 4 * (len(stages) + 2)
    finally:
        four.close()
    _assert_bits_equal(z4, z, "logits, four groups")
    _assert_bits_equal(p4, p, "p, four groups")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        z_d, p_d = clf.forward_padded_device(torch.as_tensor(ids).cuda(), torch.as_tensor(starts).cuda(),
                                             torch.as_tensor(ends).cuda(), stream=s)
    s.synchronize()
    clf.check_errors()
    _assert_bits_equal(z_d, z, "logits, device pointers")
    _assert_bits_equal(p_d, p, "p, device pointers")
    n0 = clf.launch_count
    pooled = clf._call(ids, starts, ends, pooled=True)
    assert clf.launch_count - n0 == 2
    _check_pool_rows(clf, ids, starts, ends, pooled, list(range(915, 928)) + list(range(1275, 1280)))
    _assert_bits_equal(z, TR.head_f32(torch.as_tensor(pooled).cuda(), stages), "logits of the pool")


# ---------------------------------------------------------------------------------------------------- fp32 vs torch
# Measured on an H100 80GB HBM3 at 700 W (DESIGN.md section 10): largest error over the largest magnitude, fp32 mode
# 6.0e-6 (pool) and 6.2e-5 (logits), default mode 2.5e-3 and 2.8e-2.  The threshold is 8x the larger fp32 figure.
FP32_TOL = 5e-4


def test_fp32_mode_is_closer_to_torch_than_the_default_mode():
    calib = np.vstack(R.synthetic_ids(32, 60, seed=9, vocab_sz=SMALL["vocab_sz"]))
    ref = TR.make_classifier(seed=31, n_class=5, lin_ftrs=[40], calib_ids=calib, **SMALL)
    docs = R.synthetic_ids(24, 300, seed=12, vocab_sz=SMALL["vocab_sz"], min_len=1)
    want_pool = np.vstack([ref.pooled(np.asarray(d)[None, :]).numpy() for d in docs])
    want_z = np.vstack([ref(np.asarray(d)[None, :]).numpy() for d in docs])
    err = {}
    for mode, flags in MODES.items():
        clf = TextClassifier.from_state_dict(ref.fastai_state_dict(), flags=flags)
        try:
            pool, z = clf.pooled_features(docs), clf.predict_logits(docs)
        finally:
            clf.close()
        err[mode] = dict(pool=float(np.abs(pool - want_pool).max() / np.abs(want_pool).max()),
                         z=float(np.abs(z - want_z).max() / np.abs(want_z).max()))
    print("max error relative to the largest magnitude, against torch f32:", err)
    assert err["fp32"]["pool"] < err["bf16"]["pool"] and err["fp32"]["z"] < err["bf16"]["z"], err
    assert err["fp32"]["pool"] <= FP32_TOL and err["fp32"]["z"] <= FP32_TOL, err
