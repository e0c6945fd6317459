"""Development aid: a tiny run of every kernel (persistent recurrent kernel, per-timestep fallback, both GEMMs, gather /
table / finalize, MLP head, the label-MLP trainer and its group form) for compute-sanitizer (memcheck / racecheck /
synccheck), checked against the oracle or, for the group trainer, against the single-model fits.

    IE_SPIN_LIMIT_MS=600000 compute-sanitizer --tool memcheck python tools/sanitize_tiny.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from code_intelligence_b200 import IssueEncoder
from code_intelligence_b200.mlp import MLPHead
from oracle import awd_lstm_ref as R
from oracle import lstm_numpy as N

cfg = (2, 64, 128, 300)
ref = R.make_encoder(5, cfg[3], cfg[1], cfg[2], cfg[0], scale=2.0)
weights = ref.export_weights()
docs = R.synthetic_ids(300, 5, seed=1, vocab_sz=cfg[3], min_len=1)
T = 5
ids = np.full((len(docs), T), 1, dtype=np.int64)
for i, d in enumerate(docs):
    ids[i, :len(d)] = d
lengths = np.array([len(d) for d in docs], dtype=np.int32)
want = R.encode_padded(ref, ids, lengths)
for name, env in (("persistent (last layer fused)", {}), ("persistent, hoisted last layer", {"IE_FUSE_LAST": "0"}), ("fallback+gather", {"IE_SEQ": "0", "IE_EMB_PROJ": "0"}), ("chunked", {"IE_CHUNK_T": "2"})):
    os.environ.update(env)
    enc = IssueEncoder(*cfg, 1, 0).load_weights(*weights)
    for k in env:
        os.environ.pop(k)
    got = enc.encode_ids(ids, lengths)
    m = R.parity_metrics(got, want)
    print(name, "rel_l2 %.2e" % m["rel_l2"], "launches", enc.launch_count, flush=True)
    assert m["rel_l2"] < 1e-2
    enc.close()
rng = np.random.default_rng(0)
coefs = [rng.standard_normal((24, 32)).astype(np.float32) * 0.2, rng.standard_normal((32, 5)).astype(np.float32) * 0.2]
ints = [rng.standard_normal(32).astype(np.float32) * 0.1, rng.standard_normal(5).astype(np.float32) * 0.1]
X = rng.standard_normal((300, 24)).astype(np.float32)
head = MLPHead(coefs, ints)
assert np.abs(head.predict_proba(X) - N.mlp_forward(X, coefs, ints)).max() < 5e-3
head.close()
import warnings

from code_intelligence_b200 import mlp_train as MT
# group trainer: 2 shapes x 3 models over stacked slots, short last batches of two sizes, early stopping, each fit
# equal to its own single-handle fit
Xg = rng.standard_normal((150, 40)).astype(np.float32)
Yg = (Xg[:, :3] > 0).astype(int)
folds = [np.arange(0, 100), np.arange(50, 150), np.arange(0, 101)]
jobs = [(MT.DeviceMLPClassifier(hidden_layer_sizes=h, max_iter=3, random_state=s, batch_size=32,
                                early_stopping=s == 1), f) for h in ((24,), (20, 12)) for s, f in enumerate(folds)]
with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    trained = MT._train_groups(jobs, Xg, Yg)
    for (est, rows), rec in zip(jobs, trained):
        want = MT.DeviceMLPClassifier(**est.get_params()).fit(Xg[rows], Yg[rows])
        assert rec.error is None and rec.est.loss_curve_ == want.loss_curve_
        assert all(np.array_equal(a, b) for a, b in zip(rec.est.coefs_ + rec.est.intercepts_,
                                                          want.coefs_ + want.intercepts_))
print("group trainer: 6 fits equal to their single fits", flush=True)
print("sanitize_tiny ok")
