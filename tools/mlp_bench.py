"""BASELINE.json configs[4]: Label_Microservice head, 2400/1600-d -> (600,600) -> labels on one H100: rows/s, labels/s,
max-abs probability difference and label-set agreement vs sklearn predict_proba (what MLPWrapper.predict_probabilities calls,
py/label_microservice/mlp.py:63).  Prints one JSON line per input width."""
import json, os, sys, time, warnings
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from sklearn.neural_network import MLPClassifier
from code_intelligence_b200.mlp import MLPHead, filter_predictions

rng = np.random.default_rng(1234)
for d_in in (1600, 2400):
    n_labels = 256
    Xtr = (rng.standard_normal((2048, d_in)) * 0.1).astype(np.float32)
    Ytr = (rng.random((2048, n_labels)) < 0.05).astype(int)
    clf = MLPClassifier(hidden_layer_sizes=(600, 600), random_state=1234, max_iter=5)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        clf.fit(Xtr, Ytr)
    head = MLPHead.from_sklearn(clf)
    n = 1 << 18
    X = (rng.standard_normal((n, d_in)) * 0.1).astype(np.float32)
    head.predict_proba(X[:4096])
    t0 = time.perf_counter(); probs = head.predict_proba(X); dt = time.perf_counter() - t0
    ns = 8192
    t0 = time.perf_counter(); ref = clf.predict_proba(X[:ns]); dt_cpu = time.perf_counter() - t0
    err = np.abs(probs[:ns] - ref)
    names = [f"l{i}" for i in range(n_labels)]
    thr = {nm: 0.5 for nm in names}
    same = sum(set(filter_predictions(names, probs[r], thr)) == set(filter_predictions(names, ref[r], thr)) for r in range(ns))
    flips = int(((probs[:ns] >= 0.5) != (ref >= 0.5)).sum())
    print(json.dumps(dict(d_in=d_in, hidden=[600, 600], n_labels=n_labels, rows=n, rows_per_s=n / dt, labels_per_s=n * n_labels / dt,
                          e2e_host_buffers=True, sklearn_rows_per_s=ns / dt_cpu, max_abs_prob_diff=float(err.max()),
                          label_set_agreement=same / ns, label_flips=flips, labels_checked=ns * n_labels)), flush=True)
