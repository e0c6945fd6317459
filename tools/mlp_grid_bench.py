"""Grid-search time: DeviceGridSearchCV (every fit of the search trained in lockstep groups on the device) against the
serial GridSearchCV(DeviceMLPClassifier, n_jobs=1) and sklearn's host MLPClassifier search, on the reference's default
grid (6 hidden sizes x 5 alphas x 2 learning-rate modes x 3 initial rates = 180 candidates, cv = 5).

Data: tools/mlp_train_bench.py's seeded synthetic multilabel set (D = 1600, L = 60) with n rows.  Per n, one JSON line:
  batched   wall time of the whole search, split into device training (the group runner) and the rest (sklearn's host
            scoring and bookkeeping, the refit); per lockstep epoch call its group size G, steps, device ms (CUDA
            events) and launches, summarised as device ms per step against G and launches per step
  serial    GridSearchCV(DeviceMLPClassifier, n_jobs=1) on the first --serial-candidates candidates, and that time
            extrapolated to the whole grid (labelled "extrapolated")
  host      sklearn GridSearchCV(MLPClassifier, n_jobs=-1) on the first --host-candidates candidates, extrapolated
  sweep     (--g-sweep G1,G2,...) device ms per lockstep step and launches per step of one epoch call against the
            group size G, at 1600 -> 400 -> 60 and 1600 -> 200 -> 200 -> 60, b = 200, each model on its own 80 % fold of
            the n rows, next to one ie_mlp_train handle's epoch on the same rows (--no-search skips the searches)
The card name and power limit are read in the same run.  --max-iter caps every fit's epochs (the grid's own estimator
keeps sklearn's default of 200); the cap is part of the result.

    python tools/mlp_grid_bench.py [--sizes 5000,50000] [--max-iter 200] [--serial-candidates 6] [--host-candidates 0]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

GRID = {"hidden_layer_sizes": [(100,), (200,), (400,), (50, 50), (100, 100), (200, 200)],
        "alpha": [.001, .01, .1, 1, 10],
        "learning_rate": ["constant", "adaptive"],
        "learning_rate_init": [.001, .01, .1]}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def subset(k):
    from sklearn.model_selection import ParameterGrid
    return [{key: [v] for key, v in p.items()} for p in list(ParameterGrid(GRID))[:k]]


def sweep(X, Y, Gs, bs=200):
    """Device ms and launches per lockstep step against G, and a single handle's on the same rows."""
    from code_intelligence_b200.mlp_train import DeviceGroupSteps, DeviceSteps
    rng = np.random.default_rng(0)
    n = X.shape[0]
    out = []
    for hidden in ((400,), (200, 200)):
        units = [X.shape[1], *hidden, Y.shape[1]]
        coefs = [(rng.standard_normal((units[l], units[l + 1])) * np.sqrt(2 / units[l])).astype(np.float32)
                 for l in range(len(units) - 1)]
        ints = [np.zeros(units[l + 1], np.float32) for l in range(len(units) - 1)]
        rows = rng.permutation(n)[: int(0.8 * n)]
        steps = -(-len(rows) // bs)
        lrs = np.full(steps, 1e-4)
        single = DeviceSteps(units)
        single.set_params(coefs, ints)
        single.set_data(X[rows], Y[rows])
        order = np.arange(len(rows))
        single.epoch(order, bs, lrs, 1e-4, 0.9, 0.999, 1e-8)
        n0 = single.launches
        single.epoch(order, bs, lrs, 1e-4, 0.9, 0.999, 1e-8)
        res = dict(hidden=list(hidden), batch=bs, steps=steps,
                   single_ms_per_step=round(single.last_epoch_ms() / steps, 4),
                   single_launches_per_step=(single.launches - n0) / steps, by_G={})
        single.close()
        for G in Gs:
            g = DeviceGroupSteps(units, G, bs)
            g.set_data(X, Y)
            for j in range(G):
                g.set_model(j, coefs, ints, 1e-4, 0.9, 0.999, 1e-8)
            folds = [rows] * G
            g.epoch(list(range(G)), folds, [lrs] * G)
            n0 = g.launches
            g.epoch(list(range(G)), folds, [lrs] * G)
            ms = g.last_epoch_ms() / steps
            res["by_G"][G] = dict(ms_per_step=round(ms, 4), ms_per_model_step=round(ms / G, 5),
                                  launches_per_step=(g.launches - n0) / steps)
            g.close()
        out.append(res)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="5000,50000")
    ap.add_argument("--max-iter", type=int, default=200)
    ap.add_argument("--serial-candidates", type=int, default=6)
    ap.add_argument("--host-candidates", type=int, default=0)
    ap.add_argument("--g-sweep", default="")
    ap.add_argument("--no-search", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from mlp_train_bench import teacher
    from sklearn.model_selection import GridSearchCV
    from sklearn.neural_network import MLPClassifier

    from code_intelligence_b200 import mlp_train as MT
    gpu = card()
    rows = []
    for n in [int(s) for s in a.sizes.split(",")]:
        X, Y = teacher(n)
        if a.g_sweep:
            for res in sweep(X, Y, [int(g) for g in a.g_sweep.split(",")]):
                res.update(n=n, gpu=gpu)
                print(json.dumps(res), flush=True)
                rows.append(res)
        if a.no_search:
            continue
        base = dict(random_state=0, max_iter=a.max_iter)
        stats = []
        orig = MT._train_groups
        dev = [0.0]

        def timed(*args, **kw):
            t0 = time.perf_counter()
            try:
                return orig(*args, stats=stats, **kw)
            finally:
                dev[0] += time.perf_counter() - t0

        MT._train_groups = timed
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                t0 = time.perf_counter()
                search = MT.DeviceGridSearchCV(MT.DeviceMLPClassifier(**base), GRID, cv=5).fit(X, Y)
                wall = time.perf_counter() - t0
        finally:
            MT._train_groups = orig
        per_g = {}
        launches = []
        prev = None
        for G, steps, ms, count in stats:
            per_g.setdefault(G, []).append(ms / steps)
            if prev is not None and prev[0] == G:
                launches.append((count - prev[1]) / steps)
            prev = (G, count)
        res = dict(n=n, gpu=gpu, max_iter=a.max_iter, candidates=180, folds=5, batched_wall_s=round(wall, 2),
                   batched_device_training_s=round(dev[0], 2), batched_host_rest_s=round(wall - dev[0], 2),
                   epoch_calls=len(stats),
                   device_ms_per_step_by_G={int(G): round(float(np.median(v)), 4) for G, v in sorted(per_g.items())},
                   launches_per_step_median=float(np.median(launches)) if launches else None,
                   best_params=search.best_params_, best_score=float(search.best_score_))
        if a.serial_candidates:
            k = a.serial_candidates
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                t0 = time.perf_counter()
                GridSearchCV(MT.DeviceMLPClassifier(**base), subset(k), cv=5, n_jobs=1).fit(X, Y)
                s = time.perf_counter() - t0
            res.update(serial_candidates=k, serial_s=round(s, 2), serial_full_grid_s_extrapolated=round(s * 180 / k, 1))
        if a.host_candidates:
            k = a.host_candidates
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                t0 = time.perf_counter()
                GridSearchCV(MLPClassifier(**base), subset(k), cv=5, n_jobs=-1).fit(X.astype(np.float64), Y)
                s = time.perf_counter() - t0
            res.update(host_candidates=k, host_cores=os.cpu_count(), host_s=round(s, 2),
                       host_full_grid_s_extrapolated=round(s * 180 / k, 1))
        print(json.dumps(res), flush=True)
        rows.append(res)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
