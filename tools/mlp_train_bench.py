"""Label-MLP training time: DeviceMLPClassifier.fit against sklearn's float64 MLPClassifier.fit on the host, at the
RepoMLP configuration (hidden (600, 600), alpha 1e-4, early stopping on 10 %, patience 5, random_state 1234).

Seeded synthetic multilabel data (D = 1600, L = 60: a 16-d latent factor under noise, labels the top 10 % of a
fixed random linear teacher on it) with n training rows
and 2000 held-out rows.  Per n: the device fit's wall time (a host clock around fit, which ends in a synchronise),
epochs, Adam steps per second, the device time of each epoch from CUDA events (ie_mlp_train_last_epoch_ms) and the
kernels launched per step; the host fit's wall time with all cores; the held-out micro-averaged AUC of both.  The card
name and power limit, the CPU model and its core count are read in the same run.  One JSON line per n.

    python tools/mlp_train_bench.py [--sizes 5000,50000] [--no-host] [--out results.json]
"""
import argparse
import json
import os
import platform
import subprocess
import sys
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

REPO_MLP = dict(solver="adam", activation="relu", hidden_layer_sizes=(600, 600), alpha=1e-4, early_stopping=True,
                validation_fraction=0.1, n_iter_no_change=5, max_iter=3000, random_state=1234, learning_rate="adaptive")


def teacher(n, seed=0, D=1600, L=60, k=16):
    """A learnable multilabel set: 1600-d inputs carrying a 16-d latent factor under noise, labels the top 10 % of a
    fixed random linear teacher on the factor."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((k, D))
    W = rng.standard_normal((k, L))
    Z = rng.standard_normal((n, k))
    X = (Z @ A / np.sqrt(k) + 0.5 * rng.standard_normal((n, D))).astype(np.float32)
    logits = Z @ W
    return X, (logits > np.quantile(logits, 0.9, axis=0)).astype(int)


def cpu_model():
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return platform.processor()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="5000,50000")
    ap.add_argument("--no-host", action="store_true", help="skip the sklearn fits")
    ap.add_argument("--out", default=None, help="also write every row to this JSON file")
    args = ap.parse_args()
    import torch
    from sklearn.metrics import roc_auc_score
    from sklearn.neural_network import MLPClassifier
    from code_intelligence_b200.mlp_train import DeviceMLPClassifier, DeviceSteps
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this benchmark measures the device fit and has no CPU fallback")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    machine = {"gpu": q[0] if q else torch.cuda.get_device_name(0), "cpu": cpu_model(), "cpu_cores": os.cpu_count()}
    print(json.dumps(machine), flush=True)

    class Timed(DeviceSteps):
        epochs = []

        def epoch(self, order, batch_size, *a):
            l0 = self.launches
            r = super().epoch(order, batch_size, *a)
            Timed.epochs.append((self.last_epoch_ms(), len(r), self.launches - l0))
            return r

    with warnings.catch_warnings():   # warm-up: module load, the GEMM's first launches
        warnings.simplefilter("ignore")
        Xw, Yw = teacher(600, seed=9)
        DeviceMLPClassifier(**dict(REPO_MLP, max_iter=2))._fit_with(Xw, Yw, Timed)
    rows = []
    for n in [int(s) for s in args.sizes.split(",")]:
        X, Y = teacher(n + 2000, seed=1)
        Xtr, Ytr, Xte, Yte = X[:n], Y[:n], X[n:], Y[n:]
        Timed.epochs = []
        dev = DeviceMLPClassifier(**REPO_MLP)
        t0 = time.perf_counter()
        dev._fit_with(Xtr, Ytr, Timed)
        wall = time.perf_counter() - t0
        ms = [e[0] for e in Timed.epochs]
        steps = sum(e[1] for e in Timed.epochs)
        row = {"n": n, "device_fit_s": round(wall, 3), "epochs": dev.n_iter_, "steps": steps,
               "steps_per_s": round(steps / wall, 1), "epoch_device_ms_median": round(float(np.median(ms)), 3),
               "step_device_ms": round(sum(ms) / steps, 4),
               "launches_per_step": round(sum(e[2] for e in Timed.epochs) / steps, 2),
               "auc_device": round(float(roc_auc_score(Yte, dev.predict_proba(Xte), average="micro")), 5)}
        if not args.no_host:
            sk = MLPClassifier(**REPO_MLP)
            t0 = time.perf_counter()
            sk.fit(Xtr.astype(np.float64), Ytr)
            row["host_fit_s"] = round(time.perf_counter() - t0, 3)
            row["host_epochs"] = sk.n_iter_
            row["host_s_per_epoch"] = round(row["host_fit_s"] / sk.n_iter_, 3)
            row["auc_host"] = round(float(roc_auc_score(Yte, sk.predict_proba(Xte.astype(np.float64)), average="micro")), 5)
        row.update(machine)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"machine": machine, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
