"""Throughput of the text classifier (fastai text_classifier_learner, 06_FineTune's shape: 4 x 2400 AWD-LSTM, emb_sz
800, head 2400 -> 50 -> n_class) on one H100, next to the encoder alone on the same handle:

* issues/s of TextClassifier.predict_proba (per-item mode, host id lists) and of IssueEncoder.encode_id_list, at the
  bench shape (1280 issues x 512 tokens) and on var-len issues of 64-512 tokens;
* device time (CUDA events) of one 1280 x 512 device-pointer call of each, whose difference is what the pool, the head
  and the f32 state store cost over the encoder's own pool.

Random weights (throughput does not depend on their values).  Prints one JSON line per measurement, the card's name,
power limit and max SM clock first."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from code_intelligence_b200 import IssueEncoder
from code_intelligence_b200.text_classifier import TextClassifier

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=1280)
ap.add_argument("--T", type=int, default=512)
ap.add_argument("--n-class", type=int, default=28)
ap.add_argument("--reps", type=int, default=3)
args = ap.parse_args()

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True)
print(json.dumps(dict(gpu=q.stdout.strip())), flush=True)

rng = np.random.default_rng(0)
V, E, H, L = 60000, 800, 2400, 4
enc = IssueEncoder(L, E, H, V, 1, 0)
emb = rng.uniform(-0.1, 0.1, (V, E)).astype(np.float32)
layers = []
for l in range(L):
    n_in, n_out = (E if l == 0 else H), (H if l < L - 1 else E)
    k = 2.0 / np.sqrt(n_out)
    layers.append(dict(w_ih=rng.uniform(-k, k, (4 * n_out, n_in)).astype(np.float32),
                       w_hh=rng.uniform(-k, k, (4 * n_out, n_out)).astype(np.float32),
                       b_ih=rng.uniform(-k, k, 4 * n_out).astype(np.float32),
                       b_hh=rng.uniform(-k, k, 4 * n_out).astype(np.float32)))
enc.load_weights(emb, layers)
dims = [3 * E, 50, args.n_class]
stages = [dict(bn_weight=1 + 0.1 * rng.standard_normal(a).astype(np.float32),
               bn_bias=0.1 * rng.standard_normal(a).astype(np.float32),
               bn_mean=0.05 * rng.standard_normal(a).astype(np.float32),
               bn_var=(0.01 + 0.01 * rng.random(a)).astype(np.float32),
               weight=(rng.standard_normal((b, a)) / np.sqrt(a)).astype(np.float32),
               bias=np.zeros(b, np.float32)) for a, b in zip(dims[:-1], dims[1:])]
clf = TextClassifier(enc, stages)


def docs_of(lengths):
    out = []
    for n in lengths:
        d = rng.integers(2, V, size=int(n)).astype(np.int64)
        d[0] = 2
        out.append(d)
    return out


def rate(fn, docs):
    fn(docs)                                              # warm-up: every shape, workspace grown
    ts = []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(docs)
        ts.append(time.perf_counter() - t0)
    return len(docs) / float(np.median(ts)), [round(len(docs) / t, 1) for t in ts]


for name, lengths in (("fixed", np.full(args.rows, args.T)), ("varlen_64_512", rng.integers(64, args.T + 1, args.rows))):
    docs = docs_of(lengths)
    r_clf, all_clf = rate(clf.predict_proba, docs)
    r_enc, all_enc = rate(enc.encode_id_list, docs)
    print(json.dumps(dict(shape=name, issues=len(docs), tokens=int(np.sum(lengths)),
                          classifier_issues_per_s=round(r_clf, 1), classifier_repeats=all_clf,
                          encoder_issues_per_s=round(r_enc, 1), encoder_repeats=all_enc,
                          classifier_over_encoder=round(r_clf / r_enc, 4))), flush=True)

# device time of one device-pointer call of each on the same ids
ids = torch.as_tensor(np.vstack(docs_of(np.full(args.rows, args.T)))).cuda()
lengths = torch.full((args.rows,), args.T, dtype=torch.int32, device="cuda")
starts = torch.zeros(args.rows, dtype=torch.int32, device="cuda")
ends = lengths.clone()


def event_ms(fn):
    fn()
    ms = []
    for _ in range(args.reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), [round(m, 2) for m in ms]


enc_ms, enc_all = event_ms(lambda: enc.encode_ids_device(ids, lengths))
clf_ms, clf_all = event_ms(lambda: clf.forward_padded_device(ids, starts, ends))
state_gb = args.rows * args.T * 832 * 4 / 1e9
print(json.dumps(dict(shape=f"{args.rows}x{args.T} device pointers", encoder_ms=round(enc_ms, 2), encoder_repeats=enc_all,
                      classifier_ms=round(clf_ms, 2), classifier_repeats=clf_all,
                      classifier_extra_ms=round(clf_ms - enc_ms, 2), f32_states_gb=round(state_gb, 2),
                      classifier_launches_per_call=len(dims) + 1)), flush=True)

# the classifier's own kernels in one device-pointer call, from a profiler trace (a run of its own, after the timing)
from torch.profiler import ProfilerActivity, profile
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    clf.forward_padded_device(ids, starts, ends)
    torch.cuda.synchronize()
kernels = {}
for ev in prof.key_averages():
    if "clas_" in ev.key:
        name = ev.key.split("clas_")[1].split("(")[0].split("<")[0]
        kernels[name] = round(getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1e3, 3)
pool_ms = kernels.get("pool_kernel", 0.0)
print(json.dumps(dict(shape=f"{args.rows}x{args.T} classifier kernels (profiler)", kernel_ms=kernels,
                      pool_state_read_gb_per_s=round(state_gb / (pool_ms / 1e3), 1) if pool_ms else None)), flush=True)
clf.check_errors()
clf.close()
enc.close()
