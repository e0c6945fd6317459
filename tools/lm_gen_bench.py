"""Text generation from the language model at the deployed shape (4 x 2400 AWD-LSTM, emb_sz 800, vocabulary 60000) on
one H100, in the default (bf16) and the fp32-accurate mode:

* ``predict`` from a 64-token prompt for 256 words: ms per word and words/s (host clock around the call, which ends
  with its one copy back);
* ``beam_search`` at top_k = 10, beam_sz = 1000 for 8 words: ms per step;
* each step's device time split into the encoder (recurrent kernels, input projections, copies), the logits GEMM,
  top-k / sampling, and the beam's selection and state gather, from a separate torch.profiler run (32 words of
  predict, 4 beam steps), by kernel name.

Random seeded weights (the time does not depend on their values).  Prints one JSON line per measurement, the card's
name, power limit and max SM clock first."""
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from code_intelligence_b200 import IssueEncoder
from code_intelligence_b200._lib import IE_CFG_FP32
from code_intelligence_b200.language_model import LanguageModel

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True)
print(json.dumps(dict(gpu=q.stdout.strip())), flush=True)

V, E, H, L = 60000, 800, 2400, 4


def build(flags):
    rng = np.random.default_rng(0)
    enc = IssueEncoder(L, E, H, V, 1, 0, flags)
    emb = rng.uniform(-0.1, 0.1, (V, E)).astype(np.float32)
    layers = []
    for l in range(L):
        i, o = (E if l == 0 else H), (H if l < L - 1 else E)
        s = 1 / np.sqrt(o)
        layers.append(dict(w_ih=rng.uniform(-s, s, (4 * o, i)).astype(np.float32),
                           w_hh=rng.uniform(-s, s, (4 * o, o)).astype(np.float32),
                           b_ih=rng.uniform(-s, s, 4 * o).astype(np.float32),
                           b_hh=rng.uniform(-s, s, 4 * o).astype(np.float32)))
    enc.load_weights(emb, layers)
    return LanguageModel(enc, emb * 20, rng.standard_normal(V).astype(np.float32), owns_encoder=True)


def stage(name: str) -> str:
    if "lm_topk" in name or "lm_sample" in name:
        return "topk_sample"
    if "beam_select" in name or "gather_rows" in name:
        return "select"
    if "gemm_bf16_kernel<float, 0, false" in name:
        return "logits_gemm"
    return "encoder"


def split(fn, steps):
    """ms of device time per step by stage, from one profiled call of fn."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ms = defaultdict(float)
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            ms[stage(e.key)] += t / 1000.0
    return {k: round(v / steps, 3) for k, v in sorted(ms.items())}


prompt = np.concatenate([[2], np.random.default_rng(1).integers(5, V, 63)]).astype(np.int64)
for mode, flags in (("bf16", 0), ("fp32", IE_CFG_FP32)):
    lm = build(flags)
    lm.predict(prompt, 4, seed=0)           # warm up every shape the timed calls use
    lm.beam_search(prompt, 2, seed=0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    lm.predict(prompt, 256, seed=1)
    dt = time.perf_counter() - t0
    print(json.dumps(dict(what="predict", mode=mode, prompt=64, words=256, ms_per_word=round(dt * 1e3 / 256, 3),
                          words_per_s=round(256 / dt, 1))), flush=True)
    t0 = time.perf_counter()
    lm.beam_search(prompt, 8, top_k=10, beam_sz=1000, seed=1)
    dt = time.perf_counter() - t0
    print(json.dumps(dict(what="beam_search", mode=mode, top_k=10, beam_sz=1000, words=8,
                          ms_per_step=round(dt * 1e3 / 8, 2))), flush=True)
    one = split(lambda: lm.predict(prompt[-1:], 32, seed=2), 32)
    print(json.dumps(dict(what="predict step split (device ms per word, 1 row)", mode=mode, **one)), flush=True)
    # steady beam steps: the first of the 4 runs 10 rows, the rest 100 and 1000
    beam = split(lambda: lm.beam_search(prompt[-1:], 4, top_k=10, beam_sz=1000, seed=2), 4)
    print(json.dumps(dict(what="beam step split (device ms per step, mean of 10/100/1000/1000 rows)", mode=mode,
                          **beam)), flush=True)
    lm.close()
