"""BASELINE.json configs[2]: var-len bucketed sweep, seq_len 64..2048, bf16 tensor-core path vs the fp32 CPU oracle.
Per bucket: 1280 issues (five batches of 256 per launch), lengths uniform in (T/2, T], right padded to T; parity of four
rows against the live oracle (the full-size goldens of tests/golden cover 32..256 rows per shape in the test-suite).
Prints one JSON line per bucket."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from code_intelligence_b200 import IssueEncoder
from oracle import awd_lstm_ref as R

torch.set_num_threads(min(16, os.cpu_count()))
ref = R.make_encoder(1234)
emb, layers = ref.export_weights()
enc = IssueEncoder().load_weights(emb, layers)
rng = np.random.default_rng(5)
for T in (64, 128, 256, 512, 1024, 2048):
    B = enc.max_batch
    lengths = rng.integers(T // 2 + 1, T + 1, size=B).astype(np.int32)
    ids = np.full((B, T), 1, dtype=np.int64)
    for b in range(B):
        a = rng.integers(0, 60000, size=lengths[b]); a[a == 1] = 0; a[0] = 2
        ids[b, :lengths[b]] = a
    ids_d = torch.from_numpy(ids).cuda(); len_d = torch.from_numpy(lengths).cuda()
    out = torch.empty((B, 2400), device="cuda")
    for _ in range(2):
        enc.encode_ids_device(ids_d, len_d, out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 3
    e0.record()
    for _ in range(n):
        enc.encode_ids_device(ids_d, len_d, out)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    got = out.cpu().numpy()
    sub = [0, 1, 300, B - 1]
    want = R.encode_padded(ref, ids[sub], lengths[sub])
    m = R.parity_metrics(got[sub], want)
    valid_tokens = int(lengths.sum())
    print(json.dumps(dict(seq_len=T, issues=B, ms=ms, issues_per_s=B / ms * 1e3, valid_tokens_per_s=valid_tokens / ms * 1e3,
                          tflops_valid=266.24e6 * valid_tokens / ms / 1e9, tflops_padded=266.24e6 * B * T / ms / 1e9,
                          min_cosine=m["min_cosine"], max_abs=m["max_abs"], rel_l2=m["rel_l2"],
                          phase_ms=enc.last_phase_ms(), phase_sm_mhz=enc.last_phase_mhz())), flush=True)
