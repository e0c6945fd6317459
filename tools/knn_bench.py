"""Similar-issue search throughput: IssueIndex.search against the f32 torch baseline, one JSON line per case.

Seeded corpus N x D on the device (clustered, with a common offset like pooled AWD-LSTM features), k = 10,
nq in {1, 256, 1280}, both metrics.  Device time per search from CUDA events after a warm-up, averaged over windows
of at least --window seconds.  Reports the algorithmic 2 nq N D FLOP/s, the rate of the MMAs actually issued (x3 for
split-bf16, queries padded to 128-row tiles), the bytes bound (the split-bf16 corpus read once) and the same search as
torch f32 (TF32 off): cdist / normalised Q @ X^T + topk, and both answers' top-k agreement with a float64 brute force
on a sample of queries.  The card name and its power limit are printed beside the numbers.

    python tools/knn_bench.py [--n 1000000] [--dim 1600] [--window 1.0]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timed(fn, window):
    fn()
    torch.cuda.synchronize()
    reps, ms = 1, 0.0
    while True:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b)
        if ms >= 1000 * window:
            return ms / reps
        reps = max(reps * 2, int(reps * 1.2 * 1000 * window / max(ms, 1e-3)))


def f64_topk(X, Q, k, metric):
    out = []
    for q in Q.double():
        best_d, best_i = None, None
        for r0 in range(0, X.shape[0], 1 << 17):
            x = X[r0:r0 + (1 << 17)].double()
            if metric == "euclidean":
                d = ((x - q) ** 2).sum(1).sqrt()
            else:
                d = 0.5 * ((x / x.norm(dim=1, keepdim=True) - q / q.norm()) ** 2).sum(1)
            i = torch.arange(r0, r0 + x.shape[0], device=X.device)
            best_d = d if best_d is None else torch.cat([best_d, d])
            best_i = i if best_i is None else torch.cat([best_i, i])
            o = torch.argsort(best_d, stable=True)[: 4 * k]
            best_d, best_i = best_d[o], best_i[o]
        out.append(best_i[:k])
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1600)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--nq", default="1,256,1280")
    ap.add_argument("--sample", type=int, default=8)
    args = ap.parse_args()
    from code_intelligence_b200.knn import IssueIndex
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    g = torch.Generator(device="cuda").manual_seed(0)
    N, D, k = args.n, args.dim, args.k
    centres = torch.randn(1000, D, device="cuda", generator=g) * 0.05 + 0.3
    X = torch.empty(N, D, device="cuda")
    for r0 in range(0, N, 1 << 17):
        r1 = min(N, r0 + (1 << 17))
        lab = torch.randint(0, 1000, (r1 - r0,), device="cuda", generator=g)
        X[r0:r1] = centres[lab] + 0.02 * torch.randn(r1 - r0, D, device="cuda", generator=g)
    print(json.dumps({"card": card, "power_limit": power, "N": N, "D": D, "k": k}), flush=True)
    for metric in ("cosine", "euclidean"):
        index = IssueIndex(D, metric).add(X)
        torch.cuda.synchronize()
        Xn = X / X.norm(dim=1, keepdim=True) if metric == "cosine" else None
        for nq in [int(v) for v in args.nq.split(",")]:
            Q = X[torch.randint(0, N, (nq,), device="cuda", generator=g)] + \
                0.01 * torch.randn(nq, D, device="cuda", generator=g)
            ms = timed(lambda: index.search(Q, k), args.window)

            def baseline():
                if metric == "cosine":
                    s = (Q / Q.norm(dim=1, keepdim=True)) @ Xn.T
                    return torch.topk(s, k, dim=1)
                return torch.topk(-torch.cdist(Q, X), k, dim=1)
            ms_t = timed(baseline, args.window)
            m = min(nq, args.sample)
            want = f64_topk(X, Q[:m], k, metric)
            got = index.search(Q[:m], k)[1]
            base = baseline()[1][:m]
            flop = 2.0 * nq * N * D
            mma = 2.0 * 3 * ((nq + 127) // 128 * 128) * ((N + 255) // 256 * 256) * ((D + 63) // 64 * 64)
            bytes_bound_ms = N * ((D + 63) // 64 * 64) * 4 / 3.35e12 * 1e3   # split-bf16 corpus at the 3.35 TB/s data-sheet rate
            print(json.dumps({
                "metric": metric, "nq": nq, "search_ms": round(ms, 3), "torch_f32_ms": round(ms_t, 3),
                "speedup": round(ms_t / ms, 2), "algorithmic_tflops": round(flop / ms / 1e9, 1),
                "mma_issued_tflops": round(mma / ms / 1e9, 1), "bytes_bound_ms": round(bytes_bound_ms, 3),
                "agree_exact": float((got == want).float().mean()), "torch_f32_agree": float((base == want).float().mean()),
                "card": card, "power_limit": power}), flush=True)
        index.close()


if __name__ == "__main__":
    main()
