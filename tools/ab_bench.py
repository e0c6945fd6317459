"""Development aid: A/B comparison of two source trees on the flagship benchmark, in one process tree on one GPU.

    python tools/ab_bench.py --a path/to/parent --b . [--repeats 3] [--steps 15] [--warmup 5] [--out DIR]

Each tree must already be built (``python -c "import __graft_entry__ as g; g.build()"`` inside it).  The script runs
``bench.py`` of A and of B alternately, ``--repeats`` times each, with ``--dump-outputs`` into DIR (a temporary
directory by default), so that drift of the clock or of other work on the host hits both sides alike.  It prints per
side the ``value`` of every repeat, its median and max - min spread, the median phase times of the last timed launch
(``roofline.phase_ms_last_call``) and the SM clocks the recurrent kernels saw; then the B / A ratio of the medians and whether
the last-step embeddings of every repeat of B are bit-equal (``np.array_equal``) to those of the first repeat of A.
Read the card's name and power limit (``nvidia-smi --query-gpu=name,power.limit --format=csv``) in the same call:
under a power cap the clock, not the kernel, may set the pace.

Neither tree is written to, except for what bench.py itself writes (nothing: its caches go to a temporary
directory).  A parent commit can be extracted into a directory with ``git archive <rev> | tar -x -C DIR``.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np


def run_bench(tree, args, dump):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(args.steps),
           "--warmup", str(args.warmup), "--dump-outputs", dump] + (["--no-extra"] if args.no_extra else [])
    p = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-2000:] + p.stderr[-4000:])
        raise SystemExit(f"bench.py of {tree} failed with exit code {p.returncode}")
    line = [l for l in p.stdout.splitlines() if l.startswith("{")][-1]
    return json.loads(line)


def summary(name, recs):
    vals = [r["value"] for r in recs]
    out = {"tree": name, "values": [round(v, 1) for v in vals], "median": round(statistics.median(vals), 1),
           "spread": round(max(vals) - min(vals), 1)}
    phases = [r.get("roofline", {}).get("phase_ms_last_call") for r in recs]
    if all(phases):
        def med(get):
            return round(statistics.median(get(p) for p in phases), 2)
        L = len(phases[0]["steps"])
        out["phase_ms_median"] = {"gemm": [med(lambda p, l=l: p["gemm"][l]) for l in range(L)],
                                  "steps": [med(lambda p, l=l: p["steps"][l]) for l in range(L)]}
    mhz = [r.get("roofline", {}).get("phase_sm_mhz") for r in recs]
    if all(mhz):
        out["steps_sm_mhz"] = [m["steps"] for m in mhz]
    for key in ("single_batch", "e2e"):
        if key in recs[0]:
            out[key] = [round(r[key]["value"], 1) for r in recs]
    ex = [r.get("extra", {}) for r in recs]
    for key in ("fp32_mode", "n3", "mlp_1600", "mlp_2400"):
        if all(isinstance(e.get(key), dict) and "value" in e[key] for e in ex):
            out[key] = [round(e[key]["value"], 1) for e in ex]
    bv = [e.get("bulk_varlen", {}).get("bit_equal_to_single_gpu") for e in ex]
    if any(b is not None for b in bv):
        out["bulk_varlen_bit_equal"] = bv
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", required=True, help="baseline tree (e.g. the parent commit, extracted and built)")
    ap.add_argument("--b", required=True, help="tree under test")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-extra", action="store_true", help="pass --no-extra to bench.py (value and phases only)")
    ap.add_argument("--out", default=None, help="directory for the dumped embeddings (default: a temporary one)")
    args = ap.parse_args()
    trees = {"A": os.path.abspath(args.a), "B": os.path.abspath(args.b)}
    tmp = None if args.out else tempfile.TemporaryDirectory(prefix="ab_bench_")
    root = args.out or tmp.name
    recs = {"A": [], "B": []}
    dumps = {"A": [], "B": []}
    for i in range(args.repeats):
        for side in ("A", "B"):
            d = os.path.join(root, f"{side}{i}")
            recs[side].append(run_bench(trees[side], args, d))
            dumps[side].append(os.path.join(d, "embeddings.npy"))
            print(json.dumps({"side": side, "repeat": i, "value": round(recs[side][-1]["value"], 1)}), flush=True)
    ref = np.load(dumps["A"][0])
    equal = [bool(np.array_equal(ref, np.load(p))) for p in dumps["A"][1:] + dumps["B"]]
    a, b = summary(trees["A"], recs["A"]), summary(trees["B"], recs["B"])
    for side, rec in (("A", a), ("B", b)):
        print(json.dumps({"side": side, **rec}), flush=True)
    print(json.dumps({"b_over_a": round(b["median"] / a["median"], 4), "embeddings_bit_equal_to_first_A": equal,
                      "shape": list(ref.shape)}), flush=True)
    if tmp is not None:
        tmp.cleanup()


if __name__ == "__main__":
    main()
