"""Development aid: board power / SM clock / achieved TFLOP/s of a workload run back to back for a few seconds, to
compare energy per FLOP of the encoder paths with cuBLAS (the chip sits at its power cap under all of them,
the kernels run at the board's power cap).

    python tools/power_probe.py --what cublas,enc,enc:IE_GX_BF16=0,enc256 --seconds 4 [--T 512]

    cublas            : torch.matmul bf16 8192^3 (the driver's MEASURED_PEAKS recipe)
    enc[:K=V[+K=V]]   : encoder path at max_batch rows x T per call, created under the given development knobs
    enc256[:...]      : same with 256 rows per call (one batch per launch)
    PROBE_IDS=seq|zipf: token ids whose rows of the per-token table are neighbours / follow a Zipf law (default: uniform
                        random ids, the worst case for the table's DRAM locality: layer 0 then runs ~3 ms slower per call)
Reports, per workload: median SM clock / board power (nvidia-smi), TFLOP/s, pJ/FLOP, the phase times of the last call
and the SM clock each layer's recurrent kernel saw (clock64 / globaltimer stamps inside the kernel).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
FLOP_PER_TOKEN = 266.24e6   # R4 encoder, SURVEY.md section 8d


class Sampler:
    def __init__(self, gpu=0, ms=50):
        self.rows, self.p = [], None
        self.cmd = ["nvidia-smi", "--query-gpu=clocks.sm,power.draw,temperature.gpu,clocks_event_reasons.sw_power_cap",
                    "--format=csv,noheader,nounits", "-i", str(gpu), "-lms", str(ms)]

    def __enter__(self):
        self.p = subprocess.Popen(self.cmd, stdout=subprocess.PIPE, text=True)
        threading.Thread(target=self._read, daemon=True).start()
        return self

    def _read(self):
        for line in self.p.stdout:
            self.rows.append((time.perf_counter(), [c.strip() for c in line.split(",")]))

    def __exit__(self, *a):
        self.p.terminate()

    def summary(self, t0, t1):
        clk, pw, temp, cap = [], [], [], 0
        for (t, r) in self.rows:
            if t0 + 0.5 <= t <= t1:       # skip the ramp
                try:
                    clk.append(float(r[0])); pw.append(float(r[1])); temp.append(float(r[2]))
                    cap += r[3].lower().startswith("active")
                except Exception:
                    pass
        med = lambda v: sorted(v)[len(v) // 2] if v else None
        return dict(samples=len(clk), sm_mhz=med(clk), power_w=med(pw), temp_c=med(temp), power_cap_samples=cap)


def rand_weights(seed=1234):
    import numpy as np
    rng = np.random.default_rng(seed)
    emb = rng.uniform(-0.1, 0.1, (60000, 800)).astype(np.float32)
    layers = []
    for l in range(4):
        n_in, n_out = (800 if l == 0 else 2400), (800 if l == 3 else 2400)
        k = 1.0 / np.sqrt(n_out)
        layers.append({n: rng.uniform(-k, k, s).astype(np.float32) for n, s in
                       (("w_ih", (4 * n_out, n_in)), ("w_hh", (4 * n_out, n_out)), ("b_ih", 4 * n_out), ("b_hh", 4 * n_out))})
    return emb, layers


def run(what, seconds, T):
    import torch
    if what == "cublas":
        a = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
        b = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
        step = lambda: torch.matmul(a, b)
        flop = 2 * 8192 ** 3
        extra = {}
    else:
        from code_intelligence_b200 import IssueEncoder
        name, _, knobs = what.partition(":")
        env = dict(kv.split("=") for kv in knobs.split("+")) if knobs else {}
        os.environ.update(env)
        enc = IssueEncoder().load_weights(*rand_weights())
        B = 256 if name == "enc256" else enc.max_batch
        ids = torch.randint(2, 60000, (B, T), dtype=torch.int64, device="cuda")
        if os.environ.get("PROBE_IDS") == "seq":    # neighbouring rows read neighbouring rows of the per-token table
            ids = ((torch.arange(B, device="cuda")[:, None] + 257 * torch.arange(T, device="cuda")[None, :]) % 59000 + 2).to(torch.int64)
        elif os.environ.get("PROBE_IDS") == "zipf":  # a few hot tokens, like text
            w = 1.0 / torch.arange(1, 59999, dtype=torch.float64) ** 1.1
            ids = (torch.multinomial(w / w.sum(), B * T, replacement=True).view(B, T) + 2).to(torch.int64).cuda()
        lengths = torch.full((B,), T, dtype=torch.int32, device="cuda")
        out = torch.empty((B, enc.out_dim), dtype=torch.float32, device="cuda")
        step = lambda: enc.encode_ids_device(ids, lengths, out)
        flop = FLOP_PER_TOKEN * B * T
        extra = {"rows": B, "T": T}
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    with Sampler() as s:
        t0 = time.perf_counter()
        n = 0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        while time.perf_counter() - t0 < seconds:
            for _ in range(4):
                step()
            n += 4
            torch.cuda.synchronize()
        e1.record()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        ms = e0.elapsed_time(e1)
        time.sleep(0.1)
        rec = s.summary(t0, t1)
    tflops = flop * n / (ms * 1e-3) / 1e12
    rec.update(what=what, calls=n, ms_per_call=round(ms / n, 3), tflops=round(tflops, 1), **extra)
    if rec["power_w"]:
        rec["pj_per_flop"] = round(rec["power_w"] / (tflops * 1e12) * 1e12, 3)
    if what != "cublas":
        rec["issues_per_s"] = round(extra["rows"] * n / (ms * 1e-3), 1)
        rec["phases_last_call"] = {k: ([round(x, 2) for x in v] if isinstance(v, list) else round(v, 2))
                                   for k, v in enc.last_phase_ms().items()}
        rec["phase_sm_mhz"] = {k: [round(x) for x in v] for k, v in enc.last_phase_mhz().items()}
        for k in env:
            os.environ.pop(k, None)
        enc.close()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="cublas,enc")
    ap.add_argument("--seconds", type=float, default=4.0)
    ap.add_argument("--T", type=int, default=512)
    a = ap.parse_args()
    for w in a.what.split(","):
        print(json.dumps(run(w, a.seconds, a.T)), flush=True)
        time.sleep(1.0)   # let the board cool between workloads


if __name__ == "__main__":
    main()
