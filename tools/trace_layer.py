"""Development aid: per-item timeline of the persistent recurrent kernel (csrc/lstm_layer.cu).

Slots the kernel writes per (cta, item k), %globaltimer ns: 0 step counter seen by the h producer, 1 last h tile
issued, 2 first h_{t-1} stage landed (first consumer warpgroup), 3 that warpgroup's MMAs complete, 6 item published.
The other slots of a record stay 0.
"""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from code_intelligence_b200 import IssueEncoder

ap = argparse.ArgumentParser()
ap.add_argument("--T", type=int, default=128)
ap.add_argument("--layer", type=int, default=1)
ap.add_argument("--B", type=int, default=1280)
ap.add_argument("--preroll", type=float, default=0.0, help="seconds of back-to-back encodes before the traced call (sustained clocks)")
a = ap.parse_args()
g = torch.Generator().manual_seed(1)
dims = [((800 if l == 0 else 2400), (2400 if l != 3 else 800)) for l in range(4)]
emb = (torch.rand(60000, 800, generator=g) * 0.2 - 0.1).numpy()
layers = []
for i, o in dims:
    k = 1.0 / np.sqrt(o)
    u = lambda *s: ((torch.rand(*s, generator=g) * 2 - 1) * k).numpy()
    layers.append(dict(w_ih=u(4 * o, i), w_hh=u(4 * o, o), b_ih=u(4 * o), b_hh=u(4 * o)))
enc = IssueEncoder().load_weights(emb, layers)
ids = torch.randint(2, 60000, (a.B, a.T), generator=g, dtype=torch.int64).numpy()
enc.encode_ids(ids)   # warm
if a.preroll > 0:
    import time
    ids_d = torch.from_numpy(ids).cuda()
    len_d = torch.full((a.B,), a.T, dtype=torch.int32, device="cuda")
    out_d = torch.empty((a.B, 2400), device="cuda")
    t0 = time.perf_counter()
    while time.perf_counter() - t0 < a.preroll:
        for _ in range(4):
            enc.encode_ids_device(ids_d, len_d, out_d)
        torch.cuda.synchronize()
enc._lib.ie_debug_seq_trace(enc._h, a.layer, None, 0)
if a.preroll > 0:
    for _ in range(3):      # the trace of the LAST call is read back; the ones before keep the device busy
        enc.encode_ids_device(ids_d, len_d, out_d)
    torch.cuda.synchronize()
    print("phase ms", enc.last_phase_ms(), "mhz", enc.last_phase_mhz())
else:
    enc.encode_ids(ids)
ng = (a.B + 255) // 256
tiles = 38 if a.layer < 3 else 13
C = ng * 2 * tiles                          # items per timestep: batches x row halves x column tiles
ctas = min(torch.cuda.get_device_properties(0).multi_processor_count, a.T * C)   # one item per CTA per round
items = (a.T * C + ctas - 1) // ctas
buf = np.zeros((ctas, items, 12), dtype=np.int64)
n = enc._lib.ie_debug_seq_trace(enc._h, -1, buf.ctypes.data, buf.size)
print("records", n, "ctas", ctas, "items/cta", items, "ng", ng, "tiles", tiles)
tr = buf.astype(np.float64)
sel = slice(8, items - 3)
us = 1e-3
span = (tr[:, :, 6].max() - tr[:, 0, 0].min()) * us
print(f"layer span {span / 1e3:.3f} ms = {span / a.T:.2f} us per timestep = {span / a.T / ng:.2f} us per batch-step")
period = np.diff(tr[:, :, 6], axis=1)[:, sel] * us
print(f"item period per CTA (publish to publish): mean {period.mean():.2f} us  p10 {np.percentile(period, 10):.2f}  p90 {np.percentile(period, 90):.2f}")
mma = (tr[:, :, 3] - tr[:, :, 2])[:, sel] * us
print(f"recurrent MMA phase (first h stage landed -> MMAs complete): mean {mma.mean():.2f} us  max {mma.max():.2f}")
ep = (tr[:, :, 6] - tr[:, :, 3])[:, sel] * us
print(f"epilogue + publish (MMAs complete -> published): mean {ep.mean():.2f} us  max {ep.max():.2f}")
idle = (tr[:, 1:, 2] - tr[:, :-1, 6])[:, sel] * us
print(f"published k -> first h stage of k+1 landed: mean {idle.mean():.2f} us  p90 {np.percentile(idle, 90):.2f}")
print(f"first h stage landed after counter seen: mean {((tr[:, :, 2] - tr[:, :, 0])[:, sel] * us).mean():.2f} us")
# dependency slack: item n needs every item of (t-1, g); when was the LAST of them published relative to our counter-seen time
pub_t = np.zeros((a.T, ng))
for p in range(ctas):
    for k in range(items):
        nidx = p + k * ctas
        if nidx >= a.T * C:
            break
        t, c = divmod(nidx, C)
        pub_t[t, c // (2 * tiles)] = max(pub_t[t, c // (2 * tiles)], tr[p, k, 6])
lat = []
for p in range(0, ctas, 7):
    for k in range(8, items - 3):
        nidx = p + k * ctas
        if nidx >= a.T * C:
            break
        t, c = divmod(nidx, C)
        if t > 0:
            lat.append(tr[p, k, 0] - pub_t[t - 1, c // (2 * tiles)])
lat = np.array(lat) * us
print(f"counter seen after the last publish of (t-1, g): mean {lat.mean():.2f} us  p10 {np.percentile(lat, 10):.2f}  p90 {np.percentile(lat, 90):.2f}")
