"""GPU tests of every element of the one-batch launches (ng = 1: B <= 256, b_pad = 256): one issue per call (the /text
endpoint, bench.py's online_b1), bench.py's single_batch arm (B = 256), and long issues across the time chunk, which at
b_pad = 256 is 2^20 / 256 = 4096 steps (2048 with f32 input projections).  Teacher-forced against
oracle/device_numerics.py on ALL valid rows, steps, units and layers, as tests/test_gpu_bench_shape_numerics.py does
for the 1280 x 512 launch, and tied to the production calls bit for bit:

  * the pooled encode (encode_ids_device) equals device_numerics.pool of the hook's last-layer states on every row, and
    raw_features equals the hook's last layer;
  * T <= 512: the result of the one-batch call equals the same issues' rows inside a B = 1280 call (ng = 5) padded
    with pad_idx to T = 512;
  * around a chunk boundary: the pooled row of each length equals a call on ids[:, :len] alone (prefix property);
  * the long issue: the pooled mean lies within the error bound of a sequential f32 sum of the float64 mean of the
    same states -- the one check of that mean against a high-precision value rather than a restatement.

Before every checked call the handle encodes different ids of the same shape.  The oracle mutants of the bench-shape
file are applied to the rows of batch 0 / row half 0; the item-local ones at the chunk boundary where there is one.

test_long_issue_workspace_is_released pins the raw-state workspace: only the B valid rows are stored (a 20 000-token
issue at the deployed shape fits), and a handle that served a long issue gives its workspace back after four calls far
below it.
"""
import json
import time

import numpy as np
import pytest
import torch

from oracle import awd_lstm_ref as R
from oracle import device_numerics as D
from test_gpu_bench_shape_numerics import R4, _device_used_gb, _mutants
from test_gpu_parity import _make

pytestmark = pytest.mark.gpu

PAD = 1


def _cuda():
    return torch.device("cuda", 0)


def _ids(seed, B, T, lengths, same=False):
    """Random ids right-padded with pad_idx; same: every row holds row 0's tokens."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, R4[3], (1 if same else B, T), generator=g, dtype=torch.int64)
    ids[:, 0] = 2
    ids = ids.expand(B, T).clone()
    ids[torch.arange(T)[None, :] >= torch.from_numpy(lengths).long()[:, None]] = PAD
    return ids


# tag -> (B, T, weight scale, flags, lengths (None: all T), step of the item-local mutants, (max cap, RMS cap))
# Observed on an H100 SXM 80 GB HBM3 (power limit 700 W), max / RMS of |dh| / bound over every element: text 128
#   0.689 / 0.0130, text 512 0.777 / 0.0149, text 512 fp32 0.064 / 0.0253, single batch 0.872 / 0.0132, one row over
#   0.855 / 0.0152, chunk edge 0.820 / 0.0151, chunk edge fp32 0.064 / 0.0253, long issue 0.836 / 0.0151.  The largest
#   ratio is in layer 2 (layer 3 in the fp32 mode, at t = 0) and nowhere near a chunk boundary.  Caps are about twice
#   that, never above 1 (the bound itself).  The long issue's pooled mean uses 0.64 % of its float64 bound.
# Wall time 5-44 s per configuration (the file: about 3 minutes); device memory in use at the checked calls 3.3 GB
# (text 128) to 35 GB (the chunk edges and the long issue: 31 GB of encoder workspace, the time chunk at b_pad = 256
# being 2^20 rows); torch's peak 20 GB (the oracle on 256 rows).
CONFIGS = {
    "text 128": (1, 128, 1.0, 0, None, 100, (1.0, 0.026)),
    "text 512": (1, 512, 2.0, 0, None, 300, (1.0, 0.03)),
    "text 512 fp32": (1, 512, 1.0, D.IE_CFG_FP32, None, 300, (0.13, 0.05)),
    "single batch": (256, 512, 1.0, 0, None, 300, (1.0, 0.027)),
    "one row over": (257, 300, 2.0, 0, None, 200, (1.0, 0.03)),
    "chunk edge": (4, 4100, 2.0, 0, (4095, 4096, 4097, 4100), 4096, (1.0, 0.03)),
    "chunk edge fp32": (4, 2050, 1.0, D.IE_CFG_FP32, (2047, 2048, 2049, 2050), 2048, (0.13, 0.05)),
    "long issue": (1, 12300, 2.0, 0, None, 12288, (1.0, 0.03)),
}
# Mutants that break the caps by less than 4x.  The f/o swap touches one unit of the checked rows; with one row of 128
# steps at weight scale 1 it reaches max 2.85 (2.9x the cap; 20x at T = 512, 4.6x on the 128 rows of single batch).
WEAK_MUTANTS = {("text 128", "swap_fo")}


def _pooled_mean_vs_f64(h, n, got_mean):
    """|device mean - float64 mean| over the bound of a sequential f32 sum of n terms (gamma_{n-1} sum |h|) scaled by
    f32(1/n), plus the two roundings of the scaling -> largest fraction of the bound used."""
    h = h[:n].double()
    m64 = h.sum(0) / n
    u = D.U24
    gamma = (n - 1) * u / (1 - (n - 1) * u)
    bound = gamma * h.abs().sum(0) / n * (1 + 3 * u) + 3 * u * m64.abs() + D.TINY
    return float(((torch.from_numpy(got_mean).double().to(h.device) - m64).abs() / bound).max())


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_every_element_of_the_one_batch_launches(tag, monkeypatch):
    """Every layer, valid row, step and unit of one configuration under its caps, its mutants, and the production calls
    (pooled encode, raw_features, the same issues inside a five-batch launch, shorter prefixes) tied to the checked
    states bit for bit."""
    B, T, scale, flags, ends, t_mut, (max_cap, rms_cap) = CONFIGS[tag]
    t_start = time.perf_counter()
    dev = _cuda()
    emb, layers = R.make_encoder(1234, n_layers=R4[0], scale=scale).export_weights()
    lengths = np.full(B, T, dtype=np.int32) if ends is None else np.asarray(ends, dtype=np.int32)
    same = ends is not None
    ids, poison = _ids(11, B, T, lengths, same).to(dev), _ids(12, B, T, lengths, same).to(dev)
    len_dev = torch.from_numpy(lengths).to(dev)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)

    enc = _make(R4, (emb, layers), monkeypatch, None, flags)
    states = []
    for l in range(R4[0]):
        enc.encode_ids_device(poison, len_dev)
        states.append(enc._debug_layer_states(l, ids))
        enc.check_errors()
    enc.encode_ids_device(poison, len_dev)
    raw = enc.raw_features(ids.cpu())
    enc.encode_ids_device(poison, len_dev)
    pooled = enc.encode_ids_device(ids, len_dev).cpu().numpy()
    enc.check_errors()
    torch.cuda.synchronize(dev)
    mem_gb = _device_used_gb()
    ws_gb = enc._debug_workspace_bytes() / 1e9

    ties = {}
    if T <= 512:
        # ng = 1 (or 2) against ng = 5: the rows at the end of a full launch of other issues, padded to 512
        rows = np.arange(1280 - B, 1280)
        big_len = np.random.default_rng(3).integers(1, 513, 1280).astype(np.int32)
        big_len[rows] = lengths
        big = _ids(13, 1280, 512, big_len)
        big[rows, :T] = ids.cpu()
        big[rows, T:] = PAD
        five = enc.encode_ids_device(big.to(dev), torch.from_numpy(big_len).to(dev)).cpu().numpy()
        enc.check_errors()
        ties["five_batch_equal"] = bool(np.array_equal(five[rows], pooled))
    if ends is not None:
        prefix = []
        for i, n in enumerate(lengths):
            enc.encode_ids_device(poison[i:i + 1, :n].contiguous(), len_dev[i:i + 1].clone().fill_(int(n)))
            one = enc.encode_ids_device(ids[i:i + 1, :n].contiguous(), len_dev[i:i + 1].clone().fill_(int(n)))
            prefix.append(bool(np.array_equal(one.cpu().numpy(), pooled[i:i + 1])))
        enc.check_errors()
        ties["prefix_equal"] = prefix
    enc.close()
    del enc
    torch.cuda.empty_cache()

    # the production calls are the checked one: pooled output = pool of the hook's states, raw = the hook's last layer
    last = states[-1].cpu().numpy()
    want = D.pool(last, lengths)
    ties["pool_equal"] = bool(np.array_equal(pooled, want))
    ties["raw_equal"] = bool(np.array_equal(raw, last))
    del raw, last
    if tag == "long issue":
        ties["mean_f64_bound_used"] = _pooled_mean_vs_f64(states[-1][0], int(lengths[0]), pooled[0, :R4[1]])

    modes = D.layer_modes(R4[0], flags)
    xs = [torch.from_numpy(emb).to(dev)[ids]] + states[:-1]
    design = [D.blocked_layer_stats(xs[l], states[l], layers[l], modes[l]) for l in range(R4[0])]
    mx = max(s["max"] for s in design)
    rms = max(s["rms"] for s in design)
    top = max(range(R4[0]), key=lambda l: design[l]["max"])
    items = [s["items"] for s in design]
    it_layer = max(range(R4[0]), key=lambda l: float(items[l].max()))
    it_idx = np.unravel_index(int(items[it_layer].argmax()), tuple(items[it_layer].shape))

    block = range(0, min(B, D.ITEM_ROWS))   # batch 0, row half 0
    mutants = {}
    block_design = {}
    for name, (l, mode) in _mutants(modes, t_mut).items():
        assert mode != modes[l], name
        if l not in block_design:
            block_design[l] = D.blocked_layer_stats(xs[l], states[l], layers[l], modes[l], rows=block)
        m = D.blocked_layer_stats(xs[l], states[l], layers[l], mode, rows=block)
        layer_rms = ((design[l]["sumsq"] - block_design[l]["sumsq"] + m["sumsq"]) / design[l]["n"]) ** 0.5
        mutants[name] = (m["max"], max([layer_rms] + [design[k]["rms"] for k in range(R4[0]) if k != l]))
    wall = time.perf_counter() - t_start
    print("NUMERICS " + json.dumps(dict(
        kind="one_batch", config=tag, B=B, T=T, caps=[max_cap, rms_cap], max=mx, rms=rms,
        argmax=dict(layer=top, row=design[top]["argmax"][0], t=design[top]["argmax"][1], unit=design[top]["argmax"][2]),
        above_half=sum(s["above_half"] for s in design), elements=sum(s["n"] for s in design),
        per_layer=[[s["max"], s["rms"]] for s in design],
        item_max=dict(value=float(items[it_layer].max()), layer=it_layer, t=int(it_idx[0]), g=int(it_idx[1]),
                      half=int(it_idx[2]), j=int(it_idx[3])),
        mutants=mutants, ties=ties, device_used_gb=round(mem_gb, 2), workspace_gb=round(ws_gb, 2),
        torch_peak_gb=round(torch.cuda.max_memory_allocated(dev) / 1e9, 2), wall_s=round(wall, 1))), flush=True)
    del states, xs
    torch.cuda.empty_cache()

    np.testing.assert_array_equal(pooled, want)
    assert ties["raw_equal"], tag
    assert ties.get("five_batch_equal", True), tag
    assert all(ties.get("prefix_equal", [True])), (tag, ties["prefix_equal"])
    assert ties.get("mean_f64_bound_used", 0.0) <= 1.0, (tag, ties["mean_f64_bound_used"])
    assert mx <= max_cap and rms <= rms_cap, (tag, mx, rms, (max_cap, rms_cap))
    for name, (m_mx, m_rms) in mutants.items():
        margin = 1 if (tag, name) in WEAK_MUTANTS else 4
        assert m_mx > margin * max_cap or m_rms > margin * rms_cap, (tag, name, m_mx, m_rms, (max_cap, rms_cap))


def test_long_issue_workspace_is_released(monkeypatch):
    """raw_features of one 12 300-token issue, then four bench-shape encodes: the handle holds no more workspace than a
    fresh handle after the same four encodes (the long call's buffers were given back).  raw_features of one
    20 000-token issue at the deployed shape succeeds (only the valid row's states are stored) and its pool is the
    pooled encode of the issue.  Measured on an H100: a fresh handle holds 19.3 GB after the four encodes; the long
    call's handle holds 30.9 GB (the 2^20-row time chunk of b_pad = 256) through the first three and 0.12 GB after the
    fourth; at T = 20 000 the workspace is 31.0 GB (storing the padding rows too took another 50 GB)."""
    dev = _cuda()
    emb, layers = R.make_encoder(1234, n_layers=R4[0], scale=2.0).export_weights()
    bench_len = torch.full((1280,), 512, dtype=torch.int32, device=dev)
    bench_ids = _ids(21, 1280, 512, np.full(1280, 512, dtype=np.int32)).to(dev)
    torch.cuda.empty_cache()

    fresh = _make(R4, (emb, layers), monkeypatch)
    for _ in range(4):
        fresh.encode_ids_device(bench_ids, bench_len)
    fresh.check_errors()
    fresh_bytes = fresh._debug_workspace_bytes()
    fresh.close()
    torch.cuda.empty_cache()

    enc = _make(R4, (emb, layers), monkeypatch)
    long_ids = _ids(22, 1, 12300, np.array([12300], dtype=np.int32))
    raw = enc.raw_features(long_ids)
    long_bytes = enc._debug_workspace_bytes()
    counts = []
    for _ in range(4):
        enc.encode_ids_device(bench_ids, bench_len)
        enc.check_errors()
        counts.append(enc._debug_workspace_bytes())

    T = 20000
    ids = _ids(23, 1, T, np.array([T], dtype=np.int32))
    raw = enc.raw_features(ids)
    big_bytes = enc._debug_workspace_bytes()
    pooled = enc.encode_ids(ids)
    used_gb = _device_used_gb()
    enc.close()
    print("WORKSPACE " + json.dumps(dict(fresh_after_4_encodes=fresh_bytes, after_raw_12300=long_bytes,
                                         after_each_encode=counts, after_raw_20000=big_bytes,
                                         device_used_gb=round(used_gb, 2))), flush=True)
    assert counts[-1] <= fresh_bytes, (counts, fresh_bytes)
    assert raw.shape == (1, T, R4[1]) and np.isfinite(raw).all()
    np.testing.assert_array_equal(D.pool(raw, [T]), pooled)
