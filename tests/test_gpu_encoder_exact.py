"""GPU tests of the encoder, its input-projection GEMM and the label head, bit for bit against the exact restatement of
oracle/device_numerics.py (gemm_exact, mlp_head_exact, teacher_forced_exact): the tensor-core chain by
tc_accum.chain_exact, every f32 operation and fma correctly rounded, the gate functions the device's own through
ie_debug_gates.  The bound-based files (test_gpu_numerics, test_gpu_config_space, test_gpu_single_batch_numerics,
test_gpu_bench_shape_numerics) accept any order of the sums; here a reordered k loop, a split pass issued out of turn,
Gx folded into the accumulator, the bias moved in the fused chain or the other cell contraction fails on the first
element it touches.  The configurations are those files' tables.

  * GEMM: every epilogue x operand form at the MLP shapes, and rows of the production Gx and per-token table shapes,
    through the natural (ie_debug_gemm_ex) and the fragment-ordered store (ie_debug_gemm_frag).
  * Label head: the MLP shapes, the grid-search shapes, the production fixture and the device-pointer multi-pass call.
  * Encoder, every row, step, unit and layer: the small model under every knob and the configuration space (except the
    three largest shapes, sampled).
  * Encoder sampled (every schedule item -- step, batch, row half, column tile -- on the first and last row of each row
    half and four units of each tile, the first and last real unit included, over all steps): the production shapes, the
    benchmarked launch (B = 1280, T = 512, device pointers, bench.py's weights and ids), and the one-batch launches
    across the 4096-step (2048 in the fp32 mode) time chunk.
  * Negative controls: every Mode mutant and every order mutant (device_numerics.ORDER_MUTANTS) disagrees with the
    device.

Each check prints one EXACT line with the elements compared and the wall time.
"""
import json
import time
from dataclasses import replace

import numpy as np
import pytest
import torch

from oracle import awd_lstm_ref as R
from oracle import device_numerics as D
from oracle import lstm_numpy as N
from test_gpu_bench_shape_numerics import _bench_ids
from test_gpu_config_space import CONFIGS as SPACE
from test_gpu_config_space import _edge_ids, _handle, _lengths, _weights
from test_gpu_label_head import GRID_CASES, _head
from test_gpu_numerics import EPILOGUES, MUTANTS, OUT_TYPES, R4_CONFIGS, SMALL, SMALL_CONFIGS, _mutate
from test_gpu_parity import _make, _pad
from test_gpu_single_batch_numerics import CONFIGS as ONE_BATCH
from test_gpu_single_batch_numerics import _ids as _one_batch_ids

pytestmark = pytest.mark.gpu

SAMPLED_SPACE = {"1 layer 800", "fastai 400/1152", "table > 6 GiB"}


def _cuda():
    return torch.device("cuda", 0)


def device_gates(name, x):
    """The device's gate function `name` (ie_debug_gates: the inline functions of ptx.cuh / lstm_common.cuh)."""
    from code_intelligence_b200 import _lib
    return _lib._debug_gates(name, x.to(_cuda(), torch.float32)).to(x.device, torch.float64)


def _mismatch(got, want):
    """Elements whose bits differ; +0 and -0 are equal only where the restatement's value is zero."""
    g = torch.as_tensor(got).to(want.device, torch.float32)
    w = want.to(torch.float32)
    same = (g.view(torch.int32) == w.view(torch.int32)) | ((g == 0) & (w == 0))
    return ~same


def _report(kind, **kw):
    print("EXACT " + json.dumps(dict(kind=kind, **kw)), flush=True)


# ------------------------------------------------------------------------------------------------ GEMM
def _gemm_data(M, N, K, bias, seed=0):
    """The operands of test_gpu_numerics._gemm_check."""
    rng = np.random.default_rng(seed + M + N + K)
    a = rng.standard_normal((M, K), dtype=np.float32)
    b = (rng.standard_normal((N, K), dtype=np.float32) / np.sqrt(K)).astype(np.float32)
    bv = rng.standard_normal(N, dtype=np.float32) if bias else None
    return a, b, bv


def _frag(a, b, bias, out_type, segs):
    from code_intelligence_b200 import _lib
    (M, K), N = a.shape, b.shape[0]
    got = np.empty((M, N), dtype=np.float32)
    _lib.check(_lib.load().ie_debug_gemm_frag(a.ctypes.data, b.ctypes.data, bias.ctypes.data, M, N, K, out_type, segs,
                                              got.ctypes.data, 0))
    return got


@pytest.mark.parametrize("segs", [1, 3])
@pytest.mark.parametrize("out,act", EPILOGUES)
@pytest.mark.parametrize("M,N,K,bias", [(129, 600, 1600, True), (1, 600, 2400, False), (129, 600, 2400, True)])
def test_gemm_epilogue_bit_exact(M, N, K, bias, out, act, segs):
    """Every store type, activation and operand form at the shapes of test_gemm_epilogues_per_element."""
    from code_intelligence_b200 import _lib
    t0 = time.perf_counter()
    a, b, bv = _gemm_data(M, N, K, bias)
    want = D.gemm_exact(a, b, bv, act, out, segs, device_gates, _cuda())
    d = _lib._debug_gemm(a, b, bv, act, OUT_TYPES[out], segs)
    bad = int(_mismatch(d, want).sum())
    _report("gemm", M=M, N=N, K=K, act=act, out=out, segs=segs, elements=want.numel(), mismatches=bad,
            wall_s=round(time.perf_counter() - t0, 2))
    assert bad == 0


def _sample_rows(M, n, seed):
    """n random rows, the first and last row of every 128-row m-block among them, and the last m-block's rows."""
    rng = np.random.default_rng(seed)
    r = rng.choice(M, n, replace=False)
    return np.unique(np.concatenate([r, r // 128 * 128, np.minimum(M - 1, r // 128 * 128 + 127), [M - 128, M - 1]]))


@pytest.mark.parametrize("out,segs", [("fp16", 1), ("f32", 3)])
@pytest.mark.parametrize("shape", ["gx", "table"])
def test_gemm_production_shapes_row_sample(shape, out, segs):
    """The middle layers' input projection (M = 128 x 37, N = 9728, K = 2432) and the layer-0 per-token table (M = 60160,
    N = 3328, K = 832) at R4, the default fp16 and the fp32 mode's f32 Gx, natural and fragment-ordered store (the
    recurrent kernel's Gx layout; it needs N % 256 == 0): every column of a row sample."""
    t0 = time.perf_counter()
    M, N, K = (128 * 37, 4 * 2432, 2432) if shape == "gx" else (60160, 4 * 832, 832)
    a, b, bv = _gemm_data(M, N, K, True)
    rows = _sample_rows(M, 12, seed=M)
    want = D.gemm_exact(a[rows], b, bv, 0, out, segs, device_gates, _cuda())
    from code_intelligence_b200 import _lib
    nat = _lib._debug_gemm(a, b, bv, 0, OUT_TYPES[out], segs)[rows]
    frag = _frag(a, b, bv, OUT_TYPES[out], segs)[rows]
    bad = int(_mismatch(nat, want).sum()) + int(_mismatch(frag, want).sum())
    _report("gemm_rows", shape=shape, out=out, segs=segs, rows=len(rows), elements=2 * want.numel(), mismatches=bad,
            wall_s=round(time.perf_counter() - t0, 2))
    assert bad == 0


# ------------------------------------------------------------------------------------------------ label head
def _head_check(probs, X, coefs, intercepts, tag):
    want = D.mlp_head_exact(X, coefs, intercepts, device_gates, _cuda())
    bad = int(_mismatch(torch.as_tensor(np.asarray(probs)), want).sum())
    _report("mlp_head", case=tag, elements=want.numel(), mismatches=bad)
    assert bad == 0, tag


@pytest.mark.parametrize("d_in", [2400, 1600])
@pytest.mark.parametrize("n_labels", [1, 17, 600])
def test_mlp_head_bit_exact(d_in, n_labels):
    """The shapes and inputs of test_mlp_head_per_element."""
    from code_intelligence_b200.mlp import MLPHead
    dims = [d_in, 600, 600, n_labels]
    coefs, intercepts, _ = N.seeded_mlp(d_in + n_labels, dims, 1)
    head = MLPHead(coefs, intercepts)
    rng = np.random.default_rng(n_labels)
    for n in (1, 127, 129):
        X = (rng.standard_normal((n, d_in)) * 0.5).astype(np.float32)
        _head_check(head.predict_proba(X), X, coefs, intercepts, f"{d_in}-600-600-{n_labels} n={n}")
    head.close()


@pytest.mark.parametrize("d_in,hidden,n_labels", GRID_CASES)
def test_mlp_head_grid_search_shapes_bit_exact(d_in, hidden, n_labels):
    """test_mlp_head_grid_search_shapes' heads and inputs (the padding cases of ie_mlp_create), host and device-pointer
    calls."""
    dims = [d_in, *hidden, n_labels]
    head, coefs, intercepts = _head(dims, sum(dims))
    rng = np.random.default_rng(len(dims) + n_labels)
    for n in (1, 129, 300):
        X = (rng.standard_normal((n, d_in)) * 0.5).astype(np.float32)
        _head_check(head.predict_proba(X), X, coefs, intercepts, f"{dims} n={n} host")
        got = head.predict_proba_device(torch.from_numpy(X).to(_cuda()))
        torch.cuda.synchronize()
        _head_check(got.cpu().numpy(), X, coefs, intercepts, f"{dims} n={n} device")
    head.close()


def test_mlp_head_device_pointers_multi_pass_bit_exact(monkeypatch):
    """Passes of 256 rows (IE_MLP_CHUNK), 700 rows, direct (n_labels 16) and staged (17) stores, as
    test_mlp_head_device_pointers_multi_pass runs them."""
    from code_intelligence_b200.mlp import MLPHead
    monkeypatch.setenv("IE_MLP_CHUNK", "256")
    rng = np.random.default_rng(3)
    for n_labels in (16, 17):
        coefs, intercepts, _ = N.seeded_mlp(40 + n_labels, [2400, 600, 600, n_labels], 1)
        head = MLPHead(coefs, intercepts)
        X = (rng.standard_normal((700, 2400)) * 0.5).astype(np.float32)
        got = head.predict_proba_device(torch.from_numpy(X).to(_cuda()))
        torch.cuda.synchronize()
        _head_check(got.cpu().numpy(), X, coefs, intercepts, f"device pointers n_labels={n_labels}")
        head.close()


def test_mlp_head_production_fixture_bit_exact(golden_dir):
    import os
    from code_intelligence_b200.mlp import MLPHead
    coefs, intercepts, X, _ = N.load_mlp_fixture(os.path.join(golden_dir, "mlp_ref_prod.npz"))
    head = MLPHead(coefs, intercepts)
    probs = head.predict_proba(X)
    head.close()
    _head_check(probs, X, coefs, intercepts, "mlp_ref_prod")


# ------------------------------------------------------------------------------------------------ encoder
def item_rows(B):
    """The first and last row of every 128-row half of every 256-row batch (item_of's rows), clipped to B."""
    rows = set()
    for g in range(0, B, D.BATCH_ROWS):
        for h0 in (g, g + D.ITEM_ROWS):
            if h0 < B:
                rows.update((h0, min(B, h0 + D.ITEM_ROWS) - 1))
    return sorted(rows)


def item_units(H):
    """Four units of every 64-unit column tile: its first, two inside and its last real unit."""
    units = set()
    for j0 in range(0, H, D.ITEM_UNITS):
        last = min(H, j0 + D.ITEM_UNITS) - 1
        units.update(u for u in (j0, j0 + 21, j0 + 42, last) if u <= last)
    return sorted(units)


def _states(enc, n_layers, ids, poison=None, len_dev=None):
    """Every layer's states from the device-pointer hook; with `poison`, a production encode of other ids before each
    call, so that stale buffers hold wrong values."""
    out = []
    for l in range(n_layers):
        if poison is not None:
            enc.encode_ids_device(poison, len_dev)
        out.append(enc._debug_layer_states(l, ids))
        enc.check_errors()
    return out


def _exact_layers(emb, layers, ids, states, modes, rows=None, sample_units=False, tag=""):
    """teacher_forced_exact of every layer against the device states -> (elements, mismatches per layer)."""
    t0 = time.perf_counter()
    counts, bad = 0, []
    for l, (w, mode) in enumerate(zip(layers, modes)):
        H = states[l].shape[2]
        units = item_units(H) if sample_units else None
        x, kw = (emb, {"ids": ids}) if l == 0 else (states[l - 1], {})
        h, _ = D.teacher_forced_exact(x, states[l], w, mode, rows, units, device_gates, **kw)
        got = states[l][torch.as_tensor(rows, device=states[l].device)] if rows is not None else states[l]
        if units is not None:
            got = got[:, :, units]
        m = _mismatch(got, h)
        bad.append(int(m.sum()))
        counts += h.numel()
        if bad[-1]:
            r, t, u = (int(v[0]) for v in torch.nonzero(m, as_tuple=True))
            print(f"layer {l}: first mismatch at row {r} t {t} unit {u}: device {float(got[r, t, u])!r} "
                  f"exact {float(h[r, t, u])!r}", flush=True)
    _report("encoder", config=tag, elements=counts, mismatches=bad, wall_s=round(time.perf_counter() - t0, 1))
    return counts, bad


def _controls(emb, layers, ids, states, modes, rows, tag):
    """Every Mode mutant of test_gpu_numerics and every order mutant that applies to a layer of this model must
    disagree with the device (on `rows`, every unit)."""
    n, width = len(layers), states[0].shape[2]
    names = list(MUTANTS) + ["stale_c_at", "stale_h_at", "carry_lost_at"] + list(D.ORDER_MUTANTS)
    T = states[0].shape[1]
    agree = []
    for name in names:
        for l in range(n):
            mode = modes[l]
            if name in MUTANTS:
                mut = _mutate(mode, l, name, n, width)
            elif name == "stale_c_at":
                mut = replace(mode, stale_c_at=(T // 2, (0, 1)))
            elif name == "stale_h_at":
                mut = replace(mode, stale_h_at=(T // 2, (0, 1)))
            elif name == "carry_lost_at":
                mut = replace(mode, carry_lost_at=T // 2)
            else:
                applies = {"interleaved": mode.segs == 3, "bias_early": mode.gx == "fused",
                           "gx_init": mode.gx != "fused", "gx_rz": mode.gx == "fp16"}.get(name, True)
                mut = replace(mode, order=name) if applies else mode
            if mut == mode:
                continue
            x, kw = (emb, {"ids": ids}) if l == 0 else (states[l - 1], {})
            h, _ = D.teacher_forced_exact(x, states[l], layers[l], mut, rows, None, device_gates, **kw)
            if not _mismatch(states[l][torch.as_tensor(rows, device=states[l].device)], h).any():
                agree.append((name, l))
    _report("controls", config=tag, mutants=names, agreeing=agree)
    assert not agree, (tag, agree)


@pytest.mark.parametrize("tag", list(SMALL_CONFIGS))
def test_small_model_every_element(tag, monkeypatch):
    """test_recurrent_kernel_teacher_forced_small's model, ids and knobs: B = 700, T = 23, every row, step, unit and
    layer bit for bit.  The default and the fp32 mode also run the negative controls."""
    env, flags, _ = SMALL_CONFIGS[tag]
    emb, layers = R.make_encoder(7, SMALL[3], SMALL[1], SMALL[2], SMALL[0], scale=2.0).export_weights()
    enc = _make(SMALL, (emb, layers), monkeypatch, env, flags)
    ids, _ = _pad(R.synthetic_ids(700, 23, seed=11, vocab_sz=SMALL[3], min_len=1), 23)
    states = _states(enc, SMALL[0], torch.from_numpy(ids).to(_cuda()))
    enc.close()
    modes = D.layer_modes(SMALL[0], flags, env)
    _, bad = _exact_layers(emb, layers, ids, states, modes, tag=tag)
    assert not any(bad), (tag, bad)
    if tag in ("default", "IE_CFG_FP32"):
        _controls(emb, layers, ids, states, modes, item_rows(700), tag)


@pytest.mark.parametrize("tag", list(SPACE))
def test_configuration_space(tag, monkeypatch):
    """Every configuration of test_gpu_config_space with its ids (edge tokens, lengths on chunk boundaries): every
    element, or for the three largest shapes every schedule item on its sample of rows and units."""
    shape, scale, B, T, knobs, flags, _ = SPACE[tag]
    n_layers, emb_sz, n_hid, vocab, pad_idx = shape
    _, (emb, layers) = _weights(shape, scale)
    enc = _handle(shape, (emb, layers), monkeypatch, knobs, flags)
    lengths = _lengths(B, T, int(knobs.get("IE_CHUNK_T", 5)), seed=B + T)
    ids, _ = _edge_ids(B, T, vocab, pad_idx, lengths, seed=T)
    states = _states(enc, n_layers, torch.from_numpy(ids).to(_cuda()))
    enc.close()
    modes = D.layer_modes(n_layers, flags, knobs)
    sampled = tag in SAMPLED_SPACE
    _, bad = _exact_layers(emb, layers, ids, states, modes, item_rows(B) if sampled else None, sampled, tag)
    assert not any(bad), (tag, bad)


@pytest.mark.parametrize("tag", list(R4_CONFIGS))
def test_production_shape_items(tag, monkeypatch):
    """test_recurrent_kernel_teacher_forced_production_shape's models and ids (E 800, H 2400, V 60000; B = 300,
    T = 64): every schedule item on its rows and units."""
    n_layers, scale, flags, _ = R4_CONFIGS[tag]
    cfg = (n_layers, 800, 2400, 60000)
    emb, layers = R.make_encoder(1234, n_layers=n_layers, scale=scale).export_weights()
    enc = _make(cfg, (emb, layers), monkeypatch, None, flags)
    ids, _ = _pad(R.synthetic_ids(300, 64, seed=12, min_len=1), 64)
    states = _states(enc, n_layers, torch.from_numpy(ids).to(_cuda()))
    enc.close()
    _, bad = _exact_layers(emb, layers, ids, states, D.layer_modes(n_layers, flags), item_rows(300), True, tag)
    assert not any(bad), (tag, bad)


def test_benchmarked_launch_items(monkeypatch):
    """bench.py's launch: R4 at weight scale 1, B = 1280 (five batches in one launch), T = 512, its first timed ids
    after its warm-up ids, device pointers; every schedule item on its rows and units.  The pooled production call
    equals the pool of the checked states."""
    R4 = (4, 800, 2400, 60000)
    emb, layers = R.make_encoder(1234, n_layers=R4[0], scale=1.0).export_weights()
    ids, poison, lengths = _bench_ids()
    ids, poison = ids.to(_cuda()), poison.to(_cuda())
    len_dev = torch.from_numpy(lengths).to(_cuda())
    enc = _make(R4, (emb, layers), monkeypatch, None, 0)
    assert enc.max_batch == 1280
    states = _states(enc, R4[0], ids, poison, len_dev)
    enc.encode_ids_device(poison, len_dev)
    pooled = enc.encode_ids_device(ids, len_dev).cpu().numpy()
    enc.check_errors()
    enc.close()
    np.testing.assert_array_equal(pooled, D.pool(states[-1].cpu().numpy(), lengths))
    rows = item_rows(1280)
    states = [s[rows] for s in states]   # only the checked rows are held from here on
    _, bad = _exact_layers(emb, layers, ids[rows].cpu().numpy(), states, D.layer_modes(R4[0]), None, True, "bench")
    assert not any(bad), bad


@pytest.mark.parametrize("tag", ["chunk edge", "chunk edge fp32"])
def test_time_chunk_edge_items(tag, monkeypatch):
    """test_gpu_single_batch_numerics' issues across the time chunk (4096 steps at b_pad = 256, 2048 with f32 input
    projections), every row: the cell state is recursed exactly through the chunk boundary."""
    R4 = (4, 800, 2400, 60000)
    B, T, scale, flags, ends, _, _ = ONE_BATCH[tag]
    emb, layers = R.make_encoder(1234, n_layers=R4[0], scale=scale).export_weights()
    lengths = np.asarray(ends, dtype=np.int32)
    ids = _one_batch_ids(11, B, T, lengths, True).to(_cuda())
    poison = _one_batch_ids(12, B, T, lengths, True).to(_cuda())
    enc = _make(R4, (emb, layers), monkeypatch, None, flags)
    states = _states(enc, R4[0], ids, poison, torch.from_numpy(lengths).to(_cuda()))
    enc.close()
    _, bad = _exact_layers(emb, layers, ids.cpu().numpy(), states, D.layer_modes(R4[0], flags), None, True, tag)
    assert not any(bad), (tag, bad)
