"""GPU tests of the kernels' rounding points, per element, against oracle/device_numerics.py (float64 except where the
device rounds).  Where tests/test_gpu_parity.py bounds the whole bf16 error against the fp32 oracle, these check that
the kernels round in the places DESIGN.md section 3 lists and only there:

  a. the GEMM, every epilogue (f32 / bf16 / fp16 store, relu, sigmoid) and operand form (bf16, split-bf16), at the
     production shapes: each rounded output must lie in [RNE(ref - eps), RNE(ref + eps)];
  b. the recurrent kernel, teacher-forced: every layer, step and unit of selected rows (every batch, both 128-row halves)
     predicted from the device's own inputs (ie_debug_layer_states), with max and RMS of |dh| / bound under a cap per
     configuration, and every mutant of the arithmetic rejected by at least 4x a cap (one exception, WEAK_MUTANTS);
  c. pooling, bit for bit;
  d. the MLP head, per element, with the rounding uncertainty of its bf16 hidden layers carried as intervals.
"""
import json
import os
from dataclasses import replace

import numpy as np
import pytest
import torch

from oracle import awd_lstm_ref as R
from oracle import device_numerics as D
from oracle import lstm_numpy as N
from test_gpu_parity import _make, _pad

pytestmark = pytest.mark.gpu

OUT_TYPES = {"f32": 0, "bf16": 1, "fp16": 2}
MUTANTS = ("gx_bf16", "cell_bf16", "stale_c", "swap_fo")
SMALL = (3, 96, 200, 500)


def _cuda():
    return torch.device("cuda", 0)


def _report(kind, **kw):
    print("NUMERICS " + json.dumps(dict(kind=kind, **kw)))


# ------------------------------------------------------------------------------------------------ a. GEMM
EPILOGUES = [("f32", 0), ("f32", 1), ("f32", 2), ("bf16", 0), ("bf16", 1), ("bf16", 2), ("fp16", 0)]


def _gemm_check(M, N, K, act, out, segs, bias=True, seed=0, rows=None):
    from code_intelligence_b200 import _lib
    rng = np.random.default_rng(seed + M + N + K)
    a = rng.standard_normal((M, K), dtype=np.float32)
    b = (rng.standard_normal((N, K), dtype=np.float32) / np.sqrt(K)).astype(np.float32)
    bv = rng.standard_normal(N, dtype=np.float32) if bias else None
    d = _lib._debug_gemm(a, b, bv, act, OUT_TYPES[out], segs)
    if rows is not None:
        a, d = a[rows], d[rows]
    lo, hi, ref = D.gemm_interval(a, b, bv, act, out, segs, device=_cuda())
    dd = torch.from_numpy(d).to(_cuda()).double()
    bad = int(((dd < lo) | (dd > hi)).sum())
    # f32 store: how much of the bound is used; 16-bit stores: share of elements whose interval holds two values
    used = float(((dd - ref).abs() / ((hi - lo) / 2).clamp_min(1e-30)).max()) if out == "f32" else None
    _report("gemm", M=M, N=N, K=K, act=act, out=out, segs=segs, bias=bias, outside=bad, max_ratio=used,
            two_valued=float((hi > lo).double().mean()))
    assert np.isfinite(d).all()
    assert bad == 0, (M, N, K, act, out, segs, bad)
    return a, b, bv, lo, hi


@pytest.mark.parametrize("segs", [1, 3])
@pytest.mark.parametrize("out,act", EPILOGUES)
@pytest.mark.parametrize("M,N,K,bias", [(129, 600, 1600, True), (1, 600, 2400, False), (129, 600, 2400, True)])
def test_gemm_epilogues_per_element(M, N, K, bias, out, act, segs):
    """The MLP head's shapes (K = 1600 / 2400, N = 600: not a multiple of the 256-wide tile), M = 1 and 129 (a partial
    second m-block), with and without bias, for every store type, activation and operand form."""
    _gemm_check(M, N, K, act, out, segs, bias)


@pytest.mark.parametrize("out,act,segs", [("fp16", 0, 1), ("f32", 0, 3), ("bf16", 1, 1), ("f32", 2, 1)])
def test_gemm_production_gx_shape(out, act, segs):
    """The middle layers' input projection at R4: N = 4 * 2432 = 9728, K = 2432; M = 128 * 37 m-blocks = two full L2 panels
    of 16 plus a partial one (gemm.cu decode).  fp16 store = the default Gx, f32 with split-bf16 = the fp32-accurate
    mode's Gx.  Negative control: bf16 operands must break the split-bf16 bound on most elements."""
    M, N, K = 128 * 37, 4 * 2432, 2432
    a, b, _, lo, hi = _gemm_check(M, N, K, act, out, segs)
    if segs == 3:
        from code_intelligence_b200 import _lib
        d1 = torch.from_numpy(_lib._debug_gemm(a, b, None, 0, 0, 1)).to(_cuda()).double()
        lo3, hi3, _ = D.gemm_interval(a, b, None, 0, "f32", 3, device=_cuda())
        frac = float(((d1 < lo3) | (d1 > hi3)).double().mean())
        _report("gemm_negative_control", M=M, N=N, K=K, fraction_outside=frac)
        assert frac > 0.5, frac


@pytest.mark.parametrize("out,segs", [("fp16", 1), ("f32", 3)])
def test_gemm_table_shape_row_sample(out, segs):
    """The layer-0 per-token table at R4: N = 4 * 832, K = 832, M = 60160 rows (vocabulary rounded to 256); 2048 random
    rows plus the last m-block are checked."""
    M, N, K = 60160, 4 * 832, 832
    rng = np.random.default_rng(1)
    rows = np.unique(np.concatenate([rng.choice(M, 2048, replace=False), np.arange(M - 128, M)]))
    _gemm_check(M, N, K, 0, out, segs, rows=rows)


# ------------------------------------------------------------------------------------------------ b. recurrent kernel
def _mutate(mode, layer, name, n_layers, width):
    """Mutant `name` of layer `layer`'s arithmetic: stale c on the first min(4, width) units of layer 0 (width = layer 0's
    hidden units), f/o swapped for unit 0 of layer 1 (of layer 0 in a one-layer model)."""
    if name == "gx_bf16":
        return replace(mode, gx="bf16") if mode.gx in ("fp16", "f32") else mode
    if name == "cell_bf16":
        return replace(mode, cell="bf16")
    if name == "stale_c":
        return replace(mode, stale_c=tuple(range(min(4, width)))) if layer == 0 else mode
    if name == "swap_fo":
        return replace(mode, swap_fo=(0,)) if layer == min(1, n_layers - 1) else mode
    return mode


def _rows(B, extra=4, seed=0):
    """Both 128-row halves of every 256-row batch: first and last row of each half, plus a few random rows."""
    rows = set()
    for g in range(0, B, 256):
        for r in (g, g + 127, g + 128, g + 255):
            if r < B:
                rows.add(r)
    rows.add(B - 1)
    rows.update(np.random.default_rng(seed).choice(B, size=min(B, extra), replace=False).tolist())
    return np.array(sorted(rows))


def _teacher_forced_stats(enc, emb, layers, ids, modes, rows):
    """max / RMS of |dh| / bound over every layer, step and unit of `rows`, for the design and for every mutant."""
    n_layers, width = len(layers), np.asarray(layers[0]["w_hh"]).shape[1]
    for name in MUTANTS:   # a mutant that changes no layer's arithmetic would pass as a negative control of nothing
        assert any(_mutate(modes[l], l, name, n_layers, width) != modes[l] for l in range(n_layers)), name
    states = [torch.from_numpy(enc._debug_layer_states(l, ids)[rows]).to(_cuda()) for l in range(n_layers)]
    xs = [torch.from_numpy(emb[ids[rows]]).to(_cuda())] + states[:-1]
    out = {}
    for name in (None,) + MUTANTS:
        st = [D.ratio_stats(states[l], *D.teacher_forced_layer(xs[l], states[l], layers[l],
                                                              _mutate(modes[l], l, name, n_layers, width)))
              for l in range(n_layers)]
        out[name or "design"] = (max(s["max"] for s in st), max(s["rms"] for s in st))
    return out


def _check_caps(tag, stats, max_cap, rms_cap):
    _report("teacher_forced", config=tag, caps=[max_cap, rms_cap], **{k: list(v) for k, v in stats.items()})
    mx, rms = stats["design"]
    assert mx <= max_cap and rms <= rms_cap, (tag, stats["design"], (max_cap, rms_cap))
    for name in MUTANTS:
        m_mx, m_rms = stats[name]
        margin = 1 if (tag, name) in WEAK_MUTANTS else 4
        assert m_mx > margin * max_cap or m_rms > margin * rms_cap, (tag, name, stats[name], (max_cap, rms_cap))


# (knobs, flags) -> (max cap, RMS cap) of |dh| / bound.  Observed on an H100 SXM 80 GB (power limit 400 W), max / RMS:
#   default 0.291 / 0.0065 (same with IE_CHUNK_T=5, IE_MC=1, IE_BATCHES=12: identical bits), IE_FAST_MATH=0 0.979 / 0.080,
#   IE_GX_BF16=0 0.033 / 0.0039, IE_FUSE_LAST=0 and IE_SEQ=0 0.626 / 0.0065, IE_CFG_FP32 0.159 / 0.034.
# Caps are about twice that, never above 1 (the bound itself) and never above 4x the observation.
SMALL_CONFIGS = {
    "default": ({}, 0, (0.6, 0.013)),
    "IE_FAST_MATH=0": ({"IE_FAST_MATH": 0}, 0, (1.0, 0.16)),
    "IE_GX_BF16=0": ({"IE_GX_BF16": 0}, 0, (0.07, 0.008)),
    "IE_FUSE_LAST=0": ({"IE_FUSE_LAST": 0}, 0, (1.0, 0.013)),
    "IE_SEQ=0": ({"IE_SEQ": 0}, 0, (1.0, 0.013)),
    "IE_CHUNK_T=5": ({"IE_CHUNK_T": 5}, 0, (0.6, 0.013)),
    "IE_MC=1": ({"IE_MC": 1}, 0, (0.6, 0.013)),
    "IE_BATCHES=12": ({"IE_BATCHES": 12}, 0, (0.6, 0.013)),
    "IE_CFG_FP32": ({}, 2, (0.32, 0.067)),
}

@pytest.mark.parametrize("tag", list(SMALL_CONFIGS))
def test_recurrent_kernel_teacher_forced_small(tag, monkeypatch):
    """(3, 96, 200, 500) at weight scale 2, B = 700 (three 256-row batches), T = 23, under every knob that changes a
    schedule or a rounding point."""
    env, flags, (max_cap, rms_cap) = SMALL_CONFIGS[tag]
    ref = R.make_encoder(7, SMALL[3], SMALL[1], SMALL[2], SMALL[0], scale=2.0)
    emb, layers = ref.export_weights()
    enc = _make(SMALL, (emb, layers), monkeypatch, env, flags)
    ids, _ = _pad(R.synthetic_ids(700, 23, seed=11, vocab_sz=SMALL[3], min_len=1), 23)
    stats = _teacher_forced_stats(enc, emb, layers, ids, D.layer_modes(SMALL[0], flags, env), _rows(700))
    enc.close()
    _check_caps(tag, stats, max_cap, rms_cap)


# Observed (H100 SXM, 400 W), max / RMS: R4 scale 1 0.950 / 0.018, scale 2 0.946 / 0.022, fp32 mode scale 1 0.604 / 0.113,
# scale 2 0.679 / 0.137, N3 0.941 / 0.017.
R4_CONFIGS = {
    "R4 scale 1": (4, 1.0, 0, (1.0, 0.036)),
    "R4 scale 2": (4, 2.0, 0, (1.0, 0.044)),
    "R4 scale 1 fp32": (4, 1.0, 2, (1.0, 0.23)),
    "R4 scale 2 fp32": (4, 2.0, 2, (1.0, 0.28)),
    "N3": (3, 1.0, 0, (1.0, 0.035)),
}
# Mutants that break the caps by less than 4x.  At torch's default init (scale 1) f and o of a unit are both close to
# sigmoid(0) = 0.5, so exchanging them for one unit moves h little: max ratio 3.46, RMS 0.026 (it still exceeds the max
# cap 1.0).  At scale 2 the same mutant reaches 15.
WEAK_MUTANTS = {("R4 scale 1", "swap_fo")}

@pytest.mark.parametrize("tag", list(R4_CONFIGS))
def test_recurrent_kernel_teacher_forced_production_shape(tag, monkeypatch):
    """The deployed shape (E = 800, H = 2400, V = 60000; 4 layers, and the 3-layer north-star shape), B = 300 (two
    batches), T = 64, in the default and the fp32-accurate mode."""
    n_layers, scale, flags, (max_cap, rms_cap) = R4_CONFIGS[tag]
    cfg = (n_layers, 800, 2400, 60000)
    emb, layers = R.make_encoder(1234, n_layers=n_layers, scale=scale).export_weights()
    enc = _make(cfg, (emb, layers), monkeypatch, None, flags)
    ids, _ = _pad(R.synthetic_ids(300, 64, seed=12, min_len=1), 64)
    stats = _teacher_forced_stats(enc, emb, layers, ids, D.layer_modes(n_layers, flags), _rows(300, extra=3))
    enc.close()
    _check_caps(tag, stats, max_cap, rms_cap)


@pytest.mark.parametrize("env,flags", [({}, 0), ({"IE_SEQ": 0, "IE_CHUNK_T": 4}, 0), ({"IE_MC": 1}, 0), ({}, 2)])
def test_layer_state_hook_changes_nothing(env, flags, monkeypatch):
    """The last layer's states from the hook are raw_features bit for bit, and encode outputs are the same before and
    after a hook call on any layer."""
    emb, layers = R.make_encoder(7, SMALL[3], SMALL[1], SMALL[2], SMALL[0], scale=2.0).export_weights()
    enc = _make(SMALL, (emb, layers), monkeypatch, env, flags)
    ids, lengths = _pad(R.synthetic_ids(300, 13, seed=4, vocab_sz=SMALL[3], min_len=1), 13)
    before = enc.encode_ids(ids, lengths)
    np.testing.assert_array_equal(enc._debug_layer_states(SMALL[0] - 1, ids), enc.raw_features(ids))
    for l in range(SMALL[0]):
        st = enc._debug_layer_states(l, ids)
        assert st.shape == (300, 13, SMALL[2] if l < SMALL[0] - 1 else SMALL[1]) and np.isfinite(st).all()
        np.testing.assert_array_equal(enc.encode_ids(ids, lengths), before)
    with pytest.raises(ValueError):
        enc._debug_layer_states(SMALL[0], ids)
    enc.close()


# ------------------------------------------------------------------------------------------------ c. pooling
@pytest.mark.parametrize("env,flags", [({}, 0), ({"IE_CHUNK_T": 5}, 0), ({"IE_SEQ": 0, "IE_CHUNK_T": 5}, 0), ({}, 2)])
def test_pooling_bit_exact(env, flags, monkeypatch):
    """[mean | max | last] equals device_numerics.pool of the last layer's device states bit for bit: max and last are
    exact, the mean is the sequential f32 sum times f32(1/len).  Lengths end on a time-chunk boundary (5, 10, 15, 20
    with IE_CHUNK_T=5), inside a chunk, at 1 and at T.  Pooling the bf16 ring, or a max that reads one padded step, must
    not match."""
    emb, layers = R.make_encoder(7, SMALL[3], SMALL[1], SMALL[2], SMALL[0], scale=2.0).export_weights()
    enc = _make(SMALL, (emb, layers), monkeypatch, env, flags)
    T = 23
    fixed = [1, 5, 10, 15, 20, 23, 7, 13, 2, 22, 4, 6, 11, 16, 19, 21]
    lens = np.concatenate([fixed, np.random.default_rng(2).integers(1, T + 1, 300 - len(fixed))])
    docs = [d[:n] for d, n in zip(R.synthetic_ids(300, T, seed=21, vocab_sz=SMALL[3]), lens)]
    ids, lengths = _pad(docs, T)
    pooled = enc.encode_ids(ids, lengths)
    states = enc._debug_layer_states(SMALL[0] - 1, ids)
    enc.close()
    want = D.pool(states, lengths)
    E = SMALL[1]
    np.testing.assert_array_equal(pooled[:, E:], want[:, E:])
    np.testing.assert_array_equal(pooled[:, :E], want[:, :E])
    for mutant in ("ring", "max_pad"):
        assert not np.array_equal(pooled, D.pool(states, lengths, mutant)), mutant


# ------------------------------------------------------------------------------------------------ d. MLP head
def _mlp_check(head_probs, X, coefs, intercepts, tag):
    p, lo, hi = D.mlp_head(X, coefs, intercepts, device=_cuda())
    d = torch.as_tensor(np.asarray(head_probs), device=_cuda()).double()
    bad = int(((d < lo) | (d > hi)).sum())
    half = ((hi - lo) / 2).clamp_min(1e-30)
    _report("mlp", case=tag, outside=bad, max_ratio=float(((d - p).abs() / half).max()),
            rms_ratio=float(torch.sqrt((((d - p) / half) ** 2).mean())))
    assert bad == 0, (tag, bad)


@pytest.mark.parametrize("d_in", [2400, 1600])
@pytest.mark.parametrize("n_labels", [1, 17, 600])
def test_mlp_head_per_element(d_in, n_labels):
    from code_intelligence_b200.mlp import MLPHead
    dims = [d_in, 600, 600, n_labels]
    coefs, intercepts, _ = N.seeded_mlp(d_in + n_labels, dims, 1)
    head = MLPHead(coefs, intercepts)
    rng = np.random.default_rng(n_labels)
    for n in (1, 127, 129):
        X = (rng.standard_normal((n, d_in)) * 0.5).astype(np.float32)
        _mlp_check(head.predict_proba(X), X, coefs, intercepts, f"{d_in}-600-600-{n_labels} n={n}")
    head.close()


def test_mlp_head_device_pointers_multi_pass(monkeypatch):
    """Device-pointer mode in passes of 256 rows (IE_MLP_CHUNK), 700 rows, including the direct store into the caller's
    array (n_labels = 16 is a legal store width) and the staged one (n_labels = 17)."""
    from code_intelligence_b200.mlp import MLPHead
    monkeypatch.setenv("IE_MLP_CHUNK", "256")
    rng = np.random.default_rng(3)
    for n_labels in (16, 17):
        coefs, intercepts, _ = N.seeded_mlp(40 + n_labels, [2400, 600, 600, n_labels], 1)
        head = MLPHead(coefs, intercepts)
        X = (rng.standard_normal((700, 2400)) * 0.5).astype(np.float32)
        got = head.predict_proba_device(torch.from_numpy(X).to(_cuda()))
        torch.cuda.synchronize()
        _mlp_check(got.cpu().numpy(), X, coefs, intercepts, f"device pointers n_labels={n_labels}")
        np.testing.assert_array_equal(got.cpu().numpy(), head.predict_proba(X))
        head.close()


def test_mlp_head_production_fixture_per_element(golden_dir):
    """The production-shape fixture the reference's MLPWrapper produced: per element inside the device-precision bound,
    and within 5e-3 of the reference's probabilities as test_gpu_parity checks."""
    from code_intelligence_b200.mlp import MLPHead
    coefs, intercepts, X, want = N.load_mlp_fixture(os.path.join(golden_dir, "mlp_ref_prod.npz"))
    head = MLPHead(coefs, intercepts)
    probs = head.predict_proba(X)
    head.close()
    _mlp_check(probs, X, coefs, intercepts, "mlp_ref_prod")
    assert np.abs(probs - want).max() < 5e-3
