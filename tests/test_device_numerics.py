"""CPU self-tests of oracle/device_numerics.py, the device-precision reference of tests/test_gpu_numerics.py: with every
rounding switched off it is the plain LSTM; the teacher-forced prediction of a free-running float32 emulation of the
device lies inside its own bound; each mutant of the arithmetic breaks that bound on the same data."""
from dataclasses import replace

import numpy as np
import pytest
import torch

from oracle import awd_lstm_ref as R
from oracle import device_numerics as D
from oracle import lstm_numpy as N

CFG = (3, 96, 200, 500)


@pytest.fixture(scope="module")
def small():
    ref = R.make_encoder(7, CFG[3], CFG[1], CFG[2], CFG[0], scale=2.0)
    emb, layers = ref.export_weights()
    ids = np.stack(R.synthetic_ids(32, 33, seed=3, vocab_sz=CFG[3]))
    return emb, layers, ids


# the shape classes of tests/test_gpu_config_space.py: one layer, emb_sz > n_hid, width 1 (vocab 500 rather than the
# smallest model's 3: three tokens give layer 0 three distinct inputs, too few for a per-element statistic)
SHAPES = {"1 layer": (1, 96, 8, 500), "emb > hid": (3, 200, 96, 500), "width 1": (2, 1, 1, 500)}
# Mutants that exceed the bound, but by less than 4x.  At one unit the weights and the bias are O(1) (torch init
# U(+-1/sqrt(H))), so the tanh.approx allowance (2^-11 relative) in the bound is as large as the bf16 rounding of Gx or
# of the cell state: max ratio 1.7-1.8 (gx_bf16) and 3.3 (cell_bf16) with fast gates, against a design max of 0.0001.
WEAK = {("width 1", "gx_bf16", "fast"), ("width 1", "cell_bf16", "fast")}


def _mutant(mode, layer, name, n_layers, width):
    if name == "gx_bf16":
        return replace(mode, gx="bf16") if mode.gx in ("fp16", "f32") else mode
    if name == "cell_bf16":
        return replace(mode, cell="bf16")
    if name == "stale_c":
        return replace(mode, stale_c=tuple(range(min(4, width)))) if layer == 0 else mode
    if name == "swap_fo":
        return replace(mode, swap_fo=(0,)) if layer == min(1, n_layers - 1) else mode
    return mode


def _teacher_forced(emb, layers, ids, states, modes, mutant=None):
    xs = [emb[ids]] + states[:-1]
    n, width = len(layers), layers[0]["w_hh"].shape[1]
    assert mutant is None or any(_mutant(modes[l], l, mutant, n, width) != modes[l] for l in range(n)), mutant
    stats = [D.ratio_stats(states[l], *D.teacher_forced_layer(xs[l], states[l], layers[l],
                                                            _mutant(modes[l], l, mutant, n, width)))
             for l in range(n)]
    return max(s["max"] for s in stats), max(s["rms"] for s in stats)


def test_without_rounding_it_is_the_plain_lstm(small):
    emb, layers, ids = small
    states = D.free_run(emb, layers, ids, [D.EXACT] * len(layers), torch.float64)
    _, want = N.encode(emb, layers, ids, [ids.shape[1]] * len(ids))
    np.testing.assert_allclose(states[-1].numpy(), want, rtol=0, atol=1e-12)
    # teacher forcing on exact data with exact arithmetic predicts it exactly (bound 0)
    pred, bound = D.teacher_forced_layer(emb[ids], states[0], layers[0], D.EXACT)
    np.testing.assert_allclose(pred.numpy(), states[0].numpy(), rtol=0, atol=1e-12)
    assert float(bound.max()) == 0.0


KNOB_SETS = [(0, None), (0, {"IE_FAST_MATH": 0}), (0, {"IE_GX_BF16": 0}), (0, {"IE_FUSE_LAST": 0}), (D.IE_CFG_FP32, None)]


def _emulation_inside_bound_and_mutants_outside(emb, layers, ids, flags, env, tag=None):
    modes = D.layer_modes(len(layers), flags, env)
    states = D.free_run(emb, layers, ids, modes, torch.float32)
    mx, rms = _teacher_forced(emb, layers, ids, states, modes)
    assert mx <= 1.0 and rms <= 0.05, (mx, rms)
    for name in ("gx_bf16", "cell_bf16", "stale_c", "swap_fo"):
        m_mx, m_rms = _teacher_forced(emb, layers, ids, states, modes, name)
        if (tag, name, modes[0].gates) in WEAK:
            assert m_mx > 1.0 and m_mx > 8 * mx, (name, m_mx, mx)
        else:
            assert m_mx > 4.0 or m_rms > 1.0, (name, m_mx, m_rms)


@pytest.mark.parametrize("flags,env", KNOB_SETS)
def test_free_running_emulation_inside_bound_and_mutants_outside(small, flags, env):
    """Observed here (float32 emulation, torch gates): design max ratio 0.43 (default) to 0.98 (IEEE-like gates), every
    mutant's max ratio >= 7.8 and its RMS ratio >= 1.7, i.e. at least 8x beyond the design."""
    _emulation_inside_bound_and_mutants_outside(*small, flags, env)


@pytest.mark.parametrize("tag", list(SHAPES))
@pytest.mark.parametrize("flags,env", KNOB_SETS)
def test_free_running_emulation_at_other_shape_classes(tag, flags, env):
    """The same at one layer, emb > hid and width 1.  Observed: one layer and emb > hid, design max ratio 0.004-0.98,
    every mutant's max >= 6.7 and RMS >= 1.3; width 1, see WEAK."""
    shape = SHAPES[tag]
    ref = R.make_encoder(7, shape[3], shape[1], shape[2], shape[0], scale=2.0)
    emb, layers = ref.export_weights()
    ids = np.stack(R.synthetic_ids(32, 33, seed=3, vocab_sz=shape[3]))
    _emulation_inside_bound_and_mutants_outside(emb, layers, ids, flags, env, tag)


def test_layer_modes_follow_the_knobs():
    assert [m.gx for m in D.layer_modes(4)] == ["fp16", "fp16", "fp16", "fused"]
    assert [m.gx for m in D.layer_modes(4, 0, {"IE_SEQ": 0})] == ["fp16"] * 4
    assert [m.gx for m in D.layer_modes(3, 0, {"IE_GX_BF16": 0})] == ["f32", "f32", "fused"]
    fp32 = D.layer_modes(3, D.IE_CFG_FP32, {"IE_GX_BF16": 1, "IE_FAST_MATH": 1})
    assert all(m.segs == 3 and m.gx == "f32" and m.gates == "ieee" for m in fp32)
    assert D.layer_modes(2, D.IE_CFG_ACCURATE_GATES)[0].gates == "exp"
    # one layer: layer 0 reads the fp16 per-token table and is never fused (the fused layer needs a previous layer's ring)
    assert [m.gx for m in D.layer_modes(1)] == ["fp16"]
    assert [m.gx for m in D.layer_modes(1, 0, {"IE_GX_BF16": 0})] == ["f32"]
    assert [(m.segs, m.gx) for m in D.layer_modes(1, D.IE_CFG_FP32)] == [(3, "f32")]
    assert [m.gx for m in D.layer_modes(2)] == ["fp16", "fused"]


def _small_layer(n_rows, T):
    """Layer 0 of the small model (96 -> 200 units: four column tiles, the last one partial) on n_rows rows, states
    from the float32 emulation."""
    emb, layers = R.make_encoder(7, CFG[3], CFG[1], CFG[2], CFG[0], scale=2.0).export_weights()
    ids = np.stack(R.synthetic_ids(n_rows, T, seed=5, vocab_sz=CFG[3]))
    x = torch.from_numpy(emb[ids])
    h = D.free_run_layer(x, layers[0], D.Mode(), torch.float32)
    return x, h, layers[0]


def test_blocked_statistics_equal_the_unblocked_ones():
    """300 rows (two batches, the second one ending inside its first row half) in blocks of 48 rows, which straddle the
    row-half boundaries at 128 and 256."""
    x, h, w = _small_layer(300, 7)
    pred, bound = D.teacher_forced_layer(x, h, w, D.Mode())
    r = ((h - pred).abs() / bound.clamp_min(1e-30))
    want = D.ratio_stats(h, pred, bound)
    got = D.blocked_layer_stats(x, h, w, D.Mode(), block=48)
    assert got["max"] == pytest.approx(want["max"], rel=1e-12) and got["rms"] == pytest.approx(want["rms"], rel=1e-12)
    assert got["n"] == r.numel() and got["above_half"] == int((r > 0.5).sum())
    assert got["argmax"] == tuple(int(v) for v in np.unravel_index(int(r.argmax()), r.shape))
    items = got["items"]
    assert items.shape == (7, 2, 2, 4)
    for g, half, j in np.ndindex(2, 2, 4):
        rows = r[g * 256 + half * 128:min(300, g * 256 + half * 128 + 128), :, j * 64:(j + 1) * 64]
        want_item = rows.amax((0, 2)) if rows.shape[0] else torch.zeros(7, dtype=torch.float64)
        torch.testing.assert_close(items[:, g, half, j], want_item, rtol=1e-12, atol=0)
    # a row range: the statistics of rows 128..255 only, and nothing outside them
    sub = D.blocked_layer_stats(x, h, w, D.Mode(), rows=range(128, 256), block=32)
    assert sub["max"] == pytest.approx(float(r[128:256].max()), rel=1e-12)
    assert sub["n"] == r[128:256].numel()
    assert float(sub["items"][:, 0, 0].max()) == 0 and float(sub["items"][:, 1].max()) == 0
    assert D.item_of(299, 199) == (1, 0, 3) and D.item_of(127, 64) == (0, 0, 1) and D.item_of(128, 63) == (0, 1, 0)


@pytest.mark.parametrize("name", ["stale_c_at", "stale_h_at", "carry_lost_at"])
def test_item_local_mutants_change_exactly_the_elements_they_name(name):
    """A mutant confined to (step t, units of one tile) changes the prediction of those units from step t on (the cell
    state carries the wrong value forward) and of nothing else; a lost carry at t0 changes every unit from t0 on.  Each
    also breaks the bound there."""
    x, h, w = _small_layer(40, 9)
    t, units = 4, tuple(range(64, 128))
    mutant = {"stale_c_at": D.Mode(stale_c_at=(t, units)), "stale_h_at": D.Mode(stale_h_at=(t, units)),
              "carry_lost_at": D.Mode(carry_lost_at=t)}[name]
    pred, bound = D.teacher_forced_layer(x, h, w, D.Mode())
    pred_m, bound_m = D.teacher_forced_layer(x, h, w, mutant)
    want = torch.zeros_like(pred, dtype=torch.bool)
    want[:, t:, :] = True
    if name != "carry_lost_at":
        want[:, :, :64] = want[:, :, 128:] = False
    assert torch.equal(pred_m != pred, want)
    ratio = (h - pred_m).abs() / bound_m
    assert float(ratio[:, t].max()) > 4 * float(((h - pred).abs() / bound).max())


def test_pool_restates_the_kernel_and_mutants_differ():
    rng = np.random.default_rng(0)
    h = (rng.standard_normal((6, 9, 5)) * 0.3).astype(np.float32)
    lengths = np.array([1, 4, 5, 9, 2, 7])
    got = D.pool(h, lengths)
    for b, n in enumerate(lengths):
        s = h[b, 0].copy()
        for t in range(1, n):
            s = (s + h[b, t]).astype(np.float32)
        np.testing.assert_array_equal(got[b, :5], s * (np.float32(1) / np.float32(n)))
        np.testing.assert_array_equal(got[b, 5:10], h[b, :n].max(0))
        np.testing.assert_array_equal(got[b, 10:], h[b, n - 1])
    assert not np.array_equal(D.pool(h, lengths, "ring"), got)
    assert not np.array_equal(D.pool(h, lengths, "max_pad"), got)


def test_gemm_interval_and_mlp_head_contain_float32_emulations():
    rng = np.random.default_rng(1)
    a = rng.standard_normal((40, 300)).astype(np.float32)
    b = (rng.standard_normal((24, 300)) / np.sqrt(300)).astype(np.float32)
    bias = rng.standard_normal(24).astype(np.float32)
    ab, bb = (torch.from_numpy(v).bfloat16().float() for v in (a, b))
    z32 = ab @ bb.T + torch.from_numpy(bias)
    for act, out, f in ((0, "fp16", lambda z: z.half()), (1, "bf16", lambda z: z.clamp_min(0).bfloat16()),
                        (2, "f32", torch.sigmoid)):
        lo, hi, _ = D.gemm_interval(a, b, bias, act, out, 1)
        d = f(z32).double()
        assert bool(((d >= lo) & (d <= hi)).all()), (act, out)
    lo3, hi3, _ = D.gemm_interval(a, b, None, 0, "f32", 3)
    d1 = (ab @ bb.T).double()                      # bf16 operands break the split-bf16 bound on most elements
    assert float(((d1 < lo3) | (d1 > hi3)).double().mean()) > 0.5
    coefs = [rng.uniform(-0.1, 0.1, (300, 64)).astype(np.float32), rng.uniform(-0.2, 0.2, (64, 7)).astype(np.float32)]
    ints = [rng.uniform(-0.1, 0.1, 64).astype(np.float32), rng.uniform(-1, 0, 7).astype(np.float32)]
    x = torch.from_numpy(a).bfloat16().float()
    hdn = (x @ torch.from_numpy(coefs[0]).bfloat16().float() + torch.from_numpy(ints[0])).clamp_min(0).bfloat16().float()
    p32 = torch.sigmoid(hdn @ torch.from_numpy(coefs[1]).bfloat16().float() + torch.from_numpy(ints[1])).double()
    _, lo, hi = D.mlp_head(a, coefs, ints)
    assert bool(((p32 >= lo) & (p32 <= hi)).all())
    np.testing.assert_allclose(D.mlp_head(a, coefs, ints)[0].numpy(), N.mlp_forward(a, coefs, ints), atol=5e-3)


def test_cell_bound_covers_either_contraction():
    """The compiler may fuse either product of c = f c_prev + i g (commit history: it chose differently once the IEEE
    path was compiled alone), and the test hook's instance may fuse differently from the kernel's.  With the f32 gate
    values taken as exact inputs (no gate error to absorb anything), the cell's own rounding terms must cover float32
    emulations of all three forms: fma on f c_prev (i g rounded), fma on i g (f c_prev rounded), both rounded."""
    z, cp = D.cell_grid()
    d = lambda v: v.double()   # noqa: E731
    i, f, o, g = (fn(d(torch.from_numpy(v))).float() for fn, v in ((torch.sigmoid, z[0]), (torch.sigmoid, z[1]),
                                                                    (torch.sigmoid, z[3]), (torch.tanh, z[2])))
    c32 = torch.from_numpy(cp)
    forms = {"fma f*c": (d(f) * d(c32) + d(i * g)).float(), "fma i*g": (d(f * c32) + d(i) * d(g)).float(),
             "rounded": f * c32 + i * g}
    ig = d(i) * d(g)
    zero = torch.zeros_like(ig)
    c_ref, ec = D._cell_update(ig, D.U24 * ig.abs() + D.TINY, d(f), zero, d(c32), zero, True)
    h_ref, eh = D._cell_out(c_ref, ec, d(o), zero, "exact", True)
    worst = 0.0
    for name, c in forms.items():
        h = (d(o) * torch.tanh(d(c))).float()   # the tanh exact, one rounding of the product
        rc = float(((d(c) - c_ref).abs() / ec).max())
        rh = float(((d(h) - h_ref).abs() / eh).max())
        assert rc <= 1 and rh <= 1, (name, rc, rh)
        worst = max(worst, rc)
    assert worst > 0.5   # the rounding terms are needed: the check is not slack
