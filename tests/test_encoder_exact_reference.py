"""CPU self-tests of the exact restatement the GPU file tests/test_gpu_encoder_exact.py holds the device to:

  * tc_accum.chain_exact (the vectorised chain) gives emulate's bits on every probe family and on random chains, with
    and without a starting accumulator, in bf16 and split-bf16;
  * with correctly rounded stand-ins for the gate functions, the exact GEMM, layer and label head lie inside the bounds
    of gemm_interval, teacher_forced_layer and mlp_head (the restatement is one of the roundings those bounds allow);
  * every order mutant (device_numerics.ORDER_MUTANTS) changes output bits, so that the GPU file's negative controls
    test something.
"""
from dataclasses import replace

import numpy as np
import pytest
import torch

from oracle import awd_lstm_ref as R
from oracle import device_numerics as D
from oracle import lstm_numpy as N
from oracle import tc_accum as T


def _bits_equal(got, want):
    g, w = np.asarray(got, np.float32), np.asarray(want, np.float32)
    return bool(((g.view(np.uint32) == w.view(np.uint32)) | ((g == 0) & (w == 0))).all())


def _diag_chain(a, b, p0=None):
    """chain_exact of row e of a with row e of b, for every e."""
    ta, tb = torch.from_numpy(a).double(), torch.from_numpy(b).double()
    if (b == b[:1]).all():
        return T.chain_exact([(ta, tb[:1])], None if p0 is None else p0[:, None])[:, 0]
    return torch.stack([T.chain_exact([(ta[e:e + 1], tb[e:e + 1])], None if p0 is None else p0[e:e + 1, None])[0, 0]
                        for e in range(len(a))])


@pytest.mark.parametrize("family", list(T.probes()))
def test_chain_exact_equals_emulate_on_every_probe(family):
    a, b = T.probes()[family]
    assert _bits_equal(_diag_chain(a, b), T.emulate(a, b)), family


@pytest.mark.parametrize("K,segs", [(200, 1), (832, 1), (300, 3), (77, 3)])
def test_chain_exact_equals_emulate_on_random_chains(K, segs):
    rng = np.random.default_rng(K + segs)
    a = (rng.standard_normal((24, K)) * 2.0 ** rng.integers(-8, 8, (24, 1))).astype(np.float32)
    b = rng.standard_normal((20, K)).astype(np.float32)
    if segs == 1:
        a, b = T.bf16_exact(a), T.bf16_exact(b)
    ta, tb = torch.from_numpy(a).double(), torch.from_numpy(b).double()
    got = T.chain_exact(D.passes(D.operands(ta, segs), D.operands(tb, segs), segs))
    idx = np.arange(24) % 20
    assert _bits_equal(got[np.arange(24), idx], T.emulate(a, b[idx], segs))
    # chunking and the [M, N] layout change nothing
    assert torch.equal(got, T.chain_exact(D.passes(D.operands(ta, segs), D.operands(tb, segs), segs), chunk=7))


def test_chain_exact_starting_value():
    """A starting accumulator is the state after earlier steps: chain(p0 = chain(x1, w1)) = chain([x1 | x], [w1 | w])
    for K1 a multiple of 16; and a p0 that one product forms exactly equals emulate with that product as step 0."""
    rng = np.random.default_rng(3)
    x1, w1 = T.bf16_exact(rng.standard_normal((16, 48))), T.bf16_exact(rng.standard_normal((12, 48)))
    x, w = T.bf16_exact(rng.standard_normal((16, 100))), T.bf16_exact(rng.standard_normal((12, 100)))
    t = lambda v: torch.from_numpy(v).double()
    p0 = T.chain_exact([(t(x1), t(w1))])
    assert torch.equal(T.chain_exact([(t(x), t(w))], p0),
                       T.chain_exact([(t(np.hstack([x1, x])), t(np.hstack([w1, w])))]))
    assert torch.equal(T.chain_exact([(t(x), t(w))], p0), T.chain_exact([(t(x1), t(w1)), (t(x), t(w))]))
    u, v = T.bf16_exact(rng.standard_normal(16) * 4), T.bf16_exact(rng.standard_normal(16))
    a = np.zeros((16, 116), np.float32)
    a[:, 0], a[:, 16:] = u, x
    b = np.zeros((16, 116), np.float32)
    b[:, 0], b[:, 16:] = v, w[0]
    got = T.chain_exact([(t(x), t(w[:1]))], t((u.astype(np.float64) * v)[:, None]))[:, 0]
    assert _bits_equal(got, T.emulate(a, b))


# ------------------------------------------------------------------------------------------------ inside the bounds
@pytest.mark.parametrize("segs", [1, 3])
@pytest.mark.parametrize("out,act", [("f32", 0), ("f32", 1), ("f32", 2), ("bf16", 0), ("bf16", 1), ("fp16", 0)])
def test_gemm_exact_inside_gemm_interval(out, act, segs):
    rng = np.random.default_rng(act + 7 * segs)
    a = rng.standard_normal((33, 200)).astype(np.float32)
    b = (rng.standard_normal((40, 200)) / 14).astype(np.float32)
    bias = rng.standard_normal(40).astype(np.float32)
    z = D.gemm_exact(a, b, bias, act, out, segs)
    lo, hi, _ = D.gemm_interval(a, b, bias, act, out, segs)
    assert bool(((z >= lo) & (z <= hi)).all())


def _free_run_exact(x, layer, mode, ids=None, gates=D.rounded_gates):
    """States of one layer that its exact restatement reproduces: h_t is teacher_forced_exact's prediction from
    h_0 .. h_{t-1} (the device's arithmetic run free)."""
    Rn, Tn = ids.shape if ids is not None else x.shape[:2]
    h = torch.zeros(Rn, Tn, np.asarray(layer["w_hh"]).shape[1], dtype=torch.float64)
    kw = {} if ids is None else {"ids": ids}
    for t in range(Tn):
        p, _ = D.teacher_forced_exact(x, h, layer, mode, gates=gates, **kw)
        h[:, t] = p[:, t]
    return h


def _small_model(n_hid=80, emb_sz=40):
    emb, layers = R.make_encoder(5, 60, emb_sz, n_hid, 3, scale=2.0).export_weights()
    ids = np.random.default_rng(1).integers(0, 60, (5, 6))
    return emb, layers, ids


@pytest.fixture(scope="module", params=[0, D.IE_CFG_ACCURATE_GATES, D.IE_CFG_FP32, D.IE_CFG_F32_GX])
def exact_states(request):
    """Every layer of a small 3-layer model run free under the exact restatement, per flag set."""
    flags = request.param
    emb, layers, ids = _small_model()
    modes = D.layer_modes(3, flags)
    states = []
    for l in range(3):
        x, kw = (emb, ids) if l == 0 else (states[-1], None)
        states.append(_free_run_exact(x, layers[l], modes[l], kw))
    return flags, emb, layers, ids, modes, states


def test_exact_layer_inside_teacher_forced_bound(exact_states):
    flags, emb, layers, ids, modes, states = exact_states
    for l in range(3):
        x = torch.from_numpy(emb[ids]).double() if l == 0 else states[l - 1]
        pred, bound = D.teacher_forced_layer(x, states[l], layers[l], modes[l])
        r = float(((states[l] - pred).abs() / bound).max())
        assert r <= 1.0, (flags, l, r)
        # the restatement reproduces its own states, also on a subset of rows and units and from gathered rows
        x_exact, kw = (emb, {"ids": ids}) if l == 0 else (states[l - 1], {})
        h, c = D.teacher_forced_exact(x_exact, states[l], layers[l], modes[l], **kw)
        assert torch.equal(h, states[l])
        sub, _ = D.teacher_forced_exact(x_exact, states[l], layers[l], modes[l], rows=[4, 1], units=[7, 0, 3], **kw)
        assert torch.equal(sub, states[l][[4, 1]][:, :, [7, 0, 3]])
        if l == 0:
            full, _ = D.teacher_forced_exact(x, states[l], layers[l], modes[l])
            assert torch.equal(full, h)


@pytest.mark.parametrize("mutant", D.ORDER_MUTANTS)
def test_every_order_mutant_changes_bits(exact_states, mutant):
    flags, emb, layers, ids, modes, states = exact_states
    changed = []
    applies = []
    for l in range(3):
        mode = modes[l]
        ok = {"interleaved": mode.segs == 3, "bias_early": mode.gx == "fused", "gx_init": mode.gx != "fused",
              "gx_rz": mode.gx == "fp16"}.get(mutant, True)
        if not ok:
            continue
        applies.append(l)
        x, kw = (emb, {"ids": ids}) if l == 0 else (states[l - 1], {})
        h, _ = D.teacher_forced_exact(x, states[l], layers[l], replace(mode, order=mutant), **kw)
        changed.append(int((h != states[l]).sum()))
    if not applies:
        pytest.skip(f"{mutant} has no layer to act on under flags {flags}")
    assert all(n > 0 for n in changed), (mutant, flags, changed)


def test_mlp_head_exact_inside_interval():
    dims = [200, 100, 64, 17]
    coefs, intercepts, _ = N.seeded_mlp(9, dims, 1)
    X = (np.random.default_rng(2).standard_normal((40, 200)) * 0.5).astype(np.float32)
    p = D.mlp_head_exact(X, coefs, intercepts)
    _, lo, hi = D.mlp_head(X, coefs, intercepts)
    assert bool(((p >= lo) & (p <= hi)).all())
