"""GPU tests of text generation (csrc/lm_gen.cu and the carried state behind ie_gen_*, LanguageModel.predict /
beam_search): the carried state bit for bit against one zero-state run over the whole history, the top-k and sampling
kernels against exact and float64 references, the beam selection against numpy's stable argsort, predict and
beam_search against fastai's loops restated in torch, and the encoder left as it was."""
import os
import warnings

import numpy as np
import pytest
import torch

from code_intelligence_b200 import _lib
from code_intelligence_b200._lib import IE_CFG_FP32
from code_intelligence_b200.language_model import LanguageModel
from oracle import awd_lstm_ref as R
from oracle import lm_gen_ref as G
from oracle import lm_ref as L

pytestmark = pytest.mark.gpu
MODES = {"bf16": 0, "fp32": IE_CFG_FP32}
SMALL = dict(vocab_sz=500, emb_sz=96, n_hid=200, n_layers=3)
R4 = dict(vocab_sz=60000, emb_sz=800, n_hid=2400, n_layers=4)
U = 2.0 ** -24


def device_lm(ref, flags, env=None, itos=None):
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        return LanguageModel.from_state_dict(ref.fastai_state_dict(), flags=flags, itos=itos)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def ring_bits(h32: np.ndarray, fp32: bool) -> np.ndarray:
    """[..., P, n] uint16: bf16 bits of h (round to nearest even) and, in the fp32-accurate mode, of f32(h - hi)."""
    t = torch.as_tensor(np.ascontiguousarray(h32, dtype=np.float32))
    hi = t.to(torch.bfloat16)
    planes = [hi]
    if fp32:
        planes.append((t - hi.float()).to(torch.bfloat16))
    return torch.stack([p.view(torch.int16) for p in planes], dim=-2).numpy().view(np.uint16)


def check_state(lm, state, hist: np.ndarray, fp32: bool, tag=""):
    """Every layer's exported h equals the ring's rounding of the one-shot f32 state at the history's last step."""
    enc = lm.encoder
    n = hist.shape[0]
    for l in range(enc.n_layers):
        ref = enc._debug_layer_states(l, hist)[:, -1]
        hb, _ = state.export(l, n)
        want = ring_bits(ref, fp32)
        bad = np.argwhere(hb != want)
        assert bad.size == 0, f"{tag} layer {l}: {len(bad)} h elements differ, first {bad[:3].tolist()}"


def feed(lm, state, ids):
    """One step (top 1) on host ids: the state advances by ids' width."""
    return lm.step(state, ids, 1)


# ------------------------------------------------------------------------------------------------ the carried state
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("prompt,rows", [(1, 1), (64, 10), (700, 1)])
def test_carried_state_small(mode, prompt, rows):
    """Prompts of 1, 64 and 700 tokens, then 32 single-token steps and steps of width 5, 1, 17: after every call each
    layer's h equals the ring rounding of a one-shot run over the concatenated ids (a wrong c changes every h after)."""
    ref = L.make_lm(seed=3, dec_scale=4.0, **SMALL)
    lm = device_lm(ref, MODES[mode])
    rng = np.random.default_rng(prompt + rows)
    st = lm.new_state(rows)
    try:
        hist = rng.integers(2, SMALL["vocab_sz"], (rows, prompt))
        feed(lm, st, hist)
        check_state(lm, st, hist, mode == "fp32", "prompt")
        for i, w in enumerate([1] * 32 + [5, 1, 17]):
            x = rng.integers(0, SMALL["vocab_sz"], (rows, w))
            feed(lm, st, x)
            hist = np.concatenate([hist, x], axis=1)
            if i % 8 == 7 or i >= 32:
                check_state(lm, st, hist, mode == "fp32", f"step {i}")
    finally:
        st.close()
        lm.close()


@pytest.mark.parametrize("env", [{"IE_CHUNK_T": "3"}, {"IE_SEQ": "0"}])
def test_carried_state_chunked_and_per_timestep(env):
    ref = L.make_lm(seed=4, dec_scale=4.0, **SMALL)
    for mode, flags in MODES.items():
        lm = device_lm(ref, flags, env)
        rng = np.random.default_rng(5)
        st = lm.new_state(3)
        try:
            hist = rng.integers(2, SMALL["vocab_sz"], (3, 11))
            feed(lm, st, hist)
            for w in (1, 4, 1, 7):
                x = rng.integers(2, SMALL["vocab_sz"], (3, w))
                feed(lm, st, x)
                hist = np.concatenate([hist, x], axis=1)
                check_state(lm, st, hist, mode == "fp32", f"{env} {mode} w={w}")
        finally:
            st.close()
            lm.close()


def test_carried_state_across_the_4096_chunk():
    """A 4100-token prompt on one row crosses the 4096-step chunk of a one-batch launch; then 3 steps."""
    ref = L.make_lm(seed=5, dec_scale=4.0, **SMALL)
    lm = device_lm(ref, 0)
    rng = np.random.default_rng(6)
    st = lm.new_state(1)
    try:
        hist = rng.integers(2, SMALL["vocab_sz"], (1, 4100))
        feed(lm, st, hist)
        check_state(lm, st, hist, False, "4100")
        for _ in range(3):
            x = rng.integers(2, SMALL["vocab_sz"], (1, 1))
            feed(lm, st, x)
            hist = np.concatenate([hist, x], axis=1)
        check_state(lm, st, hist, False, "4100 + 3")
    finally:
        st.close()
        lm.close()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_select_then_continue(mode):
    """select with repeated and permuted rows, then more steps: equal to one-shot runs over the gathered histories."""
    ref = L.make_lm(seed=7, dec_scale=4.0, **SMALL)
    lm = device_lm(ref, MODES[mode])
    rng = np.random.default_rng(8)
    st = lm.new_state(6)
    try:
        hist = rng.integers(2, SMALL["vocab_sz"], (4, 9))
        feed(lm, st, hist)
        parent = np.array([3, 0, 3, 1, 1, 2])
        lm.select(st, parent)
        hist = hist[parent]
        check_state(lm, st, hist, mode == "fp32", "after select")
        for w in (1, 3):
            x = rng.integers(2, SMALL["vocab_sz"], (6, w))
            feed(lm, st, x)
            hist = np.concatenate([hist, x], axis=1)
        check_state(lm, st, hist, mode == "fp32", "continued")
        # a beam row equals a one-row state with the same history, bit for bit
        one = lm.new_state(1)
        try:
            feed(lm, one, hist[2:3])
            for l in range(lm.encoder.n_layers):
                np.testing.assert_array_equal(one.export(l, 1)[0][0], st.export(l, 6)[0][2])
                np.testing.assert_array_equal(one.export(l, 1)[1][0], st.export(l, 6)[1][2])
        finally:
            one.close()
    finally:
        st.close()
        lm.close()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_carried_state_r4(mode):
    """R4 (E 800, 4 x 2400, V 60000): 1000 rows from a 64-token prompt and one step, and 10 rows for 4 more steps."""
    ref = L.make_lm(seed=9, dec_scale=20.0, bias_scale=0.5, **R4)
    lm = device_lm(ref, MODES[mode])
    rng = np.random.default_rng(10)
    try:
        st = lm.new_state(1000)
        hist = rng.integers(2, R4["vocab_sz"], (1000, 64))
        feed(lm, st, hist)
        x = rng.integers(2, R4["vocab_sz"], (1000, 1))
        feed(lm, st, x)
        check_state(lm, st, np.concatenate([hist, x], axis=1), mode == "fp32", "R4 1000 rows")
        st.close()
        st = lm.new_state(10)
        hist = hist[:10]
        feed(lm, st, hist)
        for _ in range(4):
            x = rng.integers(2, R4["vocab_sz"], (10, 1))
            feed(lm, st, x)
            hist = np.concatenate([hist, x], axis=1)
        check_state(lm, st, hist, mode == "fp32", "R4 10 rows")
        st.close()
    finally:
        lm.close()


# ------------------------------------------------------------------------------------------------ top-k
def debug_topk(z, k, exclude=-1):
    z = np.ascontiguousarray(z, dtype=np.float32)
    rows, V = z.shape
    v, i = np.empty((rows, k), np.float32), np.empty((rows, k), np.int64)
    _lib.check(_lib.load().ie_debug_gen_topk(z.ctypes.data, rows, V, k, exclude, v.ctypes.data, i.ctypes.data, 0))
    return v, i


@pytest.mark.parametrize("V", [1, 2, 255, 256, 257, 8191, 8192, 8193, 60000])
def test_topk_exact_ids(V):
    """Small-integer logits (every value exact): ids equal a stable f64 top-k for k in 1, 2, 10, 64 and the excluded id
    at 0, V - 1 and the argmax; tie storms across 256-column tiles in every other row."""
    rng = np.random.default_rng(V)
    rows = 12
    z = rng.integers(-4, 5, (rows, V)).astype(np.float32)
    z[1::2] = np.where(rng.random((rows // 2, V)) < 0.9, 3.0, z[1::2])      # storms of equal maxima
    z[2] = 0.0
    for k in (1, 2, 10, 64):
        if k > V:
            continue
        for ex in sorted({-1, 0, V - 1, int(np.argmax(z[0]))}):
            v, i = debug_topk(z, k, ex)
            zz = torch.as_tensor(z, dtype=torch.float64)
            if ex >= 0:
                zz[:, ex] = -np.inf
            _, want = G.topk_stable(zz, k)
            np.testing.assert_array_equal(i, want.numpy(), err_msg=f"V={V} k={k} exclude={ex}")
            lse = torch.logsumexp(torch.as_tensor(z, dtype=torch.float64), 1, keepdim=True)
            wv = torch.gather(zz, 1, want) - lse
            fin = np.isfinite(wv.numpy())
            assert np.array_equal(fin, np.isfinite(v))
            assert np.all(np.abs(v[fin] - wv.numpy()[fin]) <= 1e-5 * (1 + np.abs(wv.numpy()[fin])))


# ------------------------------------------------------------------------------------------------ sampling
def debug_sample(z, u, exclude=-1, temperature=1.0, min_p=0.0):
    z = np.ascontiguousarray(z, dtype=np.float32)
    u = np.ascontiguousarray(u, dtype=np.float32)
    rows, V = z.shape
    out, fl = np.empty(rows, np.int64), np.empty(rows, np.int32)
    _lib.check(_lib.load().ie_debug_gen_sample(z.ctypes.data, rows, V, u.ctypes.data, exclude, temperature, min_p,
                                               out.ctypes.data, fl.ctypes.data, 0))
    return out, fl


def sample_weights_f64(z, exclude, temperature, min_p):
    p = torch.softmax(torch.as_tensor(z, dtype=torch.float64), -1)
    if exclude >= 0:
        p[..., exclude] = 0
    warned = False
    if min_p:
        if not bool((p >= min_p).any()):
            warned = True
        else:
            p[p < min_p] = 0
    if temperature != 1.0:
        p = p ** (1 / temperature)
    return p.numpy(), warned


SAMPLE_CASES = [("plain", 300), ("no_unk", 300), ("min_p", 300), ("temperature", 300), ("min_p_none", 300),
                ("no_unk", 8193), ("min_p", 8193), ("min_p", 60000)]
EDGES = [31, 32, 63, 1023, 1024, 1025, 2047, 2048, 4095, 4096, 8191, 8192, 59391, 59392]   # warp and chunk edges


@pytest.mark.parametrize("seed,case,V", [(i, c, v) for i, (c, v) in enumerate(SAMPLE_CASES)])
def test_sampling_against_f64_inverse_cdf(seed, case, V):
    """Uniforms (0 and 1 - 2^-24 among them) on one logit row: the chosen index equals the f64 inverse CDF wherever
    u * total lies farther than the bound from the chosen index's CDF boundaries; zero-weight columns never win.  At
    V = 8193 and 60000 the CDF carries across 1024-column chunks, and the excluded or masked columns sit at warp and
    chunk edges."""
    rng = np.random.default_rng(seed)
    zrow = (rng.standard_normal(V) * 2).astype(np.float32)
    edges = [e for e in EDGES if e < V] if V > 300 else []
    zrow[edges] = -40.0
    ex, t, mp = -1, 1.0, 0.0
    if case == "no_unk":
        ex = 1024 if V > 1024 else int(np.argmax(zrow))
    if case == "min_p":
        mp = {300: 0.01, 8193: 2e-5, 60000: 1e-5}[V]
    if case == "temperature":
        t = 0.7
    if case == "min_p_none":
        mp = 0.9
    n = {300: 100000, 8193: 20000, 60000: 2000}[V]
    u = rng.random(n, dtype=np.float32)
    u[0], u[1] = 0.0, np.float32(1 - 2 ** -24)
    z = np.broadcast_to(zrow, (n, V))
    out, fl = debug_sample(z, u, ex, t, mp)
    w, warned = sample_weights_f64(zrow, ex, t, mp)
    assert np.all(fl == (1 if warned else 0))
    assert case != "min_p_none" or warned
    assert case != "min_p" or np.all(w[edges] == 0)
    assert np.all(w[out] > 0), "a zero-weight column was drawn"
    c = np.cumsum(w)
    inv_t = 1 / t
    zm = float(np.max(zrow) - np.min(zrow))
    rel = 2 * (inv_t * (U * zm + (V / 1024 + 16) * U) + (V / 1024 + 16) * U)
    tgt = u.astype(np.float64) * c[-1]
    want = np.minimum(np.searchsorted(c, tgt, side="right"), V - 1)
    lo = np.where(want > 0, c[np.maximum(want - 1, 0)], 0.0)
    clear = np.minimum(tgt - lo, c[want] - tgt) > rel * c[-1]
    assert clear.mean() > (0.99 if V == 300 else 0.5), clear.mean()
    bad = np.flatnonzero(clear & (out != want))
    assert bad.size == 0, f"{bad.size} draws differ, e.g. u={u[bad[:3]]} got {out[bad[:3]]} want {want[bad[:3]]}"
    assert out[0] == np.flatnonzero(w > 0)[0]


def test_zero_weight_columns_never_drawn():
    """The CDF scan is not monotone in rounding: with weights ~(2^-24, 2^-24, 1, 0) a lane's prefix can round one ulp
    above its left neighbour's, so a first-above-target search alone would draw the zero-weight column 3 for u near 1.
    A grid of such rows (the excluded column 3 small, zero or large) with u in {1 - 2^-24, 1 - 2^-23, 0.9999999}: the
    draw is always a column of positive weight."""
    a = np.linspace(-18.0, -15.0, 64, dtype=np.float32)
    rows = [[x, y, 0.0, c] for x in a for y in a for c in (-np.inf, 0.0, 3.0)]
    z = np.asarray(rows, np.float32)
    u = np.resize(np.array([1 - 2 ** -24, 1 - 2 ** -23, 0.9999999], np.float32), len(z))
    out, fl = debug_sample(z, u, exclude=3)
    assert np.all(fl == 0) and np.all(out != 3) and np.all(out >= 0)
    # min_p masks the two small columns: only column 2 can be drawn
    out, _ = debug_sample(z[:, :3].copy(), u, min_p=0.5)
    assert np.all(out == 2)


def test_all_zero_weights_are_reported():
    """A flat row at temperature 1e-3: every p ** 1000 underflows to 0 in f32 (fastai's torch.multinomial raises on
    it).  The kernel reports flag 2; predict raises instead of returning a token."""
    out, fl = debug_sample(np.zeros((3, 300), np.float32), np.array([0.0, 0.5, 0.9], np.float32), temperature=1e-3)
    assert np.all(fl == 2) and np.all(out == 0)
    ref = L.make_lm(seed=17, **SMALL)
    with torch.no_grad():
        ref.decoder.weight.zero_()
        ref.decoder.bias.zero_()
    lm = device_lm(ref, 0)
    try:
        with pytest.raises(ValueError, match="every weight is 0"):
            lm.predict(np.array([2, 10]), 3, temperature=1e-3, seed=0)
        assert len(lm.predict(np.array([2, 10]), 3, temperature=0.5, seed=0)) == 5
    finally:
        lm.close()


# ------------------------------------------------------------------------------------------------ beam selection
@pytest.mark.parametrize("rows,top_k", [(1, 1), (10, 10), (1000, 10), (256, 64), (3, 1), (1025, 1), (5461, 3)])
def test_beam_select_is_a_stable_argsort(rows, top_k):
    """n = rows * top_k candidates from 1 to 16383 (3, 1025 and 16383 pad the bitonic sort, and the padding keys must
    sort last), beam_sz 1, n, n + 1 and 1000, nodes of L = 3 and L = 0 columns; -0 parent scores (-0 - 0 = -0, which
    sorts as +0 and comes back as +0) and a -inf value (a +inf score) among the ties."""
    ref = L.make_lm(seed=1, vocab_sz=300, emb_sz=64, n_hid=64, n_layers=2)
    lm = device_lm(ref, 0)
    st = lm.new_state(1)
    try:
        rng = np.random.default_rng(rows * top_k)
        scores = rng.integers(0, 4, rows).astype(np.float32) * 0.5
        scores[scores == 0] = -0.0
        values = -rng.integers(0, 6, (rows, top_k)).astype(np.float32) * 0.25 + np.float32(0)   # many ties, +0
        values[0, 0] = -np.inf if rows * top_k > 1 else values[0, 0]
        tokens = rng.integers(0, 60000, (rows, top_k))
        n = rows * top_k
        for L_ in (3, 0):
            nodes = rng.integers(0, 60000, (rows, L_))
            for beam_sz in sorted({1, n, n + 1, 1000}):
                parent, token, sc, nn = lm.beam_select(st, scores, values, tokens, beam_sz, nodes if L_ else None)
                cand = (scores[:, None] - values).reshape(-1).astype(np.float32)
                order = np.argsort(cand, kind="stable")[:beam_sz]
                what = f"n={n} beam_sz={beam_sz} L={L_}"
                np.testing.assert_array_equal(parent, order // top_k, err_msg=what)
                np.testing.assert_array_equal(token, tokens.reshape(-1)[order], err_msg=what)
                np.testing.assert_array_equal(sc.view(np.int32), (cand[order] + np.float32(0)).view(np.int32),
                                              err_msg=what)
                np.testing.assert_array_equal(nn, np.concatenate([nodes[order // top_k],
                                                                  tokens.reshape(-1)[order][:, None]], 1), err_msg=what)
        assert n < 1000 or np.any(np.isposinf(cand)) and np.any(np.signbit(cand) & (cand == 0))
    finally:
        st.close()
        lm.close()


# ------------------------------------------------------------------------------------------------ end to end
def test_predict_and_beam_search_small_fp32():
    """Small config in the fp32-accurate mode against fastai's loops in torch with the same uniforms: the same tokens
    up to the first step decided inside the bound (recorded, not failed)."""
    ref = L.make_lm(seed=12, dec_scale=8.0, bias_scale=0.5, **SMALL)
    lm = device_lm(ref, IE_CFG_FP32)
    try:
        prompt = np.array([2] + list(np.random.default_rng(1).integers(5, 500, 20)))
        for kw in (dict(), dict(temperature=0.8), dict(min_p=0.02), dict(no_unk=False)):
            u = np.random.default_rng(7).random(24, dtype=np.float32)
            out = lm.predict(prompt, 24, seed=7, **kw)
            new, gaps, _ = G.predict_literal(ref, prompt, 24, u, unk=0, **kw)
            got = out[len(prompt):]
            tight = np.flatnonzero(gaps < 1e-4)
            upto = tight[0] if tight.size else 24
            np.testing.assert_array_equal(got[:upto], new[:upto], err_msg=str(kw))
            if tight.size:
                print(f"predict {kw}: step {upto} decided inside the bound (gap {gaps[upto]:.3g})")
        u = float(np.random.default_rng(3).random(dtype=np.float32))
        node = lm.beam_search(prompt, 4, top_k=5, beam_sz=50, seed=3)
        want, _, _, margins = G.beam_literal(ref, prompt, 4, u, unk=0, top_k=5, beam_sz=50)
        if min(min(m) for m in margins) > 1e-4:
            np.testing.assert_array_equal(node[1:], want)
        else:
            print("beam_search: a step decided inside the bound", margins)
    finally:
        lm.close()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_r4_decisions_against_f64(mode):
    """R4: predict 32 words from 3 prompts and beam_search with defaults for 4 words; each predict draw, the top-k of
    every step and every beam step are checked against float64 logits of the device's own states (one zero-state run
    over the history)."""
    ref = L.make_lm(seed=13, dec_scale=600.0, bias_scale=0.5, **R4)   # peaked: most draws clear the bound
    lm = device_lm(ref, MODES[mode])
    segs = 3 if mode == "fp32" else 1
    W = ref.decoder.weight.detach().numpy()
    b = ref.decoder.bias.detach().numpy()
    checked = skipped = 0
    try:
        for p, T0 in enumerate((1, 17, 64)):
            prompt = np.concatenate([[2], np.random.default_rng(p).integers(5, 60000, T0 - 1)]).astype(np.int64)
            seq = lm.predict(prompt, 32, seed=p)
            u = np.random.default_rng(p).random(32, dtype=np.float32)
            h = lm.encoder._debug_layer_states(R4["n_layers"] - 1, seq[None, :-1])[0, T0 - 1:]
            z, eps = G.logits_f64(h, W, b, segs, device="cuda")
            for i in range(32):
                w, _ = sample_weights_f64(z[i].cpu().numpy(), 0, 1.0, None)
                j, gap = G.inverse_cdf(w, float(u[i]))
                # a logit error eps moves every weight by a factor exp(+-2 eps)
                if gap > 8 * float(eps[i]) + 1e-5:
                    assert seq[T0 + i] == j, f"prompt {p} step {i}"
                    checked += 1
                else:
                    skipped += 1
            ids, _, ok, bound = G.topk_f64(z, eps, 10, 0)
            st = lm.new_state(1)
            try:
                for i in range(8):
                    v, ix = lm.step(st, seq[None, :T0] if i == 0 else seq[None, T0 + i - 1:T0 + i], 10, 0)
                    okc = bool(ok[i])
                    if okc:
                        np.testing.assert_array_equal(ix[0], ids[i].cpu().numpy())
                    zi = z[i].clone()
                    zi[0] = -np.inf
                    lse = torch.logsumexp(z[i], 0)
                    wv = (zi[torch.as_tensor(ix[0], device=zi.device)] - lse).cpu().numpy()
                    assert np.all(np.abs(v[0] - wv) <= bound[i].cpu().numpy()), f"prompt {p} step {i}"
            finally:
                st.close()
        print(f"R4 {mode}: {checked} draws checked, {skipped} inside the bound")
        assert checked >= 48
        check_beam_r4(lm, W, b, segs, mode)
    finally:
        lm.close()


def check_beam_r4(lm, W, b, segs, mode, top_k=10, beam_sz=1000, n_words=4):
    """beam_search with its defaults for 4 words, step by step through the public step / beam_select / select: every
    step's top-k ids equal the float64 top-k of the device's own states over the gathered histories (one zero-state run
    per beam row) wherever the k-boundary gap clears twice the row's bound, and the values lie within the bound; the
    survivors equal numpy's stable argsort of the device's f32 scores; the chosen node equals beam_search's."""
    prompt = np.array([2, 100, 200, 300], dtype=np.int64)
    st = lm.new_state(beam_sz)
    rows_ok = rows_all = 0
    try:
        nodes = np.tile(prompt, (top_k, 1))
        x, scores = nodes, np.zeros(top_k, np.float32)
        for k in range(n_words):
            v, ix = lm.step(st, x, top_k, 0)
            h = lm.encoder._debug_layer_states(R4["n_layers"] - 1, nodes)[:, -1]
            z, eps = G.logits_f64(h, W, b, segs, device="cuda")
            ids, vals, ok, bound = G.topk_f64(z, eps, top_k, 0)
            okn = ok.cpu().numpy()
            np.testing.assert_array_equal(ix[okn], ids.cpu().numpy()[okn], err_msg=f"beam step {k}")
            zi = z.clone()
            zi[:, 0] = -np.inf
            lse = torch.logsumexp(z, 1, keepdim=True)
            wv = (torch.gather(zi, 1, torch.as_tensor(ix, device=zi.device)) - lse).cpu().numpy()
            assert np.all(np.abs(v - wv) <= bound.cpu().numpy()), f"beam step {k}"
            rows_ok, rows_all = rows_ok + int(okn.sum()), rows_all + len(okn)
            parent, token, new_scores, new_nodes = lm.beam_select(st, scores, v, ix, beam_sz, nodes)
            cand = (scores[:, None] - v).reshape(-1).astype(np.float32)
            order = np.argsort(cand, kind="stable")[:beam_sz]
            np.testing.assert_array_equal(parent, order // top_k)
            np.testing.assert_array_equal(token, ix.reshape(-1)[order])
            np.testing.assert_array_equal(new_scores, cand[order])
            lm.select(st, parent)
            x, scores, nodes = token[:, None], new_scores, new_nodes
    finally:
        st.close()
    from code_intelligence_b200.language_model import inverse_cdf
    u = float(np.random.default_rng(1).random(dtype=np.float32))
    want = nodes[inverse_cdf(np.exp(-scores.astype(np.float64)), u)]
    np.testing.assert_array_equal(lm.beam_search(prompt, n_words, top_k=top_k, beam_sz=beam_sz, seed=1), want)
    print(f"R4 {mode} beam: top-k ids checked on {rows_ok} of {rows_all} rows")
    assert rows_ok >= rows_all // 2


def test_text_prompt_and_n_words_zero():
    ref = L.make_lm(seed=14, dec_scale=4.0, **SMALL)
    itos = ["xxunk", "xxpad", "xxbos", "xxfld", "xxmaj", "xxup", "xxrep", "xxwrep"] + \
        [f"w{i}" for i in range(SMALL["vocab_sz"] - 8)]
    lm = device_lm(ref, 0, itos=itos)
    try:
        assert lm.predict("w1 w2", 0) == "w1 w2 "
        out = lm.predict("w1 w2", 5, seed=0)
        assert out.startswith("w1 w2 ") and len(out.split()) <= 7 and "xxunk" not in out
        out = lm.beam_search("w1 w2", 3, top_k=4, beam_sz=16, seed=0)
        assert out.startswith("w1 w2 w1 w2 ") and len(out.split()) <= 7
        with pytest.raises(ValueError):
            lm.beam_search("w1", 2, beam_sz=lm.encoder.max_batch + 1)
        with pytest.raises(ValueError):
            lm.beam_search("w1", 2, top_k=65)
    finally:
        lm.close()


# ------------------------------------------------------------------------------------------------ nothing else changes
def test_encode_unchanged_next_to_a_live_state():
    ref = L.make_lm(seed=15, dec_scale=4.0, **SMALL)
    lm = device_lm(ref, 0)
    enc = lm.encoder
    ids = np.stack(R.synthetic_ids(7, 40, seed=3, vocab_sz=SMALL["vocab_sz"]))
    try:
        enc._debug_layer_states(2, ids)
        n0 = enc.launch_count
        before = enc._debug_layer_states(2, ids)
        n1 = enc.launch_count
        st = lm.new_state(7)
        feed(lm, st, ids)
        n2 = enc.launch_count
        after = enc._debug_layer_states(2, ids)
        assert enc.launch_count - n2 == n1 - n0
        np.testing.assert_array_equal(before, after)
        st.close()
    finally:
        lm.close()


def test_errors_and_refusals():
    ref = L.make_lm(seed=16, dec_scale=4.0, **SMALL)
    lm = device_lm(ref, 0)
    try:
        st = lm.new_state(4)
        V = SMALL["vocab_sz"]
        ids = torch.full((2, 3), V + 5, dtype=torch.int64, device="cuda")
        lm.step(st, ids, 3)
        with pytest.raises(ValueError, match="token id"):
            lm.check_errors()
        with pytest.raises(ValueError):
            lm.step(st, np.zeros((5, 1)), 1)                 # rows above the capacity
        for k in (0, 65):
            with pytest.raises(ValueError):
                lm.step(st, np.zeros((1, 1)), k)
        for kw in (dict(temperature=0.0), dict(min_p=0.0), dict(min_p=1.5)):
            with pytest.raises(ValueError):
                lm.sample(st, np.zeros((1, 1)), np.zeros(1), **kw)
        with pytest.raises(ValueError):
            lm.beam_select(st, np.zeros(300), np.zeros((300, 64)), np.zeros((300, 64)), 10)
        with pytest.raises(ValueError):
            lm.select(st, [4])
        with pytest.raises(ValueError):
            lm.new_state(lm.encoder.max_batch + 1)
        n = lm.launch_count
        with pytest.raises(ValueError):
            lm.step(st, np.zeros((1, 1)), 1, exclude=V)
        assert lm.launch_count == n
        st.reset()
        st.close()                                           # a state closed before its model is fine
        with pytest.raises(ValueError, match="closed"):
            lm.step(st, np.zeros((1, 1)), 1)
        other = device_lm(ref, 0)
        try:
            with pytest.raises(ValueError, match="another"):
                lm.step(other.new_state(1), np.zeros((1, 1)), 1)
            live = other.new_state(2)
            other.close()                                    # the model closes its open states first
            assert live._h is None
            with pytest.raises(ValueError, match="closed"):
                live.reset()
            del live
        finally:
            other.close()
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            lm.predict(np.array([2, 10]), 2, min_p=1.0, seed=0)
        assert sum("no item with probability" in str(r.message) for r in rec) == 2
    finally:
        lm.close()
