"""Text generation's kernels (csrc/lm_gen.cu) bit for bit against the exact float32 restatement of
oracle/lm_gen_ref.py (topk_f32_exact, sample_f32_exact), with the device's own math through ie_debug_gates: fn 9
(ex2.approx, the bare MUFU.EX2 inside inlined expf), fn 10 (logf), fn 12 (powf).  Every decision is checked, near-ties,
draws on a CDF boundary and uniforms next to 1 included; nothing is skipped.

* the restated expf against the device's standalone expf (fn 11) on every f32 x <= 0;
* the test hooks (ld = V) on V in {1, 2, 31..33, 1023..1025, 2047..2049, 8193, 60000} with real-valued and crafted
  rows, k in {1, 2, 63, 64, min(V, 64)}, the excluded column at -1, 0, V - 1, the argmax and warp and chunk edges;
  sampling at uniforms on the restated CDF boundaries (all of them up to V = 1025, then edges and random columns) and
  their f32 neighbours, u = 0 and 1 - 2^-24, min_p on a
  row's p_j exactly and out of reach, temperatures 0.5, 0.7, 2 and 1e-3 with all-zero rows in the same call;
* the production path (ld = round_up(V, 256)): logits from ie_debug_gemm_ex on the states ie_debug_layer_states gives
  for the history (tests/test_gpu_lm_generation.py pins those states to the carried ring), at SMALL and R4: step at
  1, 10, 129 and 1000 rows, sample on boundary uniforms, predict for 64 words and beam_search with its defaults;
* negative controls: every restatement mutant disagrees with the device.

Bits are compared through int32 views, so -0 against +0 is a difference."""
import functools

import numpy as np
import pytest
import torch

from code_intelligence_b200 import _lib
from code_intelligence_b200._lib import IE_CFG_FP32
from code_intelligence_b200.language_model import LanguageModel, inverse_cdf
from oracle import lm_gen_ref as G
from oracle import lm_ref as L

pytestmark = pytest.mark.gpu
MODES = {"bf16": 0, "fp32": IE_CFG_FP32}
SMALL = dict(vocab_sz=500, emb_sz=96, n_hid=200, n_layers=3)
R4 = dict(vocab_sz=60000, emb_sz=800, n_hid=2400, n_layers=4)
U_TOP = float(np.float32(1 - 2 ** -24))
CHUNK = 2048          # rows per debug-hook call


def dev_ex2(x):
    return _lib._debug_gates("lm_ex2", x)


def dev_log(x):
    return _lib._debug_gates("lm_log", x)


def dev_expf(x):
    return _lib._debug_gates("lm_expf", x)


def dev_pow(x, y):
    f = x.contiguous().view(-1)
    return _lib._debug_gates("lm_pow", torch.stack([f, torch.full_like(f, y)])).view(x.shape)


def restate_topk(z, k, ex, mutant=None):
    v, i = G.topk_f32_exact(torch.as_tensor(z).cuda(), k, ex, dev_ex2, dev_log, mutant)
    return v.cpu().numpy(), i.cpu().numpy()


def restate_scan(z, ex, min_p, inv_t, mutant=None):
    """(w, S, total, warned) of rows z on the device's math, as cuda tensors."""
    w, warned = G.sample_weights_f32(torch.as_tensor(z).cuda(), ex, min_p, inv_t, dev_ex2, dev_pow, mutant)
    S, total = G.cta_scan_f32(w, mutant)
    return w, S, total, warned


def restate_draws(scan, rows, u, mutant=None):
    """Draws and flags for row indices ``rows`` of a restate_scan at uniforms u (numpy), in pieces."""
    w, S, total, warned = scan
    rows = torch.as_tensor(np.asarray(rows), device="cuda")
    u = torch.as_tensor(np.asarray(u, np.float32), device="cuda")
    out = []
    for a in range(0, len(u), CHUNK):
        r = rows[a:a + CHUNK]
        out.append(G.draw_f32(S[r], w[r], total[r], u[a:a + CHUNK], mutant))
    ids = torch.cat(out).cpu().numpy()
    fl = torch.where(total[rows] > 0, warned[rows].int(), torch.full_like(rows, 2, dtype=torch.int32))
    return ids, fl.cpu().numpy()


def on_boundary(S, total):
    """f32 uniforms u with f32(u * total) = S (the nearest f32 u where none gives it exactly), clamped to [0, 1)."""
    t = total.double()
    u = (S.double() / t).float()
    for _ in range(2):     # step u toward the boundary where the product rounds off it
        p = (u.double() * t).float()
        u = torch.where(p < S, torch.nextafter(u, torch.ones_like(u)), torch.where(p > S, torch.nextafter(
            u, torch.zeros_like(u)), u))
    return u.clamp(0, U_TOP)


def boundary_uniforms(S, total, cols=None):
    """Uniforms on the CDF boundary S_j of each column j (of ``cols``), their f32 neighbours, 0 and 1 - 2^-24, all in
    [0, 1): numpy float32, unique."""
    u = on_boundary(S if cols is None else S[cols], total)
    u = torch.cat([u, torch.nextafter(u, torch.zeros_like(u)), torch.nextafter(u, torch.ones_like(u)),
                   torch.tensor([0.0, U_TOP], device=u.device)])
    return np.unique(u.clamp(0, U_TOP).cpu().numpy().astype(np.float32))


def debug_topk(z, k, exclude):
    z = np.ascontiguousarray(z, dtype=np.float32)
    rows, V = z.shape
    v, i = np.empty((rows, k), np.float32), np.empty((rows, k), np.int64)
    _lib.check(_lib.load().ie_debug_gen_topk(z.ctypes.data, rows, V, k, exclude, v.ctypes.data, i.ctypes.data, 0))
    return v, i


def debug_sample(z, rows, u, exclude, temperature, min_p):
    """ie_debug_gen_sample on rows z[rows] at the uniforms u, CHUNK rows per call."""
    out, fl = [], []
    for a in range(0, len(u), CHUNK):
        zz = np.ascontiguousarray(z[rows[a:a + CHUNK]], dtype=np.float32)
        uu = np.ascontiguousarray(u[a:a + CHUNK], dtype=np.float32)
        n, V = zz.shape
        o, f = np.empty(n, np.int64), np.empty(n, np.int32)
        _lib.check(_lib.load().ie_debug_gen_sample(zz.ctypes.data, n, V, uu.ctypes.data, exclude, temperature,
                                                   min_p, o.ctypes.data, f.ctypes.data, 0))
        out.append(o)
        fl.append(f)
    return np.concatenate(out), np.concatenate(fl)


def assert_bits(got, want, what):
    """Arrays [rows, ...] equal bit for bit (floats through int32 views); the first mismatching row named."""
    for g, w in zip(got, want):
        g, w = np.asarray(g), np.asarray(w)
        if g.dtype == np.float32:
            g, w = g.view(np.int32), np.ascontiguousarray(w, np.float32).view(np.int32)
        assert g.shape == w.shape, (what, g.shape, w.shape)
        bad = np.flatnonzero((g != w).reshape(len(g), -1).any(1)) if g.size else []
        assert len(bad) == 0, (what, f"{len(bad)} of {len(g)} rows differ; first row {bad[0]}", g[bad[0]], w[bad[0]])


# ------------------------------------------------------------------------------------------------ device math
def test_expf_restatement_on_every_nonpositive_f32():
    """expf_parts with fn 9's ex2, rounded as f32(scale * e), equals the device's standalone expf (fn 11) on every f32
    x <= 0 (2^31 + 1 values: the kernels evaluate expf(z - m) with z - m <= 0), -0, +0 and -inf included."""
    mant = torch.arange(1 << 23, dtype=torch.int32, device="cuda")
    n = 0
    for e in range(256):
        x = (mant | (-(1 << 31)) | (e << 23)).view(torch.float32)
        if e == 255:
            x = torch.tensor([-float("inf"), 0.0], device="cuda")
        got = dev_expf(x).view(torch.int32)
        want = G.expf_f32(x, dev_ex2).view(torch.int32)
        bad = torch.nonzero(got != want)
        assert bad.numel() == 0, (e, f"{bad.numel()} differ, first x = {float(x[bad[0, 0]])!r}",
                                  float(got[bad[0, 0]].view(torch.float32)), float(want[bad[0, 0]].view(torch.float32)))
        n += x.numel()
    print(f"expf: {n} inputs x <= 0 equal")


# ------------------------------------------------------------------------------------------------ debug hooks
V_GRID = [1, 2, 31, 32, 33, 1023, 1024, 1025, 2047, 2048, 2049, 8193, 60000]


@functools.lru_cache(maxsize=None)
def hook_rows(V):
    """Real-valued rows and crafted ones: values that collide after f32(z - lse) (one logit near 1e4 over distinct
    small ones), all-equal (s = V), integer tie storms, a spread over 88 (terms flush), the maximum in the partial last
    chunk (at V - 1), a peaked row, and near-flat rows (lse's last bits)."""
    rng = np.random.default_rng(V)
    z = (3 * rng.standard_normal((10, V))).astype(np.float32)
    z[1] = 1e-5 * rng.permutation(V)
    z[1, V // 2] = 1e4 - 0.37
    z[2] = 0.0
    z[3] = rng.integers(-4, 5, V)
    z[4] = -rng.integers(0, 200, V)
    z[4, V // 3] = 0
    z[5, V - 1] = 40.0
    z[6] = 0.5 * z[6]
    z[6, 0] = 25.0
    z[7:] = 1e-3 * z[7:]
    return z


def excludes(V, z):
    return sorted({e for e in (-1, 0, V - 1, int(np.argmax(z[0])), 31, 32, 1023, 1024) if e < V})


@pytest.mark.parametrize("V", V_GRID)
def test_topk_hook_bit_for_bit(V):
    z = hook_rows(V)
    n = 0
    for k in sorted({1, 2, 63, 64, min(V, 64)}):
        if k > V:
            continue
        for ex in excludes(V, z):
            got = debug_topk(z, k, ex)
            assert_bits(got, restate_topk(z, k, ex), (V, k, ex))
            n += 1
    print(f"V={V}: {n} calls of {len(z)} rows equal")


def sample_cases(V, z):
    """(exclude, min_p, temperature) settings: plain, an excluded column at a chunk edge, min_p equal to row 0's
    third-largest p_j exactly, min_p 1 (nobody reaches it but a one-hot row: flag 1), temperatures 0.5, 0.7, 2, 1e-3."""
    w, _, _, _ = restate_scan(z[:1], -1, 0.0, 1.0)
    p3 = float(torch.sort(w[0], descending=True).values[min(2, V - 1)])
    return [(-1, 0.0, 1.0), (min(1024, V - 1), 0.0, 1.0), (-1, p3, 1.0), (0, 1.0, 1.0), (-1, 0.0, 0.5),
            (-1, 0.0, 0.7), (-1, 0.0, 2.0), (V - 1, 0.0, 1e-3)]


# columns whose CDF boundaries are drawn on, beyond every column at V <= 1025: (the column offsets in a 1024-column
# chunk, random columns per row), so that rows x V copied to the hook stay near 2 GB per V
BOUNDARY_COLS = {2047: ((0, 31, 32, 1023), 512), 2048: ((0, 31, 32, 1023), 512), 2049: ((0, 31, 32, 1023), 512),
                 8193: ((0, 31, 32, 1023), 256), 60000: ((0, 1023), 32)}


@pytest.mark.parametrize("V", V_GRID)
def test_sample_hook_bit_for_bit(V):
    """Every row at uniforms on its restated CDF boundaries and their f32 neighbours, 0 and 1 - 2^-24: every column's
    boundary up to V = 1025; beyond, the warp and chunk edges and random columns (BOUNDARY_COLS).  Each setting runs
    in one call over all rows, so flag-2 rows (temperature 1e-3 on a flat row) sit among normal ones."""
    z = hook_rows(V)
    rng = np.random.default_rng(V + 1)
    n = 0
    for ex, mp, t in sample_cases(V, z):
        it = float(np.float32(1.0 / t))
        scan = restate_scan(z, ex, mp, it)
        rows, us = [], []
        for r in range(len(z)):
            cols = None
            if V in BOUNDARY_COLS:
                offs, n_rand = BOUNDARY_COLS[V]
                edges = [c for c in range(V) if c % 1024 in offs] + [V - 1]
                cols = torch.as_tensor(np.unique(np.concatenate([edges, rng.integers(0, V, n_rand)])), device="cuda")
            u = boundary_uniforms(scan[1][r], scan[2][r], cols)
            rows.append(np.full(len(u), r))
            us.append(u)
        rows, us = np.concatenate(rows), np.concatenate(us)
        got = debug_sample(z, rows, us, ex, t, mp)
        want = restate_draws(scan, rows, us)
        assert_bits([got[0][:, None], got[1][:, None]], [want[0][:, None], want[1][:, None]], (V, ex, mp, t))
        if mp == 1.0 and V > 1:
            assert np.any(want[1] == 1)
        if t == 1e-3 and V > 1:
            assert np.any(want[1] == 2) and np.any(want[1] == 0)
        n += len(us)
    print(f"V={V}: {n} draws equal")


def test_every_mutant_disagrees_with_the_device():
    """Negative controls on the hook data: each restatement mutant gives other bits than the device somewhere."""
    V = 2049
    z = hook_rows(V)
    topk_dev = {(k, ex): debug_topk(z, k, ex) for k, ex in ((64, -1), (10, 0))}
    scan = restate_scan(z, -1, 1e-4, 1.0)
    rows = np.concatenate([np.full(3 * V, r) for r in range(len(z))])
    us = np.concatenate([np.resize(boundary_uniforms(scan[1][r], scan[2][r]), 3 * V) for r in range(len(z))])
    dev = debug_sample(z, rows, us, -1, 1.0, 1e-4)[0]
    for mutant in G.GEN_MUTANTS:
        n = 0
        if mutant in ("one_chain", "xor_ascending", "lse_f64", "ties_high"):
            for (k, ex), got in topk_dev.items():
                want = restate_topk(z, k, ex, mutant)
                n += int((got[0].view(np.int32) != want[0].view(np.int32)).sum() + (got[1] != want[1]).sum())
        if mutant not in ("lse_f64", "ties_high"):
            n += int((dev != restate_draws(restate_scan(z, -1, 1e-4, 1.0, mutant), rows, us, mutant)[0]).sum())
        print(f"{mutant}: {n} outputs differ")
        assert n > 0, mutant


# ------------------------------------------------------------------------------------------------ production path
def device_lm(ref, flags):
    return LanguageModel.from_state_dict(ref.fastai_state_dict(), flags=flags)


@functools.lru_cache(maxsize=None)
def model(name):
    cfg = SMALL if name == "small" else R4
    # a decoder scaled so that the draws are not peaked
    return L.make_lm(seed=21, dec_scale=4.0 if name == "small" else 20.0, bias_scale=0.5, **cfg), cfg


def logits(lm, ref, hist, segs):
    """The production logits of the histories' last step: ie_debug_gemm_ex on the last layer's f32 states."""
    W = ref.decoder.weight.detach().numpy()
    b = ref.decoder.bias.detach().numpy()
    h = lm.encoder._debug_layer_states(lm.encoder.n_layers - 1, hist)[:, -1]
    return _lib._debug_gemm(h, W, b, 0, 0, segs)


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("name", ["small", "r4"])
def test_step_and_sample_bit_for_bit(name, mode):
    """step at 1, 10, 129 and 1000 rows with k = 1, 10, 64 on three successive calls: every value and id; then sample
    on 129 rows at uniforms on a CDF boundary of each row (and below and above it), plain, temperature 0.7 and min_p
    0.05 with no_unk."""
    ref, cfg = model(name)
    lm = device_lm(ref, MODES[mode])
    segs = 3 if mode == "fp32" else 1
    rng = np.random.default_rng(3)
    try:
        for rows in (1, 10, 129, 1000):
            st = lm.new_state(rows)
            try:
                hist = rng.integers(2, cfg["vocab_sz"], (rows, 5))
                x = hist
                for k in (1, 10, 64):
                    got = lm.step(st, x, k, 0)
                    z = logits(lm, ref, hist, segs)
                    assert_bits(got, restate_topk(z, k, 0), (name, mode, rows, k))
                    x = rng.integers(2, cfg["vocab_sz"], (rows, 1))
                    hist = np.concatenate([hist, x], 1)
            finally:
                st.close()
        hist = rng.integers(2, cfg["vocab_sz"], (129, 6))
        z = logits(lm, ref, hist, segs)
        for t, mp in ((1.0, None), (0.7, None), (1.0, 0.05)):
            scan = restate_scan(z, 0, mp or 0.0, float(np.float32(1.0 / t)))
            cols = torch.as_tensor(rng.integers(0, cfg["vocab_sz"], 129), device="cuda")
            u0 = on_boundary(scan[1].gather(1, cols[:, None])[:, 0], scan[2])
            for u in (u0, torch.nextafter(u0, torch.zeros_like(u0)), torch.nextafter(u0, torch.ones_like(u0))):
                u = u.clamp(0, U_TOP).cpu().numpy().astype(np.float32)
                st = lm.new_state(129)
                try:
                    got = lm.sample(st, hist, u, 0, t, mp)
                finally:
                    st.close()
                want = restate_draws(scan, np.arange(129), u)
                assert_bits([got[0][:, None], got[1][:, None]], [want[0][:, None], want[1][:, None]],
                            (name, mode, t, mp))
    finally:
        lm.close()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_r4_predict_and_beam_search_bit_for_bit(mode):
    """R4, decoder not peaked: predict for 64 words (plain, temperature 0.7, min_p 0.05), every draw equal to the
    restatement on the logits of the words before it; beam_search with its defaults for 4 words step by step through
    step / beam_select / select: every row's top-k values and ids on every step, the survivors (numpy's stable argsort
    of the device's f32 scores) and the chosen node."""
    ref, cfg = model("r4")
    lm = device_lm(ref, MODES[mode])
    segs = 3 if mode == "fp32" else 1
    try:
        prompt = np.concatenate([[2], np.random.default_rng(5).integers(5, cfg["vocab_sz"], 16)]).astype(np.int64)
        T0 = len(prompt)
        for seed, kw in enumerate((dict(), dict(temperature=0.7), dict(min_p=0.05))):
            seq = lm.predict(prompt, 64, seed=seed, **kw)
            u = np.random.default_rng(seed).random(64, dtype=np.float32)
            h = lm.encoder._debug_layer_states(cfg["n_layers"] - 1, seq[None, :-1])[0, T0 - 1:]
            z = _lib._debug_gemm(h, ref.decoder.weight.detach().numpy(), ref.decoder.bias.detach().numpy(), 0, 0, segs)
            it = float(np.float32(1.0 / kw.get("temperature", 1.0)))
            want, fl = restate_draws(restate_scan(z, 0, kw.get("min_p", 0.0), it), np.arange(64), u)
            np.testing.assert_array_equal(seq[T0:], want, err_msg=f"{mode} {kw}")
            print(f"R4 {mode} predict {kw}: 64 draws equal, {len(set(want.tolist()))} distinct words")
        top_k, beam_sz = 10, 1000
        p = np.array([2, 100, 200, 300], dtype=np.int64)
        st = lm.new_state(beam_sz)
        try:
            nodes = np.tile(p, (top_k, 1))
            x, scores = nodes, np.zeros(top_k, np.float32)
            for k in range(4):
                v, ix = lm.step(st, x, top_k, 0)
                z = logits(lm, ref, nodes, segs)
                assert_bits([v, ix], restate_topk(z, top_k, 0), (mode, "beam step", k))
                parent, token, new_scores, new_nodes = lm.beam_select(st, scores, v, ix, beam_sz, nodes)
                cand = (scores[:, None] - v).reshape(-1).astype(np.float32)
                order = np.argsort(cand, kind="stable")[:beam_sz]
                np.testing.assert_array_equal(parent, order // top_k)
                np.testing.assert_array_equal(token, ix.reshape(-1)[order])
                assert_bits([new_scores[:, None]], [cand[order][:, None] + np.float32(0)], (mode, "scores", k))
                lm.select(st, parent)
                x, scores, nodes = token[:, None], new_scores, new_nodes
        finally:
            st.close()
        u = float(np.random.default_rng(1).random(dtype=np.float32))
        want = nodes[inverse_cdf(np.exp(-scores.astype(np.float64)), u)]
        np.testing.assert_array_equal(lm.beam_search(p, 4, seed=1), want)
    finally:
        lm.close()
