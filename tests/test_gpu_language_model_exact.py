"""The language model's fused decoder (csrc/lm.cu) bit for bit against the exact float32 restatement of
oracle/lm_ref.decoder_f32_exact, in the default and the fp32-accurate mode.

* the decoder's two math functions through ie_debug_gates: ex2.approx.ftz over all 2^32 inputs and logf over every f32
  in [1, 2^24], against the figures decoder_f64 charges;
* the test hook ie_debug_lm_decode on a grid of E, V and M (up to 5120 rows at V = 60000: 320 items, so each CTA
  flushes an item and starts another) with real-valued rows and crafted ones: spreads beyond 88, maxima first in the
  last tile of a slice or in the last slice, ties across lanes, tiles and slices, all-equal logits, the maximum at
  column V - 1 inside the partial last tile, and rising rows that rescale at every tile;
* the encoder path at E = 800, V = 60000 on 4 x 2400 layers: every row of 104, 129 and 1280-row calls in three time
  chunks, the last partial, and validate() at bs = 104, bptt = 67 over three batches;
* negative controls: every mutant order of the restatement disagrees with the device on the grid.

The restatement takes the device's accumulators of h W^T from ie_debug_gemm_ex, which runs the same gemm_bf16_kernel
mainloop on the same bf16 (or split-bf16) operands; bit agreement of the outputs is the evidence that they are the
decoder's.  Bits are compared through int32 views, so -0 against +0 is a difference."""
import ctypes as C
import functools
import math
import os

import numpy as np
import pytest
import torch

from code_intelligence_b200 import IssueEncoder, _lib
from code_intelligence_b200._lib import IE_CFG_FP32, IE_FLAG_DEVICE_PTRS
from code_intelligence_b200.language_model import LanguageModel, lm_stream
from oracle import awd_lstm_ref as R
from oracle import lm_ref as L

pytestmark = pytest.mark.gpu
MODES = {"bf16": 0, "fp32": IE_CFG_FP32}
PIECE = 2048          # rows per _debug_gemm call: it returns host [rows, V] f32


def dev_ex2(x):
    return _lib._debug_gates("lm_ex2", x)


def dev_log(x):
    return _lib._debug_gates("lm_log", x)


def segs_of(mode):
    return 3 if mode == "fp32" else 1


def restate(h, W, b, targets, segs, mutant=None):
    """decoder_f32_exact on the device's accumulators of h [M, E] W^T, PIECE rows at a time -> numpy (nll, lse, pred)."""
    out = []
    for r0 in range(0, h.shape[0], PIECE):
        acc = torch.from_numpy(_lib._debug_gemm(h[r0:r0 + PIECE], W, None, 0, 0, segs)).cuda()
        o = L.decoder_f32_exact(acc, b, targets[r0:r0 + PIECE], dev_ex2, dev_log, mutant)
        out.append([v.cpu().numpy() for v in o])
        del acc, o
    return tuple(np.concatenate([p[i] for p in out]) for i in range(3))


def assert_same(got, want, what):
    """(nll, lse, pred) bit for bit; the first mismatching row named."""
    for name, g, w in zip(("nll", "lse", "pred"), got, want):
        g = np.ascontiguousarray(g).reshape(-1).view(np.int32)
        w = np.ascontiguousarray(w).reshape(-1).view(np.int32)
        bad = np.nonzero(g != w)[0]
        assert bad.size == 0, (what, name, f"{bad.size} of {g.size} differ; first rows", bad[:5].tolist(),
                               g[bad[0]], w[bad[0]])


def n_differ(got, want):
    return sum(int((np.ascontiguousarray(g).reshape(-1).view(np.int32) !=
                    np.ascontiguousarray(w).reshape(-1).view(np.int32)).sum()) for g, w in zip(got, want))


# ------------------------------------------------------------------------------------------------ math functions
def test_ex2_over_every_f32():
    """ex2.approx.ftz.f32 over all 2^32 inputs: 0 exactly below 2^-126 (no subnormal result), ex2(0) = 1,
    ex2(-inf) = 0, results <= 1 for x <= 0, and its relative error on normal results at most EXP_REL / 2, the figure
    decoder_f64 charges twice."""
    mant = torch.arange(1 << 23, dtype=torch.int32, device="cuda")
    worst, at, cut = 0.0, None, -math.inf
    for sg in (0, 1):
        for e in range(256):
            x = (mant | ((-(1 << 31) if sg else 0) | (e << 23))).view(torch.float32)
            y = dev_ex2(x)
            if e == 255:
                nan = torch.isnan(x)
                assert torch.isnan(y[nan]).all()
                assert float(y[~nan][0]) == (0.0 if sg else math.inf)
                continue
            x64, y64 = x.double(), y.double()
            ref = torch.exp2(x64)
            assert not torch.isnan(y).any(), (sg, e)
            assert ((y64 == 0) | (y64 >= 2.0 ** -126)).all(), (sg, e)       # flushed, never subnormal
            assert (y64[ref < 2.0 ** -126] == 0).all(), (sg, e)
            if sg:
                assert float(y64.max()) <= 1.0, e
                z = y64 == 0
                if bool(z.any()):
                    cut = max(cut, float(x64[z].max()))
            fin = (y64 >= 2.0 ** -126) & torch.isfinite(y64)
            r = torch.where(fin, (y64 - ref).abs() / ref, torch.zeros_like(ref))
            k = int(r.argmax())
            if float(r[k]) > worst:
                worst, at = float(r[k]), float(x64[k])
    one = dev_ex2(torch.tensor([0.0, -0.0, -math.inf], device="cuda")).tolist()
    print(f"ex2: max relative error {worst:.4g} = 2^{math.log2(worst):.3f} at x = {at!r}; largest x giving 0: {cut!r}")
    assert one == [1.0, 1.0, 0.0]
    assert worst <= L.EXP_REL / 2, (worst, at)


def test_logf_over_every_f32_in_the_range_of_s():
    """logf over every f32 in [1, 2^24] (the sum s of a row lies there): within 2 u |log s|, what decoder_f64 charges
    for the log (its 2 u |lse - max| term); logf(1) = 0 exactly."""
    mant = torch.arange(1 << 23, dtype=torch.int32, device="cuda")
    worst, at, ulps = 0.0, None, 0.0
    for e in range(127, 127 + 25):
        x = (mant | (e << 23)).view(torch.float32)
        if e == 151:
            x = x[:1]                                   # 2^24 alone
        y = dev_log(x).double()
        ref = torch.log(x.double())
        err = (y - ref).abs()
        if e == 127:
            assert float(y[0]) == 0.0
            err, ref, y, x = err[1:], ref[1:], y[1:], x[1:]
        r = err / (2 * L.U * ref)
        k = int(r.argmax())
        ulp = torch.ldexp(torch.ones_like(y), (torch.frexp(y.float()).exponent - 24).to(torch.int32))
        ulps = max(ulps, float((err / ulp).max()))
        if float(r[k]) > worst:
            worst, at = float(r[k]), float(x[k])
    print(f"logf on [1, 2^24]: max |err| / (2 u log x) = {worst:.4g} at x = {at!r}; max error {ulps:.4g} ulp")
    assert worst <= 1.0, (worst, at)


# ------------------------------------------------------------------------------------------------ debug-hook grid
def bare_lm(E, V, W, b, flags):
    enc = IssueEncoder(1, E, E, V, 1 if V > 1 else 0, 0, flags)
    return LanguageModel(enc, W, b, owns_encoder=True)


N_CRAFTED = 8


def grid_data(E, V, M, crafted):
    """h [M, E], W [V, E], b [V] or None, targets [M].  Real-valued rows; with E >= 8 and V >= 8192 column 7 of W is
    a ramp (c - V) / 256, which the odd rows take at weight one: their logits rise through every tile, so every tile
    rescales, and they span more than 88.  ``crafted`` (bias none) puts the patterns below in columns 0..7 of W and
    one-hot rows selecting them in rows 0..7."""
    rng = np.random.default_rng(E * 131 + V * 7 + M)
    h = rng.standard_normal((M, E)).astype(np.float32)
    W = (3 * rng.standard_normal((V, E)) / math.sqrt(E)).astype(np.float32)
    b = None if crafted else rng.standard_normal(V).astype(np.float32)
    if E >= N_CRAFTED and V >= 8192:
        W[:, :N_CRAFTED] = 0
        W[:, 7] = (np.arange(V) - V) / 256
        h[:, :N_CRAFTED] = 0
        h[1::2, 7] = 1
        h[1::2, N_CRAFTED:] *= 0.3
    if crafted:
        assert E >= N_CRAFTED and V >= 16385 and M >= N_CRAFTED
        h[:N_CRAFTED] = np.eye(N_CRAFTED, E, dtype=np.float32)
        last = (V - 1) // 8192 * 8192                      # first column of the last slice
        W[:, 0] = -rng.integers(0, 200, V)                 # spread 199 > 88: most terms flush to 0
        W[5, 0] = 0
        W[:, 1] = rng.standard_normal(V)                   # max first in the last tile of slice 0, tied in slice 1
        W[31 * 256 + 77, 1] = W[8192 + 300, 1] = 9
        W[:, 2] = rng.standard_normal(V)                   # max first in the last slice, tied at V - 1
        W[[last + (V - 1 - last) // 2, V - 1], 2] = 9
        W[:, 3] = rng.integers(-3, 1, V)                   # ties at 0 in every lane, tile and slice
        W[:, 4] = -1                                       # one tie per lane and across tiles and slices
        W[[8192 + 2, 8192 + 1, 8192 + 4, 8192 + 7, 8192 + 256, 16384 if V > 16384 else 8193], 4] = 2
        W[:, 5] = 0                                        # all equal: s = V exactly
        W[:, 6] = rng.standard_normal(V)                   # max at V - 1, inside the partial last tile
        W[V - 1, 6] = 9
    t = rng.integers(0, V, M)
    t[0] = -100
    t[-1] = V - 1
    return h, W, b, t


# (E, V, M, crafted): every E of {1, 64, 65, 800, 1152}, V of {1, 2, 255, 256, 257, 8191, 8192, 8193, 16385, 60000}
# and M of {1, 127, 128, 129, 5120}
GRID = [(1, 1, 1, False), (1, 2, 127, False), (64, 255, 128, False), (65, 256, 129, False), (800, 257, 127, False),
        (64, 8191, 129, False), (65, 8192, 128, False), (1152, 8193, 129, False), (64, 16385, 129, True),
        (800, 60000, 5120, False), (1152, 60000, 128, True), (65, 60000, 1, False)]


@functools.lru_cache(maxsize=None)
def grid_case(E, V, M, crafted, mode):
    h, W, b, t = grid_data(E, V, M, crafted)
    lm = bare_lm(E, V, W, b, MODES[mode])
    try:
        got = lm._debug_decode(h, t)
    finally:
        lm.close()
    return (h, W, b, t), got


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("E,V,M,crafted", GRID)
def test_debug_hook_bit_for_bit(E, V, M, crafted, mode):
    (h, W, b, t), got = grid_case(E, V, M, crafted, mode)
    want = restate(h, W, b, t, segs_of(mode))
    assert_same(got, want, (E, V, M, mode))
    if crafted:
        z = h[:N_CRAFTED].astype(np.float64) @ W.T.astype(np.float64)
        np.testing.assert_array_equal(got[2][:N_CRAFTED], np.argmax(z, 1))
        assert got[1][5] == float(dev_log(torch.tensor([float(V)], device="cuda"))[0])   # s = V, max 0
        assert got[2][6] == V - 1 and got[2][5] == 0


@pytest.mark.parametrize("mode", sorted(MODES))
def test_every_mutant_disagrees_with_the_device(mode):
    """Negative controls: each order the kernel must not have changes at least one output bit on the grid."""
    cases = [c for c in GRID if c[3] or c[1] >= 8192 and c[2] <= 129]
    for mutant in L.EXACT_MUTANTS:
        n = 0
        for c in cases:
            (h, W, b, t), got = grid_case(*c, mode)
            n += n_differ(got, restate(h, W, b, t, segs_of(mode), mutant))
            if n:
                break
        print(f"{mode} {mutant}: {n} output words differ on case {c}")
        assert n > 0, mutant


# ------------------------------------------------------------------------------------------------ the encoder path
BIG = dict(vocab_sz=60000, emb_sz=800, n_hid=2400, n_layers=4)


@functools.lru_cache(maxsize=1)
def big_ref():
    ref = L.make_lm(seed=11, dec_scale=40.0, bias_scale=1.0, **BIG)
    sd = ref.fastai_state_dict()
    return sd, sd["1.decoder.weight"].numpy(), sd["1.decoder.bias"].numpy()


def chunked_lm(mode, chunk_t):
    os.environ["IE_CHUNK_T"] = str(chunk_t)
    try:
        return LanguageModel.from_state_dict(big_ref()[0], flags=MODES[mode])
    finally:
        del os.environ["IE_CHUNK_T"]


@pytest.fixture(scope="module", params=sorted(MODES))
def big(request):
    lm = chunked_lm(request.param, 3)
    yield request.param, lm
    lm.close()


def shifted_targets(ids):
    y = np.roll(ids, -1, 1)
    y[:, -1] = -100
    return y


@pytest.mark.parametrize("B", [104, 129, 1280])
def test_encoder_path_every_row(big, B):
    """Every row of a B x 7 call in time chunks of 3, 3 and 1: the states from raw_features, the logits through
    ie_debug_gemm_ex, the outputs bit for bit."""
    mode, lm = big
    _, W, b = big_ref()
    T = 7
    ids = np.stack(R.synthetic_ids(B, T, seed=B, vocab_sz=BIG["vocab_sz"]))
    y = shifted_targets(ids)
    n0 = lm.launch_count
    got = lm.forward(ids, y)
    assert lm.launch_count - n0 == 2 * 3           # three chunks, two kernels each
    h = lm.encoder.raw_features(ids).reshape(-1, BIG["emb_sz"])
    want = restate(h, W, b, y.reshape(-1), segs_of(mode))
    assert_same(got, want, (mode, B))


def test_null_lse_and_pred_give_the_same_nll(big):
    mode, lm = big
    ids = np.stack(R.synthetic_ids(129, 7, seed=3, vocab_sz=BIG["vocab_sz"]))
    x = torch.as_tensor(ids, device="cuda")
    y = torch.as_tensor(shifted_targets(ids), device="cuda")
    full, _, _ = lm.forward_device(x, y)
    nll = torch.full_like(full, float("nan"))
    s = torch.cuda.current_stream()
    _lib.check(lm._lib.ie_lm_forward(lm._h, x.data_ptr(), y.data_ptr(), 129, 7, nll.data_ptr(), None, None,
                                     IE_FLAG_DEVICE_PTRS, C.c_void_p(s.cuda_stream)))
    lm.check_errors()
    assert torch.equal(nll.view(torch.int32), full.view(torch.int32)), mode


def test_full_batch_within_the_f64_bound(big):
    """decoder_f64 at B = 1280 on two steps: the rows beyond row 7 of a block tied to the math, not only to the
    restatement."""
    mode, lm = big
    _, W, b = big_ref()
    ids = np.stack(R.synthetic_ids(1280, 2, seed=17, vocab_sz=BIG["vocab_sz"]))
    y = np.roll(ids, -1, 1)
    nll, lse, pred = lm.forward(ids, y)
    h = lm.encoder.raw_features(ids).reshape(-1, BIG["emb_sz"])
    for r0 in range(0, h.shape[0], 640):
        sl = slice(r0, r0 + 640)
        ref = L.decoder_f64(h[sl], W, b, y.reshape(-1)[sl], segs_of(mode), device="cuda")
        v = L.check_decoder(ref, nll.reshape(-1)[sl], lse.reshape(-1)[sl], pred.reshape(-1)[sl])
        assert v["max_lse"] <= 1 and v["max_nll"] <= 1 and v["wrong_pred"] == 0, (mode, r0, v)
        torch.cuda.empty_cache()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_validate_at_bs_104_bptt_67(mode):
    """validate() over three batches of 104 x 67 with time chunks of 50: every token's nll and pred bit for bit, and
    (val_loss, accuracy) equal to validate's own float64 averaging of the restated values."""
    bs, bptt = 104, 67
    docs = R.synthetic_ids(60, 600, seed=23, vocab_sz=BIG["vocab_sz"], min_len=100)
    x, y = lm_stream(docs, bs, bptt)
    n_b = x.shape[1] // bptt
    assert n_b >= 3, n_b
    lm = chunked_lm(mode, 50)
    try:
        val_loss, acc, _ = lm.validate(docs, bs=bs, bptt=bptt)
        got = lm.forward(x, y)
        h = np.ascontiguousarray(lm.encoder.raw_features(x).reshape(-1, BIG["emb_sz"]))
    finally:
        lm.close()
    _, W, b = big_ref()
    nll, lse, pred = restate(h, W, b, y.reshape(-1), segs_of(mode))
    assert_same([got[0], got[2]], [nll, pred], (mode, "validate"))
    nll, pred = nll.reshape(y.shape), pred.reshape(y.shape)
    cols = [slice(k * bptt, (k + 1) * bptt) for k in range(n_b)]
    want_loss = float(np.mean([float(np.mean(nll[:, c], dtype=np.float64)) for c in cols]))
    want_acc = float(np.mean([float(np.mean(pred[:, c] == y[:, c])) for c in cols]))
    print(f"{mode}: validate at bs 104, bptt 67, {n_b} batches: val_loss {val_loss!r}, accuracy {acc!r}")
    assert (val_loss, acc) == (want_loss, want_acc)
