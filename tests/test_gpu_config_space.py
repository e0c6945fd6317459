"""GPU tests of the encoder across its configuration space.  tests/test_gpu_numerics.py pins the rounding points at two
shapes; the kernel instantiation and the layer geometry, though, are chosen from (n_layers, emb_sz, n_hid, vocab_sz,
pad_idx), and every other test runs with emb_sz < n_hid, n_layers >= 2, pad_idx 1 and a vocabulary under 60001.  Each
entry of CONFIGS exists for an instantiation, a layer-shape class or a path that those shapes never reach, and gets:

  a. teacher-forced per-element checks of every layer (oracle/device_numerics.py), caps on max / RMS of |dh| / bound;
  b. the four mutants of the arithmetic, each rejected by at least 4x a cap;
  c. encode_ids equal bit for bit to device_numerics.pool of the last layer's states (the only check that runs the
     pooling instantiations: the state hook runs without pooling), lengths 1, T and on time-chunk boundaries;
  d. raw_features equal bit for bit to the hook's last layer;
  e. free-running parity with the fp32 oracle on up to 32 rows, at the tolerances of tests/test_gpu_parity.py;
  f. where the design promises identical bits (IE_EMB_PROJ, IE_CHUNK_T, IE_BATCHES, IE_SEQ, IE_MC), identical bits to
     the default handle of the same configuration.

Token ids 0, vocab-1 and pad_idx sit at valid positions (t = 0 and t = len-1 included) in every configuration.  Three
more tests: the per-token table's size switch, ids at the vocabulary edges, and reloading weights on a live handle.
"""
import numpy as np
import pytest

from oracle import awd_lstm_ref as R
from oracle import device_numerics as D
from test_gpu_numerics import _check_caps, _rows, _teacher_forced_stats
from test_gpu_parity import KNOBS, REL_L2_MAX, REL_L2_MAX_SCALED, _assert_parity, _pad

pytestmark = pytest.mark.gpu

FP32 = D.IE_CFG_FP32
L1 = (1, 96, 8, 500, 1)          # one layer: out = emb_sz = 96 (two tiles, the second half padding); n_hid is unused
WIDE_OUT = (3, 200, 96, 500, 1)  # emb_sz > n_hid
BIG_VOCAB = (2, 64, 2400, 340000, 1)

# tag: ((n_layers, emb_sz, n_hid, vocab_sz, pad_idx), weight scale, B, T, knobs, flags, (max cap, RMS cap) of |dh| / bound)
# Observed on an H100 SXM 80 GB HBM3 (power limit 400 W), max / RMS:
#   one layer 0.320 / 0.0045 (identical bits with IE_SEQ=0, IE_EMB_PROJ=0, IE_CHUNK_T=5, IE_BATCHES=2, IE_MC=1),
#   IE_GX_BF16=0 0.016 / 0.0033, fp32 0.102 / 0.021; one layer 800 0.475 / 0.0082; emb > hid 0.434 / 0.0062 (same with
#   IE_FUSE_LAST=0), fp32 0.163 / 0.033; fastai 400/1152 0.814 / 0.012; 64-multiples 0.159 / 0.0041; 7/33 0.0146 / 0.0049;
#   1/1 0.0090 / 0.0051; 65/65 0.135 / 0.0035; odd tiles IE_MC=1 0.284 / 0.0046; table > 6 GiB 0.284 / 0.0069;
#   pad_idx 0 0.0151 / 0.0033, pad_idx 299 0.0153 / 0.0035.  Every mutant breaks a cap by 7.6x (f/o swap at fastai
#   400/1152, torch-default init) or more.
# Caps are about twice that, never above 1 (the bound itself) and never above 4x the observation.
CONFIGS = {
    # lstm_layer_kernel<TOK, fp16 Gx, POOL>: layer 0 reads the per-token table and carries the pooling (never fused)
    "1 layer": (L1, 2.0, 300, 23, {}, 0, (0.64, 0.009)),
    # <TOK, f32 Gx, POOL>
    "1 layer IE_GX_BF16=0": (L1, 2.0, 300, 23, {"IE_GX_BF16": 0}, 0, (0.032, 0.0066)),
    # <TOK, f32 Gx, POOL> with split-bf16 operands and IEEE gates
    "1 layer fp32": (L1, 2.0, 300, 23, {}, FP32, (0.21, 0.043)),
    # <TOK, fp16, POOL> launched once per timestep
    "1 layer IE_SEQ=0": (L1, 2.0, 300, 23, {"IE_SEQ": 0}, 0, (0.64, 0.009)),
    # <!TOK, fp16, POOL>: gather + GEMM, then the pooled layer 0
    "1 layer IE_EMB_PROJ=0": (L1, 2.0, 300, 23, {"IE_EMB_PROJ": 0}, 0, (0.64, 0.009)),
    # <TOK, POOL> over time chunks: the table row and the pooling use the global timestep
    "1 layer IE_CHUNK_T=5": (L1, 2.0, 300, 23, {"IE_CHUNK_T": 5}, 0, (0.64, 0.009)),
    # two batches per launch, 700 rows in two calls (check f)
    "1 layer IE_BATCHES=2": (L1, 2.0, 300, 23, {"IE_BATCHES": 2}, 0, (0.64, 0.009)),
    # multicast refused for the pooled layer 0 (encode); the state hook and raw_features run the multicast TOK kernel
    "1 layer IE_MC=1": (L1, 2.0, 300, 23, {"IE_MC": 1}, 0, (0.64, 0.009)),
    # one layer at the production width: out = 800 -> 13 tiles, the last one half padding
    "1 layer 800": ((1, 800, 2400, 60000, 1), 1.0, 300, 24, {}, 0, (0.96, 0.017)),
    # emb_sz > n_hid: the last layer is the widest (max_out_pad, ring y_ld, pool strides); fused with kin_pad < kh_pad
    "emb > hid": (WIDE_OUT, 2.0, 300, 23, {}, 0, (0.87, 0.013)),
    "emb > hid fp32": (WIDE_OUT, 2.0, 300, 23, {}, FP32, (0.33, 0.067)),
    "emb > hid IE_FUSE_LAST=0": (WIDE_OUT, 2.0, 300, 23, {"IE_FUSE_LAST": 0}, 0, (0.87, 0.013)),
    # fastai's default AWD_LSTM: n_hid = 1152 = 18 tiles exactly, emb_sz 400 padded to 448
    "fastai 400/1152": ((3, 400, 1152, 60000, 1), 1.0, 300, 24, {}, 0, (1.0, 0.025)),
    # every width a multiple of 64: no padded unit anywhere
    "64-multiples": ((2, 64, 256, 300, 1), 2.0, 300, 23, {}, 0, (0.32, 0.0083)),
    # emb_sz 7 (not a multiple of 8), n_hid 33 (one real unit in the second 32-unit slice), vocabulary just over 256
    "7/33 vocab 257": ((2, 7, 33, 257, 1), 2.0, 300, 23, {}, 0, (0.03, 0.0098)),
    # the smallest legal model: one real unit in a tile of 64, emb_sz 1, three tokens (M padding of the table GEMM)
    "1/1 vocab 3": ((2, 1, 1, 3, 1), 2.0, 300, 23, {}, 0, (0.018, 0.011)),
    # 65 = one real unit in the last tile of every layer
    "65/65": ((3, 65, 65, 1000, 1), 2.0, 300, 23, {}, 0, (0.27, 0.0071)),
    # n_hid 150 -> 3 tiles: multicast falls back per layer inside an IE_MC=1 handle
    "odd tiles IE_MC=1": ((3, 96, 150, 500, 1), 2.0, 300, 23, {"IE_MC": 1}, 0, (0.57, 0.0092)),
    # table of 340 224 x 4 x 2432 fp16 > 6 GiB: layer 0 falls back to gather + GEMM
    "table > 6 GiB": (BIG_VOCAB, 1.0, 300, 16, {}, 0, (0.57, 0.014)),
    # pad id at both ends of the vocabulary
    "pad_idx 0": ((2, 64, 128, 300, 0), 2.0, 300, 23, {}, 0, (0.031, 0.0066)),
    "pad_idx 299": ((2, 64, 128, 300, 299), 2.0, 300, 23, {}, 0, (0.031, 0.007)),
}
BIT_EQUAL_KNOBS = {"IE_EMB_PROJ", "IE_CHUNK_T", "IE_BATCHES", "IE_SEQ", "IE_MC"}

_weights_cache = {}


def _weights(shape, scale):
    """Oracle encoder and its exported weights, seeded by the shape (cached: the large ones take seconds to build)."""
    key = (shape[:4], scale)
    if key not in _weights_cache:
        n_layers, emb_sz, n_hid, vocab = shape[:4]
        ref = R.make_encoder(7 + n_layers + emb_sz + n_hid, vocab, emb_sz, n_hid, n_layers, scale=scale)
        _weights_cache.clear()
        _weights_cache[key] = (ref, ref.export_weights())
    return _weights_cache[key]


def _lengths(B, T, chunk, seed):
    """1, T, T-1, 2 and every multiple of the time chunk (a length ending on a chunk boundary), the rest random."""
    fixed = [1, T, T - 1, 2] + list(range(chunk, T, chunk))
    return np.concatenate([fixed, np.random.default_rng(seed).integers(1, T + 1, B - len(fixed))]).astype(np.int32)


def _edge_ids(B, T, vocab, pad_idx, lengths, seed):
    """Synthetic ids right-padded with pad_idx; ids 0, vocab-1 and pad_idx planted at t = 0, t = len-1 and inside rows."""
    docs = [d[:n] for d, n in zip(R.synthetic_ids(B, T, seed=seed, vocab_sz=vocab), lengths)]
    ids, lengths = _pad(docs, T, pad=pad_idx)
    edge = (0, vocab - 1, pad_idx)
    for r in range(min(B, 24)):
        n = int(lengths[r])
        ids[r, 0] = edge[r % 3]
        ids[r, n - 1] = edge[(r + 1) % 3]
        ids[r, n // 2] = edge[(r + 2) % 3]
    return ids, lengths


def _handle(shape, weights, monkeypatch, env=None, flags=0):
    """test_gpu_parity._make with the pad id of `shape` (its fifth entry)."""
    from code_intelligence_b200 import IssueEncoder
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, str(v))
    enc = IssueEncoder(*shape, 0, flags).load_weights(*weights)
    for k in (env or {}):
        monkeypatch.delenv(k)
    return enc


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_configuration(tag, monkeypatch):
    shape, scale, B, T, knobs, flags, (max_cap, rms_cap) = CONFIGS[tag]
    n_layers, emb_sz, n_hid, vocab, pad_idx = shape
    ref, (emb, layers) = _weights(shape, scale)
    enc = _handle(shape, (emb, layers), monkeypatch, knobs, flags)
    lengths = _lengths(B, T, int(knobs.get("IE_CHUNK_T", 5)), seed=B + T)
    ids, lengths = _edge_ids(B, T, vocab, pad_idx, lengths, seed=T)

    # c, d: pooling of the last layer's states and the raw features, bit for bit
    last = enc._debug_layer_states(n_layers - 1, ids)
    pooled = enc.encode_ids(ids, lengths)
    np.testing.assert_array_equal(pooled, D.pool(last, lengths))
    np.testing.assert_array_equal(enc.raw_features(ids), last)

    # e: free-running parity with the fp32 oracle
    sel = np.unique(np.concatenate([np.arange(24), np.linspace(0, B - 1, 8).astype(int)]))[:32]
    want = R.encode_padded(ref, ids[sel], lengths[sel])
    m = R.parity_metrics(pooled[sel], want)
    print("CONFIG parity", tag, m)
    if flags & FP32:
        assert m["rel_l2"] <= 2e-5 and m["max_abs"] <= 5e-6 and m["min_cosine"] >= 1 - 1e-9, m
    else:
        _assert_parity(pooled[sel], want, rel_l2_max=REL_L2_MAX if scale == 1.0 else REL_L2_MAX_SCALED)

    # f: identical bits to the default handle where the design promises them
    if knobs and set(knobs) <= BIT_EQUAL_KNOBS:
        base_env = {"IE_FUSE_LAST": 0} if "IE_SEQ" in knobs else {}
        exp = _handle(shape, (emb, layers), monkeypatch, dict(knobs, **base_env), flags) if base_env else enc
        base = _handle(shape, (emb, layers), monkeypatch, base_env, flags)
        np.testing.assert_array_equal(exp.encode_ids(ids, lengths), base.encode_ids(ids, lengths))
        np.testing.assert_array_equal(exp.raw_features(ids), base.raw_features(ids))
        big_ids, big_len = _edge_ids(700, 9, vocab, pad_idx, _lengths(700, 9, 5, seed=3), seed=4)
        np.testing.assert_array_equal(exp.encode_ids(big_ids, big_len), base.encode_ids(big_ids, big_len))
        base.close()
        if exp is not enc:
            exp.close()

    # a, b: teacher-forced per element, every layer, and the mutants
    stats = _teacher_forced_stats(enc, emb, layers, ids, D.layer_modes(n_layers, flags, knobs), _rows(B))
    enc.close()
    _check_caps(tag, stats, max_cap, rms_cap)


def test_table_size_switch(monkeypatch):
    """A per-token table over 6 GiB is not built: layer 0 gathers embedding rows and runs its GEMM instead.  One call
    is then 5 launches (gather, GEMM, two recurrent layers, finalize) with the table allowed or not, against 4 on the
    table path (tokens, two recurrent layers, finalize); the bits are the same either way.  The switch sits at the
    largest table that fits: 331 008 rows x 4 x 2432 x 2 bytes <= 6 GiB < 331 264 rows."""
    shape = BIG_VOCAB
    _, (emb, layers) = _weights(shape, 1.0)
    ids, lengths = _edge_ids(40, 11, shape[3], shape[4], _lengths(40, 11, 5, seed=1), seed=2)

    def launches(enc, ids, lengths):
        enc.encode_ids(ids, lengths)                 # a first call may build the table
        n0 = enc.launch_count
        got = enc.encode_ids(ids, lengths)
        return enc.launch_count - n0, got

    dflt = _handle(shape, (emb, layers), monkeypatch)
    gather = _handle(shape, (emb, layers), monkeypatch, {"IE_EMB_PROJ": 0})
    n_dflt, a = launches(dflt, ids, lengths)
    n_gather, b = launches(gather, ids, lengths)
    assert (n_dflt, n_gather) == (5, 5)
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(dflt.raw_features(ids), gather.raw_features(ids))
    dflt.close()
    gather.close()
    for vocab, want in ((331008, 4), (331009, 5)):
        small = np.minimum(ids, vocab - 1)
        enc = _handle((2, 64, 2400, vocab, 1), (emb[:vocab], layers), monkeypatch)
        n, _ = launches(enc, small, lengths)
        assert n == want, (vocab, n)
        enc.close()


@pytest.mark.parametrize("tag", ["1 layer", "1 layer IE_EMB_PROJ=0", "pad_idx 0", "pad_idx 299"])
def test_ids_at_the_vocabulary_edges(tag, monkeypatch):
    """Rows made only of ids 0, vocab-1 and pad_idx (each at t = 0 and t = len-1), through the per-token table and
    through gather + GEMM: finite, equal to the oracle at the parity tolerance, and to the same rows encoded alone.  An
    id equal to vocab_sz is refused with ValueError by encode_ids, raw_features and the state hook, and the handle stays
    usable."""
    shape, scale, B, T, knobs, flags, _ = CONFIGS[tag]
    n_layers, emb_sz, n_hid, vocab, pad_idx = shape
    ref, weights = _weights(shape, scale)
    enc = _handle(shape, weights, monkeypatch, knobs, flags)
    edge = np.array([0, vocab - 1, pad_idx])
    rng = np.random.default_rng(5)
    ids = np.stack([rng.choice(edge, 13) for _ in range(30)] + [np.full(13, v) for v in edge])
    lengths = np.concatenate([rng.integers(1, 14, 30), [13, 1, 7]]).astype(np.int32)
    got = enc.encode_ids(ids, lengths)
    _assert_parity(got, R.encode_padded(ref, ids, lengths), rel_l2_max=REL_L2_MAX_SCALED)
    np.testing.assert_array_equal(got, D.pool(enc._debug_layer_states(n_layers - 1, ids), lengths))
    for r in (0, 30, 31, 32):
        np.testing.assert_array_equal(got[r], enc.encode_ids(ids[r:r + 1, :lengths[r]])[0])
    bad = ids.copy()
    bad[3, 0] = vocab
    with pytest.raises(ValueError):
        enc.encode_ids(bad, lengths)
    with pytest.raises(ValueError):
        enc.raw_features(bad)
    with pytest.raises(ValueError):
        enc._debug_layer_states(0, bad)
    np.testing.assert_array_equal(enc.encode_ids(ids, lengths), got)
    enc.close()


@pytest.mark.parametrize("shape,flags", [(L1, 0), ((3, 96, 200, 500, 1), 0), ((3, 96, 200, 500, 1), FP32), (L1, FP32)])
def test_reload_weights_on_a_live_handle(shape, flags, monkeypatch):
    """load_weights(A), encode, load_weights(B), encode: the second result is a fresh B handle's bits (the per-token
    table and the fused last layer's [W_ih | W_hh] are rebuilt); loading A again gives A's bits back."""
    n_layers, emb_sz, n_hid, vocab, _ = shape
    wa = R.make_encoder(31, vocab, emb_sz, n_hid, n_layers, scale=2.0).export_weights()
    wb = R.make_encoder(32, vocab, emb_sz, n_hid, n_layers, scale=2.0).export_weights()
    ids, lengths = _edge_ids(300, 17, vocab, 1, _lengths(300, 17, 5, seed=6), seed=7)
    enc = _handle(shape, wa, monkeypatch, None, flags)
    a = enc.encode_ids(ids, lengths)
    raw_a = enc.raw_features(ids)
    enc.load_weights(*wb)
    b = enc.encode_ids(ids, lengths)
    fresh = _handle(shape, wb, monkeypatch, None, flags)
    np.testing.assert_array_equal(b, fresh.encode_ids(ids, lengths))
    np.testing.assert_array_equal(enc.raw_features(ids), fresh.raw_features(ids))
    assert not np.array_equal(a, b)
    enc.load_weights(*wa)
    np.testing.assert_array_equal(enc.encode_ids(ids, lengths), a)
    np.testing.assert_array_equal(enc.raw_features(ids), raw_a)
    enc.close()
    fresh.close()
