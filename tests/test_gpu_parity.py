"""GPU parity tests (run with -m gpu on an H100).  Everything goes through the C ABI (ctypes -> libissue_emb_b200.so);
the CPU oracle (oracle/) and the committed golden vectors (tests/golden/) are the checkers.

Tolerances (stated per BASELINE.json north_star: cosine >= 1 - 1e-4, max-abs reported):
  * bf16 operands, f32 accumulate / state / pooling  ->  per-issue cosine >= 1 - 1e-4 (mandated) AND, because raw
    cosine is nearly blind under random init (SURVEY.md section 7), rel-L2 <= 4e-3, centred cosine >= 0.99 and a
    negative control that must fail.
  * structural properties (batch/padding/prefix invariance, determinism) are bit-exact.
"""
import os

import numpy as np
import pytest
import torch

from oracle import awd_lstm_ref as R
from oracle import lstm_numpy as N

pytestmark = pytest.mark.gpu

COS_MIN = 1 - 1e-4
REL_L2_MAX = 4e-3          # torch-default init (|h| ~ 0.01)
REL_L2_MAX_SCALED = 1e-2   # "trained-like" weight sets (LSTM weights x2..x3, |h| ~ 0.1): bf16 rounding of h amplifies
CC_MIN_FULL = 0.985        # centred cosine at 512..2048 steps under torch-default init: the per-issue signal after
                           # removing the batch mean is ~1 % of the vector, so a rel-L2 far inside REL_L2_MAX reads only
                           # ~0.99 here; the permuted-rows negative control scores < 0.9


def _usable_cpus():
    """Affinity mask capped by the cgroup CPU quota: on the GPU boxes os.cpu_count() is far above what the container may
    use, and an oversubscribed OpenMP pool makes the CPU oracle orders of magnitude slower (tiny LSTM, 20 000 steps)."""
    import bench
    return bench.usable_cpus()


def _pad(docs, T=None, pad=1):
    T = T or max(len(d) for d in docs)
    ids = np.full((len(docs), T), pad, dtype=np.int64)
    for i, d in enumerate(docs):
        ids[i, :len(d)] = d
    return ids, np.array([len(d) for d in docs], dtype=np.int32)


def _assert_parity(got, want, cc_min=0.99, rel_l2_max=REL_L2_MAX):
    m = R.parity_metrics(got, want)
    assert np.isfinite(got).all()
    assert m["min_cosine"] >= COS_MIN, m
    assert m["rel_l2"] <= rel_l2_max, m
    if "min_centred_cosine" in m:
        assert m["min_centred_cosine"] >= cc_min, m
    return m


@pytest.fixture(scope="module")
def r4():
    """Reference-deployed shape (L=4, E=800, H=2400, V=60000), seed-1234 random init, on the GPU + its oracle."""
    from code_intelligence_b200 import IssueEncoder
    torch.set_num_threads(_usable_cpus())
    ref = R.make_encoder(1234)
    emb, layers = ref.export_weights()
    enc = IssueEncoder().load_weights(emb, layers)
    yield enc, ref
    enc.close()


def _small_from_golden(golden_dir, name):
    from code_intelligence_b200 import IssueEncoder
    z = np.load(os.path.join(golden_dir, name))
    n_layers, emb_sz, n_hid, vocab, seed = [int(x) for x in z["cfg"]]
    layers = [dict(w_ih=z[f"l{l}_w_ih"], w_hh=z[f"l{l}_w_hh"], b_ih=z[f"l{l}_b_ih"], b_hh=z[f"l{l}_b_hh"])
              for l in range(n_layers)]
    enc = IssueEncoder(n_layers, emb_sz, n_hid, vocab).load_weights(z["emb"], layers)
    return z, enc


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M,N,K,act", [(128, 16, 64, 0), (128, 80, 128, 0), (200, 240, 64, 0), (256, 480, 192, 0),
                                        (300, 600, 1600, 1), (1000, 250, 600, 2), (2048, 9600, 832, 0),
                                        (1024, 3200, 2432, 0)])
def test_tcgen05_gemm_vs_torch(M, N, K, act):
    """The wgmma GEMM behind ie_debug_gemm (the name is historical: it is the encoder's and the MLP head's GEMM)."""
    from code_intelligence_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(M + N + K)
    a = rng.standard_normal((M, K), dtype=np.float32)
    b = (rng.standard_normal((N, K), dtype=np.float32) / np.sqrt(K)).astype(np.float32)
    bias = rng.standard_normal(N, dtype=np.float32)
    d = np.zeros((M, N), dtype=np.float32)
    _lib.check(lib.ie_debug_gemm(a.ctypes.data, b.ctypes.data, bias.ctypes.data, M, N, K, act, d.ctypes.data, 0))
    ref = torch.from_numpy(a).bfloat16().double() @ torch.from_numpy(b).bfloat16().double().T + torch.from_numpy(bias).double()
    if act == 1:
        ref = ref.clamp_min(0)
    if act == 2:
        ref = torch.sigmoid(ref)
    # operands are identical (bf16-rounded); only the f32 accumulation order differs
    np.testing.assert_allclose(d, ref.numpy(), atol=2e-4 * np.sqrt(K / 64), rtol=1e-5)


# ------------------------------------------------------------------------------------------------ golden vectors
@pytest.mark.parametrize("name", ["encoder_tiny.npz", "encoder_pad_dims.npz"])
def test_golden_small(golden_dir, name):
    z, enc = _small_from_golden(golden_dir, name)
    got = enc.encode_ids(z["ids"], z["lengths"])
    assert got.shape == z["expected"].shape and got.dtype == np.float32
    _assert_parity(got, z["expected"], rel_l2_max=REL_L2_MAX if float(z["scale"]) == 1.0 else REL_L2_MAX_SCALED)
    enc.close()


@pytest.mark.parametrize("name,cc", [("encoder_r4.npz", 0.985), ("encoder_r4_varlen.npz", 0.999)])
def test_golden_r4(golden_dir, r4, name, cc):
    """encoder_r4.npz is BASELINE.json configs[0] (32 issues, seq_len 128) pushed through the GPU path."""
    enc, _ = r4
    z = np.load(os.path.join(golden_dir, name))
    scale = float(z["scale"])
    if scale != 1.0:
        from code_intelligence_b200 import IssueEncoder
        ref = R.make_encoder(1234, scale=scale)
        emb, layers = ref.export_weights()
        enc = IssueEncoder().load_weights(emb, layers)
    got = enc.encode_ids(z["ids"], z["lengths"])
    m = _assert_parity(got, z["expected"], cc_min=cc, rel_l2_max=REL_L2_MAX if scale == 1.0 else REL_L2_MAX_SCALED)
    print(name, m)
    # negative control: the same outputs against the expected vectors of *other* issues must fail the extra gates
    neg = R.parity_metrics(got, np.roll(z["expected"], 1, axis=0))
    assert neg["rel_l2"] > 2 * REL_L2_MAX
    if scale != 1.0:
        enc.close()


def test_golden_n3(golden_dir):
    """North-star wording: 3-layer AWD-LSTM (L=3, E=800, H=2400)."""
    from code_intelligence_b200 import IssueEncoder
    z = np.load(os.path.join(golden_dir, "encoder_n3.npz"))
    ref = R.make_encoder(1234, n_layers=3)
    emb, layers = ref.export_weights()
    enc = IssueEncoder(n_layers=3).load_weights(emb, layers)
    _assert_parity(enc.encode_ids(z["ids"], z["lengths"]), z["expected"])
    enc.close()


# ------------------------------------------------------------------------------------------------ live oracle
def test_r4_vs_oracle_varlen_batch(r4):
    enc, ref = r4
    docs = R.synthetic_ids(40, 72, seed=77, min_len=1)
    ids, lengths = _pad(docs, 72)
    got = enc.encode_ids(ids, lengths)
    want = R.encode_padded(ref, ids, lengths)
    m = _assert_parity(got, want)
    print("varlen", m)
    # permuted ids (negative control) must NOT pass
    wrong = enc.encode_ids(np.roll(ids, 1, axis=0), np.roll(lengths, 1))
    assert R.parity_metrics(wrong, want)["rel_l2"] > 2 * REL_L2_MAX


def test_bulk_equals_single_bit_exact(r4):
    """The reference's own invariant (04b_Inference-Batch.ipynb:369, atol 1e-5) holds exactly here: a row's result
    does not depend on its batch mates, on T, or on the pad token."""
    enc, _ = r4
    docs = R.synthetic_ids(9, 40, seed=5, min_len=1)
    bulk = enc.encode_id_list(docs, bs=4)
    single = np.concatenate([enc.encode_ids(d[None, :]) for d in docs])
    np.testing.assert_array_equal(bulk, single)
    ids, lengths = _pad(docs, 40)
    ids2, _ = _pad(docs, 57, pad=7)
    np.testing.assert_array_equal(enc.encode_ids(ids, lengths), enc.encode_ids(ids2, lengths))
    np.testing.assert_array_equal(enc.encode_ids(ids, lengths), bulk)


def test_raw_features_and_pooling_consistency(r4):
    enc, ref = r4
    docs = R.synthetic_ids(3, 33, seed=8)
    ids, lengths = _pad(docs)
    raw = enc.raw_features(ids)
    assert raw.shape == (3, 33, 800) and raw.dtype == np.float32
    want = ref(torch.as_tensor(ids)).numpy()
    assert np.abs(raw - want).max() < 2e-4 and np.linalg.norm(raw - want) / np.linalg.norm(want) < REL_L2_MAX
    pooled = enc.encode_ids(ids, lengths)
    np.testing.assert_allclose(pooled, np.concatenate([raw.mean(1), raw.max(1), raw[:, -1]], axis=1), atol=1e-6)


def test_edge_cases_and_errors(r4):
    enc, ref = r4
    one = enc.encode_ids(np.array([[2]], dtype=np.int64))                      # B=1, T=1
    want = R.encode_single(ref, np.array([2]))
    _assert_parity(one, want)
    np.testing.assert_allclose(one[0, :800], one[0, 800:1600])                 # mean == max == last for T=1
    docs = R.synthetic_ids(1500, 6, seed=3, min_len=2)                         # B > max_batch (1280) is sliced by the shim;
    ids, lengths = _pad(docs)                                                  # 1..5 batches of 256 rows ride one launch:
    got = enc.encode_ids(ids, lengths)                                         # identical bits whatever the company
    np.testing.assert_array_equal(got[256], enc.encode_ids(ids[256:257], lengths[256:257])[0])
    np.testing.assert_array_equal(got[:257], enc.encode_ids(ids[:257], lengths[:257]))
    np.testing.assert_array_equal(got[:600], enc.encode_ids(ids[:600], lengths[:600]))
    np.testing.assert_array_equal(got[1280:], enc.encode_ids(ids[1280:], lengths[1280:]))
    with pytest.raises(ValueError):
        enc.encode_ids(ids[:2], np.array([7, 1], dtype=np.int32))              # length > T
    with pytest.raises(ValueError):
        enc.encode_ids(ids[:2], np.array([0, 1], dtype=np.int32))              # length < 1
    bad = ids[:2].copy()
    bad[1, 3] = 60000
    with pytest.raises(ValueError):
        enc.encode_ids(bad, lengths[:2])                                       # token id outside the vocab
    assert np.isfinite(enc.encode_ids(ids[:2], lengths[:2])).all()            # handle still usable


KNOBS = ("IE_SEQ", "IE_COOP", "IE_EMB_PROJ", "IE_GX_BF16", "IE_BATCHES", "IE_CHUNK_T", "IE_FAST_MATH", "IE_MC",
         "IE_SPIN_LIMIT_MS", "IE_DEBUG_FAULT", "IE_FUSE_LAST")


def _make(cfg, weights, monkeypatch, env=None, flags=0):
    """Handle created under development knobs (read at ie_encoder_create; DESIGN.md section 4)."""
    from code_intelligence_b200 import IssueEncoder
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, str(v))
    enc = IssueEncoder(*cfg, 1, 0, flags).load_weights(*weights)
    for k in (env or {}):
        monkeypatch.delenv(k)
    return enc


@pytest.mark.parametrize("knobs", [{"IE_SEQ": 0}, {"IE_EMB_PROJ": 0}, {"IE_EMB_PROJ": 0, "IE_SEQ": 0}, {"IE_BATCHES": 3},
                                   {"IE_BATCHES": 8}, {"IE_CHUNK_T": 5}, {"IE_CHUNK_T": 1, "IE_EMB_PROJ": 0}, {"IE_COOP": 0},
                                   {"IE_MC": 1}, {"IE_MC": 0}, {"IE_MC": 1, "IE_BATCHES": 4, "IE_CHUNK_T": 7},
                                   {"IE_GX_BF16": 0, "_base": {"IE_GX_BF16": 0, "IE_SEQ": 0, "IE_CHUNK_T": 3}},
                                   {"IE_FAST_MATH": 0, "_base": {"IE_FAST_MATH": 0, "IE_SEQ": 0}},
                                   {"IE_BATCHES": 12, "IE_MC": 1}, {"IE_FUSE_LAST": 0, "_base": {"IE_FUSE_LAST": 0, "IE_SEQ": 0}},
                                   {"IE_FUSE_LAST": 0, "IE_BATCHES": 2, "IE_CHUNK_T": 6, "_base": {"IE_FUSE_LAST": 0}}])
def test_every_path_gives_identical_bits(knobs, monkeypatch):
    """One recurrent kernel (csrc/lstm_layer.cu), launched persistently or once per timestep (the fallback, IE_SEQ=0),
    with the cell arithmetic of csrc/lstm_common.cuh; the per-token input-projection table is the same GEMM on the same operands as gather + GEMM;
    batches per launch, time chunking and the cooperative attribute change the schedule, not the per-row arithmetic.
    All of them must reproduce the default path bit for bit, pooled and raw.  The one exception by construction: the
    persistent kernel fuses the LAST layer's input projection into its K loop (f32 sum, no fp16 Gx), which the
    per-timestep fallback cannot -- comparisons with the fallback run both sides with IE_FUSE_LAST=0
    (test_fused_last_layer covers the fused form)."""
    knobs = dict(knobs)
    base_env = knobs.pop("_base", None)
    if knobs.get("IE_SEQ") == 0 or (base_env or {}).get("IE_SEQ") == 0:
        knobs["IE_FUSE_LAST"] = 0
        base_env = dict(base_env or {}, IE_FUSE_LAST=0)
    cfg = (3, 96, 200, 500)
    weights = R.make_encoder(7, cfg[3], cfg[1], cfg[2], cfg[0]).export_weights()
    base = _make(cfg, weights, monkeypatch, base_env)
    exp = _make(cfg, weights, monkeypatch, knobs)
    for B, T in ((1, 7), (300, 19), (700, 23), (min(base.max_batch, exp.max_batch), 11)):
        docs = R.synthetic_ids(B, T, seed=B + T, vocab_sz=cfg[3], min_len=1)
        ids, lengths = _pad(docs, T)
        np.testing.assert_array_equal(exp.encode_ids(ids, lengths), base.encode_ids(ids, lengths))
        if B <= 300:
            np.testing.assert_array_equal(exp.raw_features(ids), base.raw_features(ids))
    base.close()
    exp.close()


def test_fused_last_layer(monkeypatch):
    """The last layer's input projection inside the recurrent K loop (default) against the hoisted GEMM form
    (IE_FUSE_LAST=0) and against the oracle: the fused sum W_ih x + W_hh h + b never leaves f32, so it must be at least as
    close to the oracle as the hoisted form, and the two forms agree to fp16-Gx rounding.  Shapes: padded dims (K of the
    previous layer 200 -> 256), 1..5 batches per launch, time chunks, raw features."""
    cfg = (3, 96, 200, 500)
    ref = R.make_encoder(7, cfg[3], cfg[1], cfg[2], cfg[0], scale=2.0)
    weights = ref.export_weights()
    fused = _make(cfg, weights, monkeypatch)
    hoist = _make(cfg, weights, monkeypatch, {"IE_FUSE_LAST": 0})
    chunked = _make(cfg, weights, monkeypatch, {"IE_CHUNK_T": 4, "IE_BATCHES": 2})
    for B, T in ((1, 9), (130, 19), (700, 23), (1280, 6)):
        docs = R.synthetic_ids(B, T, seed=B + T, vocab_sz=cfg[3], min_len=1)
        ids, lengths = _pad(docs, T)
        a, b = fused.encode_ids(ids, lengths), hoist.encode_ids(ids, lengths)
        assert not np.array_equal(a, b)                      # really two different code paths
        np.testing.assert_allclose(a, b, rtol=0, atol=3e-3)
        np.testing.assert_array_equal(chunked.encode_ids(ids, lengths), a)
        sel = np.arange(min(B, 32))
        want = R.encode_padded(ref, ids[sel], lengths[sel])
        ma, mb = R.parity_metrics(a[sel], want), R.parity_metrics(b[sel], want)
        assert ma["min_cosine"] >= COS_MIN and ma["rel_l2"] <= REL_L2_MAX_SCALED, ma
        assert ma["rel_l2"] <= 1.25 * mb["rel_l2"], (ma, mb)
        if B <= 130:
            np.testing.assert_allclose(fused.raw_features(ids), hoist.raw_features(ids), rtol=0, atol=3e-3)
            np.testing.assert_array_equal(fused.raw_features(ids), chunked.raw_features(ids))
    for e in (fused, hoist, chunked):
        e.close()


def test_shape_sweep_vs_oracle_and_bulk_pipeline(monkeypatch):
    """Batch sizes around every internal boundary (1, 256 +- 1, 512 +- 1, 1280 +- 1: batches per launch, slices of the host
    shim) x sequence lengths down to a single token, ragged lengths, against the oracle; then the bulk pipeline
    (length sort, pinned double-buffered staging, device un-sort) on 3000 ragged issues against row-by-row calls."""
    cfg = (2, 64, 128, 300)
    ref = R.make_encoder(11, cfg[3], cfg[1], cfg[2], cfg[0], scale=2.0)
    enc = _make(cfg, ref.export_weights(), monkeypatch)
    rng = np.random.default_rng(0)
    for B in (1, 2, 255, 256, 257, 511, 513, 1279, 1280, 1281, 1300):
        for T in (1, 2, 3, 17):
            docs = R.synthetic_ids(B, T, seed=B * 31 + T, vocab_sz=cfg[3], min_len=1)
            ids, lengths = _pad(docs, T)
            got = enc.encode_ids(ids, lengths)
            sel = rng.choice(B, size=min(B, 24), replace=False)
            want = R.encode_padded(ref, ids[sel], lengths[sel])
            m = R.parity_metrics(got[sel], want)
            assert np.isfinite(got).all() and m["min_cosine"] >= COS_MIN and m["rel_l2"] <= REL_L2_MAX_SCALED, (B, T, m)
            np.testing.assert_array_equal(got[-1], enc.encode_ids(ids[-1:, :lengths[-1]])[0])   # last row, alone, unpadded
    docs = R.synthetic_ids(3000, 40, seed=5, vocab_sz=cfg[3], min_len=1)
    bulk_out = enc.encode_id_list(docs, bs=100)
    assert bulk_out.shape == (3000, 192)
    # the result array owns its (page-locked) memory: a later bulk call of the same size must not overwrite it
    keep = bulk_out.copy()
    other = enc.encode_id_list(docs[::-1], bs=100)
    np.testing.assert_array_equal(bulk_out, keep)
    np.testing.assert_array_equal(other[::-1], keep)
    for i in rng.choice(3000, size=40, replace=False):
        np.testing.assert_array_equal(bulk_out[i], enc.encode_ids(docs[i][None, :])[0])
    with pytest.raises(ValueError):
        enc.encode_id_list([np.array([2, 5, 299, 300])])                        # token id outside the vocabulary
    enc.close()


# ------------------------------------------------------------------------------------------------ full-size goldens
def _golden_full(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name))
    return z["ids"].astype(np.int64), z["lengths"].astype(np.int32), z["expected"]


def test_golden_r4_bench_shape_all_rows(golden_dir, r4):
    """BASELINE.json configs[1] shape, 48 rows x 512 tokens of the 256-row bench batch (32 full-length, 16 var-len) against
    the committed oracle output (tests/golden/make_golden.py full): once as one call and once riding a five-batch launch
    (the mode bench.py times), where the golden rows are spread over all five batches."""
    enc, _ = r4
    ids, lengths, want = _golden_full(golden_dir, "encoder_r4_b256_t512.npz")
    got = enc.encode_ids(ids, lengths)
    m = _assert_parity(got, want, cc_min=CC_MIN_FULL)
    print("r4 48x512 single batch", m)
    neg = R.parity_metrics(got, np.roll(want, 1, axis=0))
    assert neg["rel_l2"] > 2 * REL_L2_MAX and neg["min_centred_cosine"] < 0.9
    rng = np.random.default_rng(5)
    filler = rng.integers(2, 60000, size=(enc.max_batch - len(ids), 512))
    big = np.concatenate([ids, filler])
    perm = rng.permutation(enc.max_batch)
    big_len = np.concatenate([lengths, np.full(enc.max_batch - len(ids), 512, dtype=np.int32)])
    got5 = enc.encode_ids(big[perm], big_len[perm])[np.argsort(perm)][:len(ids)]
    np.testing.assert_array_equal(got5, got)          # batch composition / position never changes a row's bits


@pytest.mark.parametrize("name,T", [("encoder_r4_t1024.npz", 1024), ("encoder_r4_t2048.npz", 2048)])
def test_golden_r4_long_buckets(golden_dir, r4, name, T):
    """BASELINE.json configs[2] buckets 1024 and 2048 (lengths in (T/2, T]), 32 issues each, against the oracle; also as
    part of a multi-batch call."""
    enc, _ = r4
    ids, lengths, want = _golden_full(golden_dir, name)
    assert ids.shape[1] == T
    got = enc.encode_ids(ids, lengths)
    m = _assert_parity(got, want, cc_min=CC_MIN_FULL)
    print(name, m)
    rep = np.concatenate([ids] * 17)[:513]            # 513 rows: three 256-row batches in one launch
    got3 = enc.encode_ids(rep, np.concatenate([lengths] * 17)[:513])
    np.testing.assert_array_equal(got3[:32], got)
    np.testing.assert_array_equal(got3[480:512], got)


def test_golden_n3_full(golden_dir):
    """North-star wording: 3-layer AWD-LSTM, 64 issues x 512 tokens."""
    from code_intelligence_b200 import IssueEncoder
    ids, lengths, want = _golden_full(golden_dir, "encoder_n3_b64_t512.npz")
    emb, layers = R.make_encoder(1234, n_layers=3).export_weights()
    enc = IssueEncoder(n_layers=3).load_weights(emb, layers)
    m = _assert_parity(enc.encode_ids(ids, lengths), want, cc_min=0.99)
    print("n3 64x512", m)
    enc.close()


# ------------------------------------------------------------------------------------------------ fp32-accurate mode
def test_fp32_accurate_mode(golden_dir, monkeypatch):
    """BASELINE.json configs[1] in fp32: IE_CFG_FP32 = split-bf16 products (hi*hi + lo*hi + hi*lo,
    f32 accumulate), f32 input projections, IEEE gates.  Stated tolerance vs the fp32 oracle: rel-L2 <= 2e-5,
    max-abs <= 2e-6, cosine >= 1 - 1e-9 (the bf16 default is ~8e-4 / 6e-5)."""
    from code_intelligence_b200 import _lib
    z, _ = None, None
    cfg = (3, 96, 200, 500)
    ref = R.make_encoder(7, cfg[3], cfg[1], cfg[2], cfg[0], scale=2.0)
    weights = ref.export_weights()
    acc = _make(cfg, weights, monkeypatch, None, flags=_lib.IE_CFG_FP32)
    fb = _make(cfg, weights, monkeypatch, {"IE_SEQ": 0, "IE_EMB_PROJ": 0, "IE_CHUNK_T": 4}, flags=_lib.IE_CFG_FP32)
    docs = R.synthetic_ids(300, 33, seed=3, vocab_sz=cfg[3], min_len=1)
    ids, lengths = _pad(docs, 33)
    got = acc.encode_ids(ids, lengths)
    want = R.encode_padded(ref, ids, lengths)
    m = R.parity_metrics(got, want)
    print("fp32 mode small", m)
    assert m["rel_l2"] <= 2e-5 and m["max_abs"] <= 5e-6 and m["min_cosine"] >= 1 - 1e-9, m
    np.testing.assert_array_equal(fb.encode_ids(ids, lengths), got)     # fallback kernel, gather + GEMM, chunked: same bits
    acc.close()
    fb.close()
    # reference shape: the 48 rows of the bench-shape golden (seq_len 512; 32 full-length, 16 var-len)
    from code_intelligence_b200 import IssueEncoder
    ids, lengths, want = _golden_full(golden_dir, "encoder_r4_b256_t512.npz")
    emb, layers = R.make_encoder(1234).export_weights()
    enc = IssueEncoder(flags=_lib.IE_CFG_FP32).load_weights(emb, layers)
    got = enc.encode_ids(ids[:48], lengths[:48])
    m = R.parity_metrics(got, want[:48])
    print("fp32 mode R4 48x512", m)
    assert m["rel_l2"] <= 2e-5 and m["max_abs"] <= 2e-6 and m["min_cosine"] >= 1 - 1e-9, m
    enc.close()


# ------------------------------------------------------------------------------------------------ robustness of the C ABI
def test_device_wait_timeout_is_an_error_code_not_a_trap(monkeypatch):
    """IE_DEBUG_FAULT drops one (step, batch) counter update inside the persistent kernel: every CTA pair that needs
    it spins.  The abort protocol (csrc/ptx.cuh) must turn that into IE_ERR_CUDA within the spin limit -- no __trap(),
    so the CUDA context survives: other handles, and new ones, keep working in the same process."""
    import time
    cfg = (2, 64, 128, 300)
    weights = R.make_encoder(5, cfg[3], cfg[1], cfg[2], cfg[0]).export_weights()
    good = _make(cfg, weights, monkeypatch)
    bad = _make(cfg, weights, monkeypatch, {"IE_DEBUG_FAULT": 1, "IE_SPIN_LIMIT_MS": 100})
    docs = R.synthetic_ids(20, 9, seed=1, vocab_sz=cfg[3])
    ids, lengths = _pad(docs, 9)
    want = good.encode_ids(ids, lengths)
    t0 = time.time()
    with pytest.raises(RuntimeError, match="wait exceeded"):
        bad.encode_ids(ids, lengths)
    assert time.time() - t0 < 20
    np.testing.assert_array_equal(good.encode_ids(ids, lengths), want)         # context not poisoned
    again = _make(cfg, weights, monkeypatch)
    np.testing.assert_array_equal(again.encode_ids(ids, lengths), want)
    for e in (good, bad, again):
        e.close()


def test_two_handles_concurrently_and_device_mode_errors(monkeypatch):
    """Two handles on one device driven from two host threads (cooperative launches serialise instead of deadlocking);
    device-pointer mode reports data-dependent errors through ie_encoder_check_errors."""
    import threading
    cfg = (2, 64, 128, 300)
    weights = R.make_encoder(5, cfg[3], cfg[1], cfg[2], cfg[0]).export_weights()
    a = _make(cfg, weights, monkeypatch)
    b = _make(cfg, weights, monkeypatch)
    docs = R.synthetic_ids(600, 40, seed=2, vocab_sz=cfg[3], min_len=3)
    ids, lengths = _pad(docs, 40)
    want = a.encode_ids(ids, lengths)
    outs = {}
    def work(name, enc):
        outs[name] = [enc.encode_ids(ids, lengths) for _ in range(6)]
    ths = [threading.Thread(target=work, args=(n, e)) for n, e in (("a", a), ("b", b))]
    [t.start() for t in ths]
    [t.join() for t in ths]
    for n in ("a", "b"):
        for o in outs[n]:
            np.testing.assert_array_equal(o, want)
    # device-pointer mode
    dev = torch.device("cuda", 0)
    ids_d = torch.as_tensor(ids[:50], device=dev)
    len_d = torch.as_tensor(lengths[:50], device=dev)
    s = torch.cuda.Stream(dev)
    with pytest.raises(ValueError, match="out must be"):
        a.encode_ids_device(ids_d, len_d, torch.empty((10, 192), device=dev))   # too small for 50 rows: refused
    out = a.encode_ids_device(ids_d, len_d, stream=s)
    a.check_errors()
    np.testing.assert_array_equal(out.cpu().numpy(), want[:50])
    bad_ids = ids_d.clone()
    bad_ids[3, 2] = 300
    a.encode_ids_device(bad_ids, len_d)
    with pytest.raises(ValueError, match="token id"):
        a.check_errors()
    bad_len = len_d.clone()
    bad_len[7] = 0
    out = a.encode_ids_device(ids_d, bad_len)
    with pytest.raises(ValueError, match="length"):
        a.check_errors()
    assert torch.isfinite(out).all()                      # the length was clamped, not divided by
    out = a.encode_ids_device(ids_d, len_d)               # state cleared, handle usable
    a.check_errors()
    np.testing.assert_array_equal(out.cpu().numpy(), want[:50])
    a.close()
    b.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs in one process")
def test_two_devices_from_one_process(monkeypatch):
    """Function attributes (dynamic shared memory opt-in) are per device: a second GPU driven from the same process
    must work (round-1 defect: a process-wide `static bool attr_set`)."""
    from code_intelligence_b200 import IssueEncoder
    cfg = (2, 64, 128, 300)
    weights = R.make_encoder(5, cfg[3], cfg[1], cfg[2], cfg[0]).export_weights()
    docs = R.synthetic_ids(300, 12, seed=4, vocab_sz=cfg[3], min_len=2)
    ids, lengths = _pad(docs, 12)
    e0 = IssueEncoder(*cfg, 1, 0).load_weights(*weights)
    e1 = IssueEncoder(*cfg, 1, 1).load_weights(*weights)
    np.testing.assert_array_equal(e0.encode_ids(ids, lengths), e1.encode_ids(ids, lengths))
    e0.close()
    e1.close()


def test_very_long_issue_is_chunked(monkeypatch):
    """A single issue longer than the round-1 cap (16384 tokens): time chunking bounds the workspace, the result equals
    the prefix-property reference (same model on the first tokens) and the oracle."""
    cfg = (2, 64, 128, 300)
    ref = R.make_encoder(9, cfg[3], cfg[1], cfg[2], cfg[0], scale=2.0)
    enc = _make(cfg, ref.export_weights(), monkeypatch)
    T = 20000
    doc = R.synthetic_ids(1, T, seed=6, vocab_sz=cfg[3])[0]
    got = enc.encode_ids(doc[None, :])
    nthreads = torch.get_num_threads()
    torch.set_num_threads(min(4, nthreads))     # 20 000 tiny steps: thread-pool barriers would dominate
    want = R.encode_single(ref, doc)
    torch.set_num_threads(nthreads)
    _assert_parity(got, want, rel_l2_max=REL_L2_MAX_SCALED)
    short = enc.encode_ids(doc[None, :], np.array([5000], dtype=np.int32))
    np.testing.assert_array_equal(short, enc.encode_ids(doc[None, :5000]))
    enc.close()


def test_full_size_batch_properties(r4):
    """BASELINE.json configs[1] shape (batch 256, seq_len 512): size-independent properties + oracle on a slice."""
    enc, ref = r4
    docs = R.synthetic_ids(256, 512, seed=99)
    ids = np.stack(docs)
    lengths = np.full(256, 512, dtype=np.int32)
    a = enc.encode_ids(ids, lengths)
    assert a.shape == (256, 2400) and np.isfinite(a).all()
    np.testing.assert_array_equal(a, enc.encode_ids(ids, lengths))                              # deterministic
    assert (a[:, 800:1600] >= a[:, :800] - 1e-6).all()                                          # max >= mean
    perm = np.random.default_rng(0).permutation(256)
    np.testing.assert_array_equal(enc.encode_ids(ids[perm], lengths)[np.argsort(perm)], a)      # row equivariance
    short = np.full(256, 100, dtype=np.int32)                                                   # prefix property
    np.testing.assert_array_equal(enc.encode_ids(ids, short), enc.encode_ids(ids[:, :100].copy(), short))
    ids2 = np.concatenate([ids, ids[::-1]])                                                     # two batches per launch
    b = enc.encode_ids(ids2, np.full(512, 512, dtype=np.int32))
    np.testing.assert_array_equal(b[:256], a)
    np.testing.assert_array_equal(b[256:], a[::-1])
    ids5 = np.concatenate([ids, ids[::-1], ids[perm], ids, ids[perm][::-1]])                    # five batches per launch
    c5 = enc.encode_ids(ids5, np.full(1280, 512, dtype=np.int32))                               # (what bench.py times)
    np.testing.assert_array_equal(c5[:256], a)
    np.testing.assert_array_equal(c5[256:512], a[::-1])
    np.testing.assert_array_equal(c5[512:768], a[perm])
    np.testing.assert_array_equal(c5[768:1024], a)
    np.testing.assert_array_equal(c5[1024:], a[perm][::-1])


def test_oom_halving_and_threads(r4, monkeypatch):
    """IE_ERR_OOM surfaces as RuntimeError, so the reference's batch-halving loop (py/code_intelligence/inference.py:214-223)
    keeps working; one handle may be driven from several host threads (calls are serialised inside the library)."""
    import threading
    enc, _ = r4
    docs = R.synthetic_ids(300, 24, seed=13, min_len=4)
    want = enc.encode_id_list(docs, bs=300, min_batches_rule=False)
    monkeypatch.setenv("IE_MAX_TOKENS", str(256 * 24))           # only B_pad = 256 fits: bs 300 -> 150
    np.testing.assert_array_equal(enc.encode_id_list(docs, bs=300, min_batches_rule=False), want)
    monkeypatch.setenv("IE_MAX_TOKENS", "128")                    # nothing with T > 1 fits: the loop gives up at bs == 1
    with pytest.raises(Exception):
        enc.encode_id_list(docs, bs=4, min_batches_rule=False)
    monkeypatch.delenv("IE_MAX_TOKENS")
    outs = [None] * 4
    def work(i):
        outs[i] = enc.encode_id_list(docs[i * 10:(i + 1) * 10], bs=10, min_batches_rule=False)
    ths = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    np.testing.assert_array_equal(np.concatenate(outs), want[:40])


# ------------------------------------------------------------------------------------------------ python surface
def test_inference_wrapper_surface(tmp_path):
    from code_intelligence_b200.inference import InferenceWrapper, text_endpoint_bytes
    ref = R.make_encoder(21, 300, 32, 48, 2)
    sd = {"encoder.weight": ref.encoder.weight.detach().numpy()}
    for l, rnn in enumerate(ref.rnns):
        sd[f"rnns.{l}.weight_hh_l0_raw"] = rnn.weight_hh_l0.detach().numpy()
        sd[f"rnns.{l}.module.weight_ih_l0"] = rnn.weight_ih_l0.detach().numpy()
        sd[f"rnns.{l}.module.weight_hh_l0"] = rnn.weight_hh_l0.detach().numpy()
        sd[f"rnns.{l}.module.bias_ih_l0"] = rnn.bias_ih_l0.detach().numpy()
        sd[f"rnns.{l}.module.bias_hh_l0"] = rnn.bias_hh_l0.detach().numpy()
    itos = ["xxunk", "xxpad", "xxbos", "xxfld", "xxmaj", "xxup", "xxrep", "xxwrep", "xxxfldtitle", "xxxfldbody"] + \
           [f"w{i}" for i in range(290)]
    np.savez(tmp_path / "enc.npz", itos=np.array(itos), **sd)
    w = InferenceWrapper(tmp_path, "enc.npz")
    text = w.process_dict({"title": "w1 w2 W3", "body": "w4 w5"})["text"]
    assert text.startswith("xxxfldtitle ") and " xxxfldbody " in text
    ids = w.numericalize_one(text)
    assert ids.shape[0] == 1 and int(ids[0, 0]) == 2
    pooled = w.get_pooled_features(text)
    assert isinstance(pooled, torch.Tensor) and tuple(pooled.shape) == (1, 96)
    raw = w.get_raw_features(text)
    assert tuple(raw.shape) == (1, ids.shape[1], 32)
    want = R.encode_single(ref, ids[0].numpy())
    _assert_parity(pooled.detach().cpu().numpy(), want, rel_l2_max=REL_L2_MAX_SCALED)
    b = text_endpoint_bytes(w, "w1 w2 W3", "w4 w5")
    assert len(b) == 96 * 4
    np.testing.assert_array_equal(np.frombuffer(b, dtype="<f4"), pooled.numpy()[0])
    import pandas as pd
    df = pd.DataFrame({"title": ["w1", "w2 w3", "W9 w8"], "body": ["w4 w5 w6", "w7", "w1 w1 w1 w1 w1"]})
    embs = w.df_to_embedding(df)
    assert embs.shape == (3, 96) and embs.dtype == np.float32
    np.testing.assert_array_equal(embs[1:2], w.get_pooled_features(w.process_dict(df.iloc[1].to_dict())["text"]).numpy())
    np.testing.assert_array_equal(w.df_to_emb(df), embs)

    # torch checkpoints with fastai 1.0.53's module tree (SURVEY.md section 8c key list): `save_encoder` writes
    # torch.save(model[0].state_dict()); `learn.save` writes {'model': SequentialRNN state dict ('0.' = encoder,
    # '1.' = decoder head), 'opt': ...}.  In both the authoritative W_hh is `weight_hh_l0_raw` -- `module.weight_hh_l0`
    # holds the last DROPPED copy of a training step, so it is filled with garbage here and must be ignored.
    class WeightDropout(torch.nn.Module):
        def __init__(self, module):
            super().__init__()
            self.module = module
            self.weight_hh_l0_raw = torch.nn.Parameter(module.weight_hh_l0.data.clone())
            module.weight_hh_l0.data.normal_()

    class EmbeddingDropout(torch.nn.Module):
        def __init__(self, emb):
            super().__init__()
            self.emb = emb

    class AwdLstmTree(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.encoder = torch.nn.Embedding(300, 32, padding_idx=1)
            self.encoder.weight.data.copy_(ref.encoder.weight.data)
            self.encoder_dp = EmbeddingDropout(self.encoder)
            rnns = []
            for l, r in enumerate(ref.rnns):
                m = torch.nn.LSTM(r.input_size, r.hidden_size, 1, batch_first=True)
                m.load_state_dict(r.state_dict())
                rnns.append(WeightDropout(m))
            self.rnns = torch.nn.ModuleList(rnns)

    tree = AwdLstmTree()
    keys = set(tree.state_dict().keys())
    assert {"encoder.weight", "encoder_dp.emb.weight", "rnns.0.weight_hh_l0_raw", "rnns.1.module.weight_ih_l0",
            "rnns.1.module.weight_hh_l0", "rnns.0.module.bias_ih_l0", "rnns.0.module.bias_hh_l0"} <= keys
    torch.save(tree.state_dict(), tmp_path / "enc_save_encoder.pth")
    full = {"0." + k: v for k, v in tree.state_dict().items()}
    full["1.decoder.weight"] = tree.encoder.weight.data.clone()
    full["1.decoder.bias"] = torch.zeros(300)
    torch.save({"model": full, "opt": {}}, tmp_path / "learn_save.pth")
    for name in ("enc_save_encoder.pth", "learn_save.pth"):
        wp = InferenceWrapper(tmp_path, name, numericalizer=w._numericalizer)
        np.testing.assert_array_equal(wp.get_pooled_features(text).numpy(), pooled.numpy())
        wp.encoder.close()


def test_bulk_api_vs_the_reference_driver_output(golden_dir, monkeypatch):
    """The CUDA path through its public bulk API against arrays the REFERENCE'S OWN df_to_embedding / batch_seq_pool
    code returned (tests/golden/reference_driver.npz; executed in the build container around the CPU oracle's nn.LSTM
    stack, make_golden.py driver): 57 / 130 / 300 ragged issues, the reference's batch-size rule, its OOM halving."""
    from test_host_logic import _driver_fixture
    z, cases = _driver_fixture(golden_dir)
    n_layers, emb_sz, n_hid, vocab = [int(v) for v in z["cfg"]]
    ref = R.make_encoder(int(z["seed"]), vocab, emb_sz, n_hid, n_layers, scale=float(z["scale"]))
    enc = _make((n_layers, emb_sz, n_hid, vocab), ref.export_weights(), monkeypatch)
    for tag, c in cases.items():
        got = enc.encode_id_list(c["docs"], bs=c["bs"])
        m = _assert_parity(got, c["expected"], rel_l2_max=REL_L2_MAX_SCALED)
        print("reference driver", tag, m)
    one = z["single_ids"].astype(np.int64)
    _assert_parity(enc.encode_ids(one[None, :]), z["single_expected"], rel_l2_max=REL_L2_MAX_SCALED)
    enc.close()


# ------------------------------------------------------------------------------------------------ MLP head
@pytest.mark.parametrize("tag", ["small", "prod"])
def test_mlp_head_vs_reference_fixture(golden_dir, tag):
    """mlp_ref_*.npz holds MLPWrapper.predict_probabilities outputs produced by the reference code itself."""
    from code_intelligence_b200.mlp import MLPHead, filter_predictions
    coefs, intercepts, X, want = N.load_mlp_fixture(os.path.join(golden_dir, f"mlp_ref_{tag}.npz"))
    head = MLPHead(coefs, intercepts)
    probs = head.predict_proba(X)
    assert probs.shape == want.shape
    err = np.abs(probs - want)
    print(tag, "max abs prob diff", err.max())
    assert err.max() < 5e-3                      # bf16 operands, f32 accumulate
    # label-set agreement after thresholding (repo_specific_model.py:138-146), away from the decision boundary
    names = [f"l{i}" for i in range(probs.shape[1])]
    thr = {nm: 0.5 for nm in names}
    agree = 0
    for r in range(probs.shape[0]):
        a = set(filter_predictions(names, probs[r], thr))
        b = set(filter_predictions(names, want[r], thr))
        near = {nm for i, nm in enumerate(names) if abs(want[r, i] - 0.5) < 5e-3}
        assert (a ^ b) <= near
        agree += a == b
    assert agree >= 0.98 * probs.shape[0]
    head.close()


def test_mlp_wrapper_matches_sklearn():
    from sklearn.neural_network import MLPClassifier
    from code_intelligence_b200.mlp import MLPWrapper
    rng = np.random.default_rng(0)
    X = rng.random((60, 12)).astype(np.float32)
    y = rng.choice([0, 1], size=(60, 4))
    clf = MLPClassifier(random_state=1234, max_iter=30)
    w = MLPWrapper(clf=clf)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        w.fit(X, y)
    Xt = rng.random((300, 12)).astype(np.float32)
    np.testing.assert_allclose(w.predict_probabilities(Xt), clf.predict_proba(Xt), atol=5e-3)


def test_reference_test_mlp_cases_on_the_gpu_wrapper():
    """The reference's own unit tests of the head (Label_Microservice/tests/test_mlp.py:7-57), body for body, with
    code_intelligence_b200.mlp.MLPWrapper (sklearn fit, GPU predict_proba + ie_pr_thresholds) in place of
    label_microservice.mlp.MLPWrapper."""
    import warnings
    from sklearn.neural_network import MLPClassifier
    from code_intelligence_b200.mlp import MLPWrapper
    warnings.simplefilter("ignore")
    # test_predict_probabilities
    n_classes, n_samples, embedding_size, random_state = 5, 20, 5, 1234
    rs = np.random.RandomState(0)
    X_train = rs.rand(n_samples, embedding_size)
    y_train = rs.choice([0, 1], size=(n_samples, n_classes))
    X_test = rs.rand(n_samples, embedding_size)
    mlp_clf = MLPClassifier(random_state=random_state)
    mlp_clf.fit(X_train, y_train)
    mlp_clf_pred = mlp_clf.predict_proba(X_test)
    mlp_wrap = MLPWrapper(clf=mlp_clf)
    mlp_wrap.fit(X_train, y_train)
    mlp_wrap_pred = mlp_wrap.predict_probabilities(X_test)
    assert mlp_clf_pred.all() == mlp_wrap_pred.all()                         # the reference's (weak) assertion ...
    np.testing.assert_allclose(mlp_wrap_pred, mlp_clf_pred, atol=5e-3)       # ... and what it means
    # test_find_probability_thresholds
    X = np.array([[0.1, 0.1], [0.2, 0.2], [0.3, 0.3], [0.4, 0.4], [0.5, 0.5], [0.6, 0.6]])
    y = np.array([[1, 0, 0], [1, 0, 0], [0, 1, 0], [0, 1, 0], [0, 0, 1], [0, 0, 1]])
    precision_threshold, recall_threshold = 0.7, 0.5
    mlp_wrap = MLPWrapper(clf=MLPClassifier(random_state=random_state), precision_threshold=precision_threshold,
                          recall_threshold=recall_threshold)
    mlp_wrap.find_probability_thresholds(X, y)
    thresholds = mlp_wrap.probability_thresholds
    precision_0, recall_0 = mlp_wrap.precisions[0], mlp_wrap.recalls[0]
    assert not thresholds[1] and not thresholds[2] and \
        precision_0 >= precision_threshold and recall_0 >= recall_threshold


def test_threshold_search_on_device_vs_reference_fixture(golden_dir):
    """ie_pr_thresholds against the thresholds / precisions / recalls the reference's own
    MLPWrapper.find_probability_thresholds computed (tests/golden/thresholds_ref.npz, make_golden.py thresholds)."""
    from code_intelligence_b200.mlp import pr_thresholds
    from test_host_logic import _check_thresholds_fixture
    _check_thresholds_fixture(pr_thresholds, golden_dir)


def test_threshold_search_on_device_matches_sklearn_loop():
    """ie_pr_thresholds (csrc/pr_curve.cu) against the reference's per-label loop on sklearn's precision_recall_curve
    (py/label_microservice/mlp.py:81-98): identical thresholds, precisions, recalls -- with ties in the scores, labels
    without positives, labels that never qualify, and n that is not a power of two."""
    from code_intelligence_b200.mlp import pr_thresholds, pr_thresholds_host
    rng = np.random.default_rng(3)
    for n, L, quant in ((37, 5, 10), (1000, 40, 50), (5000, 17, 0), (16384, 3, 1000)):
        truth = (rng.random((n, L)) < rng.uniform(0.02, 0.6, size=L)).astype(np.uint8)
        signal = rng.uniform(0.0, 3.0, size=L)                         # some labels learnable, some not
        logits = rng.standard_normal((n, L)) + signal * (truth * 2.0 - 1.0)
        scores = (1.0 / (1.0 + np.exp(-logits))).astype(np.float32)
        if quant:
            scores = (np.round(scores * quant) / quant).astype(np.float32)   # many ties
        truth[:, 0] = 0                                                 # a label without positives
        for p_thr, r_thr in ((0.7, 0.5), (0.0, 0.0), (0.99, 0.99)):
            got = pr_thresholds(scores, truth, p_thr, r_thr)
            want = pr_thresholds_host(scores, truth, p_thr, r_thr)
            assert got[0] == want[0], (n, L, quant, p_thr)
            np.testing.assert_array_equal(np.array(got[1]), np.array(want[1]))
            np.testing.assert_array_equal(np.array(got[2]), np.array(want[2]))
        assert want[0][0] is None
