"""CPU tests of the oracle itself: golden vectors, the reference's own invariant (bulk == single, atol 1e-5,
Issue_Embeddings/notebooks/04b_Inference-Batch.ipynb:369), the independent numpy restatement, padding invariance."""
import os

import numpy as np
import pytest
import torch

from oracle import awd_lstm_ref as R
from oracle import lstm_numpy as N


def _load_small(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name))
    n_layers, emb_sz, n_hid, vocab, seed = [int(x) for x in z["cfg"]]
    layers = [dict(w_ih=z[f"l{l}_w_ih"], w_hh=z[f"l{l}_w_hh"], b_ih=z[f"l{l}_b_ih"], b_hh=z[f"l{l}_b_hh"])
              for l in range(n_layers)]
    return z, (n_layers, emb_sz, n_hid, vocab, seed), layers


@pytest.mark.parametrize("name", ["encoder_tiny.npz", "encoder_pad_dims.npz"])
def test_golden_small_matches_both_restatements(golden_dir, name):
    z, (n_layers, emb_sz, n_hid, vocab, seed), layers = _load_small(golden_dir, name)
    enc = R.make_encoder(seed, vocab, emb_sz, n_hid, n_layers, scale=float(z["scale"]))
    # weights are re-derivable from the seed
    emb, lay = enc.export_weights()
    np.testing.assert_array_equal(emb, z["emb"])
    np.testing.assert_array_equal(lay[0]["w_hh"], z["l0_w_hh"])
    got = R.encode_padded(enc, z["ids"], z["lengths"])
    np.testing.assert_allclose(got, z["expected"], atol=1e-6)
    got64, _ = N.encode(z["emb"], layers, z["ids"], z["lengths"], dtype=np.float64)
    np.testing.assert_allclose(got64, z["expected"], atol=2e-6)


def test_golden_r4_config1_plumbing(golden_dir):
    """BASELINE.json configs[0]: 32 synthetic issues, seq_len 128, random-init R4 weights, CPU only."""
    z = np.load(os.path.join(golden_dir, "encoder_r4.npz"))
    n_layers, emb_sz, n_hid, vocab, seed = [int(x) for x in z["cfg"]]
    assert (n_layers, emb_sz, n_hid, vocab) == (4, 800, 2400, 60000)
    torch.set_num_threads(os.cpu_count())
    enc = R.make_encoder(seed, vocab, emb_sz, n_hid, n_layers)
    got = R.encode_padded(enc, z["ids"][:8], z["lengths"][:8])
    assert got.shape == (8, 2400) and got.dtype == np.float32
    np.testing.assert_allclose(got, z["expected"][:8], atol=1e-6)
    # single path on one issue == bulk row (the reference's invariant)
    single = R.encode_single(enc, z["ids"][3][: z["lengths"][3]])
    assert single.shape == (1, 2400)
    np.testing.assert_allclose(single[0], z["expected"][3], atol=1e-5)


def test_bulk_equals_single_and_order_restored():
    enc = R.make_encoder(5, 500, 32, 48, 3, scale=2.0)
    docs = R.synthetic_ids(45, 40, seed=9, vocab_sz=500, min_len=1)
    bulk = R.encode_bulk(enc, docs, bs=7)
    single = np.concatenate([R.encode_single(enc, d) for d in docs])
    assert np.allclose(bulk, single, atol=1e-5)
    # pool order is [mean | max | last]
    raw = enc(torch.as_tensor(docs[0])[None]).numpy()[0]
    np.testing.assert_allclose(bulk[0, :32], raw.mean(0), atol=1e-6)
    np.testing.assert_allclose(bulk[0, 32:64], raw.max(0), atol=1e-6)
    np.testing.assert_allclose(bulk[0, 64:], raw[-1], atol=1e-6)


def test_padding_and_batch_invariance():
    enc = R.make_encoder(6, 300, 16, 24, 2, scale=3.0)
    docs = R.synthetic_ids(6, 20, seed=2, vocab_sz=300, min_len=3)
    lengths = [len(d) for d in docs]
    def pad(T, pad_id):
        ids = np.full((len(docs), T), pad_id, dtype=np.int64)
        for i, d in enumerate(docs):
            ids[i, :len(d)] = d
        return ids
    a = R.encode_padded(enc, pad(20, 1), lengths)
    b = R.encode_padded(enc, pad(33, 1), lengths)       # more right padding
    c = R.encode_padded(enc, pad(20, 7), lengths)       # a different pad token
    np.testing.assert_allclose(a, b, atol=1e-6)
    np.testing.assert_allclose(a, c, atol=1e-6)


def test_negative_control_is_discriminative():
    """Raw cosine is nearly blind under random init (SURVEY.md section 7): the extra metrics must catch wrong ids."""
    enc = R.make_encoder(1, 400, 32, 64, 2)
    docs = R.synthetic_ids(8, 24, seed=3, vocab_sz=400)
    ids = np.stack(docs)
    lengths = [24] * 8
    ref = R.encode_padded(enc, ids, lengths)
    wrong = R.encode_padded(enc, np.roll(ids, 1, axis=0), lengths)
    m = R.parity_metrics(wrong, ref)
    assert m["rel_l2"] > 1e-2 and m["min_centred_cosine"] < 0.9
    ok = R.parity_metrics(ref, ref)
    assert ok["rel_l2"] == 0 and ok["min_cosine"] > 1 - 1e-12


def test_batch_seq_pool_asserts_like_reference():
    with pytest.raises(AssertionError):
        R.batch_seq_pool(np.zeros((2, 3, 4), np.float32), [3])


@pytest.mark.parametrize("tag", ["small", "prod"])
def test_mlp_numpy_restatement_matches_reference_fixture(golden_dir, tag):
    """mlp_ref_*.npz was produced by the reference's MLPWrapper.predict_probabilities."""
    coefs, intercepts, X, want = N.load_mlp_fixture(os.path.join(golden_dir, f"mlp_ref_{tag}.npz"))
    np.testing.assert_allclose(N.mlp_forward(X, coefs, intercepts), want, atol=2e-6)


def test_filter_labels_matches_reference_test_case():
    """py/label_microservice/repo_specific_model_test.py:10-33: probs [.2,.9], thresholds .5 -> {'label2': .9}."""
    out = N.filter_labels(["label1", "label2"], [.2, .9], {"label1": .5, "label2": .5})
    assert out == {"label2": .9}
    assert N.filter_labels(["a", "b"], [.9, .9], {"a": None, "b": 0}) == {}
