"""Generates the committed golden fixtures in tests/golden/.  Run in the build container:

    python tests/golden/make_golden.py

* encoder_*.npz   -- outputs of the torch-module oracle (oracle/awd_lstm_ref.py; the modules fastai 1.0.53 wraps:
                     the reference's own encoder is not importable here, SURVEY.md section 8c) on seeded inputs.
                     Small configs carry their weights; the reference-shape (R4 / N3) fixtures carry only ids and
                     expected outputs -- their weights are re-derived from the seed (torch CPU RNG is deterministic).
* mlp_ref_*.npz   -- produced by IMPORTING THE REFERENCE: label_microservice.mlp.MLPWrapper (py/label_microservice/mlp.py:56-63)
                     around an sklearn MLPClassifier; 'small' stores the fitted coefs_, intercepts_, inputs and the
                     MLPWrapper.predict_probabilities outputs, 'prod' the seed of its weights and inputs
                     (oracle.lstm_numpy.seeded_mlp) and the outputs.
* thresholds_ref.npz (`make_golden.py thresholds`) -- the reference's MLPWrapper.find_probability_thresholds (mlp.py:65-98)
                     executed on preset scores.
* reference_driver.npz (`make_golden.py driver`) -- the reference's OWN bulk driver, pooling and single-issue code
                     (py/code_intelligence/inference.py: df_to_embedding, batch_seq_pool, get_pooled_features) executed
                     around the CPU oracle's nn.LSTM stack (stand-ins only for the absent third-party imports).
* tokenizer_ref_notebook.json -- token strings the reference's pipeline printed in its notebooks (hand-collected).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
# a checkout of kubeflow/code-intelligence (the reference whose own code produces the mlp / thresholds / driver fixtures)
REFERENCE = os.environ.get('CODE_INTELLIGENCE_REFERENCE', '')


def reference_root():
    """The reference checkout, or a clear error: only the reference-pinned fixtures need it."""
    if not REFERENCE or not os.path.isdir(os.path.join(REFERENCE, 'py')):
        raise SystemExit('CODE_INTELLIGENCE_REFERENCE must name a checkout of kubeflow/code-intelligence (a directory with '
                         'py/ and Issue_Embeddings/) to regenerate the mlp / thresholds / driver fixtures; got %r' % REFERENCE)
    return REFERENCE
sys.path.insert(0, ROOT)

from oracle import awd_lstm_ref as R  # noqa: E402


def padded(docs, T, pad=1):
    ids = np.full((len(docs), T), pad, dtype=np.int64)
    for i, d in enumerate(docs):
        ids[i, :len(d)] = d
    return ids, np.array([len(d) for d in docs], dtype=np.int32)


def encoder_fixture(name, n_layers, emb_sz, n_hid, vocab, B, T, min_len, seed, scale=1.0, with_weights=True):
    torch.set_num_threads(os.cpu_count())
    enc = R.make_encoder(seed, vocab, emb_sz, n_hid, n_layers, scale=scale)
    docs = R.synthetic_ids(B, T, seed=seed + 1, vocab_sz=vocab, min_len=min_len)
    ids, lengths = padded(docs, T)
    out = R.encode_padded(enc, ids, lengths)
    d = dict(cfg=np.array([n_layers, emb_sz, n_hid, vocab, seed], dtype=np.int64), scale=np.float64(scale), ids=ids,
             lengths=lengths, expected=out.astype(np.float32))
    if with_weights:
        emb, layers = enc.export_weights()
        d['emb'] = emb
        for l, L in enumerate(layers):
            for k, v in L.items():
                d[f'l{l}_{k}'] = v
    np.savez_compressed(os.path.join(HERE, name), **d)
    print(name, out.shape, float(np.abs(out).mean()))


def mlp_fixture():
    sys.path.insert(0, os.path.join(reference_root(), 'py'))
    from label_microservice.mlp import MLPWrapper  # the reference's own wrapper
    from sklearn.neural_network import MLPClassifier
    from oracle.lstm_numpy import seeded_mlp
    import warnings
    rng = np.random.default_rng(1234)
    # 'small': a fitted classifier, stored in full
    d_in, hidden, n_labels, n_train, n_test = 24, (32, 16), 5, 200, 64
    X = (rng.standard_normal((n_train, d_in)) * 0.1).astype(np.float32)
    Y = (rng.random((n_train, n_labels)) < 0.2).astype(int)
    Xt = (rng.standard_normal((n_test, d_in)) * 0.1).astype(np.float32)
    clf = MLPClassifier(hidden_layer_sizes=hidden, random_state=1234, max_iter=8)
    w = MLPWrapper(clf=clf)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        w.fit(X, Y)
    probs = w.predict_probabilities(Xt)
    assert clf.out_activation_ == 'logistic'
    d = dict(X=Xt, probs=np.asarray(probs, dtype=np.float64), n_layers=np.int64(len(clf.coefs_)))
    for i, (W, b) in enumerate(zip(clf.coefs_, clf.intercepts_)):
        d[f'coef{i}'] = np.asarray(W, dtype=np.float32)
        d[f'intercept{i}'] = np.asarray(b, dtype=np.float32)
    np.savez_compressed(os.path.join(HERE, 'mlp_ref_small.npz'), **d)
    print('mlp small', probs.shape, float(probs.mean()))
    # 'prod' (1600 -> 600 -> 600 -> 40): the weights alone would be 5 MB, so they and the inputs come from
    # oracle.lstm_numpy.seeded_mlp; a classifier fitted for one step on a few rows supplies sklearn's attributes and
    # then receives those weights, and the reference's wrapper computes the probabilities
    dims, n_rows, seed = [1600, 600, 600, 40], 96, 4321
    coefs, intercepts, Xt = seeded_mlp(seed, dims, n_rows)
    clf = MLPClassifier(hidden_layer_sizes=tuple(dims[1:-1]), random_state=1234, max_iter=1)
    w = MLPWrapper(clf=clf)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        w.fit(Xt[:32], (rng.random((32, dims[-1])) < 0.2).astype(int))
    clf.coefs_ = [c.astype(np.float64) for c in coefs]
    clf.intercepts_ = [b.astype(np.float64) for b in intercepts]
    probs = w.predict_probabilities(Xt)
    assert clf.out_activation_ == 'logistic'
    np.savez_compressed(os.path.join(HERE, 'mlp_ref_prod.npz'), seed=np.int64(seed), dims=np.array(dims, dtype=np.int64),
                        n_rows=np.int64(n_rows), probs=np.asarray(probs, dtype=np.float64))
    print('mlp prod', probs.shape, float(probs.mean()))


def threshold_fixture():
    """Per-label probability thresholds computed by the reference's OWN loop (MLPWrapper.find_probability_thresholds,
    py/label_microservice/mlp.py:65-98) on preset scores: the classifier is a stand-in whose fit() does nothing and whose
    predict_proba() returns the preset score rows, so everything after `y_pred = ...` is the reference's code (with this
    image's sklearn precision_recall_curve).  Ties, a label without positives, labels that never qualify."""
    sys.path.insert(0, os.path.join(reference_root(), 'py'))
    from label_microservice.mlp import MLPWrapper
    rng = np.random.default_rng(77)
    out = {}
    for tag, n, L, quant, p_thr, r_thr in [('a', 400, 12, 0, 0.7, 0.5), ('b', 1500, 30, 40, 0.6, 0.3), ('c', 97, 6, 10, 0.0, 0.0)]:
        truth = (rng.random((n, L)) < rng.uniform(0.05, 0.5, size=L)).astype(int)
        truth[:, 0] = 0
        signal = rng.uniform(0.0, 3.0, size=L)
        scores = 1.0 / (1.0 + np.exp(-(rng.standard_normal((n, L)) + signal * (truth * 2.0 - 1.0))))
        scores = scores.astype(np.float32)
        if quant:
            scores = (np.round(scores * quant) / quant).astype(np.float32)

        class Stub:
            def fit(self, X, y):
                pass

            def predict_proba(self, X):
                return scores[np.asarray(X)[:, 0].astype(int)]

        w = MLPWrapper(clf=Stub(), precision_threshold=p_thr, recall_threshold=r_thr)
        X = np.arange(n)[:, None]
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            w.find_probability_thresholds(X, truth)
        from sklearn.model_selection import train_test_split
        _, X_test, _, y_test = train_test_split(X, truth, test_size=0.3, random_state=1234)
        idx = X_test[:, 0]
        thr = np.array([np.nan if w.probability_thresholds[l] is None else w.probability_thresholds[l] for l in range(L)], dtype=np.float64)
        out.update({f'{tag}_scores': scores[idx], f'{tag}_truth': y_test.astype(np.uint8), f'{tag}_p_thr': np.float64(p_thr),
                    f'{tag}_r_thr': np.float64(r_thr), f'{tag}_thresholds': thr,
                    f'{tag}_precisions': np.array([w.precisions[l] for l in range(L)], dtype=np.float64),
                    f'{tag}_recalls': np.array([w.recalls[l] for l in range(L)], dtype=np.float64)})
        print('thresholds', tag, int(np.isnan(thr).sum()), 'of', L, 'labels excluded')
    np.savez_compressed(os.path.join(HERE, 'thresholds_ref.npz'), **out)


def reference_driver_fixture():
    """Outputs of the reference's OWN bulk driver and pooling code (py/code_intelligence/inference.py:
    InferenceWrapper.df_to_embedding :138-229, batch_seq_pool :232-263, get_pooled_features :74-92) run in this
    container: the module is imported with stand-ins for its absent third-party imports (fastai, mdparse, more_itertools
    -- none of them takes part in the arithmetic of these functions), the text -> ids step is fed the numericalised docs
    directly, `.cuda()` is the identity, and `self.encoder` is the CPU oracle's stack of torch nn.LSTM (reset() + forward(x)
    -> (raw_outputs, outputs) like fastai's AWD_LSTM).  Everything else -- the batch-size rule, the length sort, pad_sequence,
    _forward_pass, batch_seq_pool, the OOM halving, the un-sort -- is the reference's code, executed."""
    import types
    import pandas as pd
    from oracle import awd_lstm_ref as R

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m
    current = {}
    mod('more_itertools', chunked=lambda it, n: [list(it)[i:i + n] for i in range(0, len(list(it)), n)])
    mod('mdparse'); mod('mdparse.parser', transform_pre_rules=[], compose=lambda fs: (lambda x: x))
    mod('fastai'); mod('fastai.text'); mod('fastai.text.transform', defaults=types.SimpleNamespace(text_pre_rules=[]))
    mod('fastai.core', PathOrStr=str, parallel=None); mod('fastai.basic_train', load_learner=None)
    mod('fastai.text.data', TokenizeProcessor=type('TokenizeProcessor', (), {}))

    class FakeLMDB:
        @staticmethod
        def from_df(**kw):
            items = current['docs']
            return types.SimpleNamespace(valid_dl=types.SimpleNamespace(x=types.SimpleNamespace(items=items)))
    sys.modules['fastai.text'].TextLMDataBunch = FakeLMDB
    torch.Tensor.cuda = lambda self, *a, **k: self
    sys.path.insert(0, os.path.join(reference_root(), 'py'))
    from code_intelligence.inference import InferenceWrapper as RefWrapper
    import importlib.util
    spec = importlib.util.spec_from_file_location('flask_app_inference', os.path.join(reference_root(), 'Issue_Embeddings/flask_app/inference.py'))
    fi = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fi)          # the flask_app copy of the wrapper (df_to_emb, FI:136-212)

    cfg = (2, 32, 48, 300)           # n_layers, emb_sz, n_hid, vocab
    ref = R.make_encoder(31, cfg[3], cfg[1], cfg[2], cfg[0], scale=2.0)

    class EncoderStub:                # fastai AWD_LSTM surface used by the reference: reset(), forward(x) -> (raw, out)
        def __init__(self, fail_above=None):
            self.fail_above, self.calls = fail_above, []

        def reset(self):
            pass

        def forward(self, x):
            self.calls.append(tuple(x.shape))
            if self.fail_above is not None and x.shape[0] > self.fail_above:
                raise RuntimeError('CUDA out of memory (stub)')
            with torch.no_grad():
                h = ref.encoder(x)
                outs = []
                for rnn in ref.rnns:
                    h, _ = rnn(h)
                    outs.append(h)
            return outs, outs

    out = {}
    for tag, n, max_len, bs, fail_above in [('a', 57, 40, 100, None), ('b', 130, 25, 100, None), ('c', 300, 20, 16, 5)]:
        docs = R.synthetic_ids(n, max_len, seed=100 + n, vocab_sz=cfg[3], min_len=1)
        current['docs'] = [np.asarray(d, dtype=np.int64) for d in docs]
        w = object.__new__(RefWrapper)
        w.encoder = EncoderStub(fail_above)
        w.pad_idx = 1
        w.path = None; w.model_tokenizer = None; w.vocab = None
        w.process_df = lambda df: df
        df = pd.DataFrame({'title': [''] * n, 'body': [''] * n})
        emb = w.df_to_embedding(df, bs=bs)
        assert emb.shape == (n, 3 * cfg[1])
        lens = np.array([len(d) for d in docs])
        out[f'{tag}_ids'] = np.concatenate(current['docs']).astype(np.int32)
        out[f'{tag}_lengths'] = lens.astype(np.int32)
        out[f'{tag}_bs'] = np.int64(bs)
        out[f'{tag}_fail_above'] = np.int64(-1 if fail_above is None else fail_above)
        out[f'{tag}_expected'] = emb.astype(np.float32)
        out[f'{tag}_batches_seen'] = np.array([c[0] for c in w.encoder.calls], dtype=np.int64)
        if fail_above is None:        # Issue_Embeddings/flask_app/inference.py:df_to_emb (chunked batches, no OOM loop)
            wf = object.__new__(fi.InferenceWrapper)
            wf.encoder = EncoderStub(None)
            wf.pad_idx = 1
            wf.path = None; wf.model_tokenizer = None; wf.vocab = None
            wf.process_df = lambda df: df
            emb_fi = wf.df_to_emb(df, bs=bs)
            out[f'{tag}_expected_flask_app'] = emb_fi.astype(np.float32)
            print('  flask_app df_to_emb vs py/code_intelligence df_to_embedding: max abs diff', float(np.abs(emb_fi - emb).max()))
        print('reference driver', tag, emb.shape, 'forward calls', len(w.encoder.calls), 'batch sizes', sorted(set(c[0] for c in w.encoder.calls)))
    # batch_seq_pool and get_pooled_features on their own
    rng = np.random.default_rng(5)
    seq = rng.standard_normal((7, 11, 6)).astype(np.float32)
    lens = np.array([11, 1, 5, 11, 3, 2, 9])
    out['pool_seq'] = seq; out['pool_lengths'] = lens.astype(np.int32)
    out['pool_expected'] = RefWrapper.batch_seq_pool(seq, lens).astype(np.float32)
    w = object.__new__(RefWrapper)
    w.encoder = EncoderStub()
    one = np.asarray(R.synthetic_ids(1, 23, seed=9, vocab_sz=cfg[3], min_len=23)[0], dtype=np.int64)
    w.numericalize_one = lambda x: torch.as_tensor(one)[None, :]
    out['single_ids'] = one.astype(np.int32)
    out['single_expected'] = w.get_pooled_features('ignored').detach().numpy().astype(np.float32)
    out['cfg'] = np.array(cfg, dtype=np.int64); out['seed'] = np.int64(31); out['scale'] = np.float64(2.0)
    np.savez_compressed(os.path.join(HERE, 'reference_driver.npz'), **out)


if __name__ == '__main__' and len(sys.argv) == 2 and sys.argv[1] == 'driver':
    reference_driver_fixture()

if __name__ == '__main__' and len(sys.argv) == 2 and sys.argv[1] == 'thresholds':
    threshold_fixture()

if __name__ == '__main__' and len(sys.argv) == 1:
    encoder_fixture('encoder_tiny.npz', 2, 64, 128, 1000, 5, 9, 2, seed=11)
    encoder_fixture('encoder_pad_dims.npz', 3, 50, 70, 300, 7, 12, 1, seed=12, scale=2.0)   # dims that need padding
    encoder_fixture('encoder_r4.npz', 4, 800, 2400, 60000, 32, 128, None, seed=1234, with_weights=False)  # config 1
    encoder_fixture('encoder_r4_varlen.npz', 4, 800, 2400, 60000, 24, 96, 5, seed=1234, scale=3.0, with_weights=False)
    encoder_fixture('encoder_n3.npz', 3, 800, 2400, 60000, 16, 64, 8, seed=1234, with_weights=False)
    mlp_fixture()


def full_size_fixture(name, n_layers, rows, T, seed, scale=1.0, keep=None):
    """Reference-shape fixtures at the shapes bench.py / the sweep measure (weights re-derived from the seed).
    rows: list of (count, min_len) groups; min_len None = fixed length T; keep: the row indices stored (every fixture
    file stays under 1 MB).  Stored compactly: int32 ids, f32 outputs."""
    torch.set_num_threads(os.cpu_count())
    enc = R.make_encoder(seed, 60000, 800, 2400, n_layers, scale=scale)
    docs = []
    for gi, (cnt, min_len) in enumerate(rows):
        docs += R.synthetic_ids(cnt, T, seed=seed + 101 + gi, vocab_sz=60000, min_len=min_len)
    ids, lengths = padded(docs, T)
    outs = []
    step = 64
    for b0 in range(0, len(docs), step):            # bounded host memory: (64, T, 2400) f32 activations per call
        tt = int(lengths[b0:b0 + step].max())
        outs.append(R.encode_padded(enc, ids[b0:b0 + step, :tt], lengths[b0:b0 + step]))
    out = np.concatenate(outs).astype(np.float32)
    if keep is not None:
        ids, lengths, out = ids[keep], lengths[keep], out[keep]
    np.savez_compressed(os.path.join(HERE, name), cfg=np.array([n_layers, 800, 2400, 60000, seed], dtype=np.int64),
                        scale=np.float64(scale), ids=ids.astype(np.int32), lengths=lengths, expected=out)
    print(name, out.shape, float(np.abs(out).mean()), flush=True)


def full_size():
    # bench shape (BASELINE configs[1]): 256 x 512; rows 0..127 full length, rows 128..255 var-len in [64, 512]; stored:
    # rows 0..31 and 128..143
    full_size_fixture('encoder_r4_b256_t512.npz', 4, [(128, None), (128, 64)], 512, seed=1234,
                      keep=np.r_[0:32, 128:144])
    # sweep buckets (configs[2]): lengths in (T/2, T]
    full_size_fixture('encoder_r4_t1024.npz', 4, [(32, 513)], 1024, seed=1234)
    full_size_fixture('encoder_r4_t2048.npz', 4, [(32, 1025)], 2048, seed=1234)
    # the north star's literal 3-layer shape
    full_size_fixture('encoder_n3_b64_t512.npz', 3, [(32, None), (32, 32)], 512, seed=1234)


if __name__ == '__main__' and len(sys.argv) > 1 and sys.argv[1] == 'full':
    full_size()
