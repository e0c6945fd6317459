"""Drop-in mirror of the reference's ``InferenceWrapper`` (Issue_Embeddings/flask_app/inference.py:27-246 and
py/code_intelligence/inference.py:25-263) with the encoder arithmetic on the H100.

Same names, argument meaning and error behaviour:

    InferenceWrapper(model_path, model_file_name)
    .parse  .process_dict  .process_df  .numericalize_one
    .get_raw_features(text)      -> torch.Tensor (1, T, 800)
    .get_pooled_features(text)   -> torch.Tensor (1, 2400)   [mean | max | last]
    .df_to_emb(df, bs=100) / .df_to_embedding(df, bs=100) -> np.ndarray (N, 2400) float32, input row order
    .batch_seq_pool(seq_emb, lengths)
    pass_through                 (module level, needed to unpickle fastai learners: app.py:10)

The contract of the GPU path starts at token ids (SURVEY.md section 8b), so every text-taking method has an
id-taking twin (``*_from_ids``).  Text -> ids needs the model's tokenizer + vocab: when fastai is importable the
exported learner's own ``one_item`` / ``TextLMDataBunch`` machinery is used exactly as in the reference; otherwise
a ``numericalizer`` callable (str -> 1-D int64 array, starting with xxbos) must be supplied, or the built-in
approximate rule tokenizer is used when the model file carries a vocab (``itos``).
"""
from __future__ import annotations

import logging
import os
import re
from pathlib import Path
from typing import Callable, List, Optional

import numpy as np

from .encoder import IssueEncoder


def pass_through(x):
    """Avoid messages when the model is deserialized in fastai library."""
    return x


# ---------------------------------------------------------------------------------------------------
# text pre-processing (boundary code; the reference composes mdparse.transform_pre_rules with fastai's
# defaults.text_pre_rules, inference.py:41-48).  mdparse is not installed here, so when it is missing only the
# fastai default pre-rules are applied (restated below from fastai 1.0.53 fastai/text/transform.py).
# ---------------------------------------------------------------------------------------------------
BOS, FLD, UNK, PAD = 'xxbos', 'xxfld', 'xxunk', 'xxpad'
TK_MAJ, TK_UP, TK_REP, TK_WREP = 'xxmaj', 'xxup', 'xxrep', 'xxwrep'


def _spec_add_spaces(t): return re.sub(r'([/#])', r' \1 ', t)
def _rm_useless_spaces(t): return re.sub(' {2,}', ' ', t)


def _replace_rep(t):
    def _r(m):
        c, cc = m.groups()
        return f' {TK_REP} {len(cc) + 1} {c} '
    return re.sub(r'(\S)(\1{3,})', _r, t)


def _replace_wrep(t):
    def _r(m):
        c, cc = m.groups()
        return f' {TK_WREP} {len(cc.split()) + 1} {c} '
    return re.sub(r'(\b\w+\W+)(\1{3,})', _r, t)


def _fix_html(x):
    re1 = re.compile(r'  +')
    x = x.replace('#39;', "'").replace('amp;', '&').replace('#146;', "'").replace('nbsp;', ' ').replace(
        '#36;', '$').replace('\\n', "\n").replace('quot;', "'").replace('<br />', "\n").replace(
        '\\"', '"').replace('<unk>', UNK).replace(' @.@ ', '.').replace(' @-@ ', '-').replace(' @,@ ', ',').replace(
        '\\', ' \\ ')
    import html
    return re1.sub(' ', html.unescape(x))


TEXT_PRE_RULES = [_fix_html, _replace_rep, _replace_wrep, _spec_add_spaces, _rm_useless_spaces]


def _replace_all_caps(toks):
    res = []
    for t in toks:
        if t.isupper() and len(t) > 1:
            res.append(TK_UP)
            res.append(t.lower())
        else:
            res.append(t)
    return res


def _deal_caps(toks):
    res = []
    for t in toks:
        if t == '':
            continue
        if t[0].isupper() and len(t) > 1 and t[1:].islower():
            res.append(TK_MAJ)
        res.append(t.lower())
    return res


TEXT_SPEC_TOK = [UNK, PAD, BOS, FLD, TK_MAJ, TK_UP, TK_REP, TK_WREP]   # fastai defaults.text_spec_tok


class RuleTokenizer:
    """Stand-in for fastai 1.0.53's ``Tokenizer(SpacyTokenizer('en'))`` when fastai/spaCy are not installed:
    ``Tokenizer.process_text`` restated -- default pre-rules, the word splitter (``tokenizer.SpacyLikeTokenizer``, a
    restatement of spaCy's rule tokenizer with fastai's special tokens registered as special cases), default
    post-rules -- then the vocab lookup of ``Vocab.numericalize`` (unknown -> xxunk).  NOT parity-pinned against
    spaCy (row f-1 of SURVEY.md section 8; no spaCy in this image)."""

    def __init__(self, itos: List[str]):
        from .tokenizer import SpacyLikeTokenizer
        self.itos = list(itos)
        self.stoi = {s: i for i, s in reversed(list(enumerate(self.itos)))}
        self.unk = self.stoi.get(UNK, 0)
        self.bos = self.stoi.get(BOS, 2)
        self.splitter = SpacyLikeTokenizer(TEXT_SPEC_TOK)

    def tokens(self, text: str) -> List[str]:
        for r in TEXT_PRE_RULES:
            text = r(text)
        toks = self.splitter(text)
        return _deal_caps(_replace_all_caps(toks))

    def __call__(self, text: str) -> np.ndarray:
        ids = [self.bos] + [self.stoi.get(t, self.unk) for t in self.tokens(text)]
        return np.asarray(ids, dtype=np.int64)


def _compose_parse():
    try:  # exactly the reference's composition when its dependencies exist
        from fastai.text.transform import defaults
        from mdparse.parser import compose, transform_pre_rules
        return compose(transform_pre_rules + defaults.text_pre_rules)
    except Exception:
        def parse(x):
            for r in TEXT_PRE_RULES:
                x = r(x)
            return x
        return parse


# ---------------------------------------------------------------------------------------------------
class InferenceWrapper:
    "Utility to aid with generating a document embedding from the Title and the Body of a GitHub Issue."

    def __init__(self, model_path, model_file_name, device: int = 0,
                 numericalizer: Optional[Callable[[str], np.ndarray]] = None, n_layers: Optional[int] = None):
        """Load the encoder from model_path/model_file_name.

        Accepted artefacts: (a) a fastai exported learner ``.pkl`` (needs fastai importable; what the reference
        loads at inference.py:33), (b) a torch ``.pth`` state dict written by fastai ``save_encoder``
        (Issue_Embeddings/README.md:84-85), (c) an ``.npz`` with the same keys (+ optional ``itos``)."""
        path = Path(model_path) / model_file_name
        self.learn = None
        self.model_tokenizer = None
        self.vocab = None
        self.pad_idx = 1
        itos = None
        if str(path).endswith('.pkl'):
            from fastai.basic_train import load_learner  # raises ImportError without fastai
            from fastai.text.data import TokenizeProcessor
            self.learn = load_learner(path=model_path, file=model_file_name)
            self.learn.model.eval()
            sd = {k: v for k, v in self.learn.model[0].state_dict().items()}
            self.pad_idx = self.learn.data.pad_idx
            self.model_tokenizer = [x.tokenizer for x in self.learn.data.processor if type(x) == TokenizeProcessor][0]
            self.vocab = self.learn.data.vocab
            itos = list(self.vocab.itos)
        elif str(path).endswith('.npz'):
            z = np.load(path, allow_pickle=False)
            sd = {k: z[k] for k in z.files if k != 'itos'}
            if 'itos' in z.files:
                itos = [str(s) for s in z['itos']]
        else:
            import torch
            sd = torch.load(path, map_location='cpu')
            if 'model' in sd and isinstance(sd['model'], dict):
                sd = sd['model']
        emb_key = [k for k in sd if k.endswith('encoder.weight')][0]
        vocab_sz, emb_sz = sd[emb_key].shape
        n_found = len({k.split('rnns.')[1].split('.')[0] for k in sd if 'rnns.' in k})
        n_layers = n_layers or n_found
        hh0 = [k for k in sd if k.endswith('rnns.0.weight_hh_l0_raw') or k.endswith('rnns.0.module.weight_hh_l0')][0]
        n_hid = sd[hh0].shape[1] if n_layers > 1 else emb_sz
        self.encoder = IssueEncoder(n_layers, emb_sz, n_hid, vocab_sz, self.pad_idx, device).load_state_dict(sd)
        self._numericalizer = numericalizer or (RuleTokenizer(itos) if itos is not None else None)
        self.path = Path(f'./inference_utils/{os.getpid()}')

    # ---- text side (boundary) ------------------------------------------------------------------
    @staticmethod
    def parse(x: str) -> str:
        """Pre-process the text (markdown annotation and cleanup) prior to tokenizing."""
        return _compose_parse()(x)

    def numericalize_one(self, x: str):
        """Convert text to a series of integers in preparation for inference -> LongTensor (1, T)."""
        import torch
        if self.learn is not None:
            return self.learn.data.one_item(x)[0]
        if self._numericalizer is None:
            raise RuntimeError("no tokenizer/vocab available: pass numericalizer= or use the *_from_ids methods")
        return torch.as_tensor(np.asarray(self._numericalizer(x), dtype=np.int64))[None, :]

    @classmethod
    def process_dict(cls, dfdict: dict) -> dict:
        """{'title','body'} -> {'text': 'xxxfldtitle ... xxxfldbody ...'}; on any exception {'text': 'xxxUnk'}."""
        assert 'title' in dfdict, 'Missing the field "title"'
        assert 'body' in dfdict, 'Missing the field "body"'
        title = dfdict['title']
        body = dfdict['body']
        try:
            text = 'xxxfldtitle ' + cls.parse(title) + ' xxxfldbody ' + cls.parse(body)
        except Exception as e:
            logging.error(f"Exception occurred in process_dict {e}")
            return {'text': 'xxxUnk'}
        return {'text': text}

    @classmethod
    def process_df(cls, dataframe):
        """Loop through a pandas DataFrame and create a single text field."""
        import pandas as pd
        lst = [cls.process_dict(d) for d in dataframe.to_dict(orient='records')]
        return pd.DataFrame(lst)

    def _forward_pass(self, x):
        """ids (B,T) right-padded -> last-layer hidden states as numpy (B,T,emb_sz), zero initial state
        (inference.py:55-57: reset(); forward(x)[-1][-1].detach().cpu().numpy()).  Kept for interface parity; the bulk
        path of this package never materialises this tensor on the host."""
        ids = np.asarray(x.cpu() if hasattr(x, 'cpu') else x, dtype=np.int64)
        return self.encoder.raw_features(ids)

    # ---- single issue ---------------------------------------------------------------------------
    def get_raw_features_from_ids(self, seq_ints):
        """ids (1,T) or (T,) -> torch.Tensor (1, T, emb_sz): hidden states of the last layer, zero initial state."""
        import torch
        ids = np.asarray(seq_ints.cpu() if hasattr(seq_ints, 'cpu') else seq_ints, dtype=np.int64).reshape(1, -1)
        return torch.from_numpy(self.encoder.raw_features(ids))

    def get_raw_features(self, x: str):
        """Get features from encoder of the language model. Returns Tensor of the shape (1, sequence_length, ndim)."""
        return self.get_raw_features_from_ids(self.numericalize_one(x))

    def get_pooled_features_from_ids(self, seq_ints):
        """ids (1,T) or (T,) -> torch.Tensor (1, 3*emb_sz) = [mean, max, last] (inference.py:90)."""
        import torch
        ids = np.asarray(seq_ints.cpu() if hasattr(seq_ints, 'cpu') else seq_ints, dtype=np.int64).reshape(1, -1)
        return torch.from_numpy(self.encoder.encode_ids(ids, np.array([ids.shape[1]], dtype=np.int32)))

    def get_pooled_features(self, x: str):
        """Get concatenation of [mean, max, last] of last hidden state -> Tensor (1, 2400)."""
        return self.get_pooled_features_from_ids(self.numericalize_one(x))

    # ---- bulk -----------------------------------------------------------------------------------
    def _numericalize_df(self, new_df) -> List[np.ndarray]:
        if self.learn is not None:  # the reference's own parallel tokenisation (inference.py:174-182)
            from fastai.text import TextLMDataBunch as lmdb
            data_lm = lmdb.from_df(path=self.path, train_df=new_df.head(), valid_df=new_df, text_cols='text',
                                   tokenizer=self.model_tokenizer, vocab=self.vocab)
            return [np.asarray(a, dtype=np.int64) for a in data_lm.valid_dl.x.items]
        if self._numericalizer is None:
            raise RuntimeError("no tokenizer/vocab available: pass numericalizer= or use encode_id_list")
        return [np.asarray(self._numericalizer(t), dtype=np.int64) for t in new_df['text']]

    def df_to_embedding(self, dataframe, bs=100) -> np.ndarray:
        """DataFrame{title, body} -> (N, 2400) float32 in input row order (py/code_intelligence/inference.py:138-229);
        batch-size rule, length sort, padding, OOM halving and unsort live in IssueEncoder.encode_id_list."""
        new_df = self.process_df(dataframe)
        docs = self._numericalize_df(new_df)
        pooled_states = self.encoder.encode_id_list(docs, bs=bs)
        assert pooled_states.shape[0] == len(docs) == len(dataframe)
        return pooled_states

    df_to_emb = df_to_embedding  # Issue_Embeddings/flask_app/inference.py:136

    def encode_id_list(self, docs: List[np.ndarray], bs=100) -> np.ndarray:
        return self.encoder.encode_id_list(docs, bs=bs)

    @classmethod
    def batch_seq_pool(cls, seq_emb, lengths):
        """Concatenate the mean, max and last hidden representations of a batch of sequences (host utility kept
        for interface parity, inference.py:215-246; the GPU path pools on the device instead)."""
        assert seq_emb.shape[0] == len(lengths), \
            'Number of elements in lengths should match the first dimension of seq_emb'
        seq_emb = np.asarray(seq_emb)
        embs = [seq_emb[i, :x, :] for i, x in enumerate(lengths)]
        features = [np.concatenate([emb.mean(axis=0), emb.max(axis=0), emb[-1, :]], axis=-1) for emb in embs]
        combined_features = np.stack(features)
        assert combined_features.shape[-1] == (seq_emb.shape[-1] * 3)
        return combined_features


def text_endpoint_bytes(wrapper: InferenceWrapper, title: str, body: str) -> bytes:
    """What ``POST /text`` returns (Issue_Embeddings/flask_app/app.py:60-69): 2400 little-endian float32, no header."""
    x = wrapper.process_dict({'title': title, 'body': body})['text']
    emb = wrapper.get_pooled_features(x).detach().numpy()
    return np.ascontiguousarray(emb, dtype='<f4').tobytes()
