"""LanguageModel: the reference's AWD-LSTM language model -- fastai 1.0.53's ``language_model_learner``, i.e.
``SequentialRNN(AWD_LSTM, LinearDecoder)`` (Issue_Embeddings/train.py) -- evaluated on the GPU: per-token
cross-entropy, argmax, and the ``learn.validate()`` pair (val_loss, accuracy) that ``SaveModelCallback`` and the
hyper-parameter sweep (objective ``val_loss``, minimize) select checkpoints by.

The decoder is csrc/lm.cu behind ``ie_lm_*`` (include/issue_emb_b200.h): logits = h W^T + b are reduced to
(logsumexp, logit of the target, argmax) inside the GEMM's epilogue, time chunk by time chunk on the encoder's ring, and
never stored.

fastai semantics restated here (from fastai 1.0.53's published text/data.py, basic_train.py, metrics.py; fastai is not
importable in this project, oracle/lm_ref.py states them literally and the CPU tests compare):

* ``LanguageModelPreLoader`` for a validation set: no shuffle, documents in order through a circular index.
  ``on_epoch_begin`` puts row ``i`` (of ``bs``) at token ``int(totalToks / bs * i)`` of the concatenated documents;
  each batch ``fill_row``s ``bptt + 1`` tokens per row with overlap 1 (a row's next batch starts at its last token), so
  row ``i`` is the ``n_b * bptt + 1`` tokens from that start, wrapping around the corpus, with
  ``n_b = ceil(totalToks / (bptt * bs))`` batches; x is a batch's first ``bptt`` columns, y its last ``bptt``.
* ``learn.validate()``: ``RNNTrainer.on_epoch_begin`` resets the state once, then the state carries from batch to
  batch; per batch ``CrossEntropyFlat()`` (mean over bs * bptt tokens) and ``accuracy`` (mean of argmax == y); both
  averaged over batches weighted by batch size, all equal here.  A state carried over the batches of a row is the state
  of one run over the whole row from zero, so one ``ie_lm_forward`` of ``bs`` rows x ``n_b * bptt`` steps computes it.

Text generation (csrc/lm_gen.cu behind ``ie_gen_state_*``): fastai 1.0.53 ``LanguageLearner.predict`` and
``beam_search`` (text/learner.py), restated literally in oracle/lm_gen_ref.py, on a recurrent state that a
:class:`LmState` carries from call to call.  Both take fastai's arguments and default ``decoder=decode_spec_tokens``.
Two deliberate deviations:

* **Sampling.**  ``torch.multinomial``'s random stream is not reproducible elsewhere.  Each draw is the inverse CDF at a
  uniform ``u`` in [0, 1): the first index of positive weight whose running sum of weights exceeds ``u`` times their
  total.  A row whose weights are all 0 (a small temperature underflows every power on a flat row) raises, as
  ``torch.multinomial`` does in fastai.  ``predict`` and ``beam_search`` take ``seed=`` or ``rng=`` (a
  ``numpy.random.Generator``) and draw every ``u`` up front: the same distribution as fastai's, with a reproducible
  choice.
* **Ties.**  torch leaves the order of ties in ``topk`` and ``argsort`` undefined.  Here ties go to the lower vocabulary
  index, and in the beam's sort to the lower candidate index (a stable sort).  This matters from the first beam step,
  where the ``top_k`` copies of the prompt give identical candidates.
"""
from __future__ import annotations

import ctypes as C
import math
import re
import warnings
import weakref
from typing import List, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import IE_FLAG_DEVICE_PTRS, check
from .encoder import IssueEncoder

IGNORE_INDEX = -100          # torch's cross_entropy ignore_index
TOKEN_CAP = 1 << 27          # the encoder's workspace cap on B_pad * T (ie_encoder_encode)


def _np32(a) -> np.ndarray:
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.float32)


def lm_stream(docs: Sequence[np.ndarray], bs: int, bptt: int):
    """(x, y) int64 [bs, n_b * bptt]: the rows fastai's LanguageModelPreLoader yields for a validation set, batch k
    being columns [k * bptt, (k + 1) * bptt)."""
    if bs < 1 or bptt < 1:
        raise ValueError(f"bs={bs} and bptt={bptt} must be >= 1")
    docs = [np.asarray(d, dtype=np.int64).reshape(-1) for d in docs]
    if not docs or any(len(d) == 0 for d in docs):
        raise ValueError("the corpus needs at least one document and no empty one")
    corpus = np.concatenate(docs)
    total = len(corpus)
    n_b = int(math.ceil(total / (bptt * bs)))
    step = total / bs
    starts = np.array([int(step * i) for i in range(bs)], dtype=np.int64)
    rows = corpus[(starts[:, None] + np.arange(n_b * bptt + 1, dtype=np.int64)[None, :]) % total]
    return rows[:, :-1], rows[:, 1:]


def decoder_keys(sd: dict):
    """(weight, bias or None) of a fastai LM state dict's LinearDecoder (``1.decoder.*``)."""
    if "1.decoder.weight" not in sd:
        raise ValueError("no decoder (key 1.decoder.weight) in the state dict")
    return sd["1.decoder.weight"], sd.get("1.decoder.bias")


TK_MAJ, TK_UP, TK_REP, TK_WREP = "xxmaj", "xxup", "xxrep", "xxwrep"
TOPK_MAX = 64          # kernels.h kLmTopkMax
BEAM_CANDIDATES = 16384  # kernels.h kLmBeamMax: rows * top_k one beam step sorts


def decode_spec_tokens(tokens: Sequence[str]) -> List[str]:
    """fastai 1.0.53's ``decode_spec_tokens`` (text/transform.py): the inverse of the caps and repetition rules.
    ``xxmaj w`` -> ``W`` (first letter up, rest down), ``xxup w`` -> ``W`` upper-cased, ``xxrep n c`` -> ``c * n``,
    ``xxwrep n w`` -> ``w`` n times; a rule whose count is not an integer is dropped with its count token."""
    new_toks, rule, arg = [], None, None
    for t in tokens:
        if t in (TK_MAJ, TK_UP, TK_REP, TK_WREP):
            rule = t
        elif rule is None:
            new_toks.append(t)
        elif rule == TK_MAJ:
            new_toks.append(t[:1].upper() + t[1:].lower())
            rule = None
        elif rule == TK_UP:
            new_toks.append(t.upper())
            rule = None
        elif arg is None:
            try:
                arg = int(t)
            except ValueError:
                rule = None
        else:
            if rule == TK_REP:
                new_toks.append(t * arg)
            else:
                new_toks += [t] * arg
            rule, arg = None, None
    return new_toks


def inverse_cdf(weights: np.ndarray, u: float) -> int:
    """The first index whose running sum (float64, in index order) exceeds ``u`` times the total: a draw from
    ``weights`` at the uniform ``u`` in [0, 1).  Used for the beam's final pick on the host."""
    w = np.asarray(weights, dtype=np.float64)
    c = np.cumsum(w)
    j = int(np.searchsorted(c, u * c[-1], side="right"))
    if j >= len(w):
        j = int(np.flatnonzero(w > 0)[-1]) if np.any(w > 0) else 0
    return j


class LmState:
    """A recurrent state carried across language-model calls (``ie_gen_state_*``): ``rows`` rows of every layer's h (as
    the encoder's ring holds it) and c (f32), zero after creation and :meth:`reset`.  Borrows the model, which closes
    its open states when it is closed itself; a closed state, or one of a closed model, refuses every call."""

    def __init__(self, lm: "LanguageModel", rows: int):
        if not 1 <= rows <= lm.encoder.max_batch:
            raise ValueError(f"rows={rows} outside [1, {lm.encoder.max_batch}] (the encoder's max_batch)")
        self.lm, self.rows, self._lib = lm, rows, lm._lib
        h = C.c_void_p()
        check(self._lib.ie_gen_state_create(lm._h, rows, C.byref(h)))
        self._h = h
        lm._states.add(self)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.ie_gen_state_destroy(self._h)   # before its model: LanguageModel.close closes its states first
            self._h = None

    def _handle(self, lm=None):
        """The C handle, after checking that the state (and its model) is open and, given ``lm``, belongs to it."""
        if not getattr(self, "_h", None) or not getattr(self.lm, "_h", None):
            raise ValueError("the state (or its language model) is closed")
        if lm is not None and lm is not self.lm:
            raise ValueError("the state belongs to another language model")
        return self._h

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self) -> None:
        """fastai's ``model.reset()``: every row back to the zero state."""
        check(self._lib.ie_gen_state_reset(self._handle()))

    def export(self, layer: int, n: Optional[int] = None):
        """Test hook ``ie_gen_state_export``: rows 0..n-1 of ``layer``: (h uint16 [n, P, out_l] bf16 bits, P = 2 planes
        hi, lo in the fp32-accurate mode, else 1; c float32 [n, out_l])."""
        n = self.rows if n is None else n
        enc = self.lm.encoder
        out_l = enc.emb_sz if layer == enc.n_layers - 1 else enc.n_hid
        planes = 2 if enc.flags & _lib.IE_CFG_FP32 else 1
        hb = np.empty((n, planes, out_l), np.uint16)
        c = np.empty((n, out_l), np.float32)
        check(self._lib.ie_gen_state_export(self._handle(), layer, n, hb.ctypes.data, c.ctypes.data))
        return hb, c


def _ids2d(ids):
    """(host int64 array or cuda int64 tensor) [n, T], device flag."""
    if hasattr(ids, "is_cuda") and ids.is_cuda:
        import torch
        if ids.dtype != torch.int64:
            raise ValueError("ids must be int64")
        ids = ids.contiguous()
        if ids.dim() == 1:
            ids = ids[None]
        return ids, True
    ids = np.ascontiguousarray(np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids), dtype=np.int64)
    if ids.ndim == 1:
        ids = ids[None]
    return ids, False


def _ptr(x, dev):
    return x.data_ptr() if dev else x.ctypes.data


class LanguageModel:
    """fastai ``language_model_learner`` in eval mode on the GPU.  Build it with :meth:`from_state_dict`, or around a
    loaded :class:`IssueEncoder` (borrowed) with the decoder's weight and bias."""

    def __init__(self, encoder: IssueEncoder, weight, bias=None, owns_encoder: bool = False,
                 itos: Optional[Sequence[str]] = None):
        self._lib = _lib.load()
        self._states = weakref.WeakSet()   # open LmStates: closed before the handle they borrow
        self.itos = list(itos) if itos is not None else None
        self._tok = None
        self.encoder, self._owns_encoder = encoder, owns_encoder
        self.vocab_sz, self.emb_sz, self.pad_idx = encoder.vocab_sz, encoder.emb_sz, encoder.pad_idx
        w = _np32(weight)
        if w.shape != (self.vocab_sz, self.emb_sz):
            raise ValueError(f"decoder weight {w.shape} != {(self.vocab_sz, self.emb_sz)}")
        b = None
        if bias is not None:
            b = _np32(bias)
            if b.shape != (self.vocab_sz,):
                raise ValueError(f"decoder bias {b.shape} != ({self.vocab_sz},)")
        h = C.c_void_p()
        check(self._lib.ie_lm_create(encoder._h, C.byref(h)))
        self._h = h
        check(self._lib.ie_lm_load_decoder(self._h, w.ctypes.data, None if b is None else b.ctypes.data))

    @classmethod
    def from_state_dict(cls, sd: dict, pad_idx: int = 1, device: int = 0, flags: int = 0,
                        itos: Optional[Sequence[str]] = None) -> "LanguageModel":
        """A fastai LM state dict (``learn.model.state_dict()``, or what ``learn.save`` writes: ``{'model': sd, ...}``):
        encoder keys ``0.encoder.weight``, ``0.rnns.{l}.*`` (AWD_LSTM names), decoder ``1.decoder.weight`` and
        ``1.decoder.bias``.  The saved decoder weight is used as is (fastai ties it to the embedding in training only).
        ``itos`` (the vocabulary, ``data.vocab.itos``): :meth:`predict` and :meth:`beam_search` then take and return
        text."""
        if "model" in sd and isinstance(sd["model"], dict):
            sd = sd["model"]
        if any(k.startswith("0.module.") for k in sd):
            raise ValueError("keys 0.module.* are a classifier's (MultiBatchEncoder); this takes a language model's")
        enc_sd = {k[2:]: v for k, v in sd.items() if k.startswith("0.")}
        if "encoder.weight" not in enc_sd:
            raise ValueError("no encoder (key 0.encoder.weight) in the state dict")
        weight, bias = decoder_keys(sd)
        vocab_sz, emb_sz = tuple(enc_sd["encoder.weight"].shape)
        n_layers = len({int(m.group(1)) for k in enc_sd for m in [re.match(r"rnns\.(\d+)\.", k)] if m})
        if n_layers < 1:
            raise ValueError("no LSTM layers (keys 0.rnns.*) in the state dict")
        n_hid = enc_sd["rnns.0.weight_hh_l0_raw"].shape[1] if n_layers > 1 else emb_sz
        if tuple(weight.shape) != (vocab_sz, emb_sz):
            raise ValueError(f"1.decoder.weight {tuple(weight.shape)} != encoder.weight {(vocab_sz, emb_sz)}")
        if bias is not None and tuple(bias.shape) != (vocab_sz,):
            raise ValueError(f"1.decoder.bias {tuple(bias.shape)} != ({vocab_sz},)")
        enc = IssueEncoder(n_layers, emb_sz, n_hid, vocab_sz, pad_idx, device, flags)
        try:
            enc.load_state_dict(enc_sd)
            return cls(enc, weight, bias, owns_encoder=True, itos=itos)
        except BaseException:
            enc.close()
            raise

    # ------------------------------------------------------------------ lifetime
    def close(self):
        for st in list(getattr(self, "_states", ())):
            st.close()
        if getattr(self, "_h", None):
            self._lib.ie_lm_destroy(self._h)
            self._h = None
        if getattr(self, "_owns_encoder", False) and self.encoder is not None:
            self.encoder.close()
            self.encoder = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launch_count(self) -> int:
        """Kernels this handle launched (two per time chunk); the encoder counts its own."""
        return int(self._lib.ie_lm_launch_count(self._h))

    def check_errors(self) -> None:
        """Waits for the last call and raises what its device-side checks found (device-pointer calls)."""
        check(self._lib.ie_lm_check_errors(self._h))

    # ------------------------------------------------------------------ calls
    def forward(self, ids, targets=None):
        """ids (B, T) int64, any B (slices of ``encoder.max_batch`` rows) -> (nll, lse, pred): f32, f32, int32 (B, T).
        Every row from a zero state.  targets default to ids shifted left with the last column -100."""
        ids = np.ascontiguousarray(np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids), dtype=np.int64)
        if ids.ndim != 2:
            raise ValueError("ids must be (B, T)")
        B, T = ids.shape
        if targets is None:
            targets = np.full_like(ids, IGNORE_INDEX)
            targets[:, :-1] = ids[:, 1:]
        targets = np.ascontiguousarray(np.asarray(targets), dtype=np.int64)
        if targets.shape != ids.shape:
            raise ValueError(f"targets {targets.shape} != ids {ids.shape}")
        nll = np.empty((B, T), np.float32)
        lse = np.empty((B, T), np.float32)
        pred = np.empty((B, T), np.int32)
        mb = self.encoder.max_batch
        for b0 in range(0, B, mb):
            b1 = min(B, b0 + mb)
            x, y = np.ascontiguousarray(ids[b0:b1]), np.ascontiguousarray(targets[b0:b1])
            o = [np.empty((b1 - b0, T), a.dtype) for a in (nll, lse, pred)]
            check(self._lib.ie_lm_forward(self._h, x.ctypes.data, y.ctypes.data, b1 - b0, T, o[0].ctypes.data,
                                          o[1].ctypes.data, o[2].ctypes.data, 0, None))
            nll[b0:b1], lse[b0:b1], pred[b0:b1] = o
        return nll, lse, pred

    def forward_padded(self, ids, targets=None):
        """``learn.model(x)`` with ``CrossEntropyFlat(reduction='none')`` and the argmax on one batch: (nll, pred)."""
        nll, _, pred = self.forward(ids, targets)
        return nll, pred

    def forward_device(self, ids, targets, nll=None, lse=None, pred=None, stream=None):
        """Asynchronous device-resident call: ids, targets cuda int64 (B, T), B <= encoder.max_batch; outputs cuda
        float32 / float32 / int32 (B, T) (allocated when None).  Runs on ``stream`` (default: torch's current stream);
        data-dependent errors are reported by :meth:`check_errors`.  Returns (nll, lse, pred)."""
        import torch
        if not (ids.is_cuda and targets.is_cuda and ids.dtype == torch.int64 and targets.dtype == torch.int64):
            raise ValueError("ids and targets must be cuda int64")
        ids, targets = ids.contiguous(), targets.contiguous()
        if ids.dim() != 2 or targets.shape != ids.shape:
            raise ValueError("ids and targets must be (B, T) of one shape")
        B, T = ids.shape
        outs = []
        for t, dt in ((nll, torch.float32), (lse, torch.float32), (pred, torch.int32)):
            if t is None:
                t = torch.empty((B, T), dtype=dt, device=ids.device)
            if not t.is_cuda or t.dtype != dt or tuple(t.shape) != (B, T) or not t.is_contiguous():
                raise ValueError(f"outputs must be contiguous cuda tensors of shape ({B}, {T})")
            outs.append(t)
        s = stream if stream is not None else torch.cuda.current_stream(ids.device)
        check(self._lib.ie_lm_forward(self._h, ids.data_ptr(), targets.data_ptr(), B, T, outs[0].data_ptr(),
                                      outs[1].data_ptr(), outs[2].data_ptr(), IE_FLAG_DEVICE_PTRS,
                                      C.c_void_p(s.cuda_stream)))
        return tuple(outs)

    def _debug_decode(self, h, targets):
        """Test hook ``ie_debug_lm_decode``: the decoder kernels on states h (M, emb_sz) (rounded as the ring holds
        them) with targets (M,) -> (nll, lse, pred)."""
        h = _np32(h)
        targets = np.ascontiguousarray(targets, dtype=np.int64)
        M = h.shape[0]
        if h.shape != (M, self.emb_sz) or targets.shape != (M,):
            raise ValueError(f"h must be (M, {self.emb_sz}) and targets (M,)")
        nll, lse, pred = np.empty(M, np.float32), np.empty(M, np.float32), np.empty(M, np.int32)
        check(self._lib.ie_debug_lm_decode(self._h, h.ctypes.data, targets.ctypes.data, M, nll.ctypes.data,
                                           lse.ctypes.data, pred.ctypes.data))
        return nll, lse, pred

    def validate(self, docs: Sequence[np.ndarray], bs: int = 64, bptt: int = 70):
        """``learn.validate()`` on numericalised documents: (val_loss, accuracy, perplexity = exp(val_loss))."""
        x, y = lm_stream(docs, bs, bptt)
        b_pad = 256 * ((bs + 255) // 256)
        if b_pad * x.shape[1] > TOKEN_CAP:
            raise ValueError(f"a stream of {bs} rows x {x.shape[1]} steps exceeds the encoder's cap of B_pad * T <= "
                             f"2^27 tokens (B_pad = {b_pad}); validate it in parts")
        if bs > self.encoder.max_batch:
            raise ValueError(f"bs={bs} > the encoder's max_batch {self.encoder.max_batch}")
        nll, _, pred = self.forward(x, y)
        n_b = x.shape[1] // bptt
        losses = [float(np.mean(nll[:, k * bptt:(k + 1) * bptt], dtype=np.float64)) for k in range(n_b)]
        accs = [float(np.mean(pred[:, k * bptt:(k + 1) * bptt] == y[:, k * bptt:(k + 1) * bptt])) for k in range(n_b)]
        val_loss, acc = float(np.mean(losses)), float(np.mean(accs))
        return val_loss, acc, math.exp(val_loss)

    # ------------------------------------------------------------------ generation
    def new_state(self, rows: int = 1) -> LmState:
        """A zero recurrent state of ``rows`` rows (<= ``encoder.max_batch``) for :meth:`step` / :meth:`sample`."""
        return LmState(self, rows)

    def _unk(self) -> int:
        if self.itos is not None and "xxunk" in self.itos:
            return self.itos.index("xxunk")
        return 0   # fastai's defaults put xxunk first

    def _exclude(self, no_unk: bool) -> int:
        return self._unk() if no_unk else -1

    def step(self, state: LmState, ids, k: int = 1, exclude: int = -1, values=None, idx=None, stream=None):
        """Feed ids [n, T] (n <= state.rows) to rows 0..n-1 of ``state`` and return the top ``k`` of each row's
        log_softmax at the last position: (values float32 [n, k] descending, idx int64 [n, k]), ties to the lower id.
        ``exclude`` (fastai's no_unk) counts in the softmax and is -inf among the values.  Host arrays: synchronous,
        numpy results.  Cuda int64 ids: asynchronous on ``stream``, cuda results (``values``/``idx`` may be given);
        errors come from :meth:`check_errors`, which must be called before the next call on this model: each call
        clears the device error words of the one before."""
        ids, dev = _ids2d(ids)
        n, T = ids.shape
        if not 1 <= k <= min(TOPK_MAX, self.vocab_sz):
            raise ValueError(f"k={k} outside [1, {min(TOPK_MAX, self.vocab_sz)}]")
        if dev:
            import torch
            values = torch.empty((n, k), dtype=torch.float32, device=ids.device) if values is None else values
            idx = torch.empty((n, k), dtype=torch.int64, device=ids.device) if idx is None else idx
            s = stream if stream is not None else torch.cuda.current_stream(ids.device)
            check(self._lib.ie_gen_topk(state._handle(self), ids.data_ptr(), n, T, k, exclude, values.data_ptr(),
                                              idx.data_ptr(), IE_FLAG_DEVICE_PTRS, C.c_void_p(s.cuda_stream)))
            return values, idx
        values, idx = np.empty((n, k), np.float32), np.empty((n, k), np.int64)
        check(self._lib.ie_gen_topk(state._handle(self), ids.ctypes.data, n, T, k, exclude, values.ctypes.data,
                                          idx.ctypes.data, 0, None))
        return values, idx

    def sample(self, state: LmState, ids, u, exclude: int = -1, temperature: float = 1.0, min_p=None, out=None,
               flags=None, stream=None):
        """Feed ids [n, T] to rows 0..n-1 of ``state`` and draw one id per row from fastai's predict weights at the
        last position (softmax; ``exclude`` zeroed; entries below ``min_p`` zeroed unless none reaches it; then
        ``** (1 / temperature)``) at the uniforms ``u`` [n] in [0, 1); an id of weight 0 is never drawn.  Returns (ids
        int64 [n], flags int32 [n]: 1 where no entry reached min_p, so nothing was masked; 2 where every weight was 0 --
        nothing to draw from, id 0 written -- which a host call raises as ValueError).  Host or cuda, as :meth:`step`;
        in device mode the flags keep every call's outcome, the error words only the last call's."""
        ids, dev = _ids2d(ids)
        n, T = ids.shape
        mp = 0.0 if min_p is None else float(min_p)
        if min_p is not None and not 0.0 < mp <= 1.0:
            raise ValueError(f"min_p={min_p} outside (0, 1]")
        if not temperature > 0 or not math.isfinite(temperature):
            raise ValueError(f"temperature={temperature} must be finite and > 0")
        if dev:
            import torch
            out = torch.empty(n, dtype=torch.int64, device=ids.device) if out is None else out
            flags = torch.empty(n, dtype=torch.int32, device=ids.device) if flags is None else flags
            s = stream if stream is not None else torch.cuda.current_stream(ids.device)
            check(self._lib.ie_gen_sample(state._handle(self), ids.data_ptr(), n, T, u.data_ptr(), exclude,
                                          float(temperature), mp, out.data_ptr(), flags.data_ptr(),
                                          IE_FLAG_DEVICE_PTRS, C.c_void_p(s.cuda_stream)))
            return out, flags
        u = np.ascontiguousarray(u, dtype=np.float32).reshape(-1)
        if u.shape != (n,):
            raise ValueError(f"u must hold {n} uniforms")
        out, flags = np.empty(n, np.int64), np.empty(n, np.int32)
        check(self._lib.ie_gen_sample(state._handle(self), ids.ctypes.data, n, T, u.ctypes.data, exclude,
                                      float(temperature), mp, out.ctypes.data, flags.ctypes.data, 0, None))
        return out, flags

    def select(self, state: LmState, idx, stream=None) -> None:
        """fastai's ``select_hidden``: rows 0..n-1 of ``state`` become its rows ``idx`` [n] (host, or a cuda int32
        tensor: asynchronous on ``stream``)."""
        if hasattr(idx, "is_cuda") and idx.is_cuda:
            import torch
            if idx.dtype != torch.int32:
                raise ValueError("device select indices must be int32")
            idx = idx.contiguous()
            s = stream if stream is not None else torch.cuda.current_stream(idx.device)
            check(self._lib.ie_gen_select(state._handle(self), idx.data_ptr(), idx.numel(), IE_FLAG_DEVICE_PTRS,
                                                C.c_void_p(s.cuda_stream)))
            return
        idx = np.ascontiguousarray(np.asarray(idx), dtype=np.int32).reshape(-1)
        check(self._lib.ie_gen_select(state._handle(self), idx.ctypes.data, len(idx), 0, None))

    def beam_select(self, state: LmState, scores, values, tokens, beam_sz: int, nodes=None, stream=None):
        """One beam step (``ie_gen_beam_select``): candidate j = r * top_k + c scores f32(scores[r] - values[r, c]); the
        min(beam_sz, rows * top_k) lowest in stable-sort order survive.  Returns (parent int32, token int64, score
        float32, nodes int64 [m, L + 1] = the parent's nodes [rows, L] plus the token).  Host or cuda arrays."""
        dev = hasattr(values, "is_cuda") and values.is_cuda
        rows, top_k = values.shape
        if rows * top_k > BEAM_CANDIDATES:
            raise ValueError(f"rows * top_k = {rows * top_k} candidates exceed {BEAM_CANDIDATES}")
        m = min(beam_sz, rows * top_k)
        if dev:
            import torch
            d = values.device
            L = 0 if nodes is None else nodes.shape[1]
            outs = (torch.empty(m, dtype=torch.int32, device=d), torch.empty(m, dtype=torch.int64, device=d),
                    torch.empty(m, dtype=torch.float32, device=d), torch.empty((m, L + 1), dtype=torch.int64, device=d))
            s = stream if stream is not None else torch.cuda.current_stream(d)
            check(self._lib.ie_gen_beam_select(state._handle(self), scores.data_ptr(),
                                               values.contiguous().data_ptr(),
                                               tokens.contiguous().data_ptr(), rows, top_k, beam_sz,
                                               None if nodes is None else nodes.contiguous().data_ptr(), L,
                                               *[o.data_ptr() for o in outs], IE_FLAG_DEVICE_PTRS,
                                               C.c_void_p(s.cuda_stream)))
            return outs
        scores = np.ascontiguousarray(scores, dtype=np.float32).reshape(-1)
        values = np.ascontiguousarray(values, dtype=np.float32)
        tokens = np.ascontiguousarray(tokens, dtype=np.int64)
        if scores.shape != (rows,) or tokens.shape != (rows, top_k):
            raise ValueError("scores [rows] and tokens [rows, top_k] must match values")
        nodes = None if nodes is None else np.ascontiguousarray(nodes, dtype=np.int64)
        L = 0 if nodes is None else nodes.shape[1]
        outs = (np.empty(m, np.int32), np.empty(m, np.int64), np.empty(m, np.float32), np.empty((m, L + 1), np.int64))
        check(self._lib.ie_gen_beam_select(state._handle(self), scores.ctypes.data, values.ctypes.data,
                                           tokens.ctypes.data, rows,
                                           top_k, beam_sz, None if nodes is None else nodes.ctypes.data, L,
                                           *[o.ctypes.data for o in outs], 0, None))
        return outs

    def _prompt(self, text_or_ids):
        """(prompt ids int64 [T], text or None)."""
        if isinstance(text_or_ids, str):
            if self.itos is None:
                raise ValueError("a text prompt needs the vocabulary: build the model with itos=")
            if self._tok is None:
                from .inference import RuleTokenizer
                self._tok = RuleTokenizer(self.itos)
            return self._tok(text_or_ids), text_or_ids
        ids = np.asarray(text_or_ids.cpu() if hasattr(text_or_ids, "cpu") else text_or_ids, dtype=np.int64).reshape(-1)
        if ids.size == 0:
            raise ValueError("the prompt is empty")
        if ids.min() < 0 or ids.max() >= self.vocab_sz:
            raise ValueError(f"a prompt id is outside [0, {self.vocab_sz})")
        return ids, None

    def _decode(self, ids, decoder) -> List[str]:
        toks = [self.itos[int(i)] for i in ids]
        return decoder(toks) if decoder is not None else toks

    def predict(self, text_or_ids, n_words: int = 1, no_unk: bool = True, temperature: float = 1.0, min_p=None,
                sep: str = " ", decoder=decode_spec_tokens, seed=None, rng=None):
        """fastai's ``LanguageLearner.predict``: ``n_words`` ids drawn one by one from the carried state, each from the
        softmax at the last position with no_unk, min_p (a warning when no entry reaches it, as fastai warns) and
        temperature applied.  Each draw is the inverse CDF at a uniform from ``rng`` (or ``numpy.random.default_rng(seed)``)
        -- the module docstring's deviation.  A text prompt (needs ``itos``) returns ``text + sep + sep.join(decoder(new
        tokens))`` as fastai does (``text + sep`` for n_words = 0); an id prompt returns the prompt's ids followed by the
        new ones.  The words stay on the device between steps; one copy back at the end."""
        import torch
        prompt, text = self._prompt(text_or_ids)
        if n_words < 0:
            raise ValueError("n_words must be >= 0")
        if min_p is not None and not 0.0 < float(min_p) <= 1.0:
            raise ValueError(f"min_p={min_p} outside (0, 1]")
        if not temperature > 0 or not math.isfinite(temperature):
            raise ValueError(f"temperature={temperature} must be finite and > 0")
        rng = rng if rng is not None else np.random.default_rng(seed)
        new = np.empty(0, np.int64)
        if n_words > 0:
            dev = torch.device("cuda", self.encoder.device)
            u = torch.as_tensor(rng.random(n_words, dtype=np.float32), device=dev)
            toks = torch.empty(n_words, dtype=torch.int64, device=dev)
            flags = torch.empty(n_words, dtype=torch.int32, device=dev)
            x = torch.as_tensor(prompt[None], device=dev)
            state = self.new_state(1)
            try:
                ex = self._exclude(no_unk)
                for i in range(n_words):
                    self.sample(state, x, u[i:i + 1], ex, temperature, min_p, out=toks[i:i + 1], flags=flags[i:i + 1])
                    x = toks[i:i + 1][None]
                new, fl = toks.cpu().numpy(), flags.cpu().numpy()
                # the flags keep every step's outcome; the device error words only the last step's
                if np.any(fl == 2):
                    i = int(np.flatnonzero(fl == 2)[0])
                    msg = (f"word {i}: every weight is 0 after no_unk / min_p / temperature={temperature} (the powers "
                           f"underflow in float32), so there is nothing to draw from")
                    try:
                        self.check_errors()            # collects (and clears) what the last step reported
                    except ValueError as e:
                        raise ValueError(msg) from e
                    raise ValueError(msg)
                self.check_errors()
            finally:
                state.close()
            for _ in range(int(np.sum(fl == 1))):
                warnings.warn(f"There is no item with probability >= {min_p}, try a lower value.")
        if text is None:
            return np.concatenate([prompt, new])
        return text + sep + sep.join(self._decode(new, decoder))

    def beam_search(self, text_or_ids, n_words: int, no_unk: bool = True, top_k: int = 10, beam_sz: int = 1000,
                    temperature: float = 1.0, sep: str = " ", decoder=decode_spec_tokens, seed=None, rng=None):
        """fastai's ``LanguageLearner.beam_search``: the prompt repeated ``top_k`` times; per word the top ``top_k`` of
        each row's log_softmax (no_unk: xxunk at -inf), candidate scores ``parent score - value``, the ``beam_sz``
        lowest kept (stable order: the module docstring's deviation), the state's rows gathered by parent
        (``select_hidden``).  At the end the scores are divided by ``temperature`` and one node is drawn with weights
        ``exp(-score)`` by the inverse CDF at a uniform from ``rng`` / ``seed``.  fastai returns that node without its
        first id -- the prompt after xxbos, then the new words -- so a text prompt gives ``text + sep + sep.join(
        decoder(those tokens))``; an id prompt returns the whole node (the prompt's ids, then the new ones)."""
        import torch
        prompt, text = self._prompt(text_or_ids)
        if n_words < 0:
            raise ValueError("n_words must be >= 0")
        if not 1 <= top_k <= min(TOPK_MAX, self.vocab_sz):
            raise ValueError(f"top_k={top_k} outside [1, {min(TOPK_MAX, self.vocab_sz)}]")
        if not 1 <= beam_sz <= self.encoder.max_batch:
            raise ValueError(f"beam_sz={beam_sz} outside [1, {self.encoder.max_batch}] (the encoder's max_batch)")
        if not temperature > 0 or not math.isfinite(temperature):
            raise ValueError(f"temperature={temperature} must be finite and > 0")
        rows = top_k
        for _ in range(n_words):
            if rows * top_k > BEAM_CANDIDATES:
                raise ValueError(f"{rows} beams x top_k={top_k} exceed {BEAM_CANDIDATES} candidates per step")
            rows = min(beam_sz, rows * top_k)
        rng = rng if rng is not None else np.random.default_rng(seed)
        u = float(rng.random(dtype=np.float32))
        if n_words == 0:
            nodes, scores = np.tile(prompt, (top_k, 1)), np.zeros(1, np.float32)
        else:
            dev = torch.device("cuda", self.encoder.device)
            x = torch.as_tensor(np.tile(prompt, (top_k, 1)), device=dev)
            nodes = x
            scores = torch.zeros(top_k, dtype=torch.float32, device=dev)
            state = self.new_state(max(top_k, min(beam_sz, rows)))
            try:
                ex = self._exclude(no_unk)
                for _ in range(n_words):
                    values, idx = self.step(state, x, top_k, ex)
                    parent, token, scores, nodes = self.beam_select(state, scores, values, idx, beam_sz, nodes)
                    self.select(state, parent)
                    x = token[:, None]
                nodes, scores = nodes.cpu().numpy(), scores.cpu().numpy()
                self.check_errors()
            finally:
                state.close()
        s = scores / np.float32(temperature) if temperature != 1.0 else scores
        node = nodes[inverse_cdf(np.exp(-s.astype(np.float64)), u)]
        if text is None:
            return node
        return text + sep + sep.join(self._decode(node[1:], decoder))
