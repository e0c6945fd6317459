"""TextClassifier: the reference's fine-tuned issue labeller -- fastai 1.0.53's ``text_classifier_learner`` over the
AWD-LSTM encoder (Issue_Embeddings/notebooks/06_FineTune.ipynb) -- run in eval mode on the GPU.

The model is ``SequentialRNN(MultiBatchEncoder(bptt, max_len, AWD_LSTM), PoolingLinearClassifier)``:

* the encoder runs every step from a zero state (the ``IssueEncoder`` handle this class owns or borrows);
* the pool is ``masked_concat_pool`` = ``[last | max | mean]`` over the window of kept bptt chunks (chunk ``i`` is kept
  when ``i > sl - max_len``), masked where ``ids == pad_idx``;
* the head is ``BatchNorm1d -> (Dropout) -> Linear`` per stage, ReLU between stages, then sigmoid (multi-label,
  ``BCEWithLogitsFlat``) or softmax (single-label, ``CrossEntropyFlat``).

Pool, head and activation are the kernels of csrc/clas.cu behind ``ie_clas_*`` (include/issue_emb_b200.h).
"""
from __future__ import annotations

import ctypes as C
import re
from typing import List, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import IE_FLAG_DEVICE_PTRS, check
from .encoder import IssueEncoder

IE_CLAS_SIGMOID, IE_CLAS_SOFTMAX = 0, 1
_BN_KEYS = ("weight", "bias", "running_mean", "running_var")


def _np32(a) -> np.ndarray:
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.float32)


def window_start(sl: int, bptt: int = 70, max_len: int = 1400) -> int:
    """First step MultiBatchEncoder(bptt, max_len) keeps of a sequence of ``sl`` steps (``ie_clas_window``): chunk
    ``i`` (``i = 0, bptt, ...``) is kept when ``i > sl - max_len``.  ValueError when no chunk is kept (fastai fails in
    ``torch.cat`` there; only possible with ``max_len <= bptt``)."""
    s = C.c_int32()
    check(_lib.load().ie_clas_window(int(sl), int(bptt), int(max_len), C.byref(s)))
    return int(s.value)


def head_stages(sd: dict, in_width: int) -> List[dict]:
    """The head stages of a fastai classifier state dict (keys ``1.layers.{k}.*``; ``{'model': sd}`` accepted), inferred
    from the tensors: a BatchNorm1d has weight, bias, running_mean, running_var (and num_batches_tracked), a Linear a
    2-D weight; Dropout and ReLU have no parameters, so the indices shift with the dropout probabilities and nothing is
    assumed about positions.  Each stage is ``dict(bn_weight, bn_bias, bn_mean, bn_var, weight, bias)``; the first
    stage must take ``in_width`` = 3 * emb_sz inputs and each stage the previous one's outputs (ValueError)."""
    if "model" in sd and isinstance(sd["model"], dict):
        sd = sd["model"]
    mods = {}
    for k, v in sd.items():
        m = re.fullmatch(r"1\.layers\.(\d+)\.(\w+)", k)
        if m:
            mods.setdefault(int(m.group(1)), {})[m.group(2)] = v
    if not mods:
        raise ValueError("no head parameters (keys 1.layers.*) in the state dict")
    stages, bn = [], None
    for idx in sorted(mods):
        p = mods[idx]
        if all(n in p for n in _BN_KEYS):
            if bn is not None:
                raise ValueError(f"1.layers.{idx}: two BatchNorm1d without a Linear between them")
            bn = {n: _np32(p[n]) for n in _BN_KEYS}
        elif "weight" in p and np.ndim(_np32(p["weight"])) == 2:
            if bn is None:
                raise ValueError(f"1.layers.{idx}: Linear without a BatchNorm1d before it (bn_drop_lin has bn=True)")
            w = _np32(p["weight"])
            b = _np32(p["bias"]) if "bias" in p else np.zeros(w.shape[0], np.float32)
            n_in = in_width if not stages else stages[-1]["weight"].shape[0]
            if w.shape[1] != n_in or any(bn[n].shape != (n_in,) for n in _BN_KEYS) or b.shape != (w.shape[0],):
                raise ValueError(f"1.layers.{idx}: stage {len(stages)} takes {w.shape[1]} inputs (BatchNorm "
                                 f"{bn['weight'].shape}), expected {n_in}")
            stages.append(dict(bn_weight=bn["weight"], bn_bias=bn["bias"], bn_mean=bn["running_mean"],
                               bn_var=bn["running_var"], weight=w, bias=b))
            bn = None
        else:
            raise ValueError(f"1.layers.{idx}: parameters {sorted(p)} are neither a BatchNorm1d nor a Linear")
    if bn is not None:
        raise ValueError("the head ends with a BatchNorm1d")
    return stages


class TextClassifier:
    """fastai ``text_classifier_learner`` in eval mode on the GPU.  Build it with :meth:`from_state_dict`."""

    def __init__(self, encoder: IssueEncoder, stages: Sequence[dict], bptt: int = 70, max_len: int = 1400,
                 activation: str = "sigmoid", classes: Optional[Sequence[str]] = None, itos=None,
                 bn_eps: float = 1e-5, owns_encoder: bool = False):
        """encoder: a loaded IssueEncoder (borrowed: several classifiers may share one); stages: ``head_stages``."""
        if activation not in ("sigmoid", "softmax"):
            raise ValueError(f"activation {activation!r} is neither 'sigmoid' nor 'softmax'")
        window_start(bptt, bptt, max_len)   # a sequence of bptt steps keeps no chunk iff max_len <= bptt: ValueError
        self._lib = _lib.load()
        self.encoder, self.bptt, self.max_len, self.activation = encoder, int(bptt), int(max_len), activation
        self.pad_idx = encoder.pad_idx
        self._owns_encoder = owns_encoder
        dims = [3 * encoder.emb_sz] + [int(s["weight"].shape[0]) for s in stages]
        for k, s in enumerate(stages):
            if s["weight"].shape[1] != dims[k]:
                raise ValueError(f"stage {k} takes {s['weight'].shape[1]} inputs, expected {dims[k]}")
        self.dims, self.n_class = dims, dims[-1]
        self.classes = list(classes) if classes is not None else None
        if self.classes is not None and len(self.classes) != self.n_class:
            raise ValueError(f"{len(self.classes)} class names for {self.n_class} outputs")
        self._tok = None
        if itos is not None:
            from .inference import RuleTokenizer
            self._tok = RuleTokenizer(itos)
        d = (C.c_int32 * len(dims))(*dims)
        h = C.c_void_p()
        check(self._lib.ie_clas_create(encoder._h, len(stages), d,
                                       IE_CLAS_SIGMOID if activation == "sigmoid" else IE_CLAS_SOFTMAX, C.byref(h)))
        self._h = h
        for k, s in enumerate(stages):
            a = [_np32(s[n]) for n in ("bn_weight", "bn_bias", "bn_mean", "bn_var", "weight", "bias")]
            check(self._lib.ie_clas_load_stage(self._h, k, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data,
                                               a[3].ctypes.data, float(bn_eps), a[4].ctypes.data, a[5].ctypes.data))

    @classmethod
    def from_state_dict(cls, sd: dict, bptt: int = 70, max_len: int = 1400, pad_idx: int = 1,
                        activation: str = "sigmoid", classes=None, itos=None, device: int = 0,
                        flags: int = 0) -> "TextClassifier":
        """A fastai classifier state dict (``learn.model.state_dict()``, or what ``learn.save`` writes:
        ``{'model': sd, 'opt': ...}``): encoder keys ``0.module.*`` (AWD_LSTM names), head keys ``1.layers.*``."""
        if "model" in sd and isinstance(sd["model"], dict):
            sd = sd["model"]
        enc_sd = {k[len("0.module."):]: v for k, v in sd.items() if k.startswith("0.module.")}
        if "encoder.weight" not in enc_sd:
            raise ValueError("no encoder (key 0.module.encoder.weight) in the state dict")
        vocab_sz, emb_sz = tuple(enc_sd["encoder.weight"].shape)
        n_layers = len({int(m.group(1)) for k in enc_sd for m in [re.match(r"rnns\.(\d+)\.", k)] if m})
        n_hid = enc_sd["rnns.0.weight_hh_l0_raw"].shape[1] if n_layers > 1 else emb_sz
        stages = head_stages(sd, 3 * emb_sz)
        enc = IssueEncoder(n_layers, emb_sz, n_hid, vocab_sz, pad_idx, device, flags)
        try:
            enc.load_state_dict(enc_sd)
            return cls(enc, stages, bptt, max_len, activation, classes, itos, owns_encoder=True)
        except BaseException:
            enc.close()
            raise

    # ------------------------------------------------------------------ lifetime
    def close(self):
        if getattr(self, "_h", None):
            self._lib.ie_clas_destroy(self._h)
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
        """Kernels this classifier launched (pool, head stages, activation); the encoder counts its own."""
        return int(self._lib.ie_clas_launch_count(self._h))

    def check_errors(self) -> None:
        """Waits for the last call and raises what its device-side checks found (device-pointer calls)."""
        check(self._lib.ie_clas_check_errors(self._h))

    # ------------------------------------------------------------------ windows
    def windows(self, lengths, T: int):
        """(starts, ends) int32 of rows whose last step is ``lengths[b] - 1``: fastai's chunk rule on each length."""
        ends = np.ascontiguousarray(lengths, dtype=np.int32)
        starts = np.array([window_start(int(e), self.bptt, self.max_len) for e in ends], dtype=np.int32)
        return starts, ends

    # ------------------------------------------------------------------ calls on one padded batch
    def _call(self, ids, starts, ends, pooled: bool):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        B, T = ids.shape
        starts = np.ascontiguousarray(starts, dtype=np.int32)
        ends = np.ascontiguousarray(ends, dtype=np.int32)
        if starts.shape != (B,) or ends.shape != (B,):
            raise ValueError(f"starts / ends must have shape ({B},)")
        if pooled:
            out = np.empty((B, self.dims[0]), np.float32)
            check(self._lib.ie_clas_pool(self._h, ids.ctypes.data, starts.ctypes.data, ends.ctypes.data, B, T,
                                         out.ctypes.data, 0, None))
            return out
        out = np.empty((B, self.n_class), np.float32)
        logits = np.empty((B, self.n_class), np.float32)
        check(self._lib.ie_clas_forward(self._h, ids.ctypes.data, starts.ctypes.data, ends.ctypes.data, B, T,
                                        out.ctypes.data, logits.ctypes.data, 0, None))
        return out, logits

    def _per_item(self, docs: Sequence[np.ndarray], pooled: bool):
        """Each issue on its own (what ``learn.predict`` gives one at a time): sorted by length, right-padded with
        pad_idx into buckets of up to ``max_batch`` rows, each row's window from its own length; input order out."""
        docs = [np.asarray(d, dtype=np.int64).reshape(-1) for d in docs]
        n = len(docs)
        width = self.dims[0] if pooled else self.n_class
        out = np.empty((n, width), np.float32)
        logits = None if pooled else np.empty((n, width), np.float32)
        if any(len(d) == 0 for d in docs):
            raise ValueError("an issue has no tokens")
        order = np.argsort([len(d) for d in docs], kind="stable")
        mb = self.encoder.max_batch
        for b0 in range(0, n, mb):
            rows = order[b0:b0 + mb]
            T = max(len(docs[i]) for i in rows)
            ids = np.full((len(rows), T), self.pad_idx, dtype=np.int64)
            lengths = np.empty(len(rows), np.int32)
            for r, i in enumerate(rows):
                ids[r, :len(docs[i])] = docs[i]
                lengths[r] = len(docs[i])
            starts, ends = self.windows(lengths, T)
            got = self._call(ids, starts, ends, pooled)
            if pooled:
                out[rows] = got
            else:
                out[rows], logits[rows] = got
        return out if pooled else (out, logits)

    # ------------------------------------------------------------------ public
    def predict_proba(self, docs: Sequence[np.ndarray]) -> np.ndarray:
        """Numericalised issues -> (n, n_class) float32 activated outputs, input order, each issue as if alone."""
        return self._per_item(docs, pooled=False)[0]

    def predict_logits(self, docs: Sequence[np.ndarray]) -> np.ndarray:
        """The last Linear's outputs of :meth:`predict_proba`."""
        return self._per_item(docs, pooled=False)[1]

    def forward_padded(self, ids):
        """``learn.model(ids)`` on one batch as ``pad_collate(pad_first=True)`` builds it: ids (B, T) with the pads in
        front, every step through the LSTM, the window from T for all rows.  Returns (logits, activated) (B, n_class)."""
        ids = np.ascontiguousarray(np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids), dtype=np.int64)
        if ids.ndim != 2:
            raise ValueError("ids must be (B, T)")
        B, T = ids.shape
        s = window_start(T, self.bptt, self.max_len)
        out = np.empty((B, self.n_class), np.float32)
        logits = np.empty((B, self.n_class), np.float32)
        mb = self.encoder.max_batch
        for b0 in range(0, B, mb):
            b1 = min(B, b0 + mb)
            o, z = self._call(ids[b0:b1], np.full(b1 - b0, s, np.int32), np.full(b1 - b0, T, np.int32), False)
            out[b0:b1], logits[b0:b1] = o, z
        return logits, out

    def forward_padded_device(self, ids, starts, ends, out=None, logits=None, stream=None):
        """Asynchronous device-resident call: ids cuda int64 (B, T), starts / ends cuda int32 (B,), out / logits cuda
        float32 (B, n_class) (allocated when None); B <= encoder.max_batch.  Runs on ``stream`` (default: torch's
        current stream); data-dependent errors are reported by :meth:`check_errors`.  Returns (logits, out)."""
        import torch
        if not (ids.is_cuda and starts.is_cuda and ends.is_cuda and ids.dtype == torch.int64
                and starts.dtype == torch.int32 and ends.dtype == torch.int32):
            raise ValueError("ids must be cuda int64, starts / ends cuda int32")
        ids, starts, ends = ids.contiguous(), starts.contiguous(), ends.contiguous()
        B, T = ids.shape
        if tuple(starts.shape) != (B,) or tuple(ends.shape) != (B,):
            raise ValueError(f"starts / ends must have shape ({B},)")
        bufs = []
        for t in (out, logits):
            if t is None:
                t = torch.empty((B, self.n_class), dtype=torch.float32, device=ids.device)
            if (not t.is_cuda or t.dtype != torch.float32 or tuple(t.shape) != (B, self.n_class)
                    or not t.is_contiguous()):
                raise ValueError(f"out / logits must be contiguous cuda float32 tensors of shape ({B}, {self.n_class})")
            bufs.append(t)
        out, logits = bufs
        s = stream if stream is not None else torch.cuda.current_stream(ids.device)
        check(self._lib.ie_clas_forward(self._h, ids.data_ptr(), starts.data_ptr(), ends.data_ptr(), B, T,
                                        out.data_ptr(), logits.data_ptr(), IE_FLAG_DEVICE_PTRS,
                                        C.c_void_p(s.cuda_stream)))
        return logits, out

    def pooled_features(self, docs=None, ids=None) -> np.ndarray:
        """The head's input ``[last | max | mean]`` alone: per issue for ``docs`` (as :meth:`predict_proba`), or for
        one front-padded batch ``ids`` (as :meth:`forward_padded`).  (n, 3 * emb_sz) float32."""
        if (docs is None) == (ids is None):
            raise ValueError("pass exactly one of docs, ids")
        if docs is not None:
            return self._per_item(docs, pooled=True)
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        B, T = ids.shape
        s = window_start(T, self.bptt, self.max_len)
        return self._call(ids, np.full(B, s, np.int32), np.full(B, T, np.int32), True)

    def numericalize(self, text: str) -> np.ndarray:
        if self._tok is None:
            raise RuntimeError("no vocabulary: pass itos= to from_state_dict")
        return self._tok(text)

    def predict(self, text: str):
        """``learn.predict(text)``: (labels, y, probs).  Multi-label (sigmoid): y is the 0/1 vector at 0.5 and labels
        the class names at or above it; single-label (softmax): y is the argmax and labels its class name."""
        probs = self.predict_proba([self.numericalize(text)])[0]
        names = self.classes if self.classes is not None else [str(i) for i in range(self.n_class)]
        if self.activation == "sigmoid":
            y = (probs >= 0.5).astype(np.float32)
            return [names[i] for i in np.flatnonzero(y)], y, probs
        y = int(np.argmax(probs))
        return names[y], y, probs
