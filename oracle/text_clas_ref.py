"""ORACLE (test infrastructure, NOT product code) for the text classifier: fastai 1.0.53's text_classifier_learner on
the AWD-LSTM encoder (Issue_Embeddings/notebooks/06_FineTune.ipynb) in eval mode, restated on torch modules, plus the
float64 restatement of the device's pool and head with their per-element bounds, and the exact float32 restatement of
the same kernels (their bits) with relative bounds for the activations.

fastai is not installed; the semantics below are restated from fastai 1.0.53's published source (text/learner.py,
text/models/awd_lstm.py, layers.py), nothing is copied:

* ``get_text_classifier(arch, vocab_sz, n_class, bptt=70, max_len=1400, config, drop_mult, lin_ftrs=None, ps=None,
  pad_idx=1)`` = ``SequentialRNN(MultiBatchEncoder(bptt, max_len, AWD_LSTM(vocab_sz, **config)),
  PoolingLinearClassifier([3 * emb_sz] + lin_ftrs + [n_class], [output_p] + ps))``; ``lin_ftrs`` defaults to ``[50]``,
  ``ps`` to ``[0.1] * len(lin_ftrs)``.
* ``MultiBatchEncoder.forward(input)``: ``bs, sl = input.size()``; reset the AWD_LSTM state to zero; for
  ``i in range(0, sl, bptt)`` run ``input[:, i:min(i + bptt, sl)]`` with the state carried from the previous chunk, and
  keep that chunk's outputs (and ``mask = input == pad_idx`` over it) only when ``i > sl - max_len`` (strict).  The
  chunked run is the same arithmetic as one run over all ``sl`` steps; with no chunk kept ``torch.cat`` fails.
* ``masked_concat_pool(outputs, mask)`` on the last layer's kept outputs ``o`` [B, W, emb_sz]:
  ``avg = o.masked_fill(mask, 0).mean(1)``, then ``avg *= W / (W - mask.sum(1))`` (an f32 tensor division: one rounding
  of the factor, one of the product); ``mx = o.masked_fill(mask, -inf).max(1)``; ``last = o[:, -1]``;
  ``x = cat([last, mx, avg], 1)``.  An all-pad window gives NaN / -inf.
* ``PoolingLinearClassifier``: per stage ``bn_drop_lin(n_in, n_out, p, actn)`` = ``BatchNorm1d(n_in)``, ``Dropout(p)``
  only when ``p != 0``, ``Linear(n_in, n_out)``, ``ReLU`` on every stage but the last -- in ``nn.Sequential`` order, so
  the state-dict indices ``1.layers.{k}`` shift with the zeros among the ``p``.  Eval BatchNorm uses the running
  statistics with eps = 1e-5.  Its forward returns (logits, raw_outputs, outputs); ``learn.predict`` applies the loss
  function's activation: sigmoid for ``BCEWithLogitsFlat`` (multi-label, 06), softmax for ``CrossEntropyFlat``.
* ``learn.save`` writes ``{'model': state_dict, 'opt': ...}``; the encoder's keys are ``0.module.encoder.weight``,
  ``0.module.encoder_dp.emb.weight``, ``0.module.rnns.{l}.weight_hh_l0_raw``, ``0.module.rnns.{l}.module.*_l0``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch
from torch import nn

from . import awd_lstm_ref as R

U = 2.0 ** -24      # unit roundoff of f32


def kept_chunks(sl: int, bptt: int = 70, max_len: int = 1400) -> List[int]:
    """MultiBatchEncoder's loop written out: the starts of the chunks whose outputs it keeps."""
    return [i for i in range(0, sl, bptt) if i > sl - max_len]


def window_start(sl: int, bptt: int = 70, max_len: int = 1400) -> int:
    kept = kept_chunks(sl, bptt, max_len)
    if not kept:
        raise ValueError(f"no chunk of bptt={bptt} is kept at sl={sl} with max_len={max_len}")
    return kept[0]


def masked_concat_pool(o: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """fastai's pool on o [B, W, E] f32 and mask [B, W] bool."""
    if bool(mask.all(1).any()):
        raise ValueError("a window is entirely pad (fastai pools NaN / -inf there)")
    avg = o.masked_fill(mask[:, :, None], 0).mean(dim=1)
    avg *= o.size(1) / (o.size(1) - mask.type(avg.dtype).sum(dim=1))[:, None]
    mx = o.masked_fill(mask[:, :, None], -float("inf")).max(dim=1)[0]
    return torch.cat([o[:, -1], mx, avg], 1)


def head_layers(layers: Sequence[int], ps: Sequence[float]) -> nn.Sequential:
    """PoolingLinearClassifier's nn.Sequential for sizes ``layers`` and dropouts ``ps``."""
    if len(ps) != len(layers) - 1:
        raise ValueError("need one dropout probability per stage")
    mods = []
    for k, (n_in, n_out, p) in enumerate(zip(layers[:-1], layers[1:], ps)):
        mods.append(nn.BatchNorm1d(n_in))
        if p != 0:
            mods.append(nn.Dropout(p))
        mods.append(nn.Linear(n_in, n_out))
        if k < len(layers) - 2:
            mods.append(nn.ReLU(inplace=True))
    return nn.Sequential(*mods)


class ClassifierRef(nn.Module):
    """Eval-mode restatement of get_text_classifier's model around ``AWDLSTMEncoderRef``."""

    def __init__(self, enc: R.AWDLSTMEncoderRef, n_class: int, lin_ftrs=(50,), ps=None, output_p=0.4,
                 bptt: int = 70, max_len: int = 1400):
        super().__init__()
        lin_ftrs = list(lin_ftrs)
        ps = [0.1] * len(lin_ftrs) if ps is None else list(ps)
        self.enc, self.bptt, self.max_len, self.pad_idx = enc, bptt, max_len, enc.pad_idx
        self.layers = head_layers([3 * enc.emb_sz] + lin_ftrs + [n_class], [output_p] + ps)
        self.eval()

    @torch.no_grad()
    def encode_chunked(self, ids: torch.Tensor):
        """MultiBatchEncoder literally: chunks of bptt with the (h, c) of every layer carried; the kept chunks' outputs
        and masks concatenated."""
        B, sl = ids.shape
        state = [None] * len(self.enc.rnns)
        outs, masks = [], []
        for i in range(0, sl, self.bptt):
            x = self.enc.encoder(ids[:, i:min(i + self.bptt, sl)])
            for l, rnn in enumerate(self.enc.rnns):
                x, state[l] = rnn(x, state[l])
            if i > sl - self.max_len:
                outs.append(x)
                masks.append(ids[:, i:min(i + self.bptt, sl)] == self.pad_idx)
        if not outs:
            raise ValueError("no chunk kept")
        return torch.cat(outs, 1), torch.cat(masks, 1)

    @torch.no_grad()
    def encode(self, ids: torch.Tensor):
        """The same window from one run over all steps."""
        s = window_start(ids.shape[1], self.bptt, self.max_len)
        return self.enc(ids)[:, s:], ids[:, s:] == self.pad_idx

    @torch.no_grad()
    def pooled(self, ids, chunked: bool = False) -> torch.Tensor:
        ids = torch.as_tensor(np.asarray(ids, dtype=np.int64))
        o, mask = self.encode_chunked(ids) if chunked else self.encode(ids)
        return masked_concat_pool(o, mask)

    @torch.no_grad()
    def forward(self, ids, chunked: bool = False) -> torch.Tensor:
        """The batched forward (``learn.model(x)[0]``): logits [B, n_class]."""
        return self.layers(self.pooled(ids, chunked))

    @torch.no_grad()
    def predict_one(self, ids, activation="sigmoid") -> np.ndarray:
        """``learn.predict``'s probabilities for one numericalised issue (a batch of one, no padding)."""
        z = self.forward(np.asarray(ids, dtype=np.int64)[None, :])
        return (torch.sigmoid(z) if activation == "sigmoid" else torch.softmax(z, 1))[0].numpy()

    def fastai_state_dict(self) -> dict:
        """The state dict ``learn.model.state_dict()`` has for this model (WeightDropout keeps the raw W_hh and the
        module's copy; EmbeddingDropout shares the embedding)."""
        sd = {"0.module.encoder.weight": self.enc.encoder.weight.detach().clone(),
              "0.module.encoder_dp.emb.weight": self.enc.encoder.weight.detach().clone()}
        for l, rnn in enumerate(self.enc.rnns):
            sd[f"0.module.rnns.{l}.weight_hh_l0_raw"] = rnn.weight_hh_l0.detach().clone()
            for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"):
                sd[f"0.module.rnns.{l}.module.{n}"] = getattr(rnn, n).detach().clone()
        for k, v in self.layers.state_dict().items():
            sd["1.layers." + k] = v.detach().clone()
        return sd

    def stages(self) -> List[dict]:
        """(BatchNorm1d, Linear) of each stage as float32 arrays."""
        bns = [m for m in self.layers if isinstance(m, nn.BatchNorm1d)]
        lins = [m for m in self.layers if isinstance(m, nn.Linear)]
        f = lambda t: t.detach().numpy().astype(np.float32)
        return [dict(bn_weight=f(b.weight), bn_bias=f(b.bias), bn_mean=f(b.running_mean), bn_var=f(b.running_var),
                     weight=f(L.weight), bias=f(L.bias)) for b, L in zip(bns, lins)]


def make_classifier(seed=5, vocab_sz=500, emb_sz=96, n_hid=200, n_layers=3, n_class=3, lin_ftrs=(50,), ps=None,
                    output_p=0.4, bptt=70, max_len=1400, scale=2.0, calib_ids=None) -> ClassifierRef:
    """A random classifier with non-trivial BatchNorm statistics: each stage's running mean / variance are those of its
    input over ``calib_ids`` (as training leaves them; random around the unit ones without), weight / bias random."""
    enc = R.make_encoder(seed, vocab_sz, emb_sz, n_hid, n_layers, scale=scale)
    clf = ClassifierRef(enc, n_class, lin_ftrs, ps, output_p, bptt, max_len)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        x = clf.pooled(calib_ids) if calib_ids is not None else None
        for m in clf.layers:
            if isinstance(m, nn.BatchNorm1d):
                n = m.num_features
                if x is not None:
                    m.running_mean.copy_(x.mean(0))
                    m.running_var.copy_(x.var(0) + 1e-4)
                else:
                    m.running_mean.copy_(0.1 * torch.randn(n, generator=g))
                    m.running_var.copy_(0.5 + torch.rand(n, generator=g))
                m.weight.copy_(1 + 0.2 * torch.randn(n, generator=g))
                m.bias.copy_(0.1 * torch.randn(n, generator=g))
                m.num_batches_tracked.fill_(1000)
            if x is not None:
                x = m(x)
    clf.eval()
    return clf


# ---------------------------------------------------------------------------------------------------
# float64 restatement of the device's pool and head (csrc/clas.cu), with the per-element bounds of DESIGN.md
# ---------------------------------------------------------------------------------------------------
def pool_f64(raw: np.ndarray, ids: np.ndarray, starts, ends, pad_idx: int):
    """raw [B, T, E] f32 (the device's states), window [starts[b], ends[b]): (last, max, avg64, bound) with last and max
    exact (what the device must return bit for bit) and |avg_device - avg64| <= bound, where avg64 = (sum / W) * factor
    in float64 over the f32 states and factor = f32(W / (W - n_masked)) as fastai rounds it.  The device sums the n
    unmasked steps in step order (n - 1 roundings), divides by W and multiplies by factor (two more):
    bound = 1.01 * factor * (n + 2) * u * sum|x| / W."""
    B, T, E = raw.shape
    last = np.empty((B, E), np.float32)
    mx = np.empty((B, E), np.float32)
    avg = np.empty((B, E))
    bound = np.empty((B, E))
    for b in range(B):
        s, e = int(starts[b]), int(ends[b])
        keep = ids[b, s:e] != pad_idx
        w, n = e - s, int(keep.sum())
        if n == 0:
            raise ValueError(f"row {b}: window entirely pad")
        x = raw[b, s:e][keep].astype(np.float64)
        factor = float(np.float32(w) / np.float32(n))        # W / (W - n_masked), one f32 rounding
        last[b] = raw[b, e - 1]
        mx[b] = raw[b, s:e][keep].max(0)
        avg[b] = x.sum(0) / w * factor
        bound[b] = 1.01 * factor * (n + 2) * U * np.abs(x).sum(0) / w
    return last, mx, avg, bound


def head_f64(x: np.ndarray, stages: Sequence[dict], activation: str = "sigmoid", eps: float = 1e-5):
    """The head in float64 on the f32 pooled input x [B, 3E], BatchNorm from its raw parameters:
    (logits64, logit_bound, p64, p_bound), the bounds holding for the device's f32 values element by element.

    Per stage, input bound e (0 for the pool's own output): the device folds BatchNorm into alpha = f32(f32(1 / f32(
    sqrt(f32(var + eps)))) * w), beta = f32(b - mean * alpha), xn = f32(x * alpha + beta) -- within 8 u (|x alpha| + |beta|
    + |mean alpha|) + |alpha| e of the exact xn; the Linear is a sequential fma chain over K plus the bias, within
    (K + 2) u (sum|xn W| + |bias|) + sum |W| e_xn; ReLU keeps the bound.  Sigmoid: e / 4 + 8 u.  Softmax:
    p (2 max e + u |z - max| + max_j u |z_j - max| + (N + 8) u) * 1.01 + 2^-126."""
    a = np.asarray(x, np.float64)
    e = np.zeros_like(a)
    for k, st in enumerate(stages):
        w, b, m, v = (np.asarray(st[n], np.float64) for n in ("bn_weight", "bn_bias", "bn_mean", "bn_var"))
        W, bias = np.asarray(st["weight"], np.float64), np.asarray(st["bias"], np.float64)
        alpha = w / np.sqrt(v + eps)
        xn = (a - m) * alpha + b
        ea = np.abs(alpha)
        e_xn = ea * e + 8 * U * ((np.abs(a) + e) * ea + np.abs(b - m * alpha) + np.abs(m) * ea)
        z = xn @ W.T + bias
        K = W.shape[1]
        e = e_xn @ np.abs(W).T + (K + 2) * U * ((np.abs(xn) + e_xn) @ np.abs(W).T + np.abs(bias))
        a = np.maximum(z, 0) if k < len(stages) - 1 else z
    z, ez = a, e
    if activation == "sigmoid":
        p = 1 / (1 + np.exp(-z))
        ep = ez / 4 + 8 * U
    else:
        d = z - z.max(1, keepdims=True)
        p = np.exp(d) / np.exp(d).sum(1, keepdims=True)
        N = z.shape[1]
        ep = p * (2 * ez.max(1, keepdims=True) + U * np.abs(d) + U * np.abs(d).max(1, keepdims=True)
                  + (N + 8) * U) * 1.01 + 2.0 ** -126
    return z, ez, p, ep


# ---------------------------------------------------------------------------------------------------
# exact float32 restatement of csrc/clas.cu: the device's pool and logits bit for bit
# ---------------------------------------------------------------------------------------------------
# Every function below takes and returns torch tensors and runs on the CPU or the GPU alike.  Values are held in float64
# and rounded to float32 after each operation, one eager op per step, so nothing contracts into an fma.  For +, -, *, /
# and sqrt that double rounding is innocuous: 53 >= 2 * 24 + 2 bits, so f32(f64(a op b)) is the correctly rounded f32
# result (Figueroa, "When is double rounding innocuous?", 1995).  An fma has no such guarantee and goes through fma_f32.

def _f32(t: torch.Tensor) -> torch.Tensor:
    """Round to the nearest f32 (ties to even), kept in float64."""
    return t.to(torch.float32).to(torch.float64)


def _t64(a, device=None) -> torch.Tensor:
    t = torch.as_tensor(a, device=device)
    if t.dtype != torch.float32 and t.dtype != torch.float64:
        raise TypeError(f"expected float32 values, got {t.dtype}")
    return t.to(torch.float64)


def fma_f32(a, b, c) -> torch.Tensor:
    """The correctly rounded f32 fma(a, b, c) of f32 values (held in float64), elementwise with broadcasting.

    The product of two f32 values is exact in float64; s = p + c is rounded once and TwoSum gives its exact error.  When
    that error is non-zero and s has an even last bit, s steps one float64 ulp toward the error: s is then p + c rounded
    to odd at 53 bits, and rounding a round-to-odd value of 53 >= 24 + 2 bits to f32 is the correctly rounded result
    (Boldo & Melquiond, 2008).  The plain f32(f64(a * b) + c) rounds twice and can land on the wrong side of an f32
    midpoint: a = b = 1 + 2^-12, c = 2^-80 gives the midpoint 1 + 2^-11 + 2^-24 after the first rounding, which then goes
    down to even while the exact sum lies above it."""
    a, b, c = torch.broadcast_tensors(_t64(a), _t64(b), _t64(c))
    p = a * b
    s = p + c
    bv = s - p
    err = (p - (s - bv)) + (c - bv)
    even = (s.view(torch.int64) & 1) == 0
    toward = torch.where(err > 0, torch.full_like(s, float("inf")), torch.full_like(s, -float("inf")))
    s = torch.where((err != 0) & even & torch.isfinite(s), torch.nextafter(s, toward), s)
    return _f32(s)


def bn_fold_f32(stage: dict, eps: float = 1e-5, device=None):
    """(alpha, beta) float64 tensors holding what ie_clas_load_stage computes on the host in f32:
    alpha = f32(f32(1 / f32(sqrt(f32(var + f32(eps))))) * w), beta = fma(-mean, alpha, b)."""
    w, b, m, v = (_t64(np.asarray(stage[n], np.float32), device) for n in ("bn_weight", "bn_bias", "bn_mean", "bn_var"))
    invstd = _f32(1.0 / _f32(torch.sqrt(_f32(v + float(np.float32(eps))))))
    alpha = _f32(invstd * w)
    return alpha, fma_f32(-m, alpha, b)


def pool_f32(raw, ids, starts, ends, pad_idx: int, pairwise: bool = False) -> torch.Tensor:
    """clas_pool_kernel bit for bit: raw [B, T, E] f32 states, ids [B, T], window [starts[b], ends[b]) -> [B, 3E]
    float64 holding f32 values [last | max | avg].  last = raw[e - 1] (masked or not); max over the unmasked steps; the
    unmasked steps summed in step order from +0, mean = f32(sum / f32(W)), factor = f32(f32(W) / f32(W - n_masked)),
    avg = f32(mean * factor).  ``pairwise=True`` is a negative control: the same sum over two accumulators (even and odd
    steps of the window) added at the end, an order the kernel must not have."""
    raw = _t64(raw)
    dev = raw.device
    B, T, E = raw.shape
    ids = torch.as_tensor(ids, device=dev)
    st = torch.as_tensor(starts, device=dev).long()
    en = torch.as_tensor(ends, device=dev).long()
    if bool(((st < 0) | (en > T) | (st >= en)).any()):
        raise ValueError("a window is empty or outside [0, T]")
    t = torch.arange(T, device=dev)
    inside = (t[None, :] >= st[:, None]) & (t[None, :] < en[:, None])
    keep = inside & (ids != pad_idx)
    n = keep.sum(1)
    if bool((n == 0).any()):
        raise ValueError("a window is entirely pad")
    rows = torch.arange(B, device=dev)
    last = raw[rows, en - 1]
    mx = torch.where(keep[:, :, None], raw, torch.full_like(raw, -float("inf"))).amax(1)
    acc = [torch.zeros(B, E, dtype=torch.float64, device=dev) for _ in range(2)]
    odd = (t[None, :] - st[:, None]) % 2 == 1
    for i in range(int(st.min()), int(en.max())):
        sels = (keep[:, i] & ~odd[:, i], keep[:, i] & odd[:, i]) if pairwise else (keep[:, i],)
        for j, sel in enumerate(sels):
            acc[j] = torch.where(sel[:, None], _f32(acc[j] + raw[:, i]), acc[j])
    total = _f32(acc[0] + acc[1]) if pairwise else acc[0]
    w = _f32((en - st).to(torch.float64))[:, None]
    mean = _f32(total / w)
    factor = _f32(w / _f32(n.to(torch.float64))[:, None])
    return torch.cat([last, mx, _f32(mean * factor)], 1)


def linear_f32(x, alpha, beta, W, bias, relu: bool, reverse: bool = False) -> torch.Tensor:
    """clas_linear_kernel bit for bit: x [B, K] f32 -> [B, N] float64 holding f32 values.  xn = fma(x, alpha, beta);
    acc = +0, then acc = fma(xn[k], W[j, k], acc) for k = 0 .. K - 1; v = f32(acc + bias[j]); ReLU as the kernel writes
    it (v < 0 -> +0, so NaN and -0 pass through).  ``reverse=True`` is a negative control: the chain from k = K - 1 down."""
    x = _t64(x)
    dev = x.device
    alpha, beta, bias = (_t64(a, dev) for a in (alpha, beta, bias))
    W = _t64(W, dev)
    xn = fma_f32(x, alpha[None, :], beta[None, :])
    K = xn.shape[1]
    acc = torch.zeros(x.shape[0], W.shape[0], dtype=torch.float64, device=dev)
    Wt = W.t().contiguous()
    for k in (range(K - 1, -1, -1) if reverse else range(K)):
        acc = fma_f32(xn[:, k, None], Wt[k][None, :], acc)
    v = _f32(acc + bias[None, :])
    if relu:
        v = torch.where(v < 0, torch.zeros_like(v), v)
    return v


def head_f32(pooled, stages: Sequence[dict], eps: float = 1e-5, reverse: bool = False) -> torch.Tensor:
    """The exact logits [B, n_class] (float64 holding f32 values) of the head on the pooled input: per stage the
    BatchNorm fold of ``bn_fold_f32`` and ``linear_f32``, ReLU on every stage but the last."""
    x = _t64(pooled)
    for k, st in enumerate(stages):
        alpha, beta = bn_fold_f32(st, eps, x.device)
        W = torch.as_tensor(np.asarray(st["weight"], np.float32), device=x.device)
        b = torch.as_tensor(np.asarray(st["bias"], np.float32), device=x.device)
        x = linear_f32(x, alpha, beta, W, b, relu=k < len(stages) - 1, reverse=reverse)
    return x


def sigmoid_bound(z):
    """(p64, bound) for clas_activate_kernel's sigmoid on exact logits z (f32 values): |p_device - p64| <= bound.

    The device computes e = expf(-z), q = f32(1 + e), p = f32(1 / q).  expf is within 2 ulp (CUDA C++ Programming Guide,
    single-precision mathematical functions), at most 4u |e| for a normal e; p = 1 / (1 + e) has dp / p = -(e / (1 + e))
    de / e, so that is at most 4u relative in p.  The add and the division add u each: 6u p to first order, times 1.01
    for the second-order terms.  Where -z > 88.72 expf overflows to inf and the device gives 0 for a p below 3e-39, and a
    subnormal e or p is off by at most a subnormal ulp: the absolute term 2^-126 covers both."""
    z = _t64(z)
    p = 1.0 / (1.0 + torch.exp(-z))
    return p, 1.01 * 6 * U * p + 2.0 ** -126


def softmax_bound(z):
    """(p64, bound) for clas_activate_kernel's softmax on exact logits z [B, N] (f32 values), row by row.

    Device: m = max z (exact); d_j = f32(z_j - m), off by at most u |d_j|, which moves expf's result by a relative
    u |d_j| (first order); e_j = expf(d_j) adds 4u (2 ulp); each lane sums its L = ceil(N / 32) terms from +0 (L - 1
    roundings: the first add is exact), the xor butterfly adds five more, all of positive terms: the sum S is within
    (L + 4) u + 4u + u max|d| relative.  p_j = f32(e_j / S) adds u to e_j's own 4u + u |d_j|.  So p_j is within
    p_j ((L + 13) u + u |d_j| + u max|d|) to first order (times 1.01), plus 2^-126 absolute for terms expf flushes to a
    subnormal or zero once d < -87.3."""
    z = _t64(z)
    d = z - z.max(1, keepdim=True).values
    e = torch.exp(d)
    p = e / e.sum(1, keepdim=True)
    L = -(-z.shape[1] // 32)
    ad = d.abs()
    return p, 1.01 * p * ((L + 13) * U + U * ad + U * ad.max(1, keepdim=True).values) + 2.0 ** -126
