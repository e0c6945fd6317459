"""ORACLE (test infrastructure, NOT product code) for the language model: fastai 1.0.53's ``language_model_learner``
(``get_language_model`` = ``SequentialRNN(AWD_LSTM, LinearDecoder)``) in eval mode restated on torch modules, a literal
``LanguageModelPreLoader`` and validate loop, and the float64 restatement of the device's fused decoder with its
per-element bounds.

fastai is not installed; the semantics below are restated from fastai 1.0.53's published source (text/data.py,
text/models/awd_lstm.py, basic_train.py, callbacks/rnn.py, metrics.py), nothing is copied:

* ``LinearDecoder(n_out, n_hid, output_p, tie_encoder, bias=True)``: ``nn.Linear(n_hid, n_out)`` on the last layer's
  outputs (output dropout off in eval); with ``tie_weights`` its weight is the embedding's during training, and the
  saved state dict holds it as ``1.decoder.weight`` next to ``0.encoder.weight``.
* ``LanguageModelPreLoader.on_epoch_begin``: ``step = totalToks / bs``; for row ``i`` walk the documents (in order, a
  ``Circularindex``) until the one holding token ``int(step * i)``: ``ro[i]`` the offset inside it, ``ri[i]`` its index.
  ``__getitem__`` fills the row's ``bptt + 1`` buffer with ``fill_row(forward, items, idx, row, ro, ri, overlap=1)``:
  copy from document ``ri`` at ``ro`` on, continuing at offset 0 of the next documents (circularly) until the buffer is
  full; the next fill starts at the buffer's last token.  ``ite_len = bs * ceil(totalToks / (bptt * bs))``.
* ``learn.validate()``: ``RNNTrainer.on_epoch_begin`` resets the model (zero state) once; ``loss_batch`` per batch with
  the state carried; ``CrossEntropyFlat`` mean and ``accuracy`` = mean of ``argmax(-1) == y``; the epoch's values are the
  batch values averaged with weights = batch size.
"""
from __future__ import annotations

import math
from typing import List, Sequence

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from . import awd_lstm_ref as R
from . import device_numerics as DN

U = 2.0 ** -24          # f32 unit roundoff
EXP_REL = 2.0 ** -21    # ex2.approx.ftz.f32 relative error (lm.cu ex2_approx): twice the 2^-22.7 measured on an H100
SLICE_TILES = 32        # kernels.h kLmSliceTiles


class LanguageModelRef(nn.Module):
    """Eval-mode ``get_language_model``: ``AWDLSTMEncoderRef`` plus the decoder ``nn.Linear(emb_sz, vocab_sz)``."""

    def __init__(self, enc: R.AWDLSTMEncoderRef, tied: bool = True):
        super().__init__()
        self.enc = enc
        self.decoder = nn.Linear(enc.emb_sz, enc.vocab_sz)
        with torch.no_grad():
            if tied:
                self.decoder.weight.copy_(enc.encoder.weight)
            self.decoder.bias.zero_()
        self.eval()

    @torch.no_grad()
    def forward(self, ids) -> torch.Tensor:
        """ids (B, T) -> logits (B, T, V), zero state."""
        return self.decoder(self.enc(torch.as_tensor(np.asarray(ids, dtype=np.int64))))

    def fastai_state_dict(self) -> dict:
        """The state dict ``learn.model.state_dict()`` has for this model."""
        sd = {"0.encoder.weight": self.enc.encoder.weight.detach().clone(),
              "0.encoder_dp.emb.weight": self.enc.encoder.weight.detach().clone()}
        for l, rnn in enumerate(self.enc.rnns):
            sd[f"0.rnns.{l}.weight_hh_l0_raw"] = rnn.weight_hh_l0.detach().clone()
            for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"):
                sd[f"0.rnns.{l}.module.{n}"] = getattr(rnn, n).detach().clone()
        sd["1.decoder.weight"] = self.decoder.weight.detach().clone()
        sd["1.decoder.bias"] = self.decoder.bias.detach().clone()
        return sd


def make_lm(seed=5, vocab_sz=500, emb_sz=96, n_hid=200, n_layers=3, tied=False, dec_scale=1.0, bias_scale=0.0,
            scale=2.0) -> LanguageModelRef:
    """A random LM.  A random-init decoder gives near-uniform softmaxes; ``dec_scale`` multiplies the decoder weight so
    that a share of tokens have clear margins, ``bias_scale`` draws a random bias."""
    enc = R.make_encoder(seed, vocab_sz, emb_sz, n_hid, n_layers, scale=scale)
    lm = LanguageModelRef(enc, tied=tied)
    g = torch.Generator().manual_seed(seed + 7)
    with torch.no_grad():
        if not tied:
            lm.decoder.weight.copy_(torch.randn(vocab_sz, emb_sz, generator=g) / math.sqrt(emb_sz))
        lm.decoder.weight.mul_(dec_scale)
        lm.decoder.bias.copy_(bias_scale * torch.randn(vocab_sz, generator=g))
    return lm


# ------------------------------------------------------------------------------------------------ the preloader
class PreLoaderRef:
    """``LanguageModelPreLoader`` for a validation set (forward, no shuffle), written out as fastai runs it."""

    def __init__(self, docs: Sequence[np.ndarray], bs: int, bptt: int):
        self.items = [np.asarray(d, dtype=np.int64) for d in docs]
        self.lengths = np.array([len(d) for d in self.items])
        self.bs, self.bptt = bs, bptt
        self.totalToks = int(self.lengths.sum())
        self.ite_len = bs * int(math.ceil(self.totalToks / (bptt * bs)))
        self.idx = list(range(len(self.items)))
        self.batch = np.zeros((bs, bptt + 1), dtype=np.int64)

    def on_epoch_begin(self):
        self.ro = np.zeros(self.bs, dtype=np.int64)
        self.ri = np.zeros(self.bs, dtype=np.int64)
        step = self.totalToks / self.bs
        ln_rag, countTokens, i_rag = 0, 0, -1
        for i in range(self.bs):
            while ln_rag + countTokens <= int(step * i):
                countTokens += ln_rag
                i_rag += 1
                ln_rag = self.lengths[self.idx[i_rag]]
            self.ro[i] = int(step * i) - countTokens
            self.ri[i] = i_rag

    def fill_row(self, row, ro, ri, overlap=1):
        ibuf = n = 0
        ri -= 1
        while ibuf < row.size:
            ri += 1
            ri %= len(self.idx)
            rag = self.items[self.idx[ri]]
            ro = 0 if ibuf else ro
            n = min(self.lengths[self.idx[ri]] - ro, row.size - ibuf)
            row[ibuf:ibuf + n] = rag[ro:ro + n]
            ibuf += n
        return ro + n - overlap, ri

    def batches(self):
        """The epoch's (x, y) batches, [bs, bptt] each."""
        self.on_epoch_begin()
        for k in range(self.ite_len):
            j = k % self.bs
            self.ro[j], self.ri[j] = self.fill_row(self.batch[j], self.ro[j], self.ri[j])
            if j == self.bs - 1:
                yield self.batch[:, :-1].copy(), self.batch[:, 1:].copy()


@torch.no_grad()
def validate_literal(lm: LanguageModelRef, docs, bs: int, bptt: int):
    """``learn.validate()`` as fastai runs it: one reset, the (h, c) of every layer carried from batch to batch, per
    batch the mean cross-entropy and accuracy, then their batch-size-weighted means.  (val_loss, accuracy)."""
    state = [None] * len(lm.enc.rnns)
    losses, accs, nums = [], [], []
    for x, y in PreLoaderRef(docs, bs, bptt).batches():
        h = lm.enc.encoder(torch.as_tensor(x))
        for l, rnn in enumerate(lm.enc.rnns):
            h, state[l] = rnn(h, state[l])
        logits = lm.decoder(h)
        yt = torch.as_tensor(y)
        losses.append(float(F.cross_entropy(logits.reshape(-1, logits.shape[-1]), yt.reshape(-1))))
        accs.append(float((logits.argmax(-1) == yt).float().mean()))
        nums.append(x.shape[0])
    return float(np.average(losses, weights=nums)), float(np.average(accs, weights=nums))


@torch.no_grad()
def validate_one_run(lm: LanguageModelRef, x, y, bptt: int):
    """The same pair from one zero-state run over whole rows (the device's design)."""
    logits = lm(x)
    nll = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), torch.as_tensor(y).reshape(-1),
                          reduction="none").reshape(y.shape)
    pred = logits.argmax(-1).numpy()
    n_b = x.shape[1] // bptt
    cols = [slice(k * bptt, (k + 1) * bptt) for k in range(n_b)]
    return (float(np.mean([nll[:, c].double().mean() for c in cols])),
            float(np.mean([(pred[:, c] == y[:, c]).mean() for c in cols])))


# ------------------------------------------------------------------------------------------------ the decoder in f64
def decoder_f64(h, W, b, targets, segs: int, device=None) -> dict:
    """The fused decoder (csrc/lm.cu) in float64 from the device's operands: h [M, E] the f32 states (the ring holds
    bf16(h), or split-bf16), W [V, E], b [V] f32, targets [M] (-100 ignored).  Returns float64 numpy arrays per row:
    lse, nll, pred (argmax, ties to the lowest index), margin (top-1 minus top-2 logit), eps (the largest logit bound
    of the row), b_lse and b_nll (bounds on |device - value|).

    Bounds.  A logit is the MMA chain of the device's operands (device_numerics.chain / acc_err, the tensor-core model
    measured in tests/test_gpu_primitives.py) plus the bias add (one f32 rounding); lse moves by at most the largest
    logit error.  The kernel's sum of exp(x - m) carries per term ex2.approx's error at its own exp and at every rescale
    it meets (at most SLICE_TILES + 3: the tiles of its slice, two quad merges, the slice combine) and the rounding of
    its exponent argument (x - m) * log2(e), which telescopes to 2.5 u (M - x) over those steps; the f32 additions
    along the longest chain (64 terms of a thread's tile, one per tile, two merges, S slices) each add u of the sum; the
    log, the final add and the nll subtraction one rounding each."""
    h, W = DN._t(h, device), DN._t(W, device)
    bt = DN._t(b, h.device)
    P, A, S = DN.chain(DN.passes(DN.operands(h, segs), DN.operands(W, segs), segs))
    z = P + bt
    eps = DN.acc_err(S, A) + U * z.abs()
    del P, A, S
    V = z.shape[1]
    top2 = torch.topk(z, min(2, V), dim=1).values
    M = top2[:, 0]
    margin = (top2[:, 0] - top2[:, 1]) if V > 1 else torch.full_like(M, math.inf)
    pred = torch.argmax(z, dim=1)          # first maximum: the lowest index
    lse = torch.logsumexp(z, dim=1)
    R_ = M - z.min(dim=1).values
    n_sl = (V + 256 * SLICE_TILES - 1) // (256 * SLICE_TILES)
    delta = (SLICE_TILES + 4) * EXP_REL + 2.5 * U * R_ + (64 + SLICE_TILES + 4 + n_sl) * U + V * 2.0 ** -126
    e_row = eps.max(dim=1).values
    b_lse = e_row + delta / (1 - delta) + 2 * U * (lse - M).abs() + 2.0 ** -126 + U * lse.abs()
    t = torch.as_tensor(np.asarray(targets, dtype=np.int64), device=h.device)
    ign = t == -100
    ti = t.clamp_min(0)
    zt = z.gather(1, ti[:, None])[:, 0]
    et = eps.gather(1, ti[:, None])[:, 0]
    nll = torch.where(ign, torch.zeros_like(lse), lse - zt)
    b_nll = torch.where(ign, torch.zeros_like(lse), b_lse + et + U * nll.abs())
    f = lambda x: x.detach().cpu().numpy()
    return dict(lse=f(lse), nll=f(nll), pred=f(pred), margin=f(margin), eps=f(e_row), b_lse=f(b_lse), b_nll=f(b_nll))


# ------------------------------------------------------------------------------------------------ the decoder in f32
# The fused decoder (csrc/lm.cu) bit for bit from the f32 accumulators of h W^T.  Every step is one eager torch op on
# float32 tensors (IEEE round to nearest, no contraction: torch evaluates each op alone), except the rescale, which the
# kernel contracts into an fma and which goes through text_clas_ref.fma_f32.  The order below is the one lm.cu's SASS
# has (tests/test_language_model_reference.py pins it): x - m, then a multiply by log2(e) as f32 (0x3fb8aa3b), then
# ex2; ts a left-to-right chain of adds; s = fma(s, scale, ts) the only contraction; merge two products and one add.
LOG2E_F32 = float(np.float32(1.4426950408889634))   # lm.cu kLog2e
NO_ARG = 0x7fffffff
EXACT_MUTANTS = ("tiles_desc", "no_fma", "quad_pairs", "slices_desc", "one_lane", "log_f64")


def ex2_rn(x: torch.Tensor) -> torch.Tensor:
    """A correctly rounded stand-in for ex2.approx.ftz.f32: 2^x rounded to f32, results below 2^-126 flushed to 0."""
    y = torch.exp2(x.double())
    return torch.where(y < 2.0 ** -126, torch.zeros_like(y), y).float()


def logf_rn(x: torch.Tensor) -> torch.Tensor:
    """A correctly rounded stand-in for logf."""
    return torch.log(x.double()).float()


def _exp_sub(x, m, ex2):
    """lm.cu exp_sub: ex2(f32(f32(x - m) * log2(e)))."""
    return ex2((x - m) * torch.tensor(LOG2E_F32, dtype=torch.float32, device=x.device))


def _merge(a, b, ex2):
    """lm.cu merge of partials a = (m, s, arg) and b: max, s = f32(s_a * e_a) + f32(s_b * e_b) (two products, one add),
    argmax with ties to the lower index; unchanged a where both maxima are -inf."""
    (m, s, arg), (m2, s2, arg2) = a, b
    ninf = -math.inf
    mn = torch.maximum(m, m2)
    dead = mn == ninf
    mn0 = torch.where(dead, torch.zeros_like(mn), mn)
    ea = _exp_sub(torch.where(m == ninf, mn0, m), mn0, ex2)
    eb = _exp_sub(torch.where(m2 == ninf, mn0, m2), mn0, ex2)
    pa = torch.where(m == ninf, torch.zeros_like(s), s * ea)
    pb = torch.where(m2 == ninf, torch.zeros_like(s2), s2 * eb)
    arg_n = torch.where(m2 > m, arg2, torch.where(m > m2, arg, torch.minimum(arg, arg2)))
    return (torch.where(dead, m, mn), torch.where(dead, s, pa + pb), torch.where(dead, arg, arg_n))


def decoder_f32_exact(acc, bias, targets, ex2, logf, mutant=None):
    """The outputs of csrc/lm.cu bit for bit: acc [M, V] f32 the rows' accumulators of h W^T (the GEMM mainloop's
    bits), bias [V] f32 or None, targets [M] (-100 ignored), ex2 / logf callables on f32 tensors (the device's through
    ie_debug_gates, or ex2_rn / logf_rn).  Returns torch (nll f32, lse f32, pred int32) [M] on acc's device.

    * logit = f32(acc + bias); columns >= V are -inf.
    * Per row, 256-column tile n and quad lane q, the lane's 64 columns 256 n + 8 jg + 2 q + e in (jg, e) order: mx the
      lane's max and am its first column; mn = max(m, mx); ts = the left-to-right f32 sum of exp_sub(x, mn); scale = 0
      while m = -inf, else exp_sub(m, mn); s = fma(s, scale, ts); arg = am where mx > m; m = mn.  A lane whose columns
      are all -inf skips the tile.  The tiles of a slice (32) run in order, the running maxima as a cummax.
    * Per slice, the quad merges lanes (0, 1) and (2, 3), then the two results.
    * The slices merge in order; lse = f32(m + logf(s)), nll = f32(lse - logit[y]) or 0 for y = -100; pred = arg.

    ``mutant`` names an order the kernel must not have (negative controls, EXACT_MUTANTS): ``tiles_desc`` the tiles of
    a slice in descending order, ``no_fma`` the rescale rounded twice, ``quad_pairs`` the quad merged as (0, 2), (1, 3),
    ``slices_desc`` the slices combined in descending order, ``one_lane`` one 256-column chain per tile, ``log_f64``
    lse = f32(m + log(s)) with the log and the add in float64."""
    if mutant is not None and mutant not in EXACT_MUTANTS:
        raise ValueError(f"unknown mutant {mutant!r}")
    from .text_clas_ref import _f32, fma_f32
    acc = torch.as_tensor(acc)
    if acc.dtype != torch.float32 or acc.dim() != 2:
        raise TypeError("acc must be a float32 [M, V] tensor")
    dev = acc.device
    M, V = acc.shape
    ninf = -math.inf
    b = torch.zeros(V, dtype=torch.float32, device=dev) if bias is None else \
        torch.as_tensor(np.asarray(bias, np.float32)).to(dev)
    t = torch.as_tensor(np.asarray(targets, np.int64)).to(dev)
    if bool(((t != -100) & ((t < 0) | (t >= V))).any()):
        raise ValueError("a target outside [0, V) other than -100")
    logit = acc + b[None, :]
    NT = -(-V // 256)
    S = -(-NT // SLICE_TILES)
    NTp = S * SLICE_TILES
    x = torch.full((M, NTp * 256), ninf, dtype=torch.float32, device=dev)
    x[:, :V] = logit
    # lanes [M, tile, lane, k] and each entry's column inside its tile
    if mutant == "one_lane":
        lanes = x.view(M, NTp, 1, 256)
        tcol = torch.arange(256, device=dev)[None, :]
    else:
        lanes = x.view(M, NTp, 32, 4, 2).permute(0, 1, 3, 2, 4).reshape(M, NTp, 4, 64)
        jg, e = torch.arange(64, device=dev) // 2, torch.arange(64, device=dev) % 2
        tcol = 8 * jg[None, :] + 2 * torch.arange(4, device=dev)[:, None] + e[None, :]
    del x
    Q, K = lanes.shape[2], lanes.shape[3]
    tix = torch.arange(NTp, device=dev)                      # processing position -> tile
    if mutant == "tiles_desc":
        tix = tix.view(S, SLICE_TILES).flip(1).reshape(-1)
        lanes = lanes[:, tix]
    mx, kk = lanes.amax(dim=3), lanes.argmax(dim=3)          # argmax: the first maximal index, as `v > mx` keeps
    am = (256 * tix[None, :, None] + tcol[torch.arange(Q, device=dev)[None, None, :], kk]).int()
    mx, am = mx.view(M, S, SLICE_TILES, Q), am.view(M, S, SLICE_TILES, Q)
    skip = mx == ninf
    m_after = torch.cummax(mx, dim=2).values
    m_prev = torch.cat([torch.full_like(m_after[:, :, :1], ninf), m_after[:, :, :-1]], 2)
    mn = torch.where(skip, torch.zeros_like(m_after), m_after)   # skipped lanes: any finite value, masked below
    terms = _exp_sub(lanes.view(M, S, SLICE_TILES, Q, K), mn[..., None], ex2)
    del lanes
    ts = terms[..., 0]
    for k in range(1, K):
        ts = ts + terms[..., k]
    del terms
    first = m_prev == ninf
    scale = torch.where(first, torch.zeros_like(mn), _exp_sub(torch.where(first, mn, m_prev), mn, ex2))
    s = torch.zeros(M, S, Q, dtype=torch.float64, device=dev)
    for p in range(SLICE_TILES):
        sc, tp = scale[:, :, p].double(), ts[:, :, p].double()
        new = _f32(_f32(s * sc) + tp) if mutant == "no_fma" else fma_f32(s, sc, tp)
        s = torch.where(skip[:, :, p], s, new)
    s = s.float()
    m = m_after[:, :, -1]
    hit = (mx == m[:, :, None, :]) & ~skip
    arg = am.gather(2, hit.to(torch.uint8).argmax(2, keepdim=True))[:, :, 0]
    arg = torch.where(m == ninf, torch.full_like(arg, NO_ARG), arg)
    lane = [(m[..., q], s[..., q], arg[..., q]) for q in range(Q)]
    if Q == 1:
        part = lane[0]
    elif mutant == "quad_pairs":
        part = _merge(_merge(lane[0], lane[2], ex2), _merge(lane[1], lane[3], ex2), ex2)
    else:
        part = _merge(_merge(lane[0], lane[1], ex2), _merge(lane[2], lane[3], ex2), ex2)
    order = range(S - 1, -1, -1) if mutant == "slices_desc" else range(S)
    tot = None
    for k in order:
        pk = tuple(v[:, k] for v in part)
        tot = pk if tot is None else _merge(tot, pk, ex2)
    m, s, arg = tot
    if mutant == "log_f64":
        lse = (m.double() + torch.log(s.double())).float()
    else:
        lse = m + logf(s)
    zt = logit.gather(1, t.clamp_min(0)[:, None])[:, 0]
    nll = torch.where(t == -100, torch.zeros_like(lse), lse - zt)
    return nll, lse, arg.int()


def check_decoder(ref: dict, nll, lse, pred) -> dict:
    """Per-element verdict of the device's outputs against ``decoder_f64``: ratios of |error| to bound, the rows whose
    argmax is decided (margin > 2 eps) and how many of those the device got wrong."""
    r_lse = np.abs(lse - ref["lse"]) / ref["b_lse"]
    r_nll = np.abs(nll - ref["nll"]) / np.maximum(ref["b_nll"], 1e-300)
    r_nll[ref["b_nll"] == 0] = np.where(nll[ref["b_nll"] == 0] == 0, 0.0, np.inf)
    decided = ref["margin"] > 2 * ref["eps"]
    return dict(max_lse=float(r_lse.max()), max_nll=float(r_nll.max()), decided=int(decided.sum()),
                wrong_pred=int((pred[decided] != ref["pred"][decided]).sum()), rows=len(nll))
