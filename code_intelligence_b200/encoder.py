"""IssueEncoder: thin Python owner of an `ie_encoder` handle (include/issue_emb_b200.h).

Token ids -> 2400-d [mean | max | last] vectors, i.e. the arithmetic behind
``InferenceWrapper._forward_pass`` + ``batch_seq_pool`` (Issue_Embeddings/flask_app/inference.py:55-57,
215-246) executed by the sm_90a kernels in csrc/.  torch is used only for pinned host buffers, device tensors
and streams.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence

import numpy as np

from . import _lib
from ._lib import IE_FLAG_DEVICE_PTRS, check, ie_config


def _layer_dims(n_layers, emb_sz, n_hid):
    return [((emb_sz if l == 0 else n_hid), (n_hid if l != n_layers - 1 else emb_sz)) for l in range(n_layers)]


def _f32c(a) -> np.ndarray:
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.float32)


class IssueEncoder:
    """AWD-LSTM encoder of the reference's deployed shape by default
    (Embedding(60000,800) -> LSTM 800->2400->2400->2400->800, notebooks/04_Inference.ipynb:157-187)."""

    def __init__(self, n_layers: int = 4, emb_sz: int = 800, n_hid: int = 2400, vocab_sz: int = 60000,
                 pad_idx: int = 1, device: int = 0, flags: int = 0):
        """flags: IE_CFG_* bits of include/issue_emb_b200.h (``_lib.IE_CFG_FP32`` = the split-bf16 fp32-accurate mode,
        ``IE_CFG_ACCURATE_GATES``, ``IE_CFG_F32_GX``); 0 = bf16 operands / f32 accumulate."""
        self._lib = _lib.load()
        self.n_layers, self.emb_sz, self.n_hid, self.vocab_sz, self.pad_idx, self.device = \
            n_layers, emb_sz, n_hid, vocab_sz, pad_idx, device
        self.out_dim = 3 * emb_sz
        self.flags = flags
        cfg = ie_config(n_layers, emb_sz, n_hid, vocab_sz, pad_idx, device, flags)
        h = C.c_void_p()
        check(self._lib.ie_encoder_create(C.byref(cfg), C.byref(h)))
        self._h = h

    # ------------------------------------------------------------------ lifetime
    def close(self):
        if getattr(self, "_h", None):
            self._lib.ie_encoder_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ weights
    def load_weights(self, emb, layers: Sequence[dict]) -> "IssueEncoder":
        """emb [V,E]; layers[l] = dict(w_ih [4*out,in], w_hh [4*out,out], b_ih [4*out], b_hh [4*out]) in
        torch.nn.LSTM layout (gate rows i|f|g|o)."""
        emb = _f32c(emb)
        if emb.shape != (self.vocab_sz, self.emb_sz):
            raise ValueError(f"embedding shape {emb.shape} != {(self.vocab_sz, self.emb_sz)}")
        if len(layers) != self.n_layers:
            raise ValueError(f"expected {self.n_layers} layers, got {len(layers)}")
        check(self._lib.ie_encoder_load_embedding(self._h, emb.ctypes.data))
        for l, ((n_in, n_out), L) in enumerate(zip(_layer_dims(self.n_layers, self.emb_sz, self.n_hid), layers)):
            w_ih, w_hh, b_ih, b_hh = (_f32c(L[k]) for k in ("w_ih", "w_hh", "b_ih", "b_hh"))
            if w_ih.shape != (4 * n_out, n_in) or w_hh.shape != (4 * n_out, n_out) or b_ih.shape != (4 * n_out,) \
                    or b_hh.shape != (4 * n_out,):
                raise ValueError(f"layer {l}: bad weight shapes {w_ih.shape} {w_hh.shape} {b_ih.shape} {b_hh.shape}")
            check(self._lib.ie_encoder_load_layer(self._h, l, w_ih.ctypes.data, w_hh.ctypes.data, b_ih.ctypes.data,
                                                  b_hh.ctypes.data))
        return self

    def load_state_dict(self, sd: dict) -> "IssueEncoder":
        """Accepts the fastai 1.0.53 AWD_LSTM encoder key layout (``save_encoder`` .pth / ``learn.model[0]``;
        Issue_Embeddings/README.md:84-85): ``encoder.weight``, ``rnns.{l}.weight_hh_l0_raw`` (authoritative
        W_hh in eval mode), ``rnns.{l}.module.weight_ih_l0``, ``rnns.{l}.module.bias_{ih,hh}_l0``.  Keys with a
        leading ``0.`` (full SequentialRNN state dict) are accepted too."""
        def get(*names):
            for n in names:
                for pre in ("", "0."):
                    if pre + n in sd:
                        return sd[pre + n]
            raise KeyError(names[0])
        layers = []
        for l in range(self.n_layers):
            layers.append(dict(
                w_ih=get(f"rnns.{l}.module.weight_ih_l0", f"rnns.{l}.weight_ih_l0"),
                w_hh=get(f"rnns.{l}.weight_hh_l0_raw", f"rnns.{l}.module.weight_hh_l0", f"rnns.{l}.weight_hh_l0"),
                b_ih=get(f"rnns.{l}.module.bias_ih_l0", f"rnns.{l}.bias_ih_l0"),
                b_hh=get(f"rnns.{l}.module.bias_hh_l0", f"rnns.{l}.bias_hh_l0")))
        return self.load_weights(get("encoder.weight", "encoder_dp.emb.weight"), layers)

    # ------------------------------------------------------------------ hot path
    def encode_ids(self, ids, lengths=None) -> np.ndarray:
        """ids (B,T) int64 right-padded with pad_idx, lengths (B,) -> (B, 3*emb_sz) float32 numpy.
        B may exceed `max_batch` (IE_MAX_BATCH by default); it is then processed in slices of that many rows."""
        ids = np.ascontiguousarray(np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids), dtype=np.int64)
        if ids.ndim != 2:
            raise ValueError("ids must be (B, T)")
        B, T = ids.shape
        if lengths is None:
            lengths = np.full(B, T, dtype=np.int32)
        lengths = np.ascontiguousarray(np.asarray(lengths), dtype=np.int32)
        assert lengths.shape[0] == B, 'Number of elements in lengths should match the first dimension of ids'
        out = np.empty((B, self.out_dim), dtype=np.float32)
        mb = self.max_batch
        for b0 in range(0, B, mb):
            b1 = min(B, b0 + mb)
            sl = np.ascontiguousarray(ids[b0:b1])
            ln = np.ascontiguousarray(lengths[b0:b1])
            o = out[b0:b1]
            check(self._lib.ie_encoder_encode(self._h, sl.ctypes.data, ln.ctypes.data, b1 - b0, T, o.ctypes.data, 0,
                                              None))
        return out

    def encode_ids_device(self, ids, lengths, out=None, stream=None):
        """Asynchronous device-resident variant: ids cuda int64 (B,T), lengths cuda int32 (B,), out cuda float32
        (B, 3*emb_sz); B <= max_batch.  Runs on `stream` (default: torch's current stream).  Data-dependent errors
        (token id out of range, bad length, device wait timeout) are reported by ``check_errors()``."""
        import torch
        assert ids.is_cuda and lengths.is_cuda and ids.dtype == torch.int64 and lengths.dtype == torch.int32
        ids, lengths = ids.contiguous(), lengths.contiguous()
        B, T = ids.shape
        if tuple(lengths.shape) != (B,):
            raise ValueError(f"lengths has shape {tuple(lengths.shape)}, expected ({B},)")
        if out is None:
            out = torch.empty((B, self.out_dim), dtype=torch.float32, device=ids.device)
        # the library writes B rows through a raw pointer: the buffer must be exactly that
        if (not out.is_cuda or out.dtype != torch.float32 or tuple(out.shape) != (B, self.out_dim)
                or not out.is_contiguous()):
            raise ValueError(f"out must be a contiguous cuda float32 tensor of shape ({B}, {self.out_dim})")
        s = stream if stream is not None else torch.cuda.current_stream(ids.device)
        check(self._lib.ie_encoder_encode(self._h, ids.data_ptr(), lengths.data_ptr(), B, T, out.data_ptr(),
                                          IE_FLAG_DEVICE_PTRS, C.c_void_p(s.cuda_stream)))
        return out

    def check_errors(self) -> None:
        """Waits for the last call on this handle and raises what its device-side checks found (ValueError for a token
        id / length out of range, RuntimeError for a device wait timeout).  Host-buffer calls do this themselves."""
        check(self._lib.ie_encoder_check_errors(self._h))

    def raw_features(self, ids) -> np.ndarray:
        """Last layer hidden states (B,T,emb_sz) float32 -- get_raw_features (inference.py:59-68)."""
        ids = np.ascontiguousarray(np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids), dtype=np.int64)
        if ids.ndim != 2:
            raise ValueError("ids must be (B, T)")
        B, T = ids.shape
        if B > self.max_batch:
            raise ValueError(f"B={B} > {self.max_batch}")
        raw = np.empty((B, T, self.emb_sz), dtype=np.float32)
        check(self._lib.ie_encoder_raw_features(self._h, ids.ctypes.data, B, T, raw.ctypes.data, 0, None))
        return raw

    def _debug_layer_states(self, layer: int, ids):
        """Test hook ``ie_debug_layer_states``: hidden states of ``layer`` (B, T, out_l) float32 as its recurrent kernel
        computed them (the ring holds their bf16 rounding); for the last layer identical to ``raw_features``.
        Host ids give a numpy array.  CUDA int64 ids give a CUDA tensor written in place on torch's current stream
        (IE_FLAG_DEVICE_PTRS: nothing passes through host memory, where one 1280 x 512 x 2400 layer takes 6.3 GB);
        ``check_errors()`` reports that call's data-dependent errors."""
        on_device = getattr(ids, "is_cuda", False)
        if not on_device:
            ids = np.ascontiguousarray(np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids), dtype=np.int64)
        if ids.ndim != 2:
            raise ValueError("ids must be (B, T)")
        B, T = ids.shape
        if B > self.max_batch:
            raise ValueError(f"B={B} > {self.max_batch}")
        if not 0 <= layer < self.n_layers:
            raise ValueError(f"layer {layer} outside [0, {self.n_layers})")
        out_l = self.emb_sz if layer == self.n_layers - 1 else self.n_hid
        if on_device:
            import torch
            if ids.dtype != torch.int64:
                raise ValueError("device ids must be int64")
            ids = ids.contiguous()
            out = torch.empty((B, T, out_l), dtype=torch.float32, device=ids.device)
            s = torch.cuda.current_stream(ids.device)
            check(self._lib.ie_debug_layer_states(self._h, layer, ids.data_ptr(), B, T, out.data_ptr(),
                                                  IE_FLAG_DEVICE_PTRS, C.c_void_p(s.cuda_stream)))
            return out
        out = np.empty((B, T, out_l), dtype=np.float32)
        check(self._lib.ie_debug_layer_states(self._h, layer, ids.ctypes.data, B, T, out.ctypes.data, 0, None))
        return out

    @property
    def max_batch(self) -> int:
        """Rows one C-ABI encode call takes: 256 x batches per launch (1280 by default, IE_BATCHES=n changes it)."""
        return int(self._lib.ie_encoder_max_batch(self._h))

    @property
    def launch_count(self) -> int:
        return int(self._lib.ie_encoder_launch_count(self._h))

    def last_phase_ms(self) -> dict:
        """CUDA-event device time of each phase of the last encode call (waits for it):
        {'gather', 'gemm': [per layer], 'steps': [per layer], 'finalize'} in ms."""
        buf = np.zeros(4 + 2 * self.n_layers, dtype=np.float32)
        n = self._lib.ie_encoder_last_phase_ms(self._h, buf.ctypes.data, buf.size)
        if n < 0:
            check(n)
        v = buf[:n].tolist()
        return dict(gather=v[0], gemm=v[1:1 + 2 * self.n_layers:2], steps=v[2:2 + 2 * self.n_layers:2],
                    finalize=v[1 + 2 * self.n_layers] if n > 1 + 2 * self.n_layers else 0.0)

    def last_phase_mhz(self) -> list:
        """SM clock (MHz) the recurrent kernel ('steps') and the input-projection GEMM ('gemm') of each layer ran at in
        the last call (clock64 / globaltimer stamps taken by the kernels themselves; nvidia-smi cannot resolve phases)."""
        buf = np.zeros(2 * self.n_layers, dtype=np.float32)
        n = self._lib.ie_encoder_last_phase_mhz(self._h, buf.ctypes.data, buf.size)
        if n < 0:
            check(n)
        return dict(steps=buf[:self.n_layers].tolist(), gemm=buf[self.n_layers:n].tolist())

    # ------------------------------------------------------------------ bulk (df_to_embedding on token ids)
    def encode_id_list(self, docs: List[np.ndarray], bs: int = 100, min_batches_rule: bool = True,
                       coalesce: bool = True) -> np.ndarray:
        """The bulk loop of ``df_to_embedding`` (py/code_intelligence/inference.py:171-229) from the
        numericalised docs on: bs = min(bs, N//20+1), argsort by length, right-pad each batch to its own max
        with pad_idx, encode, unsort with argsort(argsort); on RuntimeError (CUDA OOM) halve bs and retry.
        ``coalesce`` (default): consecutive sorted batches are merged into calls of ``max_batch`` rows -- results are
        independent of batch composition here, so the reference's default ``bs=100`` still reaches full launches.
        The loop runs as a device pipeline (pinned double-buffered staging, H2D of batch k+1 under the kernels of batch k,
        un-sort on the device): ``bulk.encode_sorted_batches_device``.  Returns (N, 3*emb_sz) float32 in input order."""
        from .bulk import encode_sorted_batches_device
        return encode_sorted_batches_device(docs, self, bs=bs, min_batches_rule=min_batches_rule, coalesce=coalesce)
