"""ORACLE (test infrastructure, NOT product code): the encoder's and the MLP head's arithmetic at the device's precision.

Everything is float64 except at the rounding points the kernels perform.  Each rounding point is stated once, here,
with the kernel line that performs it (paths relative to code_intelligence_b200/csrc/):

  operands       bf16 RNE of the embedding, the weights and the layer inputs      misc.cu convert_rows_kernel
                 split-bf16 in the fp32-accurate mode: hi = bf16(x), lo = bf16(x - hi),
                 products hi*hi + lo*hi + hi*lo (the lo*lo term is dropped)        gemm.cu / lstm_layer.cu K loops
  bias           f32(b_ih + b_hh), summed on the host in f32                       api.cu ie_encoder_load_layer
  Gx             fp16 RNE of f32(x W_ih^T + bias): the layer-0 per-token table and
                 the middle layers' input projections                              gemm.cu pack_f16x2 (epilogue store)
                 f32 with IE_GX_BF16=0 / IE_CFG_F32_GX / IE_CFG_FP32
                 none in the fused last layer: z = x W_ih^T + h W_hh^T + bias in f32  lstm_layer.cu FUSE epilogue
  gates          tanh.approx.f32 (rel err 2^-11), ex2+rcp (abs ~1e-7) or IEEE      lstm_common.cuh lstm_cell1
  cell state     f32, never rounded further                                        lstm_layer.cu __stcg(cp, cnew)
  ring           h_t stored bf16 RNE (hi + lo in the fp32-accurate mode): the next
                 step's and the next layer's operand                               lstm_common.cuh store_h1
  pooling        over the f32 h: sum sequential in t order in f32, mean = sum * f32(1/len),
                 max and last exact                                                lstm_common.cuh pool_accumulate1,
                                                                                   misc.cu pool_finalize_kernel
  MLP head       bf16 X and weights, f32 accumulate + bias, relu, bf16 hidden store,
                 sigmoid_acc on the f32 output                                     api.cu ie_mlp_predict_proba, gemm.cu

Teacher forcing.  A free-running reference cannot separate these rounding points from each other: rounding flips of the
bf16 ring carry forward through the recurrence, and their effect is as large as the effect of a wrong rounding point.
``teacher_forced_layer`` therefore predicts h_t of one layer from the device's OWN inputs -- bf16(h^{l-1}_t) and
bf16(h^l_{t-1}) as the ring holds them -- so that only one step of arithmetic separates prediction and device, and
returns a per-element error bound for that step.  The products of all (row, t) run as one batched GEMM (on whatever
torch device the inputs live on); only the float64 cell-state recursion is sequential, and its error is carried as
e_c,t = f_t e_c,t-1 + ... because the device's cell state is not observed.

Mutants (``Mode`` fields and ``pool(..., mutant=)``) are deliberately wrong variants of the arithmetic; tests use them
as negative controls that the bound must reject.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

U24 = 2.0 ** -24                 # f32 unit roundoff
TANH_APPROX_REL = 2.0 ** -10.9   # tanh.approx.f32: maximum relative error 2^-10.987 (PTX ISA)
SPLIT_REL = 2.0 ** -16           # split-bf16 products vs the f32 operands, relative to sum |a b|
ACC_ULPS = 8.0                   # f32 tensor-core accumulation: |error| <= ACC_ULPS * 2^-24 * sum_k |x_k w_k| per pass

IE_CFG_ACCURATE_GATES, IE_CFG_FP32, IE_CFG_F32_GX = 1, 2, 4   # include/issue_emb_b200.h


# ------------------------------------------------------------------------------------------------ rounding points
def _t(x, device=None) -> torch.Tensor:
    if isinstance(x, torch.Tensor):
        return x.to(device=device or x.device, dtype=torch.float64)
    return torch.as_tensor(np.asarray(x), dtype=torch.float64, device=device)


def rne_bf16(x: torch.Tensor) -> torch.Tensor:
    """Round to nearest even bf16 (misc.cu convert_rows_kernel, lstm_common.cuh store_h1, gemm.cu pack_bf16x2)."""
    return x.to(torch.bfloat16).to(x.dtype)


def rne_fp16(x: torch.Tensor) -> torch.Tensor:
    """Round to nearest even IEEE half (gemm.cu pack_f16x2: the Gx / per-token table store)."""
    return x.to(torch.float16).to(x.dtype)


def rne_f32(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).to(x.dtype)


def split_bf16(x: torch.Tensor):
    """hi = bf16(x), lo = bf16(x - hi) of the f32 value x (misc.cu convert_rows_kernel lo_off, store_h1 lo_off)."""
    x = rne_f32(x)
    hi = rne_bf16(x)
    return hi, rne_bf16(x - hi)


def operands(x: torch.Tensor, segs: int):
    """The values the tensor cores read for x: [x] (segs 0, exact), [bf16(x)] (segs 1) or [hi, lo] (segs 3)."""
    if segs == 0:
        return [x]
    if segs == 1:
        return [rne_bf16(rne_f32(x))]
    return list(split_bf16(x))


def products(x_ops, w_ops, segs: int):
    """(sum_k x_k w_k as the device forms it, sum_k |x_k w_k|) for x [M, K], w [N, K]; split-bf16: hi*hi + lo*hi +
    hi*lo.  Products of bf16 values are exact in f64, the f64 sum is exact to 2^-53."""
    if segs == 3:
        (xh, xl), (wh, wl) = x_ops, w_ops
        return xh @ wh.T + xl @ wh.T + xh @ wl.T, xh.abs() @ wh.abs().T
    x, w = x_ops[0], w_ops[0]
    return x @ w.T, x.abs() @ w.abs().T


def acc_err(a: torch.Tensor, segs: int, acc_ulps: float = ACC_ULPS) -> torch.Tensor:
    """Bound of the f32 accumulation of one GEMM pass over sum|xw| = a (three passes in split-bf16)."""
    return acc_ulps * U24 * a * (3 if segs == 3 else 1)


def round_interval(lo: torch.Tensor, hi: torch.Tensor, out_type: str):
    """[RNE(lo), RNE(hi)] in the output type: where a value known to lie in [lo, hi] must land after the store."""
    rnd = {"f32": rne_f32, "bf16": rne_bf16, "fp16": rne_fp16}[out_type]
    return rnd(lo), rnd(hi)


# ------------------------------------------------------------------------------------------------ gates
def sig_err(x: torch.Tensor, s: torch.Tensor, kind: str) -> torch.Tensor:
    """|device sigmoid - sigmoid| at x (s = sigmoid(x))."""
    if kind == "fast":    # ptx.cuh sigmoid_fast = fma(0.5, tanh.approx(0.5 x), 0.5)
        return 0.5 * TANH_APPROX_REL * torch.tanh(0.5 * x).abs() + U24
    if kind == "exp":     # ptx.cuh sigmoid_acc = __fdividef(1, 1 + __expf(-x))
        return 2.0 ** -22 + 2.0 ** -22 * x.abs() * s * (1 - s)
    if kind == "ieee":    # lstm_common.cuh sigmoid_ieee = 1 / (1 + expf(-x))
        return 2.0 ** -22 * s + 2.0 ** -23 * x.abs() * s * (1 - s)
    return torch.zeros_like(x)


def tanh_err(x: torch.Tensor, t: torch.Tensor, kind: str) -> torch.Tensor:
    """|device tanh - tanh| at x (t = tanh(x))."""
    if kind == "fast":    # ptx.cuh tanh_fast = tanh.approx.f32
        return TANH_APPROX_REL * t.abs()
    if kind == "exp":     # ptx.cuh tanh_acc = 1 - __fdividef(2, __expf(2x) + 1)
        return 2.0 ** -22 + 2.0 ** -22 * x.abs() * (1 - t * t)
    if kind == "ieee":    # lstm_common.cuh tanh_ieee (expm1f near 0)
        return 2.0 ** -22 * t.abs() + 2.0 ** -23 + 2.0 ** -23 * x.abs() * (1 - t * t)
    return torch.zeros_like(x)


# ------------------------------------------------------------------------------------------------ modes
@dataclass(frozen=True)
class Mode:
    """Arithmetic of one layer.  segs: 0 exact f64 operands, 1 bf16, 3 split-bf16.  gx: 'fp16' | 'f32' | 'fused' |
    'exact' (mutant: 'bf16').  gates: 'fast' | 'exp' | 'ieee' | 'exact'.  cell: 'f32' | 'exact' (mutant: 'bf16').
    Mutants: stale_c -- units that read c_{t-2} instead of c_{t-1} (a lost-ordering race); swap_fo -- units whose f and o
    gates are exchanged (a permutation slip)."""
    segs: int = 1
    gx: str = "fp16"
    gates: str = "fast"
    cell: str = "f32"
    stale_c: tuple = ()
    swap_fo: tuple = ()


EXACT = Mode(segs=0, gx="exact", gates="exact", cell="exact")


def layer_modes(n_layers: int, flags: int = 0, env: dict | None = None):
    """The Mode of every layer for an encoder created with `flags` under the development knobs `env`, as
    api.cu ie_encoder_create / run_encoder choose them (assumes the persistent grid is co-resident)."""
    env = {k: str(v) for k, v in (env or {}).items()}
    if flags & IE_CFG_FP32:
        segs, gx, gates = 3, "f32", "ieee"
    else:
        segs = 1
        gates = "exp" if flags & IE_CFG_ACCURATE_GATES else "fast"
        gx = "f32" if flags & IE_CFG_F32_GX else "fp16"
        if "IE_GX_BF16" in env:
            gx = "fp16" if int(env["IE_GX_BF16"]) else "f32"
        if "IE_FAST_MATH" in env:
            gates = "fast" if int(env["IE_FAST_MATH"]) else "exp"
    persistent = int(env.get("IE_SEQ", "1")) != 0
    fuse_last = int(env.get("IE_FUSE_LAST", "1")) != 0
    modes = []
    for l in range(n_layers):
        fused = persistent and fuse_last and segs == 1 and l == n_layers - 1 and l > 0
        modes.append(Mode(segs=segs, gx="fused" if fused else gx, gates=gates))
    return modes


def _bias(w, mode: Mode, device):
    b_ih, b_hh = np.asarray(w["b_ih"]), np.asarray(w["b_hh"])
    if mode.gx == "exact":
        return _t(b_ih.astype(np.float64) + b_hh.astype(np.float64), device)
    return _t(b_ih.astype(np.float32) + b_hh.astype(np.float32), device)   # api.cu: f32 sum on the host


def _preactivation(px, ax, ph, ah, bias, mode: Mode, acc_ulps: float):
    """z = x W_ih^T + h W_hh^T + bias with the Gx rounding point of `mode`, and the bound of |z_device - z|."""
    s = mode.segs
    if mode.gx == "exact":
        z = px + bias + ph
        return z, torch.zeros_like(z)
    if mode.gx == "fused":
        z = px + ph + bias
        return z, acc_err(ax + ah, s, acc_ulps) + 2 * U24 * z.abs()
    g = px + bias
    eg = acc_err(ax, s, acc_ulps) + U24 * g.abs()
    if mode.gx in ("fp16", "bf16"):
        rnd = rne_fp16 if mode.gx == "fp16" else rne_bf16
        gq = rnd(g)
        # the device rounds its own f32 value, which lies within eg of g: at most the neighbouring 16-bit value
        eg = torch.maximum((rnd(g - eg) - gq).abs(), (rnd(g + eg) - gq).abs())
        g = gq
    z = ph + g
    return z, acc_err(ah, s, acc_ulps) + eg + U24 * z.abs()


def _gate_views(z: torch.Tensor, H: int, swap_fo=()):
    """(.., 4H) in torch gate order i|f|g|o -> four (.., H) views; swap_fo exchanges f and o of the listed units."""
    zi, zf, zg, zo = (z[..., k * H:(k + 1) * H] for k in range(4))
    if swap_fo:
        u = list(swap_fo)
        zf, zo = zf.clone(), zo.clone()
        zf[..., u], zo[..., u] = z[..., 3 * H:][..., u], z[..., H:2 * H][..., u]
    return zi, zf, zg, zo


def _cell_loop(z, ez, H, mode: Mode, T: int):
    """Gates and the sequential f64 cell recursion over t of z [R, T, 4H] -> (h [R, T, H], bound [R, T, H])."""
    zi, zf, zg, zo = _gate_views(z, H, mode.swap_fo)
    ei, ef, eg_, eo = _gate_views(ez, H, mode.swap_fo)
    k = mode.gates
    i, f, o, g = torch.sigmoid(zi), torch.sigmoid(zf), torch.sigmoid(zo), torch.tanh(zg)
    ei = i * (1 - i) * ei + sig_err(zi, i, k)
    ef = f * (1 - f) * ef + sig_err(zf, f, k)
    eo = o * (1 - o) * eo + sig_err(zo, o, k)
    eg_ = (1 - g * g) * eg_ + tanh_err(zg, g, k)
    R = z.shape[0]
    c1 = torch.zeros(R, H, dtype=z.dtype, device=z.device)   # c_{t-1}
    c2 = torch.zeros_like(c1)                                   # c_{t-2} (stale-read mutant)
    ec = torch.zeros_like(c1)
    hs, eh = torch.empty(R, T, H, dtype=z.dtype, device=z.device), torch.empty(R, T, H, dtype=z.dtype, device=z.device)
    rnd = mode.cell != "exact"
    for t in range(T):
        cp = c1
        if mode.stale_c:
            cp = c1.clone()
            cp[:, list(mode.stale_c)] = c2[:, list(mode.stale_c)]
        ig = i[:, t] * g[:, t]
        c = f[:, t] * cp + ig                                   # lstm_common.cuh lstm_cell1: cnew = f c + i g (f32)
        if mode.cell == "bf16":
            c = rne_bf16(c)
        ec = (f[:, t] * ec + cp.abs() * ef[:, t] + g[:, t].abs() * ei[:, t] + i[:, t].abs() * eg_[:, t]
              + (U24 * (ig.abs() + c.abs()) if rnd else 0))
        tc = torch.tanh(c)
        h = o[:, t] * tc                                        # hn = o tanh(cnew)
        hs[:, t] = h
        eh[:, t] = (tc.abs() * eo[:, t] + o[:, t] * ((1 - tc * tc) * ec + tanh_err(c, tc, k))
                    + (U24 * h.abs() if rnd else 0))
        c2, c1 = c1, c
    return hs, eh


# ------------------------------------------------------------------------------------------------ one layer
def teacher_forced_layer(x_in, h_dev, weights: dict, mode: Mode, acc_ulps: float = ACC_ULPS):
    """Predict every h_t of one layer from the device's own inputs.

    x_in  [R, T, in]  the layer's input as f32 values: Emb[ids] for layer 0, the previous layer's device states after it
    h_dev [R, T, out] this layer's device states (f32); h_{t-1} of the prediction is their ring rounding
    weights       dict(w_ih [4 out, in], w_hh [4 out, out], b_ih, b_hh) in torch.nn.LSTM layout
    Returns (h_pred, bound) float64 [R, T, out] on the device of h_dev (torch tensors): |h_dev - h_pred| <= bound is
    expected of a kernel that rounds where `mode` says and only there."""
    h_dev = _t(h_dev)
    dev = h_dev.device
    x_in = _t(x_in, dev)
    R, T, H = h_dev.shape
    x = x_in.reshape(R * T, -1)
    hprev = torch.cat([torch.zeros(R, 1, H, dtype=h_dev.dtype, device=dev), h_dev[:, :-1]], 1).reshape(R * T, H)
    s = mode.segs
    px, ax = products(operands(x, s), operands(_t(weights["w_ih"], dev), s), s)
    ph, ah = products(operands(hprev, s), operands(_t(weights["w_hh"], dev), s), s)
    z, ez = _preactivation(px, ax, ph, ah, _bias(weights, mode, dev), mode, acc_ulps)
    return _cell_loop(z.reshape(R, T, 4 * H), ez.reshape(R, T, 4 * H), H, mode, T)


def free_run_layer(x_in, weights: dict, mode: Mode, dtype=torch.float32):
    """Free-running emulation of one layer: the rounding points of `mode` with the arithmetic between them done in
    `dtype` (float32: a stand-in for the device; float64 with EXACT: the plain LSTM of oracle.lstm_numpy).
    x_in [R, T, in] -> h [R, T, out] float64 (values of `dtype`)."""
    x_in = _t(x_in)
    dev = x_in.device
    R, T, _ = x_in.shape
    w_hh = _t(weights["w_hh"], dev)
    H = w_hh.shape[1]
    s = mode.segs

    def prod(a, w):
        ops_a, ops_w = operands(a, s), operands(w, s)
        if s == 3:
            (ah, al), (wh, wl) = [[o.to(dtype) for o in v] for v in (ops_a, ops_w)]
            return (ah @ wh.T + al @ wh.T + ah @ wl.T).double()
        return (ops_a[0].to(dtype) @ ops_w[0].to(dtype).T).double()

    cast = (lambda v: v) if dtype == torch.float64 else rne_f32
    bias = _bias(weights, mode, dev)
    px = prod(x_in.reshape(R * T, -1), _t(weights["w_ih"], dev)).reshape(R, T, 4 * H)
    if mode.gx not in ("fused", "exact"):
        px = cast(px + bias)
        if mode.gx == "fp16":
            px = rne_fp16(px)
        elif mode.gx == "bf16":
            px = rne_bf16(px)
    h = torch.zeros(R, H, dtype=torch.float64, device=dev)
    c = torch.zeros_like(h)
    out = torch.empty(R, T, H, dtype=torch.float64, device=dev)
    for t in range(T):
        ph = prod(h, w_hh)
        z = cast(px[:, t] + ph + bias) if mode.gx in ("fused", "exact") else cast(px[:, t] + ph)
        zi, zf, zg, zo = (v.to(dtype) for v in _gate_views(z, H, mode.swap_fo))
        c_new = torch.sigmoid(zf) * c.to(dtype) + torch.sigmoid(zi) * torch.tanh(zg)
        if mode.cell == "bf16":
            c_new = c_new.to(torch.bfloat16).to(dtype)
        h = (torch.sigmoid(zo) * torch.tanh(c_new)).double()
        c = c_new.double()
        out[:, t] = h
    return out


def free_run(emb, layers, ids, modes, dtype=torch.float32):
    """All layers of a free-running emulation: ids [B, T] -> list of per-layer states [B, T, out_l] float64."""
    x = _t(np.asarray(emb)[np.asarray(ids)])
    states = []
    for w, m in zip(layers, modes):
        x = free_run_layer(x, w, m, dtype)
        states.append(x)
    return states


# ------------------------------------------------------------------------------------------------ pooling
def pool(h, lengths, mutant: str | None = None) -> np.ndarray:
    """[mean | max | last] of the last layer's f32 states h [B, T, E] over the first lengths[b] steps, as the kernel
    forms them: sum sequential in t order in f32 (lstm_common.cuh pool_accumulate1: store at t = 0, red.add.f32 after),
    mean = sum * (1.0f / len) (misc.cu pool_finalize_kernel), running max and last exact.
    Mutants: 'ring' pools the bf16 ring instead of the f32 h; 'max_pad' lets the max read one padded step."""
    h = np.asarray(h, dtype=np.float32)
    if mutant == "ring":
        h = torch.from_numpy(h).to(torch.bfloat16).float().numpy()
    B, T, E = h.shape
    lengths = np.asarray(lengths, dtype=np.int64)
    s = h[:, 0].copy()
    for t in range(1, T):
        live = (t < lengths)[:, None]
        s = np.where(live, s + h[:, t], s)                      # f32 + f32: round to nearest even
    inv = np.float32(1.0) / lengths.astype(np.float32)          # IEEE division in f32
    out = np.empty((B, 3 * E), dtype=np.float32)
    out[:, :E] = s * inv[:, None]
    for b in range(B):
        n = int(lengths[b])
        m = n + 1 if (mutant == "max_pad" and n < T) else n
        out[b, E:2 * E] = h[b, :m].max(0)
        out[b, 2 * E:] = h[b, n - 1]
    return out


# ------------------------------------------------------------------------------------------------ GEMM
def gemm_interval(a, b, bias, act: int, out_type: str, segs: int, acc_ulps: float = ACC_ULPS, device=None):
    """Where each element of act(a b^T + bias), computed by the library's GEMM and stored as out_type, must lie.
    segs 1: the f64 product of the bf16-rounded operands +- the accumulation bound; segs 3: the f64 product of the
    ORIGINAL f32 operands +- SPLIT_REL * sum|a b| (split-bf16 drops lo*lo and the residual of x - hi - lo).
    Returns (lo, hi, ref) float64 torch tensors [M, N]; ref is the unrounded value."""
    a, b = _t(a, device), _t(b, device)
    if segs == 3:
        z, sab = a @ b.T, a.abs() @ b.abs().T
        eps = SPLIT_REL * sab
    else:
        z, sab = products(operands(a, 1), operands(b, 1), 1)
        eps = acc_err(sab, 1, acc_ulps)
    if bias is not None:
        z = z + _t(bias, a.device)
    eps = eps + 2 * U24 * z.abs()
    lo, hi = z - eps, z + eps
    if act == 1:
        lo, hi, z = lo.clamp_min(0), hi.clamp_min(0), z.clamp_min(0)
    elif act == 2:
        sl, sh, z = torch.sigmoid(lo), torch.sigmoid(hi), torch.sigmoid(z)
        lo, hi = sl - sig_err(lo, sl, "exp"), sh + sig_err(hi, sh, "exp")
    lo, hi = round_interval(lo, hi, out_type)
    return lo, hi, z


# ------------------------------------------------------------------------------------------------ MLP head
def mlp_head(X, coefs, intercepts, acc_ulps: float = ACC_ULPS, device=None):
    """The MLP head at device precision with interval propagation: X f32 -> bf16 (misc.cu convert_rows_vec_kernel),
    weights bf16 (api.cu ie_mlp_load_layer), f32 accumulate + bias, relu, bf16 hidden store (gemm.cu pack_bf16x2), the
    last layer sigmoid_acc on f32.  A hidden value whose interval straddles a bf16 rounding boundary may be either
    neighbour on the device; that uncertainty is carried into the next layer.
    Returns (p, lo, hi) float64 torch tensors [n, n_labels]: the device's probabilities must lie in [lo, hi]."""
    x = rne_bf16(_t(np.asarray(X, dtype=np.float32), device))
    rad = torch.zeros_like(x)
    n = len(coefs)
    for l, (W, bvec) in enumerate(zip(coefs, intercepts)):
        w = rne_bf16(_t(np.asarray(W, dtype=np.float32), x.device))          # [fan_in, fan_out]
        z = x @ w + _t(np.asarray(bvec, dtype=np.float32), x.device)
        eps = acc_err((x.abs() + rad) @ w.abs(), 1, acc_ulps) + rad @ w.abs() + 2 * U24 * z.abs()
        if l < n - 1:
            lo, hi = rne_bf16((z - eps).clamp_min(0)), rne_bf16((z + eps).clamp_min(0))
            x, rad = (lo + hi) / 2, (hi - lo) / 2
        else:
            p, sl, sh = torch.sigmoid(z), torch.sigmoid(z - eps), torch.sigmoid(z + eps)
            return p, sl - sig_err(z - eps, sl, "exp"), sh + sig_err(z + eps, sh, "exp")


# ------------------------------------------------------------------------------------------------ statistics
def ratio_stats(h_dev, pred, bound) -> dict:
    """max and RMS of |h_dev - pred| / bound over every element."""
    h_dev = _t(h_dev, pred.device)
    r = (h_dev - pred).abs() / bound.clamp_min(1e-30)
    return {"max": float(r.max()), "rms": float(torch.sqrt((r * r).mean()))}
