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
as negative controls that the bound must reject.  Some apply at every step (a wrong rounding point, a permutation slip);
the ``*_at`` ones touch a single step of a few units, which is what a broken schedule does to one work item.

``blocked_layer_stats`` runs the teacher-forced check over every row of a benchmark-size launch a block of rows at a
time and reduces it to the statistics the tests cap, with the largest ratio of every schedule item of lstm_layer.cu.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

U24 = 2.0 ** -24                 # f32 unit roundoff
TANH_APPROX_REL = 2.0 ** -10.9   # tanh.approx.f32: maximum relative error 2^-10.987 (PTX ISA)
SPLIT_REL = 2.0 ** -16           # split-bf16 products vs the f32 operands, relative to sum |a b|
TINY = 2.0 ** -150               # f32 rounding below 2^-126: half the subnormal spacing (absolute)
# f32 tensor-core accumulation (oracle/tc_accum.py MODEL, measured on the H100): each k16 step aligns C and its 16
# products to the largest exponent keeping 26 bits (each of the 17 terms loses < 2^-25 of the largest) and truncates
# the sum to f32 (< 2^-23 of it).  Over a chain: |error| <= ACC_STEP * (sum_s |C_s| + sum |x w|), C_s the accumulator
# before step s (tc_accum.acc_err_bound)
ACC_STEP = 17 * 2.0 ** -25 + 2.0 ** -23

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


def passes(x_ops, w_ops, segs: int):
    """The operand pairs of the MMA chain in the order the device adds them: [(x, w)], or in split-bf16 all hi*hi
    steps, then lo*hi, then hi*lo (gemm_kernel.cuh, lstm_layer.cu K loops)."""
    if segs == 3:
        (xh, xl), (wh, wl) = x_ops, w_ops
        return [(xh, wh), (xl, wh), (xh, wl)]
    return [(x_ops[0], w_ops[0])]


def chain(pairs, p0=None, cols: int = 4096):
    """The device's MMA chain over f64 operand pairs (x [M, K], w [N, K]), k16 steps in order, every pair into one
    accumulator starting at p0 (default 0) -> (P, A, S) [M, N]: the sum (products of bf16 values are exact in f64),
    A = sum |x w| and S >= sum over the k16 steps of |P before the step|, the partial sums acc_err charges.  S is formed
    from the exact partial sums B at every 64-wide k-block (four steps): the steps of a block see at most
    4 |B| + 3 A_0 + 2 A_1 + A_2 (A_i the |products| of its i-th step), one weighted GEMM for the A_i terms.  N is taken
    `cols` columns at a time to bound the working set."""
    M, N = pairs[0][0].shape[0], pairs[0][1].shape[0]
    x0 = pairs[0][0]
    P = torch.zeros(M, N, dtype=x0.dtype, device=x0.device) if p0 is None else p0.clone()
    A, S = torch.zeros_like(P), torch.zeros_like(P)
    for c0 in range(0, N, cols):
        p, a, s = P[:, c0:c0 + cols], A[:, c0:c0 + cols], S[:, c0:c0 + cols]
        for x, w in pairs:
            wc = w[c0:c0 + cols]
            xa, wa = x.abs(), wc.abs().T
            a.addmm_(xa, wa)
            later = 3 - (torch.arange(x.shape[1], device=x.device) % 64) // 16   # steps of the block after k's
            s.addmm_(xa * later.to(x.dtype), wa)
            for k0 in range(0, x.shape[1], 64):
                s.add_(p.abs(), alpha=4)
                p.addmm_(x[:, k0:k0 + 64], wc[:, k0:k0 + 64].T)
    return P, A, S


def acc_err(s: torch.Tensor, a: torch.Tensor) -> torch.Tensor:
    """Bound of the f32 accumulation of one MMA chain from its partial sums s and sum |x w| = a (chain).  The device's
    accumulator differs from the exact partial sum by the error so far, far below 2^-10 of it."""
    return ACC_STEP * ((1 + 2.0 ** -10) * s + a)


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
    if kind == "ieee":    # lstm_common.cuh sigmoid_ieee = 1 / (1 + expf(-x)); results below 2^-126 (x < -87.3) carry
        # no relative accuracy (measured on the H100: an error of nearly the whole value 2.9e-39 at x = -88.72)
        return 2.0 ** -22 * s + 2.0 ** -23 * x.abs() * s * (1 - s) + 2.0 ** -126
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
    gates are exchanged (a permutation slip).  Confined to one step (t, units): stale_c_at -- at step t the units read
    c_{t-2}; stale_h_at -- at step t the z of the units is formed from h_{t-2} (a ring slot read before it was written);
    carry_lost_at = t0 -- at step t0 h_{t0-1} and c_{t0-1} read as zero (a lost time-chunk carry)."""
    segs: int = 1
    gx: str = "fp16"
    gates: str = "fast"
    cell: str = "f32"
    stale_c: tuple = ()
    swap_fo: tuple = ()
    stale_c_at: tuple = ()
    stale_h_at: tuple = ()
    carry_lost_at: int = -1


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


def _preactivation(px, ex, ph, eh, bias, mode: Mode):
    """z = x W_ih^T + h W_hh^T + bias with the Gx rounding point of `mode`, and the bound of |z_device - z|; ex, eh are
    the accumulation bounds of the two products (fused: ex + eh is that of the one chain over both)."""
    if mode.gx == "exact":
        z = px + bias + ph
        return z, torch.zeros_like(z)
    if mode.gx == "fused":
        z = px + ph + bias
        return z, ex + eh + 2 * U24 * z.abs()
    g = px + bias
    eg = ex + U24 * g.abs()
    if mode.gx in ("fp16", "bf16"):
        rnd = rne_fp16 if mode.gx == "fp16" else rne_bf16
        gq = rnd(g)
        # the device rounds its own f32 value, which lies within eg of g: at most the neighbouring 16-bit value
        eg = torch.maximum((rnd(g - eg) - gq).abs(), (rnd(g + eg) - gq).abs())
        g = gq
    z = ph + g
    return z, eh + eg + U24 * z.abs()


def _gate_views(z: torch.Tensor, H: int, swap_fo=()):
    """(.., 4H) in torch gate order i|f|g|o -> four (.., H) views; swap_fo exchanges f and o of the listed units."""
    zi, zf, zg, zo = (z[..., k * H:(k + 1) * H] for k in range(4))
    if swap_fo:
        u = list(swap_fo)
        zf, zo = zf.clone(), zo.clone()
        zf[..., u], zo[..., u] = z[..., 3 * H:][..., u], z[..., H:2 * H][..., u]
    return zi, zf, zg, zo


def _gates(zi, zf, zg, zo, ei, ef, eg_, eo, k: str, rnd: bool):
    """Gate values of the preactivations (with bounds ez of |z_device - z|) for gate kind k -> (i g, its bound, f, its
    bound, o, its bound)."""
    i, f, o, g = torch.sigmoid(zi), torch.sigmoid(zf), torch.sigmoid(zo), torch.tanh(zg)
    ei = i * (1 - i) * ei + sig_err(zi, i, k)
    ef = f * (1 - f) * ef + sig_err(zf, f, k)
    eo = o * (1 - o) * eo + sig_err(zo, o, k)
    eg_ = (1 - g * g) * eg_ + tanh_err(zg, g, k)
    ig = i * g
    return ig, g.abs() * ei + i.abs() * eg_ + (U24 * ig.abs() + TINY if rnd else 0), f, ef, o, eo


def _cell_update(ig, e_ig, f, ef, cp, ec, rnd: bool):
    """c = f c_{t-1} + i g (lstm_common.cuh lstm_cell1, f32) and its bound from e_c,t-1 = ec.  The compiler may round
    either product before fusing the other onto it (the fp32 mode rounds f c_{t-1}), so both roundings are charged:
    U24 |i g| in e_ig, U24 |f c_{t-1}| here, and U24 |c| for the sum."""
    c = torch.addcmul(ig, f, cp)
    ec = torch.addcmul(e_ig, f, ec).addcmul_(cp.abs(), ef)
    if rnd:
        ec.add_(c.abs(), alpha=U24).addcmul_(f, cp.abs(), value=U24).add_(2 * TINY)
    return c, ec


def _cell_out(c, ec, o, eo, k: str, rnd: bool):
    """h = o tanh(c) and its bound."""
    tc = torch.tanh(c)
    h = o * tc
    return h, tc.abs() * eo + o * ((1 - tc * tc) * ec + tanh_err(c, tc, k)) + (U24 * h.abs() + TINY if rnd else 0)


def cell_step(zi, zf, zg, zo, c_prev, kind: str):
    """One step of the cell with c_{t-1} given (exact preactivations and c_{t-1}): the arithmetic of _cell_loop for a
    single t.  -> (c, bound of c, h, bound of h) float64 for gate kind 'fast' | 'exp' | 'ieee'."""
    zi, zf, zg, zo, cp = (_t(v) for v in (zi, zf, zg, zo, c_prev))
    zero = torch.zeros_like(zi)
    ig, e_ig, f, ef, o, eo = _gates(zi, zf, zg, zo, zero, zero, zero, zero, kind, True)
    c, ec = _cell_update(ig, e_ig, f, ef, cp, zero, True)
    h, eh = _cell_out(c, ec, o, eo, kind, True)
    return c, ec, h, eh


def cell_grid(seed: int = 5):
    """Adversarial cell inputs: saturated gates (|z| up to 100), f ~ 1 with |c_prev| up to 2^15 (the cell state of a
    20000-token issue over its time chunks), +-0 and tiny c_prev.  -> (z [4, n] planes i, f, g, o; c_prev [n]) float32."""
    rng = np.random.default_rng(seed)
    zs = np.concatenate([np.float32([0, -0.0, 1e-30, -1e-30, 1e-7, 0.5, -0.5, 3, -3, 17, -17, 40, -40, 100, -100]),
                         rng.uniform(-12, 12, 40).astype(np.float32)])
    cs = np.concatenate([np.float32([0, -0.0, 1e-38, -1e-38, 1e-30, 2 ** -20, 1, -1]),
                         np.float32(2.0 ** np.arange(1, 16)) * rng.choice([-1, 1], 15).astype(np.float32),
                         rng.uniform(-300, 300, 20).astype(np.float32)])
    z = rng.choice(zs, (4, 6000)).astype(np.float32)
    z[1, :2000] = rng.uniform(8, 100, 2000)   # f ~ 1: c_prev carried almost unchanged
    cp = rng.choice(cs, 6000).astype(np.float32)
    return z, cp


def _cell_loop(z, ez, H, mode: Mode, T: int):
    """Gates and the sequential f64 cell recursion over t of z [R, T, 4H] -> (h [R, T, H], bound [R, T, H]).  Only c
    and its error bound e_c are sequential; everything else runs over all steps at once."""
    k = mode.gates
    rnd = mode.cell != "exact"
    ig, e_ig, f, ef, o, eo = _gates(*_gate_views(z, H, mode.swap_fo), *_gate_views(ez, H, mode.swap_fo), k, rnd)
    R = z.shape[0]
    c1 = torch.zeros(R, H, dtype=z.dtype, device=z.device)   # c_{t-1}
    c2 = torch.zeros_like(c1)                                   # c_{t-2} (stale-read mutants)
    ec = torch.zeros_like(c1)
    cs, ecs = torch.empty_like(ig), torch.empty_like(ig)
    for t in range(T):
        cp = c1
        if mode.stale_c:
            cp = c1.clone()
            cp[:, list(mode.stale_c)] = c2[:, list(mode.stale_c)]
        if mode.stale_c_at and mode.stale_c_at[0] == t:
            cp = c1.clone()
            cp[:, list(mode.stale_c_at[1])] = c2[:, list(mode.stale_c_at[1])]
        if mode.carry_lost_at == t:
            cp = torch.zeros_like(c1)
        c, ec = _cell_update(ig[:, t], e_ig[:, t], f[:, t], ef[:, t], cp, ec, rnd)
        if mode.cell == "bf16":
            c = rne_bf16(c)
        cs[:, t], ecs[:, t] = c, ec
        c2, c1 = c1, c
    hs, eh = _cell_out(cs, ecs, o, eo, k, rnd)
    return hs, eh


# ------------------------------------------------------------------------------------------------ one layer
def teacher_forced_layer(x_in, h_dev, weights: dict, mode: Mode):
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
    hprev = torch.cat([torch.zeros(R, 1, H, dtype=h_dev.dtype, device=dev), h_dev[:, :-1]], 1)
    if mode.carry_lost_at >= 0:
        hprev[:, mode.carry_lost_at] = 0
    hprev = hprev.reshape(R * T, H)
    s = mode.segs
    w_hh = _t(weights["w_hh"], dev)
    if mode.gx == "exact":
        px, _ = products(operands(x, s), operands(_t(weights["w_ih"], dev), s), s)
        ph, _ = products(operands(hprev, s), operands(w_hh, s), s)
        ex = eh = None
    else:
        # the input projection is its own chain (the Gx GEMM), except in the fused last layer where the recurrent
        # steps continue the chain of x W_ih^T (lstm_layer.cu FUSE: pre_nkb k-blocks first)
        px, ax, sx = chain(passes(operands(x, s), operands(_t(weights["w_ih"], dev), s), s))
        ph_pairs = passes(operands(hprev, s), operands(w_hh, s), s)
        if mode.gx == "fused":
            pz, ah, sh = chain(ph_pairs, p0=px)
            ph = pz - px
        else:
            ph, ah, sh = chain(ph_pairs)
        ex, eh = acc_err(sx, ax), acc_err(sh, ah)
        del ax, sx, ah, sh
    if mode.stale_h_at:
        t, units = mode.stale_h_at
        cols = [q * H + u for q in range(4) for u in units]
        h2 = h_dev[:, t - 2] if t >= 2 else torch.zeros_like(h_dev[:, 0])
        p2, _ = products(operands(h2, s), operands(w_hh[cols], s), s)
        ph.view(R, T, 4 * H)[:, t, cols] = p2
    z, ez = _preactivation(px, ex, ph, eh, _bias(weights, mode, dev), mode)
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
def gemm_interval(a, b, bias, act: int, out_type: str, segs: int, device=None):
    """Where each element of act(a b^T + bias), computed by the library's GEMM and stored as out_type, must lie.
    segs 1: the f64 product of the bf16-rounded operands +- the accumulation bound; segs 3: the f64 product of the
    ORIGINAL f32 operands +- what split-bf16 drops (lo*lo and the residuals of x - hi - lo), taken exactly as the
    difference from the f64 sum of the three passes' products, +- the accumulation bound of the three-pass chain.
    SPLIT_REL * sum|a b| is no bound on the dropped terms: one dominant product can lose nearly 3 * 2^-16 of itself,
    and operands whose lo part falls below bf16's normal range (|x| < 2^-118) lose more.
    Returns (lo, hi, ref) float64 torch tensors [M, N]; ref is the unrounded value."""
    a, b = _t(a, device), _t(b, device)
    _, sa, ss = chain(passes(operands(a, segs), operands(b, segs), segs))
    if segs == 3:
        z = a @ b.T
        zs, _ = products(operands(a, 3), operands(b, 3), 3)
        # the two f64 sums carry at most K * 2^-53 of sum|a b| each
        eps = (z - zs).abs() + a.shape[1] * 2.0 ** -51 * sa + acc_err(ss, sa)
    else:
        z, _ = products(operands(a, 1), operands(b, 1), 1)
        eps = acc_err(ss, sa)
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
def mlp_head(X, coefs, intercepts, device=None):
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
        # the device's x lies within rad of x: each partial sum within rad |w| of the chain's over x
        _, _, sp = chain([(x, w.T)])
        rw = rad @ w.abs()
        eps = acc_err(sp + -(-x.shape[1] // 16) * rw, (x.abs() + rad) @ w.abs()) + rw + 2 * U24 * z.abs()
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


ITEM_ROWS, ITEM_UNITS, BATCH_ROWS = 128, 64, 256   # lstm_layer.cu: kLRows rows x kLTileN / 4 units per item; one batch


def item_of(row: int, unit: int):
    """(batch g, row half, column tile j) of the schedule item that computes h[row, t, unit] at every step t."""
    return row // BATCH_ROWS, (row % BATCH_ROWS) // ITEM_ROWS, unit // ITEM_UNITS


def blocked_layer_stats(x_in, h_dev, weights: dict, mode: Mode, rows: range | None = None, block: int = 32) -> dict:
    """teacher_forced_layer over `rows` (default: all) of one layer, `block` rows at a time, reduced to statistics of
    r = |h_dev - pred| / bound (ratio_stats on every element, without holding the [R, T, 4H] float64 working set).

    x_in [R, T, in], h_dev [R, T, out] as for teacher_forced_layer (any float dtype; the work runs on h_dev's device).
    Returns max, rms, sumsq and n (so that statistics of several row sets combine), above_half (count of r > 0.5),
    argmax (row, t, unit) and items: the largest r of every schedule item, float64 [T, ng, 2, tiles] indexed by
    (t, batch g, row half, column tile j) as item_of maps rows and units (zero for items outside `rows`)."""
    R, T, H = h_dev.shape
    dev = h_dev.device
    rows = range(R) if rows is None else rows
    w = dict(weights, w_ih=_t(weights["w_ih"], dev), w_hh=_t(weights["w_hh"], dev))
    ng, tiles = -(-R // BATCH_ROWS), -(-H // ITEM_UNITS)
    items = torch.zeros(T, ng, 2, tiles, dtype=torch.float64, device=dev)
    out = {"max": -1.0, "sumsq": 0.0, "n": 0, "above_half": 0, "argmax": None}
    for r0 in range(rows.start, rows.stop, block):
        r1 = min(r0 + block, rows.stop)
        pred, bound = teacher_forced_layer(x_in[r0:r1], h_dev[r0:r1], w, mode)
        r = (_t(h_dev[r0:r1]) - pred).abs_().div_(bound.clamp_min_(1e-30))
        del pred, bound
        m = float(r.max())
        if m > out["max"]:
            k = int(r.argmax())
            out["max"], out["argmax"] = m, (r0 + k // (T * H), (k // H) % T, k % H)
        out["sumsq"] += float((r * r).sum())
        out["n"] += r.numel()
        out["above_half"] += int((r > 0.5).sum())
        per_tile = torch.nn.functional.pad(r, (0, tiles * ITEM_UNITS - H)).view(r1 - r0, T, tiles, ITEM_UNITS).amax(3)
        for q0 in range(r0, r1):   # rows of the block grouped by (batch, row half)
            if q0 > r0 and q0 % ITEM_ROWS:
                continue
            q1 = min(r1, (q0 // ITEM_ROWS + 1) * ITEM_ROWS)
            g, half, _ = item_of(q0, 0)
            items[:, g, half] = torch.maximum(items[:, g, half], per_tile[q0 - r0:q1 - r0].amax(0))
    out["rms"] = (out["sumsq"] / out["n"]) ** 0.5
    out["items"] = items
    return out
