"""The two arithmetic primitives every per-element bound of the suite rests on, measured on the device.

  * The wgmma f32 accumulator (ie_debug_gemm_ex: act 0, no bias, f32 out): the probes of oracle/tc_accum.py give the
    same bits on the device as tc_accum.emulate under tc_accum.MODEL, every other candidate model disagrees with the
    device on at least one probe, and random elements at the production shapes (the K = 2432 input projection, the
    K = 832 per-token table, the MLP's K = 1600 / 2400; bf16 and split-bf16) are bit-equal to the emulator.
  * The gate functions and the cell update (ie_debug_gates, the inline functions of ptx.cuh / lstm_common.cuh): every
    f32 bit pattern of each gate function against float64 torch, within device_numerics.sig_err / tanh_err; +-inf
    saturate exactly, NaN gives NaN, outputs stay in range, tanh_ieee is exactly odd; the cell of every gate mode on
    adversarial grids within device_numerics.cell_step's bound.  gemm_interval(act 2) and mlp_head bound their
    sigmoid_acc by sig_err(..., 'exp'), the model this sweep checks.
"""
import numpy as np
import pytest
import torch

from code_intelligence_b200 import _lib
from oracle import device_numerics as D
from oracle import knn_ref as K_REF
from oracle import tc_accum as T

pytestmark = pytest.mark.gpu


def _same(x, y):
    """Bit equality of f32 arrays (+0 and -0 equal: the sign of an exact zero sum is not modelled)."""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    return (x.view(np.uint32) == y.view(np.uint32)) | ((x == 0) & (y == 0))


@pytest.fixture(scope="module")
def probe_results():
    P = T.probes()
    return P, {k: np.diag(_lib._debug_gemm(a, b)) for k, (a, b) in P.items()}


def test_accumulator_model_equals_device_on_every_probe(probe_results):
    P, dev = probe_results
    for k, (a, b) in P.items():
        bad = ~_same(T.emulate(a, b), dev[k])
        assert not bad.any(), (k, int(bad.sum()), np.nonzero(bad)[0][:5])


def test_every_discarded_candidate_disagrees_with_device(probe_results):
    P, dev = probe_results
    order = sorted(P, key=lambda k: P[k][0].size)   # the small families first: most candidates fail there
    for m in T.candidates():
        if m == T.MODEL:
            continue
        assert any(not _same(T.emulate(*P[k], 1, m), dev[k]).all() for k in order), m


@pytest.mark.parametrize("segs", [1, 3])
@pytest.mark.parametrize("K, scale", [(2432, 1.0), (832, 1.0), (1600, 0.05), (2400, 0.05)])
def test_accumulator_model_at_production_shapes(K, scale, segs):
    rng = np.random.default_rng(K + segs)
    a = rng.standard_normal((256, K)).astype(np.float32)
    b = (scale * rng.standard_normal((256, K))).astype(np.float32)
    d = _lib._debug_gemm(a, b, segs=segs)
    idx = rng.integers(0, 256, (256, 2))
    want = T.emulate(a[idx[:, 0]], b[idx[:, 1]], segs)
    got = d[idx[:, 0], idx[:, 1]]
    assert _same(want, got).all(), np.nonzero(~_same(want, got))[0][:5]


# ------------------------------------------------------------------------------------------------ gates
KINDS = {"sigmoid_fast": ("s", "fast"), "tanh_fast": ("t", "fast"), "sigmoid_acc": ("s", "exp"),
         "tanh_acc": ("t", "exp"), "sigmoid_ieee": ("s", "ieee"), "tanh_ieee": ("t", "ieee")}


@pytest.mark.parametrize("fn", list(KINDS))
def test_gate_function_over_every_f32(fn):
    """All 2^32 inputs, one (sign, exponent) bin of 2^23 at a time."""
    ft, kind = KINDS[fn]
    mant = torch.arange(1 << 23, dtype=torch.int32, device="cuda")
    worst, at = 0.0, None
    for sg in (0, 1):
        for e in range(256):
            x = (mant | ((-(1 << 31) if sg else 0) | (e << 23))).view(torch.float32)
            y = _lib._debug_gates(fn, x).double()
            if e == 255:
                nan = torch.isnan(x)
                assert torch.isnan(y[nan]).all(), fn
                inf = float(y[~nan][0])
                assert inf == ((0.0 if sg else 1.0) if ft == "s" else (-1.0 if sg else 1.0)), (fn, sg, inf)
                continue
            x64 = x.double()
            ref = torch.sigmoid(x64) if ft == "s" else torch.tanh(x64)
            bound = D.sig_err(x64, ref, kind) if ft == "s" else D.tanh_err(x64, ref, kind)
            r = (y - ref).abs() / bound.clamp_min(1e-300)
            assert not torch.isnan(y).any(), (fn, sg, e)
            assert float(y.min()) >= (0.0 if ft == "s" else -1.0) and float(y.max()) <= 1.0, (fn, sg, e)
            if fn == "tanh_ieee" and sg == 0:
                assert torch.equal(_lib._debug_gates(fn, -x), -y.float()), e
            k = int(r.argmax())
            if float(r[k]) > worst:
                worst, at = float(r[k]), float(x64[k])
    print(f"{fn}: max |y - f| / bound = {worst:.4g} at x = {at!r}")
    assert worst <= 1.0, (fn, worst, at)


@pytest.mark.parametrize("kind", ["fast", "exp", "ieee"])
def test_cell_on_adversarial_grids(kind):
    z, cp = D.cell_grid()
    x = torch.from_numpy(np.vstack([z, cp[None]])).cuda()
    c, h = _lib._debug_gates("cell_" + kind, x).double().cpu()
    c_ref, ec, h_ref, eh = D.cell_step(*torch.from_numpy(z), torch.from_numpy(cp), kind)
    rc = ((c - c_ref).abs() / ec).max()
    rh = ((h - h_ref).abs() / eh).max()
    print(f"cell {kind}: max |dc| / bound = {float(rc):.4g}, max |dh| / bound = {float(rh):.4g}")
    assert float(rc) <= 1 and float(rh) <= 1


@pytest.mark.parametrize("K", [832, 2432, 4864])
def test_split_chain_on_coherent_f32_operands(K):
    """Split-bf16 on positive f32 operands, where every step truncates the running sum: the device equals the emulator,
    lies inside gemm_interval (SPLIT_REL plus the chain's accumulation term) and inside knn_ref's stage-1 model; the
    former SPLIT_REL-only interval is exceeded at K = 4864 (tests/test_tc_accum.py keeps the record)."""
    rng = np.random.default_rng(K)
    a = (1 + rng.random((64, K))).astype(np.float32)
    b = (1 + rng.random((64, K))).astype(np.float32)
    got = np.diag(_lib._debug_gemm(a, b, segs=3))
    assert _same(got, T.emulate(a, b, 3)).all()
    lo, hi, _ = D.gemm_interval(a, b, None, 0, "f32", 3)
    g = torch.from_numpy(got.astype(np.float64))
    assert ((g >= lo.diagonal()) & (g <= hi.diagonal())).all()
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    err = np.abs(got - (a64 * b64).sum(1))
    sab = (a64 * b64).sum(1)
    k_pad = -(-K // 64) * 64
    e_knn = (K_REF.SPLIT_PRODUCT + K_REF.PASSES * (k_pad // 16) * K_REF.ACC_STEP * (1 + 2.0 ** -6)) * sab
    print(f"K = {K}: |err| / (SPLIT_REL sum|ab|) max {(err / (D.SPLIT_REL * sab)).max():.3g}, "
          f"/ knn stage-1 bound max {(err / e_knn).max():.3g}")
    assert (err <= e_knn).all()
