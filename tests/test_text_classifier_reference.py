"""CPU tests of the text classifier's host side: fastai's window rule (oracle and ie_clas_window), the oracle against a
literal MultiBatchEncoder run, the head-layout inference of a fastai state dict, the refusals, the plain-C declarations
and the ptxas figures of csrc/clas.cu; the exact f32 restatement of the pool and head (its fma against exact rationals,
its agreement with the float64 restatement's bounds, and the negative controls the GPU checks rely on)."""
import os
import re
import subprocess
from fractions import Fraction

import numpy as np
import pytest
import torch

from code_intelligence_b200 import _lib
from code_intelligence_b200 import text_classifier as TC
from oracle import awd_lstm_ref as R
from oracle import text_clas_ref as TR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# sl -> first kept step at bptt = 70, max_len = 1400 (chunk i kept when i > sl - max_len)
WINDOWS = {1: 0, 69: 0, 70: 0, 1399: 0, 1400: 70, 1401: 70, 1469: 70, 1470: 140, 2800: 1470, 2801: 1470}


@pytest.mark.parametrize("sl", sorted(WINDOWS))
def test_window_rule_at_the_default_bptt_and_max_len(sl):
    assert TR.kept_chunks(sl)[0] == WINDOWS[sl]
    assert TR.window_start(sl) == WINDOWS[sl] == TC.window_start(sl)
    assert sl - TR.window_start(sl) <= 1400 + 69


@pytest.mark.parametrize("bptt,max_len", [(16, 40), (7, 8), (70, 71), (5, 1000)])
def test_window_rule_at_other_bptt_and_max_len(bptt, max_len):
    for sl in range(1, 3 * max_len + 2 * bptt):
        want = [i for i in range(0, sl, bptt) if i > sl - max_len][0]
        assert TR.window_start(sl, bptt, max_len) == want == TC.window_start(sl, bptt, max_len), sl


@pytest.mark.parametrize("bptt,max_len", [(70, 70), (70, 10), (16, 1)])
def test_window_rule_refuses_when_no_chunk_is_kept(bptt, max_len):
    with pytest.raises(ValueError):
        TR.window_start(bptt, bptt, max_len)
    with pytest.raises(ValueError, match="no chunk"):
        TC.window_start(bptt, bptt, max_len)
    # some lengths still keep a chunk, others do not: the classifier refuses such a configuration outright
    kept = [bool(TR.kept_chunks(sl, bptt, max_len)) for sl in range(1, 4 * bptt)]
    assert not all(kept)


def _docs_with_pads(n, T, vocab, seed, pad=1):
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, vocab, size=(n, T))
    ids[ids == pad] = 0
    ids[0, :5] = pad                       # front padding
    ids[1, T // 2] = pad                   # a pad inside the window
    ids[2, -1] = pad                       # the last step is a pad
    return ids


@pytest.mark.parametrize("sl,bptt,max_len", [(50, 8, 20), (41, 8, 20), (24, 8, 40), (33, 5, 9)])
def test_oracle_equals_a_literal_chunked_run(sl, bptt, max_len):
    clf = TR.make_classifier(seed=3, vocab_sz=300, emb_sz=24, n_hid=40, n_layers=3, n_class=4, bptt=bptt,
                             max_len=max_len)
    ids = _docs_with_pads(4, sl, 300, seed=sl)
    o1, m1 = clf.encode_chunked(torch.as_tensor(ids))
    o2, m2 = clf.encode(torch.as_tensor(ids))
    assert o1.shape == o2.shape and torch.equal(m1, m2)
    assert o1.shape[1] == sl - TR.window_start(sl, bptt, max_len)
    torch.testing.assert_close(o1, o2, rtol=0, atol=2e-6)
    torch.testing.assert_close(clf(ids, chunked=True), clf(ids), rtol=0, atol=2e-5)


def test_masked_concat_pool_by_hand():
    o = torch.tensor([[[1.0, -2.0], [3.0, 5.0], [4.0, 7.0]]])
    mask = torch.tensor([[False, True, False]])
    got = TR.masked_concat_pool(o, mask)[0]
    # last = o[-1] whatever the mask; max over unmasked; mean of masked_fill(0) over W = 3 times 3 / 2
    np.testing.assert_array_equal(got.numpy(), np.float32([4, 7, 4, 7, 2.5, 2.5]))
    with pytest.raises(ValueError, match="entirely pad"):
        TR.masked_concat_pool(o, torch.ones(1, 3, dtype=torch.bool))


def test_pool_f64_refuses_an_all_pad_window():
    raw = np.ones((1, 4, 2), np.float32)
    with pytest.raises(ValueError, match="entirely pad"):
        TR.pool_f64(raw, np.array([[1, 1, 1, 1]]), [1], [4], 1)


@pytest.mark.parametrize("lin_ftrs,ps", [([50], None), ([50], [0.0]), ([], []), ([100, 50], [0.2, 0.1]),
                                         ([100, 50], [0.0, 0.1]), ([100, 50], [0.0, 0.0])])
@pytest.mark.parametrize("output_p", [0.4, 0.0])
def test_head_layout_is_inferred_from_the_tensors(lin_ftrs, ps, output_p):
    clf = TR.make_classifier(seed=2, vocab_sz=100, emb_sz=16, n_hid=24, n_layers=2, n_class=3, lin_ftrs=lin_ftrs,
                             ps=ps, output_p=output_p)
    sd = clf.fastai_state_dict()
    idx = sorted({int(k.split(".")[2]) for k in sd if k.startswith("1.layers.")})
    n_drop = sum(p != 0 for p in [output_p] + (ps if ps is not None else [0.1] * len(lin_ftrs)))
    n_stages = len(lin_ftrs) + 1
    assert max(idx) + 1 == 2 * n_stages + n_drop + (n_stages - 1)      # BN, Linear, Dropouts, ReLUs
    for wrapped in (sd, {"model": sd, "opt": {}}):
        got = TC.head_stages(wrapped, 48)
        want = clf.stages()
        assert len(got) == len(want) == n_stages
        for g, w in zip(got, want):
            for k in w:
                np.testing.assert_array_equal(g[k], w[k])
    assert [s["weight"].shape[0] for s in got] == lin_ftrs + [3]


def test_head_layout_refusals():
    clf = TR.make_classifier(seed=2, vocab_sz=100, emb_sz=16, n_hid=24, n_layers=2, n_class=3)
    sd = clf.fastai_state_dict()
    with pytest.raises(ValueError, match="expected 60"):
        TC.head_stages(sd, 60)                                     # wrong head width (3 * emb_sz = 48)
    bad = {k: v for k, v in sd.items() if not k.startswith("1.layers.0.")}
    with pytest.raises(ValueError, match="without a BatchNorm1d"):
        TC.head_stages(bad, 48)
    with pytest.raises(ValueError, match="no head"):
        TC.head_stages({k: v for k, v in sd.items() if k.startswith("0.")}, 48)


def test_bn_fold_restates_torch_eval_batchnorm():
    """The device folds eval BatchNorm1d as torch's CPU kernel does: alpha = (1 / sqrt(var + eps)) * w,
    beta = fma(-mean, alpha, b), y = fma(x, alpha, beta) -- oracle.text_clas_ref.bn_fold_f32 and fma_f32.  Checked on
    this torch: at least 99.9 % of the elements match torch's bits and the rest differ by one ulp (torch's CPU kernel
    may be vectorised differently on other instruction sets)."""
    torch.manual_seed(0)
    n = 2048
    bn = torch.nn.BatchNorm1d(n).eval()
    with torch.no_grad():
        bn.weight.copy_(torch.randn(n))
        bn.bias.copy_(torch.randn(n))
        bn.running_mean.copy_(torch.randn(n) * 3)
        bn.running_var.copy_(torch.rand(n) * 5 + 1e-3)
    x = torch.randn(32, n) * 4
    y = bn(x).detach().numpy()
    stage = dict(bn_weight=bn.weight.detach().numpy(), bn_bias=bn.bias.detach().numpy(),
                 bn_mean=bn.running_mean.numpy(), bn_var=bn.running_var.numpy())
    alpha, beta = TR.bn_fold_f32(stage, bn.eps)
    got = TR.fma_f32(x, alpha[None, :], beta[None, :]).numpy().astype(np.float32)
    assert (got == y).mean() >= 0.999
    assert np.abs(got.view(np.int32) - y.view(np.int32)).max() <= 1
    # the fold's own rounding points: alpha is the f32 product of the f32 reciprocal square root and w
    v32 = stage["bn_var"] + np.float32(bn.eps)
    np.testing.assert_array_equal(alpha.numpy().astype(np.float32),
                                  (np.float32(1) / np.sqrt(v32)).astype(np.float32) * stage["bn_weight"])


# ------------------------------------------------------------------------- exact f32 restatement (oracle/text_clas_ref)
def _round_f32(x: Fraction) -> float:
    """A non-zero rational rounded to the nearest f32, ties to even (overflow to inf), as a float."""
    sgn = -1 if x < 0 else 1
    x = abs(x)
    e = x.numerator.bit_length() - x.denominator.bit_length()
    if x < Fraction(2) ** e:
        e -= 1                                              # now 2^e <= x < 2^(e + 1)
    q = Fraction(2) ** (max(e, -126) - 23)                  # the f32 spacing there (subnormal below 2^-126)
    v = round(x / q) * q                                    # Fraction rounds half to even
    if v >= Fraction(2) ** 128:
        return sgn * float("inf")
    return sgn * float(v)


def _fma_exact(a: np.float32, b: np.float32, c: np.float32) -> np.float32:
    """fma(a, b, c) from exact rationals: one rounding of a b + c; an exact zero is -0 only when a b and c are both
    -0 (IEEE 754 round to nearest)."""
    s = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if s != 0:
        return np.float32(_round_f32(s))
    prod_neg = np.signbit(a) != np.signbit(b)
    both_neg_zero = a * b == 0 and prod_neg and c == 0 and np.signbit(c)
    return np.float32(-0.0 if both_neg_zero else 0.0)


def _bits(x) -> np.ndarray:
    return np.asarray(x, np.float32).view(np.uint32)


def _check_fma(a, b, c):
    a, b, c = (np.asarray(t, np.float32) for t in (a, b, c))
    got = TR.fma_f32(torch.as_tensor(a), torch.as_tensor(b), torch.as_tensor(c)).numpy().astype(np.float32)
    want = np.array([_fma_exact(*t) for t in zip(a, b, c)], np.float32)
    bad = np.flatnonzero(_bits(got) != _bits(want))
    assert bad.size == 0, [(a[i], b[i], c[i], got[i], want[i]) for i in bad[:5]]


def _f32_values(rng, n, lo, hi):
    """Random f32 values of random sign with exponents uniform in [lo, hi]."""
    m = rng.uniform(1, 2, n)
    return (rng.choice([-1.0, 1.0], n) * m * 2.0 ** rng.integers(lo, hi + 1, n)).astype(np.float32)


def test_fma_f32_is_correctly_rounded_on_random_triples():
    rng = np.random.default_rng(0)
    n = 6000
    a, b = _f32_values(rng, n, -20, 20), _f32_values(rng, n, -20, 20)
    c = _f32_values(rng, n, -45, 45)
    _check_fma(a, b, c)
    # near-cancellation: c within a few ulp of -a b, so the result is the product's low bits
    p = (a.astype(np.float64) * b).astype(np.float32)
    near = np.nextafter(-p, rng.choice([-np.inf, np.inf], n).astype(np.float32)).astype(np.float32)
    _check_fma(a, b, near)
    _check_fma(a, b, -p)


def test_fma_f32_at_an_f32_midpoint_where_plain_double_rounding_fails():
    """a = b = 1 + 2^-12: a b = 1 + 2^-11 + 2^-24 is the midpoint of two f32 values.  With c = +2^-80 the exact sum lies
    above it and the fma rounds up; f32(f64(a b) + c) loses c in the first rounding and then rounds the tie down to
    even.  With c = -2^-80 both round down."""
    a = np.float32(1 + 2.0 ** -12)
    for sgn in (1, -1):
        c = np.float32(sgn * 2.0 ** -80)
        want = _fma_exact(a, a, c)
        got = TR.fma_f32(torch.tensor([a]), torch.tensor([a]), torch.tensor([c])).numpy().astype(np.float32)[0]
        assert _bits(got) == _bits(want)
        plain = np.float32(np.float64(a) * np.float64(a) + np.float64(c))
        assert (plain == want) == (sgn < 0), (sgn, plain, want)
    assert _fma_exact(a, a, np.float32(2.0 ** -80)) == np.float32(1 + 2.0 ** -11 + 2.0 ** -23)


def test_fma_f32_signed_zeros_subnormals_and_exponent_gaps():
    z, one = np.float32(0.0), np.float32(1.0)
    a, b, c = [], [], []

    def add(x, y, w):
        a.append(x), b.append(y), c.append(w)

    for x, y, w in [(one, one, -one), (-one, one, one), (z, one, -z), (-z, one, -z), (z, -one, -z), (-z, -one, -z),
                    (z, one, z), (np.float32(3), np.float32(5), np.float32(-15)), (np.float32(1.5), np.float32(-2),
                                                                                      np.float32(3))]:
        add(x, y, w)                                        # exact cancellation: +0, or -0 only from -0 + -0
    rng = np.random.default_rng(1)
    sub = np.float32(2.0 ** -149)
    for _ in range(800):
        x, y = _f32_values(rng, 2, -75, -60)                # product 2^-150 .. 2^-120: subnormal or just normal
        add(x, y, np.float32(rng.integers(-2 ** 20, 2 ** 20)) * sub)
        x, y = _f32_values(rng, 2, -10, 10)                 # a tiny or huge c against a moderate product
        add(x, y, _f32_values(rng, 1, -140, -100)[0])
        add(x, y, _f32_values(rng, 1, 60, 100)[0])
        x, y = _f32_values(rng, 2, 55, 63)                  # product near the f32 overflow threshold
        add(x, y, _f32_values(rng, 1, 100, 127)[0])
    _check_fma(a, b, c)
    zeros = TR.fma_f32(torch.tensor([1.0, -0.0]), torch.tensor([-1.0, 1.0]), torch.tensor([1.0, -0.0]))
    assert list(np.signbit(zeros.numpy())) == [False, True]


def _stages(rng, dims, x):
    """Random head stages with BatchNorm statistics calibrated on x (float64 forward between stages)."""
    stages = []
    a = x.astype(np.float64)
    for k, (K, N) in enumerate(zip(dims[:-1], dims[1:])):
        st = dict(bn_weight=(1 + 0.2 * rng.standard_normal(K)).astype(np.float32),
                  bn_bias=(0.1 * rng.standard_normal(K)).astype(np.float32),
                  bn_mean=a.mean(0).astype(np.float32), bn_var=(a.var(0) + 1e-4).astype(np.float32),
                  weight=(rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32),
                  bias=(0.1 * rng.standard_normal(N)).astype(np.float32))
        stages.append(st)
        xn = (a - st["bn_mean"]) / np.sqrt(st["bn_var"].astype(np.float64) + 1e-5) * st["bn_weight"] + st["bn_bias"]
        a = xn @ st["weight"].T.astype(np.float64) + st["bias"]
        if k < len(dims) - 2:
            a = np.maximum(a, 0)
    return stages


def _pool_inputs(rng, B, T, E, pad=1):
    raw = np.tanh(rng.standard_normal((B, T, E)) * 1.5).astype(np.float32)
    ids = rng.integers(2, 100, size=(B, T))
    starts = np.array([TR.window_start(T)] * B, np.int32)
    ends = np.full(B, T, np.int32)
    ids[0, :7] = pad                                        # pads in front of the window's first kept step
    ids[1, T // 2] = pad                                    # inside
    ids[2, -1] = pad                                        # on the last step
    ends[3] = T - 5                                         # a shorter window, right padding after it
    ids[3, T - 5:] = pad
    starts[3] = TR.window_start(T - 5)
    return raw, ids, starts, ends


@pytest.mark.parametrize("T,E", [(150, 96), (600, 800)])
def test_exact_pool_lies_within_the_float64_bound(T, E):
    rng = np.random.default_rng(T)
    raw, ids, starts, ends = _pool_inputs(rng, 4, T, E)
    got = TR.pool_f32(raw, ids, starts, ends, 1).numpy()
    assert np.array_equal(got, got.astype(np.float32))     # f32 values
    last, mx, avg, bound = TR.pool_f64(raw, ids, starts, ends, 1)
    np.testing.assert_array_equal(got[:, :E], last)
    np.testing.assert_array_equal(got[:, E:2 * E], mx)
    err = np.abs(got[:, 2 * E:] - avg)
    assert (err <= bound).all(), (err / bound).max()
    assert (err > 0).mean() > 0.3                           # the f32 sum does round


@pytest.mark.parametrize("dims", [[288, 50, 3], [2400, 50, 28], [2400, 129, 33, 5]])
def test_exact_head_lies_within_the_float64_bound(dims):
    rng = np.random.default_rng(len(dims) + dims[0])
    x = np.tanh(rng.standard_normal((24, dims[0]))).astype(np.float32)
    stages = _stages(rng, dims, x)
    z = TR.head_f32(x, stages).numpy()
    assert np.array_equal(z, z.astype(np.float32))
    z64, ez, _, _ = TR.head_f64(x, stages)
    assert (np.abs(z - z64) <= ez).all(), (np.abs(z - z64) / ez).max()
    assert np.std(z64) > 0.05


def test_reordered_sums_differ_from_the_exact_restatement():
    """The negative controls the GPU checks rest on: at the 06 shape a reversed k chain (K = 2400) and a two-accumulator
    pool sum give other bits in a non-trivial fraction of the elements, so equality with the forward restatement pins
    the order."""
    rng = np.random.default_rng(7)
    x = np.tanh(rng.standard_normal((32, 2400))).astype(np.float32)
    stages = _stages(rng, [2400, 50], x)
    fwd = TR.head_f32(x, stages).numpy()
    rev = TR.head_f32(x, stages, reverse=True).numpy()
    assert (fwd != rev).mean() > 0.2, (fwd != rev).mean()
    raw, ids, starts, ends = _pool_inputs(rng, 4, 512, 800)
    fwd = TR.pool_f32(raw, ids, starts, ends, 1).numpy()
    pw = TR.pool_f32(raw, ids, starts, ends, 1, pairwise=True).numpy()
    np.testing.assert_array_equal(fwd[:, :1600], pw[:, :1600])     # last and max do not depend on the order
    assert (fwd[:, 1600:] != pw[:, 1600:]).mean() > 0.2, (fwd[:, 1600:] != pw[:, 1600:]).mean()


def test_activation_bounds_on_exact_logits():
    """The relative bounds hold for the float32 torch forms on the same logits (a stand-in for the device: a correctly
    rounded exp is within them) and are tight enough to see a 1e-6 probability off by 1 %."""
    z = torch.linspace(-110, 110, 4001, dtype=torch.float32)
    p64, bound = TR.sigmoid_bound(z)
    p32 = (1 / (1 + torch.exp(-z))).double()
    assert ((p32 - p64).abs() <= bound).all()
    i = int(torch.argmin((p64 - 1e-6).abs()))
    assert bound[i] < 0.01 * p64[i]
    zs = torch.tensor([[0.0, -5.0, -100.0, 3.5, -120.0] * 7], dtype=torch.float32)
    p64, bound = TR.softmax_bound(zs)
    assert ((torch.softmax(zs, 1).double() - p64).abs() <= bound).all()
    assert (bound <= p64 * 1e-4 + 2.0 ** -126).all()


def test_clas_abi_from_plain_c(tmp_path):
    """include/issue_emb_b200.h's classifier declarations compile as C99 (-pedantic -Werror), every ie_clas_* entry point
    links, the window rule answers without a GPU and bad arguments are error codes (tests/c_abi/clas_abi_check.c)."""
    _lib.load()
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "clas_abi_check")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "c_abi", "clas_abi_check.c"), "-o", exe, "-L", libdir,
                    "-l:" + os.path.basename(_lib.LIB_PATH), "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "clas_symbols=8 activations=0,1" in r.stdout, r.stdout
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "issue_emb_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(ie_clas_[a-z_0-9]+)\s*\(", hdr))
    assert declared == {k for k in _lib.PROTOTYPES if k.startswith("ie_clas_")} and len(declared) == 8


def test_clas_cu_built_for_sm_90a_without_spills():
    _lib.load()
    text = open(os.path.join(ROOT, "code_intelligence_b200", "csrc", "build", "clas.ptxas.log")).read()
    assert "sm_90a" in text
    entries = re.findall(r"Compiling entry function '([^']+)'", text)
    for k in ("clas_pool_kernel", "clas_linear_kernel", "clas_activate_kernel"):
        assert any(k in e for e in entries), entries
    spills = [int(v) for v in re.findall(r"(\d+) bytes spill (?:stores|loads)", text)]
    stack = [int(v) for v in re.findall(r"(\d+) bytes stack frame", text)]
    regs = [int(r) for r in re.findall(r"Used (\d+) registers", text)]
    print("clas.cu ptxas:", [l.strip() for l in text.splitlines() if "registers" in l or "spill" in l])
    assert spills and not any(spills) and not any(stack)
    assert max(regs) <= 64


def test_product_loader_accepts_the_oracle_state_dict_keys():
    """from_state_dict's encoder half: stripping ``0.module.`` leaves the AWD_LSTM names IssueEncoder.load_state_dict
    takes, and the shapes it infers are the model's."""
    clf = TR.make_classifier(seed=2, vocab_sz=100, emb_sz=16, n_hid=24, n_layers=3, n_class=3)
    sd = clf.fastai_state_dict()
    enc_sd = {k[len("0.module."):]: v for k, v in sd.items() if k.startswith("0.module.")}
    emb, layers = clf.enc.export_weights()
    np.testing.assert_array_equal(enc_sd["encoder.weight"].numpy(), emb)
    for l, L in enumerate(layers):
        np.testing.assert_array_equal(enc_sd[f"rnns.{l}.weight_hh_l0_raw"].numpy(), L["w_hh"])
        np.testing.assert_array_equal(enc_sd[f"rnns.{l}.module.weight_ih_l0"].numpy(), L["w_ih"])
    assert tuple(enc_sd["rnns.0.weight_hh_l0_raw"].shape) == (4 * 24, 24)
    assert isinstance(R.AWDLSTMEncoderRef, type)
