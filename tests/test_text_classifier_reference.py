"""CPU tests of the text classifier's host side: fastai's window rule (oracle and ie_clas_window), the oracle against a
literal MultiBatchEncoder run, the head-layout inference of a fastai state dict, the refusals, the plain-C declarations
and the ptxas figures of csrc/clas.cu."""
import os
import re
import subprocess

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
    beta = fma(-mean, alpha, b), y = fma(x, alpha, beta).  Checked on this torch: where the fma forms are evaluated
    exactly (float64 then one rounding), at least 99.9 % of the elements match torch's bits and the rest differ by one
    ulp (torch's CPU kernel may be vectorised differently on other instruction sets)."""
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
    w, b, m, v = (t.detach().numpy() for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))
    alpha = (np.float32(1) / np.sqrt(v + np.float32(1e-5))) * w
    beta = (b.astype(np.float64) - m.astype(np.float64) * alpha).astype(np.float32)
    got = (x.numpy().astype(np.float64) * alpha + beta).astype(np.float32)
    assert (got == y).mean() >= 0.999
    assert np.abs(got.view(np.int32) - y.view(np.int32)).max() <= 1


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
