"""CPU tests of the language model's host side: the vectorised validation stream against a literal fastai
LanguageModelPreLoader, the literal stateful validate loop against one zero-state run over whole rows, the state-dict
refusals, the plain-C declarations and the ptxas figures of csrc/lm.cu; the exact float32 restatement of the decoder
against the float64 bounds, its negative controls, and the SASS facts it rests on."""
import functools
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from code_intelligence_b200 import _lib
from code_intelligence_b200 import language_model as LM
from oracle import awd_lstm_ref as R
from oracle import lm_ref as L
from oracle.sass import sass_functions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def corpus(seed, n_docs, lo, hi, vocab=50):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, vocab, size=int(rng.integers(lo, hi + 1))) for _ in range(n_docs)]


CORPORA = {
    "bs_above_docs": (corpus(1, 3, 5, 40), 8),
    "docs_below_bptt": (corpus(2, 30, 1, 6), 5),
    "single_doc": ([np.arange(1000) % 47], 7),
    "ragged_not_divisible": (corpus(3, 17, 1, 300), 13),
    "one_row": (corpus(4, 5, 10, 90), 1),
}


@pytest.mark.parametrize("bptt", [1, 67, 70])
@pytest.mark.parametrize("name", sorted(CORPORA))
def test_stream_equals_the_literal_preloader(name, bptt):
    docs, bs = CORPORA[name]
    x, y = LM.lm_stream(docs, bs, bptt)
    pre = L.PreLoaderRef(docs, bs, bptt)
    batches = list(pre.batches())
    assert len(batches) == pre.ite_len // bs == x.shape[1] // bptt
    np.testing.assert_array_equal(np.concatenate([b[0] for b in batches], 1), x)
    np.testing.assert_array_equal(np.concatenate([b[1] for b in batches], 1), y)
    assert pre.totalToks % bs != 0 or name != "ragged_not_divisible"


def test_stream_refusals():
    with pytest.raises(ValueError):
        LM.lm_stream([], 4, 70)
    with pytest.raises(ValueError):
        LM.lm_stream([np.arange(5), np.array([], np.int64)], 4, 70)
    with pytest.raises(ValueError):
        LM.lm_stream([np.arange(5)], 0, 70)


@pytest.mark.parametrize("bs,bptt", [(4, 7), (3, 1), (6, 20)])
def test_stateful_validate_equals_one_zero_state_run(bs, bptt):
    """fastai's validate carries (h, c) from batch to batch after one reset: the same as one run over each row."""
    lm = L.make_lm(seed=3, vocab_sz=60, emb_sz=16, n_hid=24, n_layers=3, dec_scale=4.0, bias_scale=0.5)
    docs = corpus(5, 9, 3, 40, vocab=60)
    x, y = LM.lm_stream(docs, bs, bptt)
    lit = L.validate_literal(lm, docs, bs, bptt)
    one = L.validate_one_run(lm, x, y, bptt)
    assert abs(lit[0] - one[0]) <= 1e-5 * abs(lit[0]) and abs(lit[1] - one[1]) <= 1e-6, (lit, one)


def test_tied_and_untied_state_dicts():
    tied = L.make_lm(seed=1, vocab_sz=40, emb_sz=8, n_hid=12, n_layers=2, tied=True).fastai_state_dict()
    untied = L.make_lm(seed=1, vocab_sz=40, emb_sz=8, n_hid=12, n_layers=2, tied=False).fastai_state_dict()
    assert torch.equal(tied["1.decoder.weight"], tied["0.encoder.weight"])
    assert not torch.equal(untied["1.decoder.weight"], untied["0.encoder.weight"])
    for sd in (tied, untied, {"model": untied}):
        w, b = LM.decoder_keys(sd.get("model", sd))
        assert tuple(w.shape) == (40, 8) and tuple(b.shape) == (40,)


def _sd():
    return L.make_lm(seed=2, vocab_sz=40, emb_sz=8, n_hid=12, n_layers=2).fastai_state_dict()


@pytest.mark.parametrize("edit,msg", [
    (lambda sd: sd.pop("1.decoder.weight"), "no decoder"),
    (lambda sd: sd.pop("0.encoder.weight"), "no encoder"),
    (lambda sd: sd.__setitem__("1.decoder.weight", torch.zeros(41, 8)), "1.decoder.weight"),
    (lambda sd: sd.__setitem__("1.decoder.weight", torch.zeros(40, 9)), "1.decoder.weight"),
    (lambda sd: sd.__setitem__("1.decoder.bias", torch.zeros(39)), "1.decoder.bias"),
    (lambda sd: sd.__setitem__("0.module.encoder.weight", torch.zeros(40, 8)), "classifier"),
    (lambda sd: [sd.pop(k) for k in list(sd) if k.startswith("0.rnns.")], "no LSTM layers"),
])
def test_state_dict_refusals(edit, msg):
    """Every refusal comes before a device handle exists."""
    sd = _sd()
    edit(sd)
    with pytest.raises(ValueError, match=msg):
        LM.LanguageModel.from_state_dict(sd)
    with pytest.raises(ValueError, match=msg):
        LM.LanguageModel.from_state_dict({"model": sd})


def test_lm_abi_from_plain_c(tmp_path):
    """include/issue_emb_b200.h's language-model declarations compile as C99 (-pedantic -Werror), every ie_lm_* entry
    point links and bad arguments are error codes (tests/c_abi/lm_abi_check.c)."""
    _lib.load()
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "lm_abi_check")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "c_abi", "lm_abi_check.c"), "-o", exe, "-L", libdir,
                    "-l:" + os.path.basename(_lib.LIB_PATH), "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "lm_symbols=7" in r.stdout, r.stdout
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "issue_emb_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(ie_(?:debug_)?lm_[a-z_0-9]+)\s*\(", hdr))
    assert declared == {k for k in _lib.PROTOTYPES if re.match(r"ie_(debug_)?lm_", k)} and len(declared) == 7


def test_lm_cu_built_for_sm_90a():
    """The combine kernel has no spills; the fused decoder's instantiation of the GEMM (128 accumulator registers of
    the 168 its launch bounds allow) spills at most 64 bytes, only around its per-item flush."""
    _lib.load()
    text = open(os.path.join(ROOT, "code_intelligence_b200", "csrc", "build", "lm.ptxas.log")).read()
    assert "sm_90a" in text
    blocks = re.split(r"Compiling entry function '", text)[1:]
    figures = {}
    for b in blocks:
        name = b.split("'")[0]
        spill = sum(int(v) for v in re.findall(r"(\d+) bytes spill stores", b))
        figures["combine" if "lm_combine_kernel" in name else "decode" if "LmEpi" in name else name] = spill
    print("lm.cu ptxas spill stores:", figures)
    assert set(figures) == {"combine", "decode"}
    assert figures["combine"] == 0 and figures["decode"] <= 64


# ------------------------------------------------------------------------------------------------ exact restatement
def _int_case(E, V, M, seed):
    rng = np.random.default_rng(seed)
    h = rng.integers(-2, 3, size=(M, E)).astype(np.float32)
    W = rng.integers(-3, 4, size=(V, E)).astype(np.float32)
    b = rng.integers(-4, 5, size=V).astype(np.float32)
    t = rng.integers(0, V, size=M)
    t[0] = -100
    t[-1] = V - 1
    return h, W, b, t


@pytest.mark.parametrize("E,V,M", [(7, 1, 3), (7, 257, 17), (16, 8193, 9), (16, 20000, 40)])
def test_exact_restatement_within_the_f64_bounds(E, V, M):
    """decoder_f32_exact with correctly rounded 2^x and log as stand-ins lies inside decoder_f64's per-element bounds
    (small-integer h and W: the logits are exact, so the accumulators are h W^T in f32), and its argmax is the f64
    argmax."""
    h, W, b, t = _int_case(E, V, M, E + V + M)
    acc = torch.from_numpy(h @ W.T)
    nll, lse, pred = (v.numpy() for v in L.decoder_f32_exact(acc, b, t, L.ex2_rn, L.logf_rn))
    ref = L.decoder_f64(h, W, b, t, 1)
    v = L.check_decoder(ref, nll, lse, pred)
    assert v["max_lse"] <= 1 and v["max_nll"] <= 1 and v["wrong_pred"] == 0, v
    np.testing.assert_array_equal(pred, np.argmax(h.astype(np.float64) @ W.T.astype(np.float64) + b, 1))
    assert nll[0] == 0


def _mixed_acc(M, V, seed):
    """Accumulators of two kinds: half the rows 4 N(0, 1) plus a bias, half a ramp (c - V) / 256 plus N(0, 1) that
    rescales at every tile and ends near 0, where lse = log(s) shows the last bits of s."""
    g = torch.Generator().manual_seed(seed)
    acc = 4 * torch.randn(M, V, generator=g, dtype=torch.float64)
    acc[M // 2:] = (torch.arange(V, dtype=torch.float64) - V) / 256 + torch.randn(M - M // 2, V, generator=g,
                                                                                 dtype=torch.float64)
    b = torch.randn(V, generator=g).float().numpy()
    t = torch.randint(0, V, (M,), generator=g).numpy()
    t[0] = -100
    return acc.float(), b, t


@functools.lru_cache(maxsize=1)
def _mixed_case():
    acc, b, t = _mixed_acc(96, 40000, 4)       # five slices
    return acc, b, t, L.decoder_f32_exact(acc, b, t, L.ex2_rn, L.logf_rn)


@pytest.mark.parametrize("mutant", L.EXACT_MUTANTS)
def test_every_mutant_changes_output_bits(mutant):
    acc, b, t, base = _mixed_case()
    mut = L.decoder_f32_exact(acc, b, t, L.ex2_rn, L.logf_rn, mutant=mutant)
    n = sum(int((x.view(torch.int32) != y.view(torch.int32)).sum()) for x, y in zip(base, mut))
    assert n > 0, mutant


def test_lm_sass_has_the_restated_order():
    """The facts decoder_f32_exact rests on, read from build/lm.o: the decoder's GEMM instantiation has exactly two
    FFMA (s = fma(s, scale, ts), one per row half); lm_combine_kernel has no FFMA but logf's own (the count in the
    test kernel of ie_debug_gates fn 10 in build/misc.o, built with the same flags), so merge is two products and an
    add; every MUFU.EX2 in both reads an FMUL by log2(e) as f32 (0x3fb8aa3b), i.e. ex2(f32(f32(x - m) * log2e)) with
    nothing contracted into it."""
    _lib.load()
    build = os.path.join(ROOT, "code_intelligence_b200", "csrc", "build")
    fns = sass_functions(os.path.join(build, "lm.o"))
    misc = sass_functions(os.path.join(build, "misc.o"))
    pick = lambda fs, key: [v for k, v in fs.items() if key in k]
    decode, combine = pick(fns, "LmEpi"), pick(fns, "lm_combine_kernel")
    logf = pick(misc, "debug_lm_math_kernelILi10E")
    assert len(decode) == len(combine) == len(logf) == 1, list(fns)
    decode, combine, logf = decode[0], combine[0], logf[0]
    count = lambda ins, op: sum(1 for o, _, _ in ins if o == op)
    assert count(decode, "FFMA") == 2, "the decoder's epilogue contracts other than s * scale + ts"
    assert count(logf, "FFMA") > 0
    assert count(combine, "FFMA") == count(logf, "FFMA"), "merge in lm_combine_kernel is contracted into an fma"
    assert count(decode, "MUFU.EX2") >= 128 and count(combine, "MUFU.EX2") > 0
    for name, ins in (("decode", decode), ("combine", combine)):
        for i, (op, args, _) in enumerate(ins):
            if op != "MUFU.EX2":
                continue
            src = args.split(",")[1].strip()
            w = next((j for j in range(i - 1, -1, -1) if ins[j][1].split(",")[0].strip() == src), None)
            assert w is not None and ins[w][0] == "FMUL" and "0x3fb8aa3b" in ins[w][2], \
                (name, "MUFU.EX2 not fed by an FMUL by log2(e)", ins[i][2], None if w is None else ins[w][2])
