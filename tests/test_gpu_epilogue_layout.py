"""GPU tests of the recurrent kernel's memory layout (DESIGN.md section 3): the hidden units a thread owns, and the
fragment order in which the input-projection GEMM stores Gx and the per-token table for it.

  * the fragment-ordered GEMM store (ie_debug_gemm_frag), undone on the host, is per-element correct and bit-equal to
    the natural store at the production Gx shape (fp16; f32 with split-bf16 operands) and at the table shape;
  * encoder outputs, pooled and raw, hash to the values an H100 produced with the natural layout of Gx and of the
    hidden units (tests/golden/epilogue_layout_hashes.json): the layout moves values, it changes none of them.

``python tests/test_gpu_epilogue_layout.py --write FILE`` recomputes the hashes with whatever build is importable.
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import awd_lstm_ref as R  # noqa: E402

HASHES = os.path.join(ROOT, "tests", "golden", "epilogue_layout_hashes.json")
KNOBS = ("IE_SEQ", "IE_COOP", "IE_EMB_PROJ", "IE_GX_BF16", "IE_BATCHES", "IE_CHUNK_T", "IE_FAST_MATH", "IE_MC",
         "IE_SPIN_LIMIT_MS", "IE_DEBUG_FAULT", "IE_FUSE_LAST")
R4 = (4, 800, 2400, 60000)
FP32 = 2  # IE_CFG_FP32

# tag: ((n_layers, emb_sz, n_hid, vocab_sz), weight scale, B, T, development knobs, config flags)
CASES = {
    "R4": (R4, 1.0, 300, 24, {}, 0),
    "R4 IE_CFG_FP32": (R4, 1.0, 300, 24, {}, FP32),
    "R4 IE_GX_BF16=0": (R4, 1.0, 300, 24, {"IE_GX_BF16": 0}, 0),
    "R4 IE_SEQ=0": (R4, 1.0, 300, 12, {"IE_SEQ": 0}, 0),
    "R4 IE_MC=1": (R4, 1.0, 300, 24, {"IE_MC": 1}, 0),
    "one layer": ((1, 96, 8, 500), 2.0, 300, 23, {}, 0),
    "emb > hid": ((3, 200, 96, 500), 2.0, 300, 23, {}, 0),
    "width 33": ((2, 7, 33, 257), 2.0, 300, 23, {}, 0),
}

_weights_cache = {}


def _weights(shape, scale):
    key = (shape, scale)
    if key not in _weights_cache:
        n_layers, emb_sz, n_hid, vocab = shape
        ref = R.make_encoder(11 + n_layers + emb_sz + n_hid, vocab, emb_sz, n_hid, n_layers, scale=scale)
        _weights_cache.clear()
        _weights_cache[key] = ref.export_weights()
    return _weights_cache[key]


def _inputs(shape, B, T):
    vocab = shape[3]
    rng = np.random.default_rng(B * 1000 + T)
    ids = rng.integers(0, vocab, size=(B, T), dtype=np.int64)
    ids[ids == 1] = 0
    ids[:, 0] = 2
    lengths = np.concatenate([[1, T, T - 1, 2], rng.integers(1, T + 1, B - 4)]).astype(np.int32)
    for r, n in enumerate(lengths):
        ids[r, n:] = 1
    return ids, lengths


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def _outputs(tag, setenv, delenv):
    """sha256 of encode_ids (pooled, var-len) and raw_features of case `tag` under its knobs."""
    from code_intelligence_b200 import IssueEncoder
    shape, scale, B, T, knobs, flags = CASES[tag]
    for k in KNOBS:
        delenv(k)
    for k, v in knobs.items():
        setenv(k, str(v))
    try:
        enc = IssueEncoder(*shape, 1, 0, flags).load_weights(*_weights(shape, scale))
    finally:
        for k in knobs:
            delenv(k)
    ids, lengths = _inputs(shape, B, T)
    try:
        pooled = enc.encode_ids(ids, lengths)
        raw = enc.raw_features(ids)
    finally:
        enc.close()
    assert np.isfinite(pooled).all() and np.isfinite(raw).all()
    return {"encode": _sha(pooled), "raw": _sha(raw)}


def _frag_index(c, elem_bytes):
    """Fragment-order position of column c of a 256-column tile (DESIGN.md section 3), written out independently."""
    q = (c % 8) // 2                                  # quad lane holding the column in a wgmma fragment
    ix = 4 * (c // 16) + 2 * ((c // 8) % 2) + c % 2    # its place in that lane's run of 64: (m, gate i f g o)
    per = 16 // elem_bytes
    return (ix // per * 4 + q) * per + ix % per


def _layout(out_units):
    import ctypes as C
    from code_intelligence_b200 import _lib
    lib = _lib.load()
    rows = lib.ie_debug_epilogue_layout(out_units, None, 0, None, None)
    perm = np.empty(rows, dtype=np.int32)
    f2 = np.empty(256, dtype=np.int32)
    f4 = np.empty(256, dtype=np.int32)
    assert lib.ie_debug_epilogue_layout(out_units, perm.ctypes.data_as(C.c_void_p), rows, f2.ctypes.data_as(C.c_void_p),
                                        f4.ctypes.data_as(C.c_void_p)) == rows
    return perm, f2, f4


@pytest.mark.parametrize("out_units", [1, 33, 64, 96, 2400, 800])
def test_unit_permutation(out_units):
    """Weight rows of the recurrent kernel: a bijection onto torch's gate-major rows plus padding (-1); each thread's
    four gates of a unit sit in its fragment, and its units of a tile come in runs of four."""
    perm, _, _ = _layout(out_units)
    out_pad = -(-out_units // 64) * 64
    assert perm.shape == (4 * out_pad,)
    real = perm[perm >= 0]
    assert np.array_equal(np.sort(real), np.arange(4 * out_units))
    assert (perm == -1).sum() == 4 * (out_pad - out_units)
    gate, unit = perm // out_units, perm % out_units
    for col in range(4 * out_pad):
        j, c = divmod(col, 256)
        m, w = divmod(c, 16)
        q, b = (w % 8) // 2, w % 2
        s, e = divmod(m, 4)
        u = j * 64 + 16 * s + 4 * q + e
        g = (0 if b == 0 else 1) if w < 8 else (2 if b == 0 else 3)
        if u < out_units:
            assert (gate[col], unit[col]) == (g, u), col
        else:
            assert perm[col] == -1, col


def test_fragment_order_round_trips():
    _, f2, f4 = _layout(64)
    for f, eb in ((f2, 2), (f4, 4)):
        assert np.array_equal(np.sort(f), np.arange(256))            # a permutation of the tile
        assert np.array_equal(f, [_frag_index(c, eb) for c in range(256)])
        inv = np.empty(256, dtype=np.int64)
        inv[f] = np.arange(256)
        assert np.array_equal(inv[f], np.arange(256))
        # a lane's 16-byte chunk k holds only its own columns, chunk k sits at chunk position 4k + q
        per = 16 // eb
        for pos in range(0, 256, per):
            cols = inv[pos:pos + per]
            q = {(c % 8) // 2 for c in cols}
            assert len(q) == 1 and (pos // per) % 4 == q.pop()


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,out_type,segs", [(1280, 9728, 2432, 2, 1),     # hoisted Gx of a 2400-wide layer, fp16
                                                 (1280, 9728, 2432, 0, 3),     # f32 Gx, split-bf16 operands
                                                 (512, 9728, 832, 2, 1),       # per-token table shape (E 800 -> H 2400)
                                                 (300, 768, 64, 0, 1)])        # partial last M tile
def test_fragment_order_gemm_store(M, N, K, out_type, segs):
    """The fragment-ordered store, put back into column order on the host, equals the natural store bit for bit and
    is per-element correct against a float64 product of the bf16 (or split-bf16) operands."""
    from code_intelligence_b200 import _lib
    rng = np.random.default_rng(M + N + K)
    a = (rng.standard_normal((M, K)) * 0.5).astype(np.float32)
    b = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = (rng.standard_normal(N) * 0.1).astype(np.float32)
    nat = _lib._debug_gemm(a, b, bias, 0, out_type, segs)
    got = np.empty((M, N), dtype=np.float32)
    _lib.check(_lib.load().ie_debug_gemm_frag(a.ctypes.data, b.ctypes.data, bias.ctypes.data, M, N, K, out_type, segs,
                                              got.ctypes.data, 0))
    assert np.array_equal(got.view(np.uint32), nat.view(np.uint32))

    def bf16(x):
        u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
        return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16 << 16).astype(np.uint32).view(np.float32)
    if segs == 3:
        ah, bh = bf16(a), bf16(b)
        al, bl = bf16(a - ah), bf16(b - bh)
        want = ah.astype(np.float64) @ bh.T.astype(np.float64) + al.astype(np.float64) @ bh.T + ah.astype(np.float64) @ bl.T
    else:
        want = bf16(a).astype(np.float64) @ bf16(b).T.astype(np.float64)
    want += bias
    tol = (2.0 ** -10 if out_type == 2 else 2.0 ** -20) * np.abs(want) + 1e-5 * np.sqrt(K)
    assert (np.abs(got - want) <= tol).all()


@pytest.mark.gpu
@pytest.mark.parametrize("tag", list(CASES))
def test_outputs_match_the_natural_layout(tag, monkeypatch):
    with open(HASHES) as f:
        want = json.load(f)["cases"][tag]
    got = _outputs(tag, monkeypatch.setenv, lambda k: monkeypatch.delenv(k, raising=False))
    assert got == want


def _write(path):
    def delenv(k):
        os.environ.pop(k, None)
    cases = {}
    for tag in CASES:
        cases[tag] = _outputs(tag, os.environ.__setitem__, delenv)
        print(tag, cases[tag], flush=True)
    with open(path, "w") as f:
        json.dump({"cases": cases}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    if len(sys.argv) != 3 or sys.argv[1] != "--write":
        raise SystemExit(__doc__)
    _write(sys.argv[2])
