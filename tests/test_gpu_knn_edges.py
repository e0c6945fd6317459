"""GPU tests of the similar-issue index where its fused top-k can go wrong (csrc/knn.cu, the ie_knn_* half of
csrc/api.cu, code_intelligence_b200/knn.py): exact-arithmetic tie storms checked bit for bit, worst-case arrival orders,
permutation and power-of-two scale invariance, the norm range, the degraded regime, multi-pass searches, the largest
merge, and lifecycle / stream / thread use of a handle.

Every search result goes through `_verify`: indices in [0, n) and distinct per row, ascending by (distance, index), and
each distance within 1 f32 ulp of the f64 distance of its (query, row) pair."""
import threading

import numpy as np
import pytest
import torch

from oracle import knn_ref as K

pytestmark = pytest.mark.gpu

EXTRA = 32


def _index(D, metric):
    from code_intelligence_b200.knn import IssueIndex
    return IssueIndex(D, metric)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _np(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else t


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _verify(dist, idx, X, Q, metric):
    dist, idx = _np(dist), _np(idx)
    n = X.shape[0]
    assert ((idx >= 0) & (idx < n)).all(), "index out of range"
    s = np.sort(idx, axis=1)
    assert (s[:, 1:] != s[:, :-1]).all(), "repeated index in a row"
    d0, d1, i0, i1 = dist[:, :-1], dist[:, 1:], idx[:, :-1], idx[:, 1:]
    assert ((d1 > d0) | ((d1 == d0) & (i1 > i0))).all(), "not ascending by (distance, index)"
    ref = K._exact(np.asarray(Q, np.float64), np.asarray(X, np.float64), idx, metric)
    tol = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    err = np.abs(dist.astype(np.float64) - ref)
    assert (err <= tol).all(), f"distance off its pair's f64 value by {(err / tol).max():.2f} ulp"


def _same(got, want, what):
    (gd, gi), (wd, wi) = (_np(got[0]), _np(got[1])), want
    assert (gi == wi).all(), f"{what}: {(gi != wi).sum()} indices differ"
    assert (_bits(gd) == _bits(wd)).all(), f"{what}: {(_bits(gd) != _bits(wd)).sum()} distances differ in bits"


def _check_lattice(index, X, Q, k, metric, what):
    """Shortlist == exact top-k' (scores bit for bit, -inf / -1 past n) and search == exact brute force."""
    score, sidx = index._shortlist(Q, k)
    wscore, widx = K.topk_exact(K.lattice_scores(X, Q, metric), k + EXTRA)
    bad = (sidx != widx).any(1) | (_bits(score) != _bits(wscore)).any(1)
    assert not bad.any(), f"{what}: shortlist differs for queries {np.flatnonzero(bad)[:8]}"
    got = index.search(Q, k)
    _verify(*got, X, Q, metric)
    _same(got, K.lattice_brute(X, Q, k, metric), what)


def _planted(n, D, seed):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((max(1, n // 50), D)) * 3.0 + 5.0
    return (centres[rng.integers(0, len(centres), n)] + rng.standard_normal((n, D))).astype(np.float32)


def _queries(X, nq, seed):
    rng = np.random.default_rng(seed)
    return (X[rng.integers(0, len(X), nq)] + rng.standard_normal((nq, X.shape[1])) * 0.5).astype(np.float32)


def _sphere(rng, q, G, metric):
    """G lattice rows at one stage-1 score for query q, most of them distinct: euclidean q with one coordinate moved
    by +-1 (|q - x| = 1), cosine q with one sign flipped (same norm, q.x = |q|^2 - 2)."""
    R = np.repeat(q[None], G, 0)
    rows = np.arange(G)
    if metric == "euclidean":
        R[rows, rng.integers(0, q.size, G)] += rng.choice(np.float32([-1, 1]), G)
    else:
        R[rows, rng.choice(np.flatnonzero(q), G)] *= -1
    return R


# ---- lattice ties, bit-exact --------------------------------------------------------------------------------------
TIES = [  # (k, n = 256 * SMs * mult + delta, nq, tie-group size G, where)
    (10, (2, 1), 8, 5000, "all"),
    (64, (2, -1), 8, 300, "all"),
    (1, (2, 600), 8, 500, "last"),
    (64, (2, 600), 130, 100, "last"),
    (10, (3, 0), 8, 0, "tiles"),
    (1, (0, 20_000), 8, 2000, "all"),
    (64, (0, 90), 3, 40, "all"),
]


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
@pytest.mark.parametrize("k,nspec,nq,G,where", TIES)
def test_lattice_ties_bit_exact(metric, k, nspec, nq, G, where):
    """Tie groups of up to 5000 rows at the k-th score (copies of the query ahead of them, so the group straddles both
    the k-th and the k'-th place), spread over every slice, confined to the last partial slice, or as whole 256-row
    tiles that equal the running threshold: ties must resolve by index however many there are."""
    sms, D = _sms(), 64
    n = 256 * sms * nspec[0] + nspec[1]
    rng = np.random.default_rng(n + k + G)
    m = min(64, n // 4)
    X = np.vstack([K.with_zero_centre(K.lattice_rows(rng, m, D, metric, -1, 1)),
                   K.lattice_rows(rng, n - 2 * m, D, metric, -1, 1)])
    Q = K.lattice_rows(rng, nq, D, metric, -1, 1)
    S, nbs, _ = K.plan(nq, n, k + EXTRA, sms)
    m1 = k // 2
    for qi in range(min(nq, 2)):
        if where == "tiles":
            for t in range(1, -(-n // 256)):
                if t % 3 != 1:
                    X[256 * t:256 * (t + 1)] = _sphere(rng, Q[qi], len(X[256 * t:256 * (t + 1)]), metric)
            X[rng.choice(np.arange(2 * m, n), m1, replace=False)] = Q[qi]
            continue
        lo = max(2 * m, (S - 1) * nbs * 256) if where == "last" else 2 * m
        pos = rng.choice(np.arange(lo, n), min(m1 + G, n - lo), replace=False)
        X[pos[:m1]] = Q[qi]
        X[pos[m1:]] = _sphere(rng, Q[qi], len(pos) - m1, metric)
    index = _index(D, metric).add(X[:2 * m]).add(X[2 * m:])
    _check_lattice(index, X, Q, k, metric, f"{metric} k={k} n={n} G={G} {where} S={S} nbs={nbs}")
    index.close()


def test_zero_rows_tie_with_exact_zero_scores():
    """Euclidean, an all-negative query: a zero row scores sum(q_i * 0) - 0, which the tensor cores may return as -0;
    rows -2 e_j score 2 - 2 = +0 by cancellation.  Both are at distance |q|, so they tie by index: the zero rows (lower
    indices) come first, in the shortlist as in the answer."""
    D, k = 32, 10
    rng = np.random.default_rng(21)
    B = 3.0 * rng.integers(0, 2, (64, D)).astype(np.float32)   # -B and B both score below 0
    B[B.sum(1) == 0, 0] = 3.0
    n_zero, n_cancel = 40, 200
    cancel = np.zeros((n_cancel, D), np.float32)
    cancel[np.arange(n_cancel), rng.integers(0, D, n_cancel)] = -2.0
    back = rng.integers(0, 2, (3000, D)).astype(np.float32)     # q.x - |x|^2/2 < 0 for every nonzero 0/1 row
    back[back.sum(1) == 0, 0] = 1.0
    X = np.vstack([K.with_zero_centre(B), np.zeros((n_zero, D), np.float32), cancel, back])
    Q = np.vstack([-np.ones((2, D), np.float32), K.lattice_rows(rng, 6, D, "euclidean", -1, 1)])
    index = _index(D, "euclidean").add(X[:128]).add(X[128:])
    _check_lattice(index, X, Q, k, "euclidean", "zero rows vs +0")
    _, idx = index.search(Q[:1], k)
    assert list(idx[0]) == list(range(128, 128 + k))
    index.close()


# ---- worst-case arrival orders ----------------------------------------------------------------------------------
def _orders(s0, n0, n, S, nbs, kp, rng):
    """Row orders of the corpus rows [n0, n) by query 0's score: increasing (every tile beats the threshold),
    decreasing, and the best kp spread one per slice (the first row of each)."""
    body = np.arange(n0, n)
    inc = body[np.lexsort((body, s0[body]))]
    yield "increasing", np.concatenate([np.arange(n0), inc])
    yield "decreasing", np.concatenate([np.arange(n0), inc[::-1]])
    top = inc[::-1][:kp]
    rest = rng.permutation(np.setdiff1d(body, top))
    order = np.empty(n, np.int64)
    order[:n0] = np.arange(n0)
    starts = [p for p in range(0, S * nbs * 256, nbs * 256) if p >= n0][:len(top)]
    free = np.setdiff1d(np.arange(n0, n), starts)
    order[starts] = top[:len(starts)]
    order[free] = np.concatenate([top[len(starts):], rest])
    yield "spread", order


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_arrival_orders(metric):
    sms, D, k, nq = _sms(), 64, 10, 4
    n = 256 * sms * 2 + 37
    S, nbs, _ = K.plan(nq, n, k + EXTRA, sms)
    rng = np.random.default_rng(31)
    # lattice: bit-exact
    X = np.vstack([K.with_zero_centre(K.lattice_rows(rng, 64, D, metric, -1, 1)),
                   K.lattice_rows(rng, n - 128, D, metric, -1, 1)])
    Q = K.lattice_rows(rng, nq, D, metric, -1, 1)
    s0 = K.lattice_scores(X, Q[:1], metric)[0]
    for name, order in _orders(s0, 128, n, S, nbs, k + EXTRA, rng):
        Xo = X[order]
        index = _index(D, metric).add(Xo[:128]).add(Xo[128:])
        _check_lattice(index, Xo, Q, k, metric, f"lattice {name}")
        index.close()
    # planted float data: against brute force
    X = _planted(n, D, 32)
    Q = _queries(X, nq, 33)
    s0, _ = K.stage1_scores(X, Q[:1], K.center(X[:4096]), metric)
    for name, order in _orders(s0[0], 4096, n, S, nbs, k + EXTRA, rng):
        Xo = X[order]
        index = _index(D, metric).add(Xo[:4096]).add(Xo[4096:])
        got = index.search(Q, k)
        _verify(*got, Xo, Q, metric)
        wd, wi = K.brute(Xo, Q, k, metric)
        assert (got[1] == wi).all(), f"planted {name}"
        index.close()


# ---- invariances ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_permutation(metric):
    n, D, k = 20_000, 96, 10
    rng = np.random.default_rng(41)
    X = _planted(n, D, 41)
    X += rng.standard_normal(X.shape).astype(np.float32) * 1e-2   # no exact or near-exact duplicates: no ties
    Q = _queries(X, 300, 42)
    perm = rng.permutation(n)
    a = _index(D, metric).add(X)
    b = _index(D, metric).add(X[perm])
    da, ia = a.search(Q, k)
    db, ib = b.search(Q, k)
    _verify(da, ia, X, Q, metric)
    assert (perm[ib] == ia).all() and (_bits(db) == _bits(da)).all()
    a.close()
    b.close()


def _bf16(x):
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def _scale_range(X, Q):
    """The powers of two 2^j for which scaling X and Q commutes with every rounding of the index: the scaled split
    parts (bf16 hi, lo), their products and the centre stay normal, every partial sum |q~||x~| and |x~|^2 stays below
    2^126, and every row norm stays inside the index's range [2^-48, 2^48]."""
    c = K.center(X).astype(np.float64)
    parts = []
    for A in (X, Q):
        t = A.astype(np.float64) - c
        hi = _bf16(t.astype(np.float32))
        parts += [hi, _bf16((t - hi).astype(np.float32))]
    tiny = min(np.abs(p[p != 0]).min() for p in parts)
    tiny = min(tiny ** 2, tiny * np.abs(c[c != 0]).min())
    big = max(np.linalg.norm(A.astype(np.float64) - c, axis=1).max() for A in (X, Q)) ** 2 * 4
    norms = np.concatenate([np.linalg.norm(A.astype(np.float64), axis=1) for A in (X, Q)])
    j_lo = max(int(np.ceil((-126 - np.log2(tiny)) / 2)), int(np.ceil(-48 - np.log2(norms.min()))))
    j_hi = min(int(np.floor((126 - np.log2(big)) / 2)), int(np.floor(48 - np.log2(norms.max()))))
    return j_lo, j_hi


def test_power_of_two_scale():
    """Scaling by 2^j commutes with bf16, f32, the f64 centre and 1/sqrt: cosine answers are bit-identical, euclidean
    indices identical with distances exactly 2^j times; shortlist scores scale by 2^j (cosine) / 2^2j (euclidean)."""
    n, D, k = 20_000, 200, 10
    X = _planted(n, D, 51)
    Q = _queries(X, 200, 52)
    j_lo, j_hi = _scale_range(X, Q)
    js = sorted({j_lo, -8, -1, 1, 8, j_hi})
    print(f"power-of-two scale: derived j range [{j_lo}, {j_hi}], tested {js}")
    assert j_lo <= -8 and j_hi >= 8
    for metric in ("cosine", "euclidean"):
        base = _index(D, metric).add(X)
        d0, i0 = base.search(Q, k)
        s0, si0 = base._shortlist(Q, k)
        base.close()
        for j in js:
            f = np.float32(2.0 ** j)
            idx = _index(D, metric).add(X * f)
            d, i = idx.search(Q * f, k)
            s, si = idx._shortlist(Q * f, k)
            idx.close()
            _verify(d, i, X * f, Q * f, metric)
            assert (i == i0).all() and (si == si0).all(), f"{metric} j={j}"
            want = d0 if metric == "cosine" else d0 * f
            assert (_bits(d) == _bits(want)).all(), f"{metric} j={j}"
            sf = np.float32(2.0 ** (j if metric == "cosine" else 2 * j))
            assert (_bits(s) == _bits(s0 * sf)).all(), f"{metric} j={j} shortlist"


# ---- the norm range ------------------------------------------------------------------------------------------
def _edge_row(D, log2_norm):
    """A +-1 row on 16 coordinates, scaled to norm exactly 2^log2_norm."""
    r = np.zeros(D, np.float32)
    r[:16] = np.where(np.arange(16) % 3 == 0, -1.0, 1.0)
    return r * np.float32(2.0 ** (log2_norm - 2))


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
@pytest.mark.parametrize("side", ["huge", "tiny"])
def test_norm_range(metric, side):
    """Rows at the limits (norm 2^48 or 2^-48, a row with subnormal entries among normal ones) are answered exactly;
    one step outside (2^49, 2^-49, a row of subnormal entries) host input is refused with ValueError and device input
    is reported by check_errors.  A finite input never yields an out-of-range index or a non-finite distance."""
    n, D, k = 3000, 64, 5
    e = 48 if side == "huge" else -48
    X = _planted(n, D, 61)
    Q = _queries(X, 60, 62)
    norms = np.linalg.norm(np.vstack([X, Q]), axis=1)
    f = np.float32(2.0 ** (e - 1 - np.ceil(np.log2(norms.max())) if e > 0 else e + 1 - np.floor(np.log2(norms.min()))))
    X, Q = X * f, np.vstack([Q * f, _edge_row(D, e)[None]])
    X[10] = _edge_row(D, e)
    X[11] = X[12]
    X[11, 5] = np.float32(1e-40)                               # a subnormal entry in a normal row
    for dev in (False, True):
        index = _index(D, metric)
        if dev:
            index.add(torch.from_numpy(X).cuda())
            d, i = index.search(torch.from_numpy(Q).cuda(), k)
            index.check_errors()
        else:
            index.add(X)
            d, i = index.search(Q, k)
        _verify(d, i, X, Q, metric)
        wd, wi = K.brute(X, Q, k, metric)
        assert (_np(i) == wi).all(), f"{side} {metric} dev={dev}"
        outside = [_edge_row(D, e + (1 if e > 0 else -1))]
        if e < 0:
            outside.append(np.full(D, 1e-40, np.float32))      # nonzero, every entry subnormal
        for row in outside:
            with pytest.raises(ValueError, match="outside the index's range"):
                index.add(row[None])
            with pytest.raises(ValueError, match="outside the index's range"):
                index.search(np.vstack([Q[:2], row[None]]), k)
            d2, i2 = index.search(torch.from_numpy(np.vstack([Q[:2], row[None]])).cuda(), k)
            torch.cuda.synchronize()
            with pytest.raises(ValueError, match="outside the index's range"):
                index.check_errors()
            index.check_errors()   # cleared
        index.add(np.zeros((1, D), np.float32))   # a zero row is always allowed
        index.close()


# ---- degraded regime ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_near_duplicate_storm(metric):
    """Storms of 60-400 near-duplicates of each query, all within 2 eps of each other: the exactness condition fails
    and the answer may differ from brute force.  The shortlist argument still bounds it.  Let s* be exact scores,
    s^ = s* +- eps the stage-1 scores, and T_i the exact top i.  If every row of T_i is shortlisted, the i-th best
    shortlisted row scores at least s*_(i).  Otherwise some t in T_i was dropped, so every shortlisted row r has
    s^_r >= s^_t, hence s*_r >= s*_t - eps_t - eps_r >= s*_(i) - 2 max eps.  Stage 2 orders the shortlist by exact
    distance (monotone in s*), so the i-th returned row scores at least s*_(i) - 2 max eps over T_k and the rows
    returned."""
    n, D, k = 20_000, 256, 10
    rng = np.random.default_rng(71)
    X = _planted(n, D, 71)
    Q = _queries(X, 50, 72)
    for qi in range(Q.shape[0]):
        G = int(rng.integers(60, 400))
        pos = rng.choice(n, G, replace=False)
        # |x - q| ~ 0.016: distinct f32 rows whose scores differ by ~1e-4, far inside eps (~0.05 here)
        X[pos] = Q[qi] + (rng.standard_normal((G, D)) * 1e-3).astype(np.float32)
    index = _index(D, metric).add(X)
    d, i = index.search(Q, k)
    _verify(d, i, X, Q, metric)
    s, eps = K.stage1_scores(X, Q, K.center(X), metric)
    held = sum(K.exactness_holds(s[r], eps[r], k) for r in range(Q.shape[0]))
    print(f"storm {metric}: the exactness condition holds for {held} of {Q.shape[0]} queries")
    assert held < Q.shape[0]
    for r in range(Q.shape[0]):
        top = np.lexsort((np.arange(n), -s[r]))[:k]
        e2 = 2 * max(eps[r, top].max(), eps[r, i[r]].max())
        assert (s[r, i[r]] >= s[r, top] - e2).all(), f"{metric} query {r}"
    index.close()


# ---- multi-pass, the largest merge, dimension edges ------------------------------------------------------------
def _lattice_brute_gpu(X, Q, k, metric, chunk=4096):
    """K.lattice_brute with the exact f64 products on the GPU (integer sums, exact in any order)."""
    Xg = torch.from_numpy(X).cuda().double()
    x2 = (Xg * Xg).sum(1)
    out_d, out_i = [], []
    for r0 in range(0, Q.shape[0], chunk):
        Qg = torch.from_numpy(Q[r0:r0 + chunk]).cuda().double()
        acc = Qg @ Xg.T
        q2 = (Qg * Qg).sum(1, keepdim=True)
        if metric == "euclidean":
            d = torch.sqrt(q2 - 2.0 * acc + x2[None])
        else:
            d = 1.0 - acc / (torch.sqrt(q2) * torch.sqrt(x2)[None])
            d = torch.where((q2 == 0) | (x2[None] == 0), torch.ones_like(d), d)
        d, i = torch.sort(d, dim=1, stable=True)
        out_d.append(d[:, :k].float().cpu().numpy())
        out_i.append(i[:, :k].cpu().numpy())
    return np.concatenate(out_d), np.concatenate(out_i)


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_multi_pass(metric):
    """nq = 128 SMs + 1 and 2 * 128 SMs + 200: two and three passes, host and device pointers, each equal to brute
    force and bit-equal to the same queries searched in chunks."""
    sms, D, k, n = _sms(), 32, 5, 3000
    rng = np.random.default_rng(81)
    X = np.vstack([K.with_zero_centre(K.lattice_rows(rng, 64, D, metric, -1, 1)),
                   K.lattice_rows(rng, n - 128, D, metric, -1, 1)])
    index = _index(D, metric).add(X[:128]).add(X[128:])
    for nq in (128 * sms + 1, 2 * 128 * sms + 200):
        Q = K.lattice_rows(rng, nq, D, metric, -1, 1)
        want = _lattice_brute_gpu(X, Q, k, metric)
        host = index.search(Q, k)
        dev = index.search(torch.from_numpy(Q).cuda(), k)
        torch.cuda.synchronize()
        chunks = [index.search(Q[r0:r0 + 5000], k) for r0 in range(0, nq, 5000)]
        chunked = (np.concatenate([c[0] for c in chunks]), np.concatenate([c[1] for c in chunks]))
        _verify(*host, X, Q, metric)
        for what, got in (("host", host), ("device", dev), ("chunked", chunked)):
            _same(got, want, f"{metric} nq={nq} {what}")
    index.close()


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_largest_merge(metric):
    """k = 64, nq <= 128, n = 256 * SMs * j: S * k' > 8192, so the merge sorts P = 16384 keys (about 130 KB of shared
    memory), on lattice data full of ties."""
    sms, D, k = _sms(), 64, 64
    for j, nq in ((1, 128), (3, 7)):
        n = 256 * sms * j
        assert K.plan(nq, n, k + EXTRA, sms)[2] == 16384
        rng = np.random.default_rng(91 + j)
        X = np.vstack([K.with_zero_centre(K.lattice_rows(rng, 64, D, metric, -1, 1)),
                       K.lattice_rows(rng, n - 128, D, metric, -1, 1)])
        Q = K.lattice_rows(rng, nq, D, metric, -1, 1)
        index = _index(D, metric).add(X[:128]).add(X[128:])
        _check_lattice(index, X, Q, k, metric, f"P=16384 n={n} nq={nq}")
        index.close()


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
@pytest.mark.parametrize("D", [63, 65, 8192])
def test_dimension_edges(metric, D):
    rng = np.random.default_rng(D)
    lo, hi = (-1, 1) if D > 2400 else (-3, 3)
    X = np.vstack([K.with_zero_centre(K.lattice_rows(rng, 32, D, metric, lo, hi)),
                   K.lattice_rows(rng, 1000, D, metric, lo, hi)])
    Q = np.vstack([K.lattice_rows(rng, 40, D, metric, lo, hi), X[100:110]])
    index = _index(D, metric).add(X[:64]).add(X[64:])
    _check_lattice(index, X, Q, 10, metric, f"D={D}")
    index.close()
    with pytest.raises(ValueError, match="not in"):
        _index(8193, metric)


# ---- lifecycle, streams, threads ------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_search_add_search_and_single_row_adds(metric):
    D, k = 48, 5
    X = _planted(7000, D, 101)
    Q = _queries(X, 100, 102)
    index = _index(D, metric).add(X[:1000])
    got = index.search(Q, k)
    _verify(*got, X[:1000], Q, metric)
    assert (got[1] == K.brute(X[:1000], Q, k, metric)[1]).all()
    index.add(X[1000:])                                   # the storage grows from 1024 rows
    got = index.search(Q, k)
    _verify(*got, X, Q, metric)
    assert (got[1] == K.brute(X, Q, k, metric)[1]).all()
    index.close()
    # 300 rows, one add at a time (the first a row and its negation: centre 0), searched after every add
    rng = np.random.default_rng(103)
    L = K.lattice_rows(rng, 300, 16, metric, -1, 1)
    L[1] = -L[0]
    Ql = K.lattice_rows(rng, 20, 16, metric, -1, 1)
    index = _index(16, metric).add(L[:2])
    for r in range(2, 301):
        kk = min(k, r)
        got = index.search(Ql, kk)
        _verify(*got, L[:r], Ql, metric)
        _same(got, K.lattice_brute(L[:r], Ql, kk, metric), f"{metric} after {r} rows")
        if r < 300:
            index.add(L[r:r + 1])
    index.close()


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_poor_centre(metric):
    """The first add is one far outlier, so the centre is that row: every query that meets the exactness condition
    with the index's actual centre gets the exact answer."""
    D, k = 64, 10
    X = _planted(10_000, D, 111)
    X[0] = X[0] + 300.0
    Q = _queries(X[1:], 200, 112)
    index = _index(D, metric).add(X[:1]).add(X[1:])
    d, i = index.search(Q, k)
    _verify(d, i, X, Q, metric)
    s, eps = K.stage1_scores(X, Q, K.center(X[:1]), metric)
    held = np.array([K.exactness_holds(s[r], eps[r], k) for r in range(Q.shape[0])])
    print(f"poor centre {metric}: the exactness condition holds for {held.sum()} of {Q.shape[0]} queries")
    wd, wi = K.brute(X, Q, k, metric)
    assert (i[held] == wi[held]).all()
    index.close()


def test_streams():
    """A device add on stream A followed at once by a search on stream B; a query tensor made by a kernel on a side
    stream and searched under that stream; back-to-back device searches of growing nq on one stream (the scratch
    buffers grow between asynchronous calls).  Every result is bit-equal to a serial host-pointer search."""
    D, k, metric = 64, 10, "euclidean"
    X = _planted(30_000, D, 121)
    Q = _queries(X, 20_000, 122)
    ref = _index(D, metric).add(X[:5000]).add(X[5000:])   # the same centre as `index`
    index = _index(D, metric).add(X[:5000])
    Xg = torch.from_numpy(X[5000:]).cuda()
    Qg = torch.from_numpy(Q).cuda()
    A, B, side = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    A.wait_stream(torch.cuda.current_stream())
    B.wait_stream(torch.cuda.current_stream())
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(A):
        index.add(Xg)
    with torch.cuda.stream(B):
        dB, iB = index.search(Qg[:500], k)
    with torch.cuda.stream(side):
        Qs = Qg[:700] * 2.0 - Qg[:700]                  # made by a kernel on `side`, equal to Q[:700]
        dS, iS = index.search(Qs, k)
    grow = []
    with torch.cuda.stream(B):
        for nq in (1, 200, 3000, 20_000):
            grow.append((nq, index.search(Qg[:nq], k)))
    torch.cuda.synchronize()
    index.check_errors()
    for what, nq, (d, i) in [("A/B", 500, (dB, iB)), ("side", 700, (dS, iS))] + [("grow", nq, r) for nq, r in grow]:
        _same((d, i), ref.search(Q[:nq], k), f"{what} nq={nq}")
    _verify(dB, iB, X, Q[:500], metric)
    index.close()
    ref.close()


def test_threads():
    """4 host threads on one handle and 2 handles searched concurrently: every result bit-equal to a serial search."""
    D, k = 64, 10
    X = _planted(20_000, D, 131)
    Q = _queries(X, 2000, 132)
    one = _index(D, "cosine").add(X)
    two = _index(D, "euclidean").add(X)
    want = {(h, t): (one if h == 0 else two).search(Q[t * 500:(t + 1) * 500], k) for h in (0, 1) for t in range(4)}
    got, errors = {}, []

    def run(h, t):
        try:
            for _ in range(3):
                got[(h, t)] = (one if h == 0 else two).search(Q[t * 500:(t + 1) * 500], k)
        except Exception as e:   # surfaced below
            errors.append(e)
    threads = [threading.Thread(target=run, args=(0, t)) for t in range(4)]
    threads += [threading.Thread(target=run, args=(1, t)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for key, res in got.items():
        _same(res, want[key], f"thread {key}")
    one.close()
    two.close()
