"""The vector stage bit for bit (run with -m gpu on an H100).

On exact-arithmetic inputs (tests/vec_spec.py) every distance the device computes is determined, so both implementations of
`Index.nns_by_vector` must reproduce R1, the float32 replica of the device formula, exactly: ids, distances and counts.
  - the GEMV path (vec_dist_kernel + topk_select_kernel): batches of fewer than 16 queries, k > 128, d > 768, d % 64 != 0;
  - the wgmma path (vec_gemm_topk_kernel + vec_merge_kernel): the rest.
B200_VEC_GEMM=0/1 forces a path where both apply and B200_VEC_SMS bounds the CTAs of the wgmma path (more slices per query tile,
or several launches).  The selection is stressed where it can go wrong: more ties at the k-th distance than the tie buffer holds,
zero queries and zero rows, duplicate docids, tiles that all survive the screen, exact ties at the reject bound, filters.  On
realistic inputs, results are checked as float64 certificates (R2)."""
import numpy as np
import pytest

from tests import vec_spec as vs
from tests.helpers import synthetic_image

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mb():
    import meilisearch_b200 as m

    m.load_library()
    return m


@pytest.fixture(scope="module")
def img():
    return synthetic_image(3000, 800, seed=31)


@pytest.fixture(scope="module")
def ix(mb, img):
    return mb.Index(img)


def _nns(ix, monkeypatch, path, q, k, cand=None, sms=None):
    """run one batch on `path` ("gemv", "wgmma" or "auto") and check that the intended kernels ran"""
    if path == "auto":
        monkeypatch.delenv("B200_VEC_GEMM", raising=False)
    else:
        monkeypatch.setenv("B200_VEC_GEMM", "1" if path == "wgmma" else "0")
    if sms is None:
        monkeypatch.delenv("B200_VEC_SMS", raising=False)
    else:
        monkeypatch.setenv("B200_VEC_SMS", str(sms))
    ix.reset_stats()
    got = ix.nns_by_vector(q, k, cand)
    kern = ix.stats()["kernels"]
    gemm = kern["vec_gemm_topk"]["count"] > 0
    if path == "wgmma":
        assert gemm, "the wgmma path did not run"
    elif path == "gemv":
        assert not gemm and kern["vec_dist"]["count"] > 0, "the GEMV path did not run"
    return got, gemm


def _same(got, want, ctx):
    gi, gd, gc = got
    wi, wd, wc = want
    assert np.array_equal(gc, wc), (ctx, "counts", np.nonzero(gc != wc)[0][:5])
    for q in range(len(wc)):
        c = int(wc[q])
        assert np.array_equal(gi[q, :c], wi[q, :c]), (ctx, q, "ids", gi[q, :c][:8], wi[q, :c][:8])
        assert np.array_equal(gd[q, :c].view(np.uint32), wd[q, :c].view(np.uint32)), (ctx, q, "distances", gd[q, :c][:8], wd[q, :c][:8])


def _exact(ix, monkeypatch, rows, docids, q, k, paths, cand=None, sms=None, ctx=None):
    assert vs.rule_margin_ok(rows, q)
    want = vs.r1(rows, docids, q, k, cand)
    for p in paths:
        got, _ = _nns(ix, monkeypatch, p, q, k, cand, sms)
        _same(got, want, (ctx, p, sms, "filtered" if cand is not None else ""))
    return want


def _filter(g, n_docs, p=0.5):
    return vs.bitmap(np.nonzero(g.rng.random(n_docs) < p)[0], (n_docs + 63) // 64)


# ------------------------------------------------------------------------------------------------ wgmma shapes, both paths
# (d, rows, queries, k, B200_VEC_SMS): k <= 8 keeps the slice's best keys in registers, k > 8 goes through run compaction;
# 600 queries with 8 CTAs take two launches
W_CASES = [
    (64, 1, 16, 1, None),
    (64, 63, 17, 7, 33),
    (128, 64, 63, 8, None),
    (128, 65, 64, 9, 8),
    (704, 127, 65, 64, None),
    (768, 129, 16, 127, 33),
    (768, 64 * 41, 17, 128, None),
    (64, 20011, 64, 9, 33),
    (128, 20011, 65, 128, None),
    (704, 20011, 16, 8, 8),
    (768, 20011, 63, 1, None),
    (128, 64 * 41, 600, 7, 8),
]


@pytest.mark.parametrize("d,n,nq,k,sms", W_CASES)
def test_wgmma_shapes_bit_exact(ix, img, monkeypatch, d, n, nq, k, sms):
    g = vs.ExactGen(d, seed=d * 7 + n + nq + k)
    rows = g.mixed_rows(n)
    docids = g.docids(n, img.n_docs)
    q = g.mixed_queries(nq, rows)
    ix.set_embeddings(rows, docids)
    for cand in (None, _filter(g, img.n_docs + 64 * 3 * max(n, 64))):
        _exact(ix, monkeypatch, rows, docids, q, k, ("wgmma", "gemv"), cand, sms, (d, n, nq, k))


# ------------------------------------------------------------------------------------------------ GEMV shapes
# (d, rows, queries, k, path): 70 001 rows are selected in several slices; at 64 queries, d = 100 / 1024 / 1536 and k > 128 fall
# back from the batched path
G_CASES = [
    (8, 70001, 1, 1, "gemv"),
    (100, 70001, 2, 129, "gemv"),
    (1024, 70001, 7, 1000, "gemv"),
    (1536, 70001, 15, 0, "gemv"),
    (1536, 70001, 1, 129, "gemv"),
    (100, 20011, 64, 100, "auto"),
    (1024, 20011, 64, 64, "auto"),
    (1536, 5000, 64, 10, "auto"),
    (64, 70001, 64, 129, "auto"),
]


@pytest.mark.parametrize("d,n,nq,k,path", G_CASES)
def test_gemv_shapes_bit_exact(ix, img, monkeypatch, d, n, nq, k, path):
    g = vs.ExactGen(d, seed=d * 5 + n + nq + k)
    rows = g.mixed_rows(n)
    docids = g.docids(n, img.n_docs)
    q = g.mixed_queries(nq, rows)
    ix.set_embeddings(rows, docids)
    for cand in (None, _filter(g, img.n_docs + 64 * 3 * n)):
        _exact(ix, monkeypatch, rows, docids, q, k, (path,), cand, None, (d, n, nq, k))
        if path == "auto":
            assert not _nns(ix, monkeypatch, "auto", q, k, cand)[1], "expected the fallback to the GEMV path"


@pytest.mark.parametrize("d,k", [(64, 8), (768, 100), (128, 128)])
def test_cross_path_one_query_vs_batch(ix, img, monkeypatch, d, k):
    """the same exact queries one at a time (GEMV) and in a batch of 16+ (wgmma): identical results"""
    g = vs.ExactGen(d, seed=100 + d)
    n = 20011
    rows = g.mixed_rows(n)
    docids = g.docids(n, img.n_docs)
    q = g.mixed_queries(20, rows)
    ix.set_embeddings(rows, docids)
    batch, gemm = _nns(ix, monkeypatch, "auto", q, k)
    assert gemm
    for i in range(len(q)):
        one, gemm = _nns(ix, monkeypatch, "auto", q[i:i + 1], k)
        assert not gemm
        _same(one, tuple(x[i:i + 1] for x in batch), (d, k, i))
    _same(batch, vs.r1(rows, docids, q, k), (d, k, "r1"))


# ------------------------------------------------------------------------------------------------ selection stress
def test_ties_past_tie_buffer_in_every_slice(ix, img, monkeypatch):
    """40 % of 70 001 rows are copies of one row (exact or scaled by 2^k): far more than 1024 ties at the k-th distance in every
    slice of the GEMV selection, with permuted docids; the k smallest docids must win"""
    d, n = 64, 70001
    g = vs.ExactGen(d, seed=41)
    rows = g.rows(n)
    src = rows[0]
    copy = g.rng.random(n) < 0.4
    rows[copy] = src
    sc = copy & (g.rng.random(n) < 0.5)
    rows[sc] = g.scaled(rows[sc], 2.0 ** -14)
    docids = g.rng.permutation(n).astype(np.uint32)
    ix.set_embeddings(rows, docids)
    q = np.concatenate([g.band(np.stack([src, -src]), 2.0 ** -8), g.queries(14)])
    for k in (1, 100, 129, 1000):
        want = _exact(ix, monkeypatch, rows, docids, q[:3], k, ("gemv",), ctx=("ties", k))
        assert (want[1][0, :k] == want[1][0, 0]).all()  # the whole top-k is one tie
    for k in (1, 9, 128):
        _exact(ix, monkeypatch, rows, docids, q, k, ("wgmma", "gemv"), ctx=("ties", k))


@pytest.mark.parametrize("n", [5000, 70001])
def test_zero_query(ix, img, monkeypatch, n):
    """every distance is 0: the result is the k smallest docids, for one query and inside a batch"""
    d = 128
    g = vs.ExactGen(d, seed=n)
    rows = g.mixed_rows(n)
    docids = g.docids(n, img.n_docs)
    ix.set_embeddings(rows, docids)
    q = np.concatenate([np.zeros((1, d), np.float32), g.queries(15)])
    for k in (1, 100, 128):
        want = _exact(ix, monkeypatch, rows, docids, q[:1], k, ("gemv",), ctx=("zero query", n, k))
        assert list(want[0][0]) == sorted(docids.tolist())[:k]
        _exact(ix, monkeypatch, rows, docids, q, k, ("wgmma", "gemv"), ctx=("zero query batch", n, k))
    _exact(ix, monkeypatch, rows, docids, q[:1], 1000, ("gemv",), ctx=("zero query", n, 1000))


def test_many_zero_rows(ix, img, monkeypatch):
    """8 000 zero rows rank first for every query (distance 0), in docid order"""
    d, n = 128, 20011
    g = vs.ExactGen(d, seed=43)
    rows = g.mixed_rows(n, zero=0)
    rows[g.rng.permutation(n)[:8000]] = 0
    docids = g.docids(n, img.n_docs)
    ix.set_embeddings(rows, docids)
    q = g.mixed_queries(16, rows)
    for k in (8, 100, 128):
        _exact(ix, monkeypatch, rows, docids, q, k, ("wgmma", "gemv"), ctx=("zero rows", k))
        _exact(ix, monkeypatch, rows, docids, q[:3], k, ("gemv",), ctx=("zero rows", k))
    _exact(ix, monkeypatch, rows, docids, q[:2], 1000, ("gemv",), ctx=("zero rows", 1000))


def test_duplicate_docids(ix, img, monkeypatch):
    d, n = 64, 20011
    g = vs.ExactGen(d, seed=44)
    rows = g.mixed_rows(n, dup=0.2)
    docids = g.docids(n, img.n_docs, dup=0.3)
    ix.set_embeddings(rows, docids)
    q = g.mixed_queries(16, rows)
    for k in (7, 64, 128):
        _exact(ix, monkeypatch, rows, docids, q, k, ("wgmma", "gemv"), ctx=("duplicate docids", k))


@pytest.mark.parametrize("k", [1, 8, 9, 128])
def test_rows_in_increasing_similarity(ix, img, monkeypatch, k):
    """rows ordered from the farthest to the nearest of every query: every tile survives the screen and the candidate runs are
    compacted over and over"""
    d, n = 128, 20011
    g = vs.ExactGen(d, seed=45)
    rows = g.rows(n)
    q0 = g.queries(1)
    q = g.band(np.concatenate([q0 * np.float32(2.0 ** s) for s in range(-6, 10)]), 2.0 ** -8)  # one direction, several norms
    order = np.argsort(-vs.r1_distances(rows, q0)[0], kind="stable")
    rows = rows[order]
    docids = g.rng.permutation(n).astype(np.uint32)
    ix.set_embeddings(rows, docids)
    for sms in (None, 8):
        _exact(ix, monkeypatch, rows, docids, q, k, ("wgmma",), sms=sms, ctx=("increasing", k))
    _exact(ix, monkeypatch, rows, docids, q[:2], k, ("gemv",), ctx=("increasing", k))


@pytest.mark.parametrize("k", [8, 64, 128])
def test_ties_at_the_reject_bound(ix, img, monkeypatch, k):
    """50 distinct rows, each repeated about 400 times (exact copies and copies scaled by 2^k) under permuted docids: the k-th
    distance of every query sits inside a run of exact ties, and the threshold the screen rejects against equals it"""
    d, n = 128, 20011
    g = vs.ExactGen(d, seed=46 + k)
    base = g.rows(50)
    rows = base[g.rng.integers(0, 50, n)]
    sc = g.rng.random(n) < 0.5
    rows[sc] = g.scaled(rows[sc], 2.0 ** -14)
    docids = g.rng.permutation(n).astype(np.uint32)
    ix.set_embeddings(rows, docids)
    q = g.queries(17)
    for sms in (None, 33):
        _exact(ix, monkeypatch, rows, docids, q, k, ("wgmma", "gemv"), sms=sms, ctx=("reject bound", k))
    _exact(ix, monkeypatch, rows, docids, q[:4], k, ("gemv",), ctx=("reject bound", k))


# ------------------------------------------------------------------------------------------------ filters, staging, empty store
def test_filters(ix, img, monkeypatch):
    """an empty bitmap, a single bit, a bitmap shorter than the largest docid, docids at or past n_docs"""
    d, n = 128, 5000
    g = vs.ExactGen(d, seed=47)
    rows = g.mixed_rows(n)
    docids = g.docids(n, img.n_docs, beyond=0.2)
    ix.set_embeddings(rows, docids)
    q = g.mixed_queries(16, rows)
    top = int(docids.max())
    filters = {
        "empty": np.zeros((top >> 6) + 1, np.uint64),
        "single": vs.bitmap([int(docids[1234])], (top >> 6) + 1),
        "short": vs.bitmap(np.nonzero(g.rng.random(top // 2) < 0.5)[0], (top // 2 >> 6) + 1),
        "beyond n_docs": vs.bitmap(docids[docids >= img.n_docs], (top >> 6) + 1),
    }
    for name, cand in filters.items():
        for k in (1, 9, 128):
            want = _exact(ix, monkeypatch, rows, docids, q, k, ("wgmma", "gemv"), cand, ctx=(name, k))
            if name == "empty":
                assert (want[2] == 0).all()
            if name == "single":
                assert (want[2] == min(k, int((docids == docids[1234]).sum()))).all()
        _exact(ix, monkeypatch, rows, docids, q[:3], 300, ("gemv",), cand, ctx=(name, 300))


@pytest.mark.parametrize("d", [64, 100, 768])
def test_f32_and_f16_staging_agree(ix, img, monkeypatch, d):
    """rows staged from f32 (converted on the device) and as fp16 give identical results; d = 100 is padded to 104"""
    g = vs.ExactGen(d, seed=48 + d)
    n = 3001
    rows = g.mixed_rows(n)
    docids = g.docids(n, img.n_docs)
    q = g.mixed_queries(16, rows)
    paths = ("gemv",) if d % 64 else ("wgmma", "gemv")
    for staged in (rows, rows.astype(np.float16)):
        ix.set_embeddings(staged, docids)
        for k in (5, 100):
            _exact(ix, monkeypatch, rows, docids, q, k, paths, ctx=("staging", staged.dtype, k))


@pytest.mark.parametrize("d", [64, 100])
def test_empty_store(ix, img, monkeypatch, d):
    ix.set_embeddings(np.zeros((0, d), np.float32), np.zeros(0, np.uint32))
    g = vs.ExactGen(d, seed=49)
    for nq in (1, 16, 70):
        q = g.queries(nq)
        for force in (None, "0", "1"):
            if force is None:
                monkeypatch.delenv("B200_VEC_GEMM", raising=False)
            else:
                monkeypatch.setenv("B200_VEC_GEMM", force)
            ids, dist, cnt = ix.nns_by_vector(q, 10)
            assert (cnt == 0).all(), (nq, force)
            ids, dist, cnt = ix.nns_by_vector(q, 10, np.full(4, ~np.uint64(0)))
            assert (cnt == 0).all(), (nq, force, "filtered")


# ------------------------------------------------------------------------------------------------ float64 certificates
@pytest.mark.parametrize("d", [128, 768, 1536])
@pytest.mark.parametrize("norms", ["unit", "random"])
def test_r2_certificates(ix, img, monkeypatch, d, norms):
    rng = np.random.default_rng(d + len(norms))
    n, k = 20011, 100
    rows = rng.standard_normal((n, d)).astype(np.float32)
    q = rng.standard_normal((16, d)).astype(np.float32)
    if norms == "unit":
        rows /= np.linalg.norm(rows, axis=1, keepdims=True)
        q /= np.linalg.norm(q, axis=1, keepdims=True)
    else:
        rows *= np.exp2(rng.uniform(-6, 6, (n, 1))).astype(np.float32)
        q *= np.exp2(rng.uniform(-6, 6, (16, 1))).astype(np.float32)
    docids = rng.permutation(n).astype(np.uint32)
    ix.set_embeddings(rows, docids)
    cand = vs.bitmap(np.nonzero(rng.random(n) < 0.3)[0], (n + 63) // 64)
    for path in ("gemv", "wgmma") if d <= 768 else ("gemv",):
        r2 = vs.r2_distances(rows, q, path)
        for cw in (None, cand):
            ids, dist, cnt = _nns(ix, monkeypatch, path, q, k, cw)[0]
            vs.check_certificate(ids, dist, cnt, docids, r2, k, d, cw, ctx=(d, norms, path))


# ------------------------------------------------------------------------------------------------ through the search path
def test_semantic_search_zero_vector(mb, img, monkeypatch):
    """a semantic search with a zero vector: every embedded document is at distance 0, so the hits are the smallest embedded
    docids (more of them than the selection's tie buffer holds)"""
    from oracle.pyoracle import OracleIndex

    monkeypatch.delenv("B200_VEC_GEMM", raising=False)
    d = 64
    g = vs.ExactGen(d, seed=50)
    n = 2500
    docids = g.rng.permutation(img.n_docs)[:n].astype(np.uint32)
    rows = g.mixed_rows(n)
    ix, o = mb.Index(img), OracleIndex(img)
    ix.set_embeddings(rows, docids)
    o.set_embeddings(rows, docids)
    vec = np.zeros((1, d), np.float32)
    got = ix.search().semantic(vec).limit(20).execute()
    want = o.search_batch(mb.TokenBatch([""]), vectors=vec, vector_only=True, limit=20)
    assert got.ids(0) == want.ids(0) == sorted(docids.tolist())[:20]
