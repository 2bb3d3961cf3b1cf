"""GPU: `Index.similar` (b200_similar_batch, Similar::execute) against the reference's known answers, against `nns_by_vector` on the
f32 copy of the target's row (bit for bit, both scan paths), and against the specification of tests/similar_spec.py (R1 bit for bit on
exact-arithmetic stores, 1e-4 on Gaussian ones) across universes, filters, offsets, thresholds, distributions, ties and the stores
the route refuses.

The known answers come from float32 vectors, the device holds them as fp16.  Every component of the golden vectors is a normal fp16
number, so rounding moves each by at most u = 2^-11 of itself and each vector v by at most u |v|, i.e. by an angle of at most
asin(u).  The cosine is 1-Lipschitz in the angle, so it moves by at most 2 asin(u) and the score (1 + cos) / 2 by at most asin(u);
the device's f32 arithmetic adds at most vs.tol(d) (tests/vec_spec.py).  SCORE_BOUND is their sum, about 5e-4 at d = 3."""
import math

import numpy as np
import pytest

import meilisearch_b200 as mb
from corpus.facets import FacetImage
from corpus.pyindexgen import IndexImage
from tests import similar_spec as ss
from tests import vec_spec as vs
from tests.filter_fixtures import geo_spec, synthetic_docs
from tests.filter_spec import FilterError, FilterSpec
from tests.test_similar_goldens import load, request

pytestmark = pytest.mark.gpu

SCORE_BOUND = math.asin(2.0 ** -11) + vs.tol(3)
N_DOCS = 3000
HOLES = set(range(5, N_DOCS, 97))  # docids outside documents_ids


def staged(rows):
    """the f32 values the device holds for f32 rows (fp16 rows)"""
    return np.asarray(rows, np.float32).astype(np.float16).astype(np.float32)


@pytest.fixture(scope="module")
def gold():
    g = load()
    img, fac = IndexImage(1), FacetImage()
    for d, doc in enumerate(g["documents"]):
        img.add_text(d, 0, "")
        fac.add_json(d, "release_year", doc["release_year"])
    fac.fid("release_year")
    img = img.build()
    fac.build()
    ix = mb.Index(img, facets=fac)
    rows = np.asarray([d["vector"] for d in g["documents"]], np.float32)
    assert np.abs(rows).min() >= 2.0 ** -14  # normal in fp16
    ix.set_embeddings(rows)
    return g, ix, rows


def test_goldens_through_the_abi(gold):
    g, ix, rows = gold
    ext = [d["id"] for d in g["documents"]]
    for c in g["cases"]:
        target, u, offset, limit, thr = request(g, c)
        flt = c["request"].get("filter")
        res = ix.similar([target], offset=offset, limit=limit, filter=flt, ranking_score_threshold=thr)
        assert res.status[0] == 0, (c, ix.last_error())
        assert [ext[h] for h in res.ids(0)] == c["hits"], c
        got = [s[0][1] for s in res.scores(0)]
        assert all(s[0][0] == "vector" for s in res.scores(0))
        if c["scores"] is not None:
            assert np.allclose(got, c["scores"], rtol=0, atol=SCORE_BOUND), (c, got)
        if c["estimatedTotalHits"] is not None:
            assert int(res.n_candidates[0]) == c["estimatedTotalHits"], c
        if thr is not None:  # no score can cross the threshold within the bound
            _, want, _ = ss.similar(rows, np.arange(len(rows)), target, u, limit=len(rows), distance=ss.f64)
            assert all(abs(float(s) - thr) > SCORE_BOUND for s in want), (c, want)


# ------------------------------------------------------------------------------------------------ the filter-capable store
@pytest.fixture(scope="module")
def fx():
    docs = synthetic_docs(N_DOCS)
    img, fac = IndexImage(1), FacetImage()
    for d, doc in enumerate(docs):
        if d in HOLES:
            continue
        img.add_text(d, 0, "")
        for k, v in doc.items():
            fac.add_json(d, k, v)
    for f in ("n", "s", "m", "flag"):
        fac.fid(f)
    fac.add_synthetic_geo(N_DOCS)
    img = img.build()
    fac.build()
    fac.build_presence()
    assert img.n_docs == N_DOCS
    docs_ids = sorted(set(range(N_DOCS)) - HOLES)
    spec = FilterSpec(fac, docs_ids, geo_spec(fac, N_DOCS))
    return mb.Index(img, facets=fac), spec, docs_ids


def stage(ix, rows, docids, distribution=None):
    ix.set_embeddings(rows, docids, distribution)
    if distribution is None:
        ix._ck(ix._l.b200_stage_distribution(ix._h, 0, 0.0, 0.0))


def set_path(monkeypatch, path):
    monkeypatch.setenv("B200_VEC_GEMM", "1" if path == "wgmma" else "0")


def check_spec(res, rows, docids, targets, universes, *, offset, limit, threshold=None, distribution=None, distance=ss.r1, tol=None,
               status=None, documents_ids=None):
    """every query against the specification: ids, counts and statuses exactly; scores bit for bit (tol None) or within tol"""
    for q, t in enumerate(targets):
        want_status = 0 if status is None else status[q]
        assert res.status[q] == want_status, (q, t, res.status[q])
        if want_status:
            assert res.n_hits[q] == 0
            continue
        ids, scores, n_cand = ss.similar(rows, docids, t, universes[q], offset=offset, limit=limit, threshold=threshold,
                                         distribution=distribution, distance=distance, documents_ids=documents_ids)
        got = res.ids(q)
        sims = res.score_sim[q, : len(got), 0]
        assert int(res.n_candidates[q]) == n_cand, (q, t, int(res.n_candidates[q]), n_cand)
        if tol is None:
            assert got == ids, (q, t, got[:8], ids[:8])
            assert np.array_equal(sims.view(np.uint32), np.asarray(scores, np.float32).view(np.uint32)), (q, t, sims[:8], scores[:8])
        else:
            assert len(got) == len(ids), (q, t)
            assert np.allclose(sims, np.asarray(scores, np.float64), rtol=0, atol=tol), (q, t)
            full = dict(zip(*ss.similar(rows, docids, t, universes[q], limit=len(rows), distance=distance)[:2]))
            for i, (a, b) in enumerate(zip(got, ids)):  # a swap is allowed only between documents the spec scores within tol
                assert a == b or abs(float(full[a]) - float(full[b])) <= tol, (q, t, i, a, b)


def exact_store(d, n, seed):
    """ExactGen rows that are also valid queries (every row is some query's target): normal rows in the query norm band, with
    exact duplicates, scaled copies, zero rows and tiny rows mixed in"""
    g = vs.ExactGen(d, seed)
    x = g.queries(n)
    kinds, src = g.rng.random(n), g.rng.integers(0, max(n, 1), n)
    dup, scaled = kinds < 0.1, (kinds >= 0.1) & (kinds < 0.15)
    x[dup] = x[src[dup]]
    x[scaled] = g.scaled(x[src[scaled]], 2.0 ** -8)
    x[(kinds >= 0.15) & (kinds < 0.17)] = 0
    tiny = (kinds >= 0.17) & (kinds < 0.19)
    x[tiny] = g.tiny(int(tiny.sum()))
    assert vs.rule_margin_ok(x, x)
    return x


# ------------------------------------------------------------------------------------------------ bit-exact equivalence with nns
@pytest.mark.parametrize("n_targets", [1, 15, 16, 64, 1024])
@pytest.mark.parametrize("path", ["gemv", "wgmma"])
@pytest.mark.parametrize("data", ["exact", "gauss"])
@pytest.mark.parametrize("d", [64, 61])
def test_similar_is_nns_of_the_row_copy(fx, monkeypatch, n_targets, path, data, d):
    ix, spec, docs_ids = fx
    n = N_DOCS
    rows = exact_store(d, n, 11 + d) if data == "exact" else np.random.default_rng(d).standard_normal((n, d)).astype(np.float32)
    stage(ix, rows, np.arange(n, dtype=np.uint32))
    rng = np.random.default_rng(n_targets)
    targets = rng.choice(docs_ids, n_targets, replace=False).astype(np.uint32)
    offset, limit = 3, 10
    picked = rng.choice(N_DOCS, N_DOCS // 2, replace=False) if n_targets == 64 else np.arange(N_DOCS)
    uni = vs.bitmap(picked, (N_DOCS + 63) // 64) if n_targets == 64 else None
    u = vs.bitmap(sorted(set(picked.tolist()) & set(docs_ids)), (N_DOCS + 63) // 64)  # U: within documents_ids
    set_path(monkeypatch, path)
    ix.reset_stats()
    res = ix.similar(targets, offset=offset, limit=limit, universes=uni)
    kern = ix.stats()["kernels"]
    if path == "wgmma":  # d = 61 is padded to 64 at staging, which the batched kernel takes
        assert kern["vec_gemm_topk"]["count"] > 0
    else:
        assert kern["vec_gemm_topk"]["count"] == 0 and kern["vec_dist"]["count"] > 0
    k = offset + limit + 2
    ids, dist, cnt = ix.nns_by_vector(staged(rows)[targets], k, u)
    for q, t in enumerate(targets):
        keep = [(int(i), dd) for i, dd in zip(ids[q, : cnt[q]], dist[q, : cnt[q]]) if i != t][: offset + limit + 1]
        want = keep[offset: offset + limit]
        assert res.status[q] == 0
        assert res.ids(q) == [i for i, _ in want], (q, int(t))
        want_sim = np.float32(1) - np.asarray([dd for _, dd in want], np.float32)
        assert np.array_equal(res.score_sim[q, : len(want), 0].view(np.uint32), want_sim.view(np.uint32)), q


# ------------------------------------------------------------------------------------------------ against the specification
def test_universes_filters_and_failing_leaves(fx, monkeypatch):
    ix, spec, docs_ids = fx
    rows = exact_store(64, N_DOCS, 5)
    docids = np.arange(N_DOCS, dtype=np.uint32)
    stage(ix, rows, docids)
    rng = np.random.default_rng(3)
    shared = vs.bitmap(rng.choice(N_DOCS, 2000, replace=False), (N_DOCS + 63) // 64)
    other = vs.bitmap(rng.choice(N_DOCS, 500, replace=False), (N_DOCS + 63) // 64)
    geo = ("or", [("geo", "radius", ["48.85", "2.35", "300000.0"]), ("cond", "n", ">", ["3"])])
    failing = ("and", [("cond", "n", "=", ["1.0"]), ("geo", "radius", ["91", "0", "10"])])
    own_out = ("cond", "flag", "=", ["true"])
    targets, unis, filters = [], [], []
    for i in range(40):
        t = int(rng.choice(docs_ids))
        kind = i % 5
        targets.append(t)
        unis.append(shared if kind in (0, 1) else (other if kind == 2 else None))
        filters.append([None, geo, failing, own_out, "s = apple OR m EXISTS"][kind])
    # a target outside its own filter: a flag-less or false-flag document filtered on flag = true
    outside = [d for d in docs_ids if d not in spec.evaluate(own_out)]
    targets[3] = outside[0]
    want_u, status, leaves = [], [], []
    for t, u, f in zip(targets, unis, filters):
        base = set(docs_ids) if u is None else set(np.nonzero(np.unpackbits(u.view(np.uint8), bitorder="little"))[0]) & set(docs_ids)
        try:
            base &= set(spec.evaluate(f)) if f is not None else base
            status.append(0)
            leaves.append(-1)
        except FilterError as e:
            status.append(-3)
            leaves.append(e.leaf)
        want_u.append(base)
    assert -3 in status and 0 in status
    for path in ("gemv", "wgmma"):
        set_path(monkeypatch, path)
        for n in (40, 16):  # both scan paths over the same groups
            res = ix.similar(targets[:n], offset=2, limit=7, universes=unis[:n], filter=filters[:n])
            check_spec(res, staged(rows), docids, targets[:n], want_u[:n], offset=2, limit=7, status=status[:n])
            assert list(res.filter_error_leaf[:n]) == leaves[:n]


@pytest.mark.parametrize("path", ["gemv", "wgmma"])
def test_offsets_limits_and_thresholds(fx, monkeypatch, path):
    ix, spec, docs_ids = fx
    rows = exact_store(64, N_DOCS, 9)
    docids = np.arange(N_DOCS, dtype=np.uint32)
    stage(ix, rows, docids)
    set_path(monkeypatch, path)
    targets = [int(x) for x in np.random.default_rng(1).choice(docs_ids, 16, replace=False)]
    U = [set(docs_ids)] * len(targets)
    for offset, limit in ((0, 20), (5, 0), (0, 0), (N_DOCS, 5), (len(docs_ids) - 3, 10), (40, 60)):
        res = ix.similar(targets, offset=offset, limit=limit)
        check_spec(res, staged(rows), docids, targets, U, offset=offset, limit=limit)
    # thresholds cutting before, at and after the offset, and one equal to a score (kept): from target 0's own scores
    _, s, _ = ss.similar(staged(rows), docids, targets[0], U[0], limit=30)
    for offset, thr in ((0, float(s[0]) + 1e-3), (5, float(s[5])), (5, float(s[4])), (5, float(s[12])), (0, float(s[9])),
                        (3, float(s[20]) - 1e-7), (0, 0.0), (0, 1.0)):
        res = ix.similar(targets, offset=offset, limit=10, ranking_score_threshold=thr)
        check_spec(res, staged(rows), docids, targets, U, offset=offset, limit=10, threshold=thr)
    # a staged distribution shifts the scores, and the threshold applies to the shifted ones
    stage(ix, rows, docids, distribution=(0.6, 0.1))
    for thr in (None, 0.5):
        res = ix.similar(targets, offset=1, limit=10, ranking_score_threshold=thr)
        check_spec(res, staged(rows), docids, targets, U, offset=1, limit=10, threshold=thr, distribution=(0.6, 0.1))


@pytest.mark.parametrize("path", ["gemv", "wgmma"])
def test_ties_zero_vectors_and_absent_targets(fx, monkeypatch, path):
    ix, spec, docs_ids = fx
    rows = exact_store(64, N_DOCS, 13)
    rows[100:1300] = rows[2000]  # 1201 rows tied with target 2000 at distance 0
    rows[2500] = 0  # a zero target: every distance 0, smallest docids first
    n_rows = N_DOCS - 50  # the last 50 documents have no row
    docids = np.arange(n_rows, dtype=np.uint32)
    stage(ix, rows[:n_rows], docids)
    set_path(monkeypatch, path)
    hole = min(HOLES)
    targets = [2000, 700, 2500, N_DOCS - 10, hole, N_DOCS + 5, 10 ** 9, 0, 1, 2, 3, 4, 6, 7, 8, 9]
    U = [set(docs_ids)] * len(targets)
    for offset, limit in ((0, 20), (1190, 20), (3, 5)):
        res = ix.similar(targets, offset=offset, limit=limit)
        check_spec(res, staged(rows[:n_rows]), docids, targets, U, offset=offset, limit=limit, documents_ids=set(docs_ids))
    res = ix.similar(targets, limit=5)
    assert res.ids(2) == [d for d in docs_ids if d != 2500][:5]  # the zero target ties with everything
    for q in (3, 4, 5, 6):  # unembedded, outside documents_ids, beyond the range: no hits, status 0
        assert res.status[q] == 0 and res.n_hits[q] == 0
    assert int(res.n_candidates[3]) == len(docs_ids) - 1 and int(res.n_candidates[4]) == len(docs_ids)


def test_small_multi_row_and_gaussian_stores(fx, monkeypatch):
    ix, spec, docs_ids = fx
    monkeypatch.delenv("B200_VEC_GEMM", raising=False)
    rows = exact_store(64, 4, 17)
    # one row, then an empty store
    stage(ix, rows[:1], np.asarray([7], np.uint32))
    res = ix.similar([7, 8])
    assert list(res.n_hits) == [0, 0] and list(res.status) == [0, 0]
    assert list(res.n_candidates) == [len(docs_ids) - 1, len(docs_ids) - 1]
    stage(ix, rows[:0], np.zeros(0, np.uint32))
    res = ix.similar([7])
    assert res.n_hits[0] == 0 and res.status[0] == 0 and int(res.n_candidates[0]) == len(docs_ids) - 1
    # a document with two rows: every query is refused alone
    stage(ix, rows, np.asarray([1, 2, 1, 3], np.uint32))
    res = ix.similar([1, 2, 3, 4], limit=3)
    assert list(res.status) == [-4] * 4 and list(res.n_hits) == [0] * 4
    # Gaussian data against the float64 specification
    g = np.random.default_rng(23).standard_normal((N_DOCS, 48)).astype(np.float32)
    docids = np.arange(N_DOCS, dtype=np.uint32)
    stage(ix, g, docids)
    targets = [int(x) for x in np.random.default_rng(2).choice(docs_ids, 20, replace=False)]
    for path in ("gemv", "wgmma"):
        set_path(monkeypatch, path)
        res = ix.similar(targets, offset=2, limit=15)
        check_spec(res, staged(g), docids, targets, [set(docs_ids)] * 20, offset=2, limit=15, distance=ss.f64, tol=1e-4)


def test_no_query_vector_crosses_pcie(fx, monkeypatch):
    ix, spec, docs_ids = fx
    d = 64
    rows = exact_store(d, N_DOCS, 19)
    stage(ix, rows, np.arange(N_DOCS, dtype=np.uint32))
    targets = np.asarray(docs_ids[:64], np.uint32)
    for path in ("gemv", "wgmma"):
        set_path(monkeypatch, path)
        ix.reset_stats()
        ix.similar(targets, limit=10)
        sim = ix.stats()["h2d_bytes"]
        ix.reset_stats()
        ix.nns_by_vector(staged(rows)[targets], 12)
        nns = ix.stats()["h2d_bytes"]
        assert sim == 4 * len(targets), (path, sim)  # the row indices only
        assert nns >= len(targets) * d * 4, (path, nns)


def test_call_errors(fx):
    ix, spec, docs_ids = fx
    stage(ix, exact_store(64, 10, 3), np.arange(10, dtype=np.uint32))
    short = np.zeros(2, np.uint64)
    with pytest.raises(mb.B200Error) as e:
        ix.similar([1], universes=[short])
    assert e.value.code == -3
    rq = mb._SimilarRequest(1, None, 0, 5)
    res = mb.SearchResult(1, 5)
    r = mb._Results(mb._p(res.documents_ids), mb._p(res.n_hits))
    assert ix._l.b200_similar_batch(ix._h, mb.C.byref(rq), mb.C.byref(r)) == -3  # NULL docids
    t = np.asarray([1], np.uint32)
    rq.docids = mb._p(t)
    cand = np.zeros((1, (N_DOCS + 63) // 64), np.uint64)
    r.candidates, r.candidates_words = mb._p(cand), cand.shape[1]
    assert ix._l.b200_similar_batch(ix._h, mb.C.byref(rq), mb.C.byref(r)) == -4  # the candidates bitmap
    img = IndexImage(1)
    img.add_text(0, 0, "")
    bare = mb.Index(img.build())
    with pytest.raises(mb.B200Error) as e:
        bare.similar([0])
    assert e.value.code == -6  # no embeddings staged
