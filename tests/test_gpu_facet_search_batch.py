"""GPU: facet search inside b200_search_batch (b200_query_batch::facet_search_*), over each query's own candidates, against the CPU
specification (tests/facet_search_spec.py): keyword searches (Skip / Detailed, every terms matching strategy), placeholder, filtered,
geo-filtered and degraded searches take the `candidates` bitmap; semantic and hybrid searches take the filtered universe."""
import numpy as np
import pytest

import meilisearch_b200 as mb
from tests.facet_search_spec import facet_search
from tests.test_gpu_facet_search import CRITERIA, EXACT, bitmap, docs_of, make

pytestmark = pytest.mark.gpu

GEO_FILTER = "_geoRadius(48.85, 2.35, 300000.0)"


@pytest.fixture(scope="module")
def env():
    img, fac = make(40_000)
    fac.add_synthetic_geo(img.n_docs)
    fac.build()
    fac.build_search()
    ix = mb.Index(img, criteria=CRITERIA, facets=fac, exact_words=EXACT)
    rng = np.random.default_rng(4)
    ix.set_embeddings(rng.standard_normal((img.n_docs, 16)).astype(np.float32))
    return img, fac, ix


REQUESTS = [("genre", "ad", "count", 3), ("genre", None, "alpha", 5), ("brand", "brnd01", "count", 10), ("model", "ab", "alpha", 100),
            ("genre", "", "count", 2), ("tags", "tag07", "alpha", 4)]


def check(fac, res, sets, name, query, order, mx):
    for q, docs in enumerate(sets):
        assert res.status[q] == 0, q
        want = facet_search(fac, fac.fields[name], docs, query, order=order, max_values=mx, exact_words=EXACT)
        assert res.facet_hits(q) == want, (q, name, query, order, mx, len(docs))


@pytest.mark.parametrize("scoring", ["skip", "detailed"])
@pytest.mark.parametrize("tms", ["last", "all", "frequency"])
def test_keyword_candidates(env, scoring, tms):
    img, fac, ix = env
    queries = img.synthetic_queries(8, seed=7)
    for name, query, order, mx in REQUESTS[:3]:
        res = (ix.search().query(queries).scoring_strategy(scoring).terms_matching_strategy(tms).with_candidates()
               .facet_search(name, query, order, mx).execute())
        plain = ix.search().query(queries).scoring_strategy(scoring).terms_matching_strategy(tms).execute()
        for q in range(len(queries)):
            assert res.ids(q) == plain.ids(q)
        check(fac, res, [docs_of(res.candidates[q], img.n_docs) for q in range(len(queries))], name, query, order, mx)


@pytest.mark.parametrize("kind", ["placeholder", "universes", "geofilter", "degraded"])
def test_other_keyword_candidates(env, kind):
    img, fac, ix = env
    n = 6
    rng = np.random.default_rng(8)
    s = ix.search().query([""] * n if kind != "degraded" else img.synthetic_queries(n, seed=9)).with_candidates()
    if kind == "universes":
        s = s.universes([bitmap(img.n_docs, rng.choice(img.n_docs, 5000, replace=False)) for _ in range(n)])
    if kind == "geofilter":
        s = s.geo_filter([GEO_FILTER])
    if kind == "degraded":
        s = s.deadline(stop_after=3)
    for name, query, order, mx in REQUESTS:
        res = s.facet_search(name, query, order, mx).execute()
        if kind == "degraded":
            assert any(res.degraded)
        check(fac, res, [docs_of(res.candidates[q], img.n_docs) for q in range(n)], name, query, order, mx)


@pytest.mark.parametrize("mode", ["semantic", "hybrid"])
def test_filtered_universe(env, mode):
    img, fac, ix = env
    n = 4
    rng = np.random.default_rng(10)
    qv = rng.standard_normal((n, 16)).astype(np.float32)
    us = [bitmap(img.n_docs, rng.choice(img.n_docs, 8000, replace=False)) for _ in range(n - 1)] + [None]
    geo, _ = ix.geo_filter([GEO_FILTER])
    for filt in ("universes", "geo"):
        s = ix.search().semantic(qv)
        if mode == "hybrid":
            s = s.query(img.synthetic_queries(n, seed=11))
        if filt == "universes":
            s = s.universes(us)
            sets = [docs_of(u, img.n_docs) if u is not None else list(range(img.n_docs)) for u in us]
        else:
            s = s.geo_filter([GEO_FILTER])
            sets = [docs_of(geo[0], img.n_docs)] * n
        for name, query, order, mx in REQUESTS[:4]:
            s = s.facet_search(name, query, order, mx)
            res = s.execute() if mode == "semantic" else s.execute_hybrid(0.5)
            check(fac, res, sets, name, query, order, mx)


def test_mixed_with_facets_and_per_query_fields(env):
    img, fac, ix = env
    queries = img.synthetic_queries(5, seed=12)
    names = ["genre", None, "brand", "model", "genre"]
    qs = ["adv", None, "brand00", None, "comedie"]
    res = ix.search().query(queries).with_candidates().facets(["brand", "price"]).facet_search(names, qs, "count", 3).execute()
    ref = ix.search().query(queries).with_candidates().facets(["brand", "price"]).execute()
    for q in range(len(queries)):
        assert res.status[q] == 0
        assert res.facet_distribution(q) == ref.facet_distribution(q)
        docs = docs_of(res.candidates[q], img.n_docs)
        want = [] if names[q] is None else facet_search(fac, fac.fields[names[q]], docs, qs[q], order="count", max_values=3, exact_words=EXACT)
        assert res.facet_hits(q) == want, q


def test_per_query_errors(env):
    img, fac, ix = env
    queries = img.synthetic_queries(3, seed=13)
    res = ix.search().query(queries).ranking_score_threshold(0.1).facet_search("genre", "ad").execute()
    assert list(res.status) == [-4, -4, -4]
    res = ix.search().query(queries).facet_search(["genre", None, "genre"], ["a" * 70, None, "ad"]).execute()
    assert list(res.status) == [-4, 0, 0]
    assert res.n_hits[0] == 0 and res.facet_hits(2)
