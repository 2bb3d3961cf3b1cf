"""GPU: the GeoSort rule of placeholder searches (geo.cu, then sort.cu for the following rules) against the reference's known
answers under every strategy and against the CPU specification (tests/geo_spec.py): docids, score tuples, candidate counts."""
import numpy as np
import pytest

import meilisearch_b200 as mb
from tests.geo_fixtures import STRATEGIES, doc_images, load_geo_goldens, spec_state, synthetic_geo_images
from tests.geo_spec import placeholder_search, sort_rules
from tests.sort_spec import universe_docs

pytestmark = pytest.mark.gpu

CRITERIA = ["words", "typo", "proximity", "attributeRank", "sort", "wordPosition", "exactness"]


@pytest.mark.parametrize("strategy,cache", STRATEGIES)
def test_geo_goldens_on_gpu(strategy, cache):
    g = load_geo_goldens()
    for t in g["tests"]:
        img, fac = doc_images(t["docs"])
        ix = mb.Index(img, criteria=g["criteria"], facets=fac)
        for c in t["cases"]:
            r = ix.search().query([""]).sort(c["sort"]).scoring_strategy("detailed").geo_strategy(strategy, cache).execute()
            assert r.status[0] == 0
            assert r.ids(0) == c["ids"], (t["name"], c["sort"])
            assert [list(s[0][2]) if s[0][2] is not None else None for s in r.scores(0)] == c["geo_values"], (t["name"], c["sort"])
            assert r.n_candidates[0] == len(t["docs"])


def test_geo_max_bucket_size_goldens():
    g = load_geo_goldens()
    m = g["max_bucket"]
    img, fac = doc_images(m["docs"])
    ext = [d["id"] for d in m["docs"]]
    ix = mb.Index(img, criteria=g["criteria"], facets=fac)
    for strategy, cache in m["strategies"]:
        r = ix.search().query([""]).sort(m["sort"]).geo_strategy(strategy, cache).geo_max_bucket_size(m["max_bucket_size"]).execute()
        ids = [ext[d] for d in r.ids(0)]
        assert len(ids) == 15 and ids[10:] == m["no_geo_ids"]
        assert all(6 <= x <= 11 for x in ids[:6]) and all(12 <= x <= 15 for x in ids[6:10])


@pytest.fixture(scope="module")
def syn():
    img, fac = synthetic_geo_images(40000)
    dbs, gix = spec_state(fac)
    return img, fac, dbs, gix


def check(ix, img, fac, dbs, gix, sorts, *, offset=0, limit=20, scoring="detailed", universes=None, strategy=("dynamic", 1000),
          max_bucket=1000, criteria=CRITERIA):
    n = len(sorts)
    s = ix.search().query([""] * n).sort(sorts).offset(offset).limit(limit).scoring_strategy(scoring)
    s = s.geo_strategy(*strategy).geo_max_bucket_size(max_bucket)
    if universes is not None:
        s = s.universes(universes)
    r = s.execute()
    for q in range(n):
        assert r.status[q] == 0, (q, sorts[q])
        u = universe_docs(img.n_docs, None if universes is None else universes[q])
        want_ids, want_sc = placeholder_search(dbs, gix, sort_rules(criteria, sorts[q], fac.fields), u, offset, limit, scoring,
                                               strategy[0], strategy[1], max_bucket)
        assert r.ids(q) == want_ids, (q, sorts[q], offset, limit, scoring, strategy)
        assert r.scores(q) == want_sc, (q, sorts[q], offset, limit, scoring, strategy)
        assert int(r.n_candidates[q]) == len(u)
    return r


SORTS = [["_geoPoint(48.85, 2.35):asc"], ["_geoPoint(48.85, 2.35):desc"], ["_geoPoint(10.0, 20.0):asc", "price:asc"],
         ["_geoPoint(0.0, 180.0):desc", "brand:desc", "price:asc"], ["_geoPoint(45.0, 7.0):asc", "tags:asc"],
         ["_geoPoint(-48.85, -177.65):asc"]]


@pytest.mark.parametrize("scoring", ["detailed", "skip"])
def test_geo_parity(syn, scoring):
    img, fac, dbs, gix = syn
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    for off, lim in ((0, 20), (7, 33), (980, 20), (0, 0), (3000, 100)):
        check(ix, img, fac, dbs, gix, SORTS, offset=off, limit=lim, scoring=scoring)


@pytest.mark.parametrize("strategy", [("iterative", 1000), ("rtree", 1000), ("dynamic", 300), ("rtree", 2)])
def test_geo_strategies(syn, strategy):
    img, fac, dbs, gix = syn
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    check(ix, img, fac, dbs, gix, SORTS[:4], offset=7, limit=40, strategy=strategy)


def _bitmap(n_docs, docs):
    w = np.zeros((n_docs + 63) // 64, np.uint64)
    for d in docs:
        w[d >> 6] |= np.uint64(1) << np.uint64(d & 63)
    return w


def test_geo_universe_sizes(syn):
    # 0, 1, 999, 1000, 1001 and 2500 geo documents: under Dynamic(1000) the last n mod 1000 come in iterative order
    img, fac, dbs, gix = syn
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    rng = np.random.default_rng(3)
    geo = np.array(sorted(gix.points))
    non = np.array(sorted(set(range(img.n_docs)) - set(gix.points)))
    us = []
    for k in (0, 1, 999, 1000, 1001, 2500):
        docs = list(rng.choice(geo, k, replace=False)) + list(rng.choice(non, 50, replace=False))
        us.append(_bitmap(img.n_docs, docs))
    sort = ["_geoPoint(48.85, 2.35):desc", "price:asc"]
    for off, lim in ((0, 20), (980, 40), (2480, 60)):
        for scoring in ("skip", "detailed"):
            check(ix, img, fac, dbs, gix, [sort] * len(us), universes=us, offset=off, limit=lim, scoring=scoring)


def test_geo_max_bucket_sizes():
    # 5000 identical points: buckets of 2, of 1000, or one of 5000
    from tests.geo_fixtures import doc_images as mk

    docs = [{"id": i, "_geo": {"lat": 1.0, "lng": 2.0}, "score": i % 7} for i in range(5000)] + [{"id": 5000 + i} for i in range(30)]
    img, fac = mk(docs)
    dbs, gix = spec_state(fac)
    ix = mb.Index(img, criteria=["sort"], facets=fac)
    for cap in (2, 1000, 10**9):
        for off, lim in ((0, 20), (990, 30), (4990, 30)):
            check(ix, img, fac, dbs, gix, [["_geoPoint(0.0, 0.0):asc", "score:desc"]], offset=off, limit=lim, max_bucket=cap,
                  criteria=["sort"])


def test_geo_errors_per_query(syn):
    img, fac, dbs, gix = syn
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    r = ix.search().query(["", "", ""]).sort([["price:asc", "_geoPoint(1.0, 2.0):asc"], ["_geoPoint(1.0, 2.0):asc", "_geoPoint(3.0, 4.0):asc"],
                                              ["_geoPoint(1.0, 2.0):asc"]]).execute()
    assert list(r.status) == [-4, -4, 0]  # GeoSort after the first rule
    ix2 = mb.Index(img, criteria=["words", "asc:price", "sort"], facets=fac)
    r = ix2.search().query([""]).sort(["_geoPoint(1.0, 2.0):asc"]).execute()
    assert r.status[0] == -4  # after a field rule from the criteria
    q = img.synthetic_queries(1, seed=3)
    r = ix.search().query([q[0], ""]).sort(["_geoPoint(1.0, 2.0):asc"]).execute()
    assert r.status[0] == -4 and r.status[1] == 0  # with query terms
    r = ix.search().query([""]).sort(["_geoPoint(1.0, 2.0):asc"]).deadline(stop_after=2).execute()
    assert r.status[0] == -4
    r = ix.search().query(["", ""]).sort([["_geoPoint(1.0, 2.0):asc"], []]).execute_hybrid(0.5)
    assert r.status[0] == -4 and r.status[1] == 0
    many = ["_geoPoint(1.0, 2.0):asc"] + [f"f{i}:asc" for i in range(12)]
    r = ix.search().query([""]).sort(many).execute()
    assert r.status[0] == -4
    emb = np.random.default_rng(0).standard_normal((img.n_docs, 16)).astype(np.float32)
    ix.set_embeddings(emb)
    qv = np.random.default_rng(1).standard_normal((2, 16)).astype(np.float32)
    r = ix.search().semantic(qv).sort([["_geoPoint(1.0, 2.0):asc"], []]).execute()
    assert r.status[0] == -4 and r.status[1] == 0 and r.n_hits[1] == 20


def test_geo_time_budget(syn):
    img, fac, dbs, gix = syn
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    sort = ["_geoPoint(48.85, 2.35):asc"]
    r = check(ix, img, fac, dbs, gix, [sort] * 2)
    assert not any(r.degraded)
    r = ix.search().query([""]).sort(sort).scoring_strategy("detailed").deadline(budget_ms=1e-6).execute()
    assert r.status[0] == 0 and r.degraded[0] and r.ids(0) == list(range(20))
    assert r.scores(0)[0] == [("skipped", 0, 1)]


def test_geo_without_geo_fields(syn):
    # no geo fields staged: every document is in the Null bucket
    img, fac, dbs, gix = syn
    ix = mb.Index(img, criteria=CRITERIA, facets=fac, geo=(0xFFFF, 0xFFFF))
    r = ix.search().query([""]).sort(["_geoPoint(1.0, 2.0):asc", "price:asc"]).scoring_strategy("detailed").execute()
    assert r.status[0] == 0 and all(s[0] == ("geo", True, None) for s in r.scores(0))


def test_geo_large_corpus():
    img, fac = synthetic_geo_images(700_000, vocab=20000, with_geo=0.3)
    dbs, gix = spec_state(fac)
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    check(ix, img, fac, dbs, gix, [["_geoPoint(48.85, 2.35):asc"], ["_geoPoint(35.68, 139.69):desc"]], offset=1500, limit=300)
    check(ix, img, fac, dbs, gix, [["_geoPoint(0.0, 180.0):asc", "price:asc"]], offset=0, limit=20)
    assert ix.stats()["kernels"]["geo"]["count"] >= 2
