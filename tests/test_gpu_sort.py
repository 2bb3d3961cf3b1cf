"""GPU: the Sort rule of placeholder searches (sort_window_kernel) against the reference's known answers and against the CPU
specification (tests/sort_spec.py) on synthetic corpora with facet fields: docids, Sort score tuples, candidate counts."""
import numpy as np
import pytest

import meilisearch_b200 as mb
from tests.sort_fixtures import golden_images, load_sort_goldens, synthetic_images
from tests.sort_spec import FacetDbs, placeholder_search, sort_rules, universe_docs

pytestmark = pytest.mark.gpu

CRITERIA = ["words", "typo", "proximity", "attributeRank", "sort", "wordPosition", "exactness"]


def test_sort_goldens_on_gpu():
    g = load_sort_goldens()
    img, fac = golden_images(g)
    ix = mb.Index(img, criteria=g["criteria"], facets=fac)
    for c in g["cases"]:
        r = ix.search().query([""]).sort(c["sort"]).scoring_strategy("detailed").limit(g["limit"]).execute()
        assert r.status[0] == 0
        assert r.ids(0) == c["ids"], c["name"]
        if c["sort_values"] is not None:
            assert [s[0][3] for s in r.scores(0)] == c["sort_values"], c["name"]
        assert r.n_candidates[0] == len(g["docs"])


@pytest.fixture(scope="module")
def syn():
    img, fac = synthetic_images(40000)
    return img, fac, FacetDbs(fac.f64_db, fac.string_db)


def check(ix, img, fac, dbs, criteria, sorts, *, offset=0, limit=20, scoring="detailed", universes=None):
    n = len(sorts)
    s = ix.search().query([""] * n).sort(sorts).offset(offset).limit(limit).scoring_strategy(scoring)
    if universes is not None:
        s = s.universes(universes)
    r = s.execute()
    for q in range(n):
        assert r.status[q] == 0, (q, sorts[q])
        u = universe_docs(img.n_docs, None if universes is None else universes[q])
        want_ids, want_sc = placeholder_search(dbs, sort_rules(criteria, sorts[q], fac.fields), u, offset, limit, scoring)
        assert r.ids(q) == want_ids, (q, sorts[q], offset, limit, scoring)
        assert r.scores(q) == want_sc, (q, sorts[q], offset, limit, scoring)
        assert int(r.n_candidates[q]) == len(u)
    return r


SORTS = [["price:asc"], ["price:desc"], ["brand:asc"], ["brand:desc"], ["tags:asc"], ["tags:desc"], ["missing:asc"],
         ["brand:asc", "price:desc"], ["tags:desc", "brand:asc", "price:asc"], ["price:asc", "price:desc"], []]


@pytest.mark.parametrize("scoring", ["detailed", "skip"])
def test_sort_parity(syn, scoring):
    img, fac, dbs = syn
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    for off, lim in ((0, 20), (7, 33), (980, 20), (0, 0), (1500, 3000)):
        check(ix, img, fac, dbs, CRITERIA, SORTS, offset=off, limit=lim, scoring=scoring)


def test_sort_universes_and_custom_criteria(syn):
    img, fac, dbs = syn
    crit = ["words", "desc:price", "sort", "asc:brand", "exactness"]
    ix = mb.Index(img, criteria=crit, facets=fac)
    rng = np.random.default_rng(5)
    words = (img.n_docs + 63) // 64
    us = [rng.integers(0, 2**63, words, dtype=np.uint64) & rng.integers(0, 2**63, words, dtype=np.uint64) for _ in range(3)] + [None]
    sorts = [["price:asc", "tags:asc"], ["brand:desc"], [], ["tags:desc"]]
    check(ix, img, fac, dbs, crit, sorts, universes=us)
    check(ix, img, fac, dbs, crit, sorts, universes=us, scoring="skip", offset=5, limit=50)


def test_sort_errors_per_query(syn):
    img, fac, dbs = syn
    ix = mb.Index(img, criteria=["words", "typo"], facets=fac)
    r = ix.search().query(["", ""]).sort([["price:asc"], []]).execute()
    assert r.status[0] == -3 and r.status[1] == 0  # SortRankingRuleMissing
    assert r.ids(1) == list(range(20))
    ix2 = mb.Index(img, criteria=CRITERIA, facets=fac)
    r = ix2.search().query(["", ""]).sort([["price:asc"], []]).execute_hybrid(0.5)
    assert r.status[0] == -4 and r.status[1] == 0
    q = img.synthetic_queries(2, seed=3)
    r = ix2.search().query([q[0], ""]).sort([["price:asc"], ["price:asc"]]).execute()
    assert r.status[0] == -4 and r.status[1] == 0  # sort with query terms: not built
    r = ix2.search().query([""]).sort(["price:asc"]).deadline(stop_after=2).execute()
    assert r.status[0] == -4


def test_sort_time_budget(syn):
    img, fac, dbs = syn
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    r = ix.search().query([""] * 4).sort(["price:desc"]).scoring_strategy("detailed").deadline(budget_ms=60000).execute()
    want, _ = placeholder_search(dbs, sort_rules(CRITERIA, ["price:desc"], fac.fields), universe_docs(img.n_docs), 0, 20, "detailed")
    for q in range(4):
        assert r.status[q] == 0 and r.ids(q) == want and not r.degraded[q]
    r = ix.search().query([""]).sort(["price:desc"]).scoring_strategy("detailed").deadline(budget_ms=1e-6).execute()
    assert r.status[0] == 0 and r.degraded[0] and r.ids(0) == list(range(20))
    assert r.scores(0)[0] == [("skipped", 0, 1)]


def test_sort_large_corpus():
    img, fac = synthetic_images(700_000, vocab=20000)
    dbs = FacetDbs(fac.f64_db, fac.string_db)
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    check(ix, img, fac, dbs, CRITERIA, [["price:asc"], ["brand:desc", "price:asc"], ["tags:asc"]], offset=3000, limit=100)
    assert ix.stats()["kernels"]["sort"]["count"] >= 1


def _bitmap(n_docs, docs):
    w = np.zeros((n_docs + 63) // 64, np.uint64)
    for d in docs:
        w[d >> 6] |= np.uint64(1) << np.uint64(d & 63)
    return w


def test_sort_skip_small_universes(syn):
    # bucket_sort.rs:196-204 under Skip: a rule universe of one document (the whole universe, or the end of a group of equal keys)
    # returns it with the scores of the rules above
    img, fac, dbs = syn
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    rng = np.random.default_rng(11)
    docs = [[5], [3, 9], [0, 1, 2], sorted(rng.choice(img.n_docs, 40, replace=False).tolist()),
            sorted(rng.choice(img.n_docs, 300, replace=False).tolist())]
    us = [_bitmap(img.n_docs, d) for d in docs]
    for sort in (["price:asc"], ["tags:desc", "brand:asc", "price:asc"], ["brand:asc", "tags:asc"]):
        for off, lim in ((0, 20), (1, 7), (7, 33)):
            check(ix, img, fac, dbs, CRITERIA, [sort] * len(us), universes=us, scoring="skip", offset=off, limit=lim)
            check(ix, img, fac, dbs, CRITERIA, [sort] * len(us), universes=us, scoring="detailed", offset=off, limit=lim)


def test_sort_two_absent_fields(syn):
    # milli deduplicates sort fields by name: two different absent fields are two rules with a Null value each
    img, fac, dbs = syn
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    sorts = [["nope:asc", "price:desc", "other:asc", "nope:desc"]]
    r = check(ix, img, fac, dbs, CRITERIA, sorts)
    assert [x[1] for x in r.scores(0)[0]] == ["nope", "price", "other"]


def test_sort_refused_in_semantic_searches(syn):
    img, fac, dbs = syn
    emb = np.random.default_rng(0).standard_normal((img.n_docs, 16)).astype(np.float32)
    qv = np.random.default_rng(1).standard_normal((2, 16)).astype(np.float32)
    ix = mb.Index(img, criteria=["words", "desc:price", "sort"], facets=fac)
    ix.set_embeddings(emb)
    r = ix.search().semantic(qv).execute()
    assert list(r.status) == [-4, -4] and list(r.n_hits) == [0, 0]  # Asc/Desc criteria in a semantic search: not built
    ix2 = mb.Index(img, criteria=["words", "typo"], facets=fac)
    ix2.set_embeddings(emb)
    r = ix2.search().semantic(qv).sort([["price:asc"], []]).execute()
    assert r.status[0] == -3 and r.status[1] == 0 and r.n_hits[1] == 20  # SortRankingRuleMissing
    ix3 = mb.Index(img, criteria=CRITERIA, facets=fac)
    ix3.set_embeddings(emb)
    r = ix3.search().semantic(qv).sort([["price:asc"], []]).execute()
    assert r.status[0] == -4 and r.status[1] == 0 and r.n_hits[1] == 20
