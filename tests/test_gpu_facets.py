"""GPU: the facet distribution and facet stats (facet.cu) of search batches and of b200_facet_distribution_batch against the CPU
specification (tests/facet_spec.py) over the same candidates."""
import numpy as np
import pytest

import meilisearch_b200 as mb
from corpus.facets import FacetImage
from corpus.pyindexgen import IndexImage
from tests.facet_spec import facet_stats, facet_values

pytestmark = pytest.mark.gpu

CRITERIA = ["words", "typo", "proximity", "attributeRank", "sort", "wordPosition", "exactness"]
FIELDS = ["price", "brand", "tags", "sku", "colour"]


def make(n_docs, vocab=2000):
    """the synthetic corpus with `price`, `brand`, `tags`, `_geo`, `sku` (a number field with more values than fit the shared-memory
    histogram, FACET_SHARED_VALUES, so its counts go through global atomics) and `colour`"""
    img = IndexImage(1)
    img.add_synthetic(n_docs, vocab)
    img.build()
    fac = FacetImage().add_synthetic(n_docs).add_synthetic_geo(n_docs)
    rng = np.random.default_rng(77)
    fac._bulk("sku", np.arange(n_docs, dtype=np.uint32), rng.integers(0, 3 * 4096, n_docs).astype(np.float64), numbers=True)
    # `colour`: originals that differ from their normalised value and from one document to the next, so each string's key depends on
    # facet_docid being the smallest candidate holding it
    originals = ["Blue", "BLUE", " blue", "Red", "red ", "RED", "Green", "GREEN"]
    for d, k in enumerate(rng.integers(0, len(originals), n_docs)):
        fac.add_facet(d, "colour", originals[k])
    fac.build()
    return img, fac


@pytest.fixture(scope="module")
def small():
    img, fac = make(40_000)
    return img, fac, mb.Index(img, criteria=CRITERIA, facets=fac)


def docs_of(bitmap, n_docs):
    return set(np.nonzero(np.unpackbits(bitmap.view(np.uint8), bitorder="little")[:n_docs])[0].tolist())


def bitmap(n_docs, docs):
    bits = np.zeros(((n_docs + 63) // 64) * 64, np.uint8)
    bits[np.asarray(sorted(docs), np.int64)] = 1
    return np.packbits(bits, bitorder="little").view(np.uint64)


def check(res, fac, img, names, max_values, queries):
    for q in queries:
        assert res.status[q] == 0, q
        cand = docs_of(res.candidates[q], img.n_docs)
        assert len(cand) == res.n_candidates[q]
        dist, stats = res.facet_distribution(q), res.facet_stats(q)
        for name in names:
            fid = fac.fields[name]
            assert dist[name] == facet_values(fac, fid, cand, max_values), (q, name, len(cand))
            want = facet_stats(fac, fid, cand)
            assert stats.get(name) == want, (q, name)


@pytest.mark.parametrize("kind", ["keyword", "placeholder", "sort", "geosort", "geofilter", "universes"])
def test_search_facets_match_spec(small, kind):
    img, fac, ix = small
    n = 12
    rng = np.random.default_rng(3)
    s = ix.search().facets(FIELDS).with_candidates().scoring_strategy("detailed")
    if kind == "keyword":
        s = s.query(img.synthetic_queries(n, seed=4))
    else:
        s = s.query([""] * n)
    if kind == "sort":
        s = s.sort(["price:desc", "brand:asc"])
    if kind == "geosort":
        s = s.sort(["_geoPoint(48.85, 2.35):asc"])
    if kind == "geofilter":
        s = s.geo_filter([[f"_geoRadius(48.85, 2.35, {2000.0 * (q + 1)!r})"] for q in range(n)])
    if kind == "universes":
        s = s.universes([bitmap(img.n_docs, rng.choice(img.n_docs, int(rng.integers(1, 9000)), replace=False)) for _ in range(n)])
    res = s.execute()
    check(res, fac, img, FIELDS, 100, range(n))
    assert ix.stats()["kernels"]["facet"]["count"] >= 1


@pytest.mark.parametrize("size", [3000, 3001])
@pytest.mark.parametrize("max_values", [0, 1, 2, 50, 100])
def test_path_switch_and_max_values(small, size, max_values):
    img, fac, ix = small
    rng = np.random.default_rng(size + max_values)
    us = [bitmap(img.n_docs, rng.choice(img.n_docs, size, replace=False)) for _ in range(3)]
    res = ix.search().query(["", "", ""]).universes(us).facets(FIELDS).max_values_per_facet(max_values).with_candidates().execute()
    assert list(res.n_candidates) == [size] * 3
    check(res, fac, img, FIELDS, max_values, range(3))


def test_levels_path_appends_every_tag_string(small):
    # `tags` has 200 numbers and 60 strings: at max 50 the numbers fill the map and every non-empty string is appended
    img, fac, ix = small
    res = ix.search().query([""]).facets(["tags"]).max_values_per_facet(50).with_candidates().execute()
    d = res.facet_distribution(0)["tags"]
    assert len(d) == 50 + 60 and d == facet_values(fac, fac.fields["tags"], set(range(img.n_docs)), 50)


def test_skip_scoring_and_identical_without_facets(small):
    img, fac, ix = small
    queries = img.synthetic_queries(16, seed=9)
    for scoring in ("skip", "detailed"):
        a = ix.search().query(queries).scoring_strategy(scoring).with_candidates().execute()
        b = ix.search().query(queries).scoring_strategy(scoring).with_candidates().facets(FIELDS).execute()
        for q in range(16):
            assert a.ids(q) == b.ids(q) and a.scores(q) == b.scores(q) and a.n_candidates[q] == b.n_candidates[q]
        assert np.array_equal(a.candidates, b.candidates)
        check(b, fac, img, FIELDS, 100, range(16))


def test_capacity_fails_its_own_query(small):
    img, fac, ix = small
    us = [bitmap(img.n_docs, range(10)), None]
    res = ix.search().query(["", ""]).universes(us).facets(["brand"]).facet_cap(12).with_candidates().execute()
    assert list(res.status) == [0, -5] and res.n_hits[0] == 10
    assert "needs" in ix.last_error()
    check(res, fac, img, ["brand"], 100, [0])


def test_unsupported_and_invalid(small):
    img, fac, ix = small
    r = ix.search().query(["", ""]).facets([["brand"], []]).facet_order("count").execute()
    assert list(r.status) == [-4, 0]
    r = ix.search().query(["", ""]).facets([["brand"], []]).ranking_score_threshold(0.5).execute()
    assert list(r.status) == [-4, 0]
    rng = np.random.default_rng(1)
    ix2 = mb.Index(img, criteria=CRITERIA, facets=fac)
    ix2.set_embeddings(rng.standard_normal((img.n_docs, 16)).astype(np.float32))
    qv = rng.standard_normal((2, 16)).astype(np.float32)
    r = ix2.search().semantic(qv).facets([["brand"], []]).execute()
    assert list(r.status) == [-4, 0] and r.n_hits[1] == 20
    r = ix2.search().query(["", ""]).semantic(qv).facets([["brand"], []]).execute_hybrid(0.5)
    assert list(r.status) == [-4, 0]
    # facet_begin without facet_fid or without the outputs: INVALID for the queries with facets
    tokens = mb.TokenBatch(["", ""])
    res = mb.SearchResult(2, 20)
    b = mb._Batch(2, mb._p(tokens.token_begin), mb._p(tokens.token_kind), mb._p(tokens.lemma_off), mb._p(tokens.lemma_bytes), 0, 0, 0, 20, 10,
                  None, 0, 0.0)
    b.stop_after = -1
    begin = np.array([0, 1, 1], np.uint32)
    b.facet_begin = mb._p(begin)
    r = mb._Results(mb._p(res.documents_ids), mb._p(res.n_hits), None, None, None, None, None, mb._p(res.n_candidates), None, mb._p(res.status))
    ix._ck(ix._l.b200_search_batch(ix._h, mb.C.byref(b), mb.C.byref(r)))
    assert list(res.status) == [-3, 0] and res.n_hits[1] == 20


def test_unknown_field(small):
    img, fac, ix = small
    r = ix.search().query([""]).facets(["nope", "brand"]).with_candidates().execute()
    assert r.status[0] == 0
    assert r.facet_distribution(0)["nope"] == [] and "nope" not in r.facet_stats(0)
    check(r, fac, img, ["brand"], 100, [0])


@pytest.mark.parametrize("max_values", [0, 3, 100])
def test_entry_point_random_bitmaps(small, max_values):
    img, fac, ix = small
    rng = np.random.default_rng(max_values)
    sets = [set(rng.choice(img.n_docs, int(k), replace=False).tolist()) for k in (0, 1, 50, 2999, 3000, 3001, 20000)]
    bms = [bitmap(img.n_docs, s) for s in sets]
    bms.append(bms[3])  # equal pointers are uploaded once
    sets.append(sets[3])
    dists, stats, status = ix.facet_distribution(bms, FIELDS, max_values=max_values)
    assert not status.any()
    for i, cand in enumerate(sets):
        for name in FIELDS:
            fid = fac.fields[name]
            assert dists[i][name] == facet_values(fac, fid, cand, max_values), (i, name)
            assert stats[i].get(name) == facet_stats(fac, fid, cand)
    _, _, status = ix.facet_distribution(bms[:2], FIELDS, order="count")
    assert list(status) == [-4, -4]
    _, _, status = ix.facet_distribution(bms[6:7], ["brand"], cap=5)
    assert list(status) == [-5]


def test_many_segments():
    # 700 k documents: the candidates of a broad keyword query span many compaction segments of the step loop
    img, fac = make(700_000, vocab=20000)
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    res = ix.search().query(img.synthetic_queries(4, seed=2) + [""]).facets(["brand", "price", "colour"]).with_candidates().execute()
    check(res, fac, img, ["brand", "price", "colour"], 100, range(5))
    assert ix.stats()["kernels"]["facet"]["count"] >= 1


def test_display_order_of_large_numbers():
    # the <= 3000 path orders numbers by their Rust Display strings: large values print their shortest digits padded with zeros
    values = [2.0, 9.0, 10.0, 1e21, 1e23, 2.0 ** 60, 1.2345678901234567e25, 1.7976931348623157e308, 0.1, -0.0, -3.25e-7]
    img = IndexImage(1)
    fac = FacetImage()
    for d, v in enumerate(values):
        img.add_text(d, 0, "")
        fac.add_facet(d, "big", v)
    img.build()
    fac.build()
    ix = mb.Index(img, facets=fac)
    cand = set(range(len(values)))
    for max_values in (0, 1, 3, 100):
        dists, stats, status = ix.facet_distribution([bitmap(len(values), cand)], ["big"], max_values=max_values)
        assert list(status) == [0]
        assert dists[0]["big"] == facet_values(fac, fac.fields["big"], cand, max_values), max_values
        assert stats[0]["big"] == facet_stats(fac, fac.fields["big"], cand)
