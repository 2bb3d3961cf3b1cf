"""GPU: filter programs (filter.cu) against the CPU specification (tests/filter_spec.py): b200_filter_batch bit for bit on random trees,
and every search mode with a filter against the same search given the specification's bitmap as `universes`."""
import numpy as np
import pytest

import meilisearch_b200 as mb
from tests.filter_fixtures import NUMS, filter_images, geo_spec, random_tree, synthetic_docs
from tests.filter_spec import FilterError, FilterSpec, Unsupported
from tests.geo_filter_spec import bitmap

pytestmark = pytest.mark.gpu

CRITERIA = ["words", "typo", "proximity", "attributeRank", "sort", "wordPosition", "exactness"]
DENIED = {("s", "comparison"), ("m", "equality"), ("flag", "null")}


def make(n_docs, vocab=500):
    docs = synthetic_docs(n_docs)
    img, fac = filter_images(docs, vocab=vocab)
    spec = FilterSpec(fac, range(img.n_docs), geo_spec(fac, img.n_docs))
    return img, fac, spec


@pytest.fixture(scope="module")
def small():
    return make(20_000)


def outcome(spec, tree, n_docs):
    try:
        return 0, bitmap(n_docs, spec.evaluate(tree, DENIED)), -1
    except FilterError as e:
        return -3, None, e.leaf
    except Unsupported as e:
        return -4, None, e.leaf


def special_trees(rng):
    deep = ("cond", "n", ">", ["1.0"])
    for k in range(12):  # depth >= 8: alternating AND / OR / NOT
        deep = [("and", [deep, ("cond", "s", "!=", ["apple"])]), ("or", [("cond", "m", "EXISTS", []), deep]), ("not", deep)][k % 3]
    big_in = ("cond", "n", "IN", [repr(float(x)) for x in rng.uniform(-10, 200, 999)] + ["42.0"])
    return [deep, big_in,
            ("and", [("not", ("cond", "s", "=", ["apple"])), ("or", [("not", ("cond", "n", "<", ["2"])), ("cond", "m", "!=", ["b"])])]),
            ("or", [("geo", "radius", ["48.85", "2.35", "50000.0"]), ("not", ("geo", "bbox", ["49.5", "3.0", "48.0", "1.5"]))]),
            ("not", ("or", [("geo", "radius", ["48.85", "2.35", "20000.0"]), ("cond", "n", "EMPTY", [])])),
            ("and", [("cond", "n", "=", ["12345"]), ("cond", "s", ">", ["a"])]),      # denied, not reached
            ("and", [("cond", "n", "=", ["1.0"]), ("cond", "s", ">", ["a"])]),        # denied, reached
            ("and", [("cond", "n", ">=", ["1e6"]), ("and", [("cond", "s", "=", ["apple"]), ("cond", "m", "=", ["x"])])]),
            ("and", [("cond", "n", "=", ["1.0"]), ("geo", "radius", ["91", "0", "10"])]),
            # a bounding box intersects with its hint, a radius does not: the denied leaf behind them is reached or not accordingly
            ("and", [("cond", "n", ">=", ["1e6"]), ("and", [("geo", "bbox", ["90", "180", "-90", "-180"]), ("cond", "m", "=", ["x"])])]),
            ("and", [("cond", "n", ">=", ["1e6"]), ("and", [("geo", "radius", ["48.85", "2.35", "2e7"]), ("cond", "m", "=", ["x"])])]),
            ("and", [("cond", "n", "=", ["12345"]), ("geo", "radius", ["91", "0", "10"])]),
            ("cond", "s", "CONTAINS", ["a"]), ("geo", "polygon", ["0", "0", "1", "1", "0", "1"]),
            ("cond", "n", "IN", []), ("and", []), ("or", [])]


@pytest.mark.parametrize("n_docs", [20_000, 700_000])
def test_filter_batch_matches_spec(small, n_docs):
    img, fac, spec = small if n_docs == 20_000 else make(n_docs, vocab=2000)
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    rng = np.random.default_rng(3)
    trees = special_trees(rng) + [random_tree(rng, int(rng.integers(1, 6))) for _ in range(2000 if n_docs == 20_000 else 200)]
    out, status, leaf = ix.filter_batch(trees, DENIED)
    seen = set()
    for i, t in enumerate(trees):
        st, want, lf = outcome(spec, t, img.n_docs)
        seen.add(st)
        assert (status[i], leaf[i]) == (st, lf), (i, t, ix.last_error())
        if st == 0:
            assert np.array_equal(out[i], want), (i, t)
    assert seen == {0, -3, -4}
    assert ix.stats()["kernels"]["filter"]["count"] >= 1


def filters_and_universes(img, spec, n):
    rng = np.random.default_rng(21)
    caller = bitmap(img.n_docs, rng.choice(img.n_docs, img.n_docs // 2, replace=False))
    trees, callers, want = [], [], []
    for q in range(n):
        t = random_tree(rng, 3)
        while outcome(spec, t, img.n_docs)[0] != 0:
            t = random_tree(rng, 3)
        u = caller if q % 3 == 1 else None
        docs = spec.evaluate(t, DENIED)
        if u is not None:
            docs &= set(np.nonzero(np.unpackbits(u.view(np.uint8), bitorder="little")[: img.n_docs])[0].tolist())
        trees.append(t)
        callers.append(u)
        want.append(bitmap(img.n_docs, docs))
    return trees, callers, want


def same(a, b, n):
    assert list(a.status) == [0] * n and list(b.status) == [0] * n
    for q in range(n):
        assert a.ids(q) == b.ids(q), q
        assert a.scores(q) == b.scores(q), q
        assert a.n_candidates[q] == b.n_candidates[q], q
    if a.candidates is not None:
        assert np.array_equal(a.candidates, b.candidates)


@pytest.mark.parametrize("mode", ["placeholder", "keyword-detailed", "keyword-skip", "sort", "geosort", "semantic", "hybrid", "geo+program"])
def test_search_modes_match_universes(small, mode):
    img, fac, spec = small
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    n = 24
    trees, callers, want = filters_and_universes(img, spec, n)
    queries = img.synthetic_queries(n, seed=5)
    rng = np.random.default_rng(2)
    if mode in ("semantic", "hybrid"):
        ix.set_embeddings(rng.standard_normal((img.n_docs, 32)).astype(np.float32))
        qv = rng.standard_normal((n, 32)).astype(np.float32)
    geo = None
    if mode == "geo+program":  # the old geo_filter_* fields and a program together
        geo = [["_geoRadius(48.85, 2.35, 200000.0)"] if q % 2 else [] for q in range(n)]
        g = spec.geo.geo_radius(48.85, 2.35, 200000.0)
        want = [bitmap(img.n_docs, set(np.nonzero(np.unpackbits(w.view(np.uint8), bitorder="little")[: img.n_docs])[0].tolist()) & (g if q % 2 else set(range(img.n_docs))))
                for q, w in enumerate(want)]
    builds = {
        "placeholder": lambda s: s.query([""] * n).scoring_strategy("detailed").limit(30).with_candidates(),
        "keyword-detailed": lambda s: s.query(queries).scoring_strategy("detailed").with_candidates(),
        "keyword-skip": lambda s: s.query(queries).scoring_strategy("skip").offset(3).limit(15),
        "sort": lambda s: s.query([""] * n).sort(["n:asc"]).scoring_strategy("detailed"),
        "geosort": lambda s: s.query([""] * n).sort(["_geoPoint(48.85, 2.35):asc"]).scoring_strategy("detailed").limit(40),
        "semantic": lambda s: s.semantic(qv).scoring_strategy("detailed"),
        "hybrid": lambda s: s.query(queries).semantic(qv).scoring_strategy("detailed"),
        "geo+program": lambda s: s.query(queries).scoring_strategy("detailed").with_candidates(),
    }
    got = builds[mode](ix.search()).filter(trees, DENIED)
    if any(u is not None for u in callers):
        got = got.universes(callers)
    if geo is not None:
        got = got.geo_filter(geo)
    ref = builds[mode](ix.search()).universes(want)
    if mode == "hybrid":
        a, b = got.execute_hybrid(0.5), ref.execute_hybrid(0.5)
    else:
        a, b = got.execute(), ref.execute()
    same(a, b, n)
    assert list(a.filter_error_leaf[:n]) == [-1] * n
    assert any(int(c) > 0 for c in a.n_candidates)


def test_errors_per_query(small):
    img, fac, spec = small
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    filters = ["n > 1", "n = 1 AND s > a", "n = 12345 AND s > a", "s CONTAINS a", "n = 1 AND _geoRadius(91, 0, 10)", None, "m IS NULL"]
    r = ix.search().query([""] * len(filters)).filter(filters, DENIED).execute()
    assert list(r.status) == [0, -3, 0, -4, -3, 0, 0]
    assert list(r.filter_error_leaf[:len(filters)]) == [-1, 2, -1, 0, 2, -1, -1]
    assert r.n_candidates[0] == len(spec.evaluate("n > 1")) and r.n_candidates[2] == 0 and r.n_candidates[5] == img.n_docs
    assert r.n_candidates[6] == len(spec.evaluate("m IS NULL"))
    # an index staged without the presence databases: only the queries that need one fail
    bare_fac = filter_images(synthetic_docs(20_000), vocab=500, presence=False)[1]
    bare = mb.Index(img, criteria=CRITERIA, facets=bare_fac)
    r = bare.search().query([""] * 3).filter(["n EXISTS", "n > 1", "NOT m IS EMPTY"]).execute()
    assert list(r.status) == [-3, 0, -3] and "which was not staged" in bare.last_error()
    assert r.n_candidates[1] == len(spec.evaluate("n > 1"))
    # no geo fields: a geo leaf's `_geo` not filterable error is raised only where evaluation reaches it
    nogeo = mb.Index(img, criteria=CRITERIA, facets=fac, geo=(0xFFFF, 0xFFFF))
    out, st, leaf = nogeo.filter_batch(["n = 12345 AND _geoRadius(48, 2, 10)", "n = 1 AND _geoRadius(48, 2, 10)"])
    assert list(st) == [0, -3] and list(leaf) == [-1, 2] and not out[0].any()
    assert nogeo.last_error() == "Attribute `_geo/_geojson` is not filterable."


def test_no_filter_unchanged(small):
    img, fac, spec = small
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    q = img.synthetic_queries(8, seed=1)
    a = ix.search().query(q).scoring_strategy("detailed").execute()
    b = ix.search().query(q).scoring_strategy("detailed").filter([None] * 8).execute()
    same(a, b, 8)
    assert ix.stats()["kernels"]["filter"]["count"] == 0
