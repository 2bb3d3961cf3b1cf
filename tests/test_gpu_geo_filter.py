"""GPU: geo filters (geo_filter.cu) against the CPU specification (tests/geo_filter_spec.py): b200_geo_filter_batch bit for bit, and
every search mode with geo clauses against the same search given the specification's bitmap as `universes`."""
import numpy as np
import pytest

import meilisearch_b200 as mb
from tests.geo_filter_spec import NOT_FILTERABLE, GeoFilterIndex, bitmap
from tests.geo_fixtures import spec_state, synthetic_geo_images

pytestmark = pytest.mark.gpu

CRITERIA = ["words", "typo", "proximity", "attributeRank", "sort", "wordPosition", "exactness"]


def make(n_docs):
    img, fac = synthetic_geo_images(n_docs, **({} if n_docs < 100_000 else {"vocab": 20000, "with_geo": 0.3}))
    dbs, gix = spec_state(fac)
    spec = GeoFilterIndex(dbs, gix, img.n_docs, fac.fields["_geo.lat"], fac.fields["_geo.lng"])
    return img, fac, gix, spec


@pytest.fixture(scope="module")
def small():
    return make(40_000)


def clause_set(gix):
    """radii around the cluster centres, a duplicated point and a sub-metre chain; boxes of every shape"""
    chain = min((p for p in gix.points.values() if p[1] == 7.0), key=lambda p: p[0])
    dup = next(p for p in gix.points.values() if p[1] == 20.0)
    one = next(p for d, p in sorted(gix.points.items()) if round(p[0], 1) == p[0] and round(p[1], 1) == p[1])
    centres = [(48.85, 2.35), (0.0, 179.99), (-48.85, -177.65), dup, chain]
    out = []
    for c in centres:
        for r in (0.0, 0.5, 1.0, 100.0, 10_000.0, 20_000_000.0, -1.0):
            out.append(f"_geoRadius({c[0]!r}, {c[1]!r}, {r!r})")
    out += ["_geoBoundingBox([49.5, 3.0], [48.0, 1.5])",      # normal
            "_geoBoundingBox([1.0, -179.5], [-1.0, 179.5])",  # wraps the antimeridian
            "_geoBoundingBox([90.0, 180.0], [60.0, -180.0])", # polar cap
            f"_geoBoundingBox([{one[0]!r}, {one[1]!r}], [{one[0]!r}, {one[1]!r}])",  # one point, inclusive edges
            "_geoBoundingBox([90.0, 180.0], [-90.0, -180.0])",  # the whole earth
            "_geoBoundingBox([48.8, 2.4], [48.8, 2.3])",      # an edge on round coordinates
            "_geoBoundingBox([10.02, 20.0], [10.0, 20.0])"]   # duplicates on both edges
    return out


@pytest.mark.parametrize("n_docs", [40_000, 700_000])
def test_geo_filter_batch_matches_spec(small, n_docs):
    img, fac, gix, spec = small if n_docs == 40_000 else make(n_docs)
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    clauses = clause_set(gix)
    out, status = ix.geo_filter(clauses)
    assert list(status) == [0] * len(clauses)
    for i, c in enumerate(clauses):
        kind, neg, args = mb.parse_geo_filter(c)
        want = bitmap(img.n_docs, spec.clause(kind, neg, args))
        assert np.array_equal(out[i], want), (c, int(np.unpackbits(out[i].view(np.uint8)).sum()), len(spec.clause(kind, neg, args)))
    assert ix.stats()["kernels"]["geo_filter"]["count"] >= 2


def filters_and_universes(img, gix, spec, n):
    """per query: its geo clauses, its caller universe (or None), and the specification's filtered universe"""
    rng = np.random.default_rng(11)
    pool = clause_set(gix)
    caller = bitmap(img.n_docs, rng.choice(img.n_docs, img.n_docs // 2, replace=False))
    filters, callers, want = [], [], []
    for q in range(n):
        k = 1 + q % 2
        fs = [("NOT " if (q + j) % 5 == 0 else "") + pool[rng.integers(len(pool))] for j in range(k)]
        if q % 7 == 3:
            fs = ["_geoRadius(48.85, 2.35, 60000.0)", "NOT _geoBoundingBox([49.0, 2.5], [48.7, 2.2])"]
        u = caller if q % 3 == 1 else None
        filters.append(fs)
        callers.append(u)
        docs = None if u is None else np.nonzero(np.unpackbits(u.view(np.uint8), bitorder="little")[: img.n_docs])[0]
        want.append(bitmap(img.n_docs, spec.filtered_universe([mb.parse_geo_filter(f) for f in fs], docs)))
    return filters, callers, want


def same(a, b, n):
    assert list(a.status) == [0] * n and list(b.status) == [0] * n
    for q in range(n):
        assert a.ids(q) == b.ids(q), q
        assert a.scores(q) == b.scores(q), q
        assert a.n_candidates[q] == b.n_candidates[q], q
    if a.candidates is not None:
        assert np.array_equal(a.candidates, b.candidates)


def both(ix, build, filters, callers, want):
    n = len(filters)
    got = build(ix.search()).geo_filter(filters)
    if any(u is not None for u in callers):
        got = got.universes(callers)
    ref = build(ix.search()).universes(want)
    return got, ref, n


@pytest.mark.parametrize("mode", ["placeholder", "keyword-detailed", "keyword-skip", "sort-box", "geosort-radius", "semantic", "hybrid"])
def test_search_modes_match_universes(small, mode):
    img, fac, gix, spec = small
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    n = 24
    filters, callers, want = filters_and_universes(img, gix, spec, n)
    queries = img.synthetic_queries(n, seed=5)
    rng = np.random.default_rng(2)
    if mode in ("semantic", "hybrid"):
        ix.set_embeddings(rng.standard_normal((img.n_docs, 32)).astype(np.float32))
        qv = rng.standard_normal((n, 32)).astype(np.float32)
    if mode == "sort-box":
        filters = [["_geoBoundingBox([49.5, 3.0], [48.0, 1.5])"] if q % 2 else ["_geoBoundingBox([1.0, -179.5], [-1.0, 179.5])"] for q in range(n)]
        want = [bitmap(img.n_docs, spec.filtered_universe([mb.parse_geo_filter(f) for f in fs],
                                                          None if u is None else np.nonzero(np.unpackbits(u.view(np.uint8), bitorder="little")[: img.n_docs])[0]))
                for fs, u in zip(filters, callers)]
    if mode == "geosort-radius":
        filters = [[f"_geoRadius(48.85, 2.35, {1000.0 * (q + 1)!r})"] for q in range(n)]
        want = [bitmap(img.n_docs, spec.filtered_universe([mb.parse_geo_filter(f) for f in fs],
                                                          None if u is None else np.nonzero(np.unpackbits(u.view(np.uint8), bitorder="little")[: img.n_docs])[0]))
                for fs, u in zip(filters, callers)]
    builds = {
        "placeholder": lambda s: s.query([""] * n).scoring_strategy("detailed").limit(30).with_candidates(),
        "keyword-detailed": lambda s: s.query(queries).scoring_strategy("detailed").with_candidates(),
        "keyword-skip": lambda s: s.query(queries).scoring_strategy("skip").offset(3).limit(15),
        "sort-box": lambda s: s.query([""] * n).sort(["price:asc"]).scoring_strategy("detailed"),
        "geosort-radius": lambda s: s.query([""] * n).sort(["_geoPoint(48.85, 2.35):asc"]).scoring_strategy("detailed").limit(40),
        "semantic": lambda s: s.semantic(qv).scoring_strategy("detailed"),
        "hybrid": lambda s: s.query(queries).semantic(qv).scoring_strategy("detailed"),
    }
    got, ref, n = both(ix, builds[mode], filters, callers, want)
    if mode == "hybrid":
        a, b = got.execute_hybrid(0.5), ref.execute_hybrid(0.5)
    else:
        a, b = got.execute(), ref.execute()
    same(a, b, n)
    assert any(int(c) > 0 for c in a.n_candidates)


def test_errors_per_query(small):
    img, fac, gix, spec = small
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    filters = [["_geoRadius(48.85, 2.35, 5000.0)"], ["_geoRadius(91.0, 2.35, 5000.0)"], ["_geoBoundingBox([1.0, 2.0], [3.0, 1.0])"],
               ["_geoRadius(48.85, 200.0, 10.0)"], ["_geoRadius(48.85, 2.35, inf)"], []]
    r = ix.search().query([""] * 6).geo_filter(filters).execute()
    assert list(r.status) == [0, -3, -3, -3, -3, 0]
    assert r.n_candidates[0] == len(spec.geo_radius(48.85, 2.35, 5000.0)) and r.n_candidates[5] == img.n_docs
    assert r.ids(0) == sorted(spec.geo_radius(48.85, 2.35, 5000.0))[:20]
    out, st = ix.geo_filter(["_geoRadius(91.0, 2.35, 5000.0)", "_geoBoundingBox([1.0, 2.0], [0.0, 1.0])"])
    assert list(st) == [-3, 0] and not out[0].any()
    assert "Bad latitude `91`" in ix.last_error()
    out, st = ix.geo_filter(["_geoBoundingBox([1.0, 2.0], [3.0, 1.0])"])
    assert st[0] == -3 and ix.last_error() == "The top latitude `1` is below the bottom latitude `3`."
    out, st = ix.geo_filter(["_geoRadius(48.85, 200.0, 10.0)"])
    assert ix.last_error().endswith("Hint: try using `-160` instead.")
    # no geo fields staged: `_geo` is not filterable, in every mode
    bare = mb.Index(img, criteria=CRITERIA, facets=fac, geo=(0xFFFF, 0xFFFF))
    r = bare.search().query(["", ""]).geo_filter([["_geoRadius(48.85, 2.35, 5000.0)"], []]).execute()
    assert list(r.status) == [-3, 0] and bare.last_error() == NOT_FILTERABLE
    out, st = bare.geo_filter(["_geoBoundingBox([1.0, 2.0], [0.0, 1.0])", "_geoRadius(95.0, 0.0, 1.0)"])
    assert list(st) == [-3, -3]
    rng = np.random.default_rng(4)
    bare.set_embeddings(rng.standard_normal((img.n_docs, 16)).astype(np.float32))
    qv = rng.standard_normal((2, 16)).astype(np.float32)
    r = bare.search().semantic(qv).geo_filter([["_geoRadius(48.85, 2.35, 5000.0)"], []]).execute()
    assert list(r.status) == [-3, 0] and r.n_hits[1] == 20
    r = bare.search().query(["", ""]).semantic(qv).geo_filter([[], ["NOT _geoRadius(48.85, 2.35, 5000.0)"]]).execute_hybrid(0.5)
    assert list(r.status) == [0, -3]


def test_null_fields_unchanged(small):
    # a batch without geo clauses runs exactly as before, and no geo filter kernel is launched
    img, fac, gix, spec = small
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    a = ix.search().query(img.synthetic_queries(8, seed=1)).scoring_strategy("detailed").execute()
    b = ix.search().query(img.synthetic_queries(8, seed=1)).scoring_strategy("detailed").geo_filter([]).execute()
    same(a, b, 8)
    assert ix.stats()["kernels"]["geo_filter"]["count"] == 0


def test_more_slots_than_one_chunk(small):
    # 1100 distinct clauses: the filter kernel accumulates its counts 1024 slots at a time
    img, fac, gix, spec = small
    ix = mb.Index(img, criteria=CRITERIA, facets=fac)
    rng = np.random.default_rng(9)
    docs = np.array(sorted(gix.points))
    lat = np.array([gix.points[d][0] for d in docs])
    lng = np.array([gix.points[d][1] for d in docs])
    n = 1100
    centre = rng.integers(0, len(docs), n)
    half = rng.uniform(0.01, 2.0, (n, 2))
    boxes = [(float(min(90.0, lat[c] + h[0])), float(min(180.0, lng[c] + h[1])), float(max(-90.0, lat[c] - h[0])), float(max(-180.0, lng[c] - h[1])))
             for c, h in zip(centre, half)]
    clauses = [f"_geoBoundingBox([{t!r}, {r!r}], [{b!r}, {l!r}])" for t, r, b, l in boxes]
    want = [docs[(lat >= b) & (lat <= t) & (lng >= l) & (lng <= r)] for t, r, b, l in boxes]
    out, status = ix.geo_filter(clauses)
    assert not status.any()
    for i in range(n):
        assert np.array_equal(out[i], bitmap(img.n_docs, want[i])), clauses[i]
    r = ix.search().query([""] * n).geo_filter([[c] for c in clauses]).limit(5).execute()
    for i in range(n):
        assert r.status[i] == 0 and int(r.n_candidates[i]) == len(want[i]) and r.ids(i) == [int(d) for d in want[i][:5]], clauses[i]
