"""GPU: GeoSort and the geo filters where a haversine decision turns on its last bits (tests/geo_edge_fixtures.py): a whole metre of
the iterative order, the 1 m margin of the bucket chain, a radius equal to a distance or one double below it, the ±180° seam, the
poles, and exact antipodes (where the reference's distance can be NaN).  One index holds every case's points; each query gets the
universe of its own case.  Searches are compared with tests/geo_spec.py (ids, score tuples, candidate counts), filters with
tests/geo_filter_spec.py bit for bit."""
import math

import numpy as np
import pytest

import meilisearch_b200 as mb
from corpus.facets import FacetImage
from corpus.pyindexgen import IndexImage
from tests import geo_edge_fixtures as F
from tests.geo_filter_spec import GeoFilterIndex, bitmap
from tests.geo_fixtures import spec_state
from tests.geo_spec import distance_between_two_points, opposite_of, placeholder_search, sort_rules

pytestmark = pytest.mark.gpu

CRITERIA = ["sort"]


class Corpus:
    """explicit points, each a document with a `price` that runs opposite to its docid"""

    def __init__(self):
        self.points = []

    def add(self, p):
        self.points.append((float(p[0]), float(p[1])))
        return len(self.points) - 1

    def build(self):
        img, fac = IndexImage(1), FacetImage()
        n = len(self.points)
        for d, (lat, lng) in enumerate(self.points):
            img.add_text(d, 0, "")
            fac.add_json(d, "_geo", {"lat": lat, "lng": lng})
            fac.add_json(d, "price", n - d)
        fac.fid("_geo.lat")
        fac.fid("_geo.lng")
        img.build()
        fac.build()
        self.img, self.fac = img, fac
        self.dbs, self.gix = spec_state(fac)
        assert self.gix.points == dict(enumerate(self.points))
        self.spec = GeoFilterIndex(self.dbs, self.gix, img.n_docs, fac.fields["_geo.lat"], fac.fields["_geo.lng"])
        self.ix = mb.Index(img, criteria=CRITERIA, facets=fac)
        return self


def _toward(t, d):
    """a point at about d metres north of t along its meridian, or over the pole beyond it"""
    ang = math.degrees(d / F.R)
    lat = t[0] + ang
    if lat <= 90.0:
        return (lat, t[1])
    return (180.0 - lat, opposite_of((0.0, t[1]))[1])


@pytest.fixture(scope="module")
def corpus():
    c = Corpus()
    c.floor = []  # (target, [L, B, H], [4 fillers near the target], [4 fillers near its antipode])
    for t, p, n, h in F.floor_edges(7, 60, steps=2):
        if n + 10.0 > math.pi * F.R:
            continue
        low, high = _toward(t, n + 0.5), _toward(t, n - 0.5)
        trip = [c.add(low), c.add(p), c.add(high)]
        near = [c.add(t) for _ in range(4)]
        far = [c.add((opposite_of(t)[0] + (1e-3 if t[0] < 0 else -1e-3), opposite_of(t)[1])) for _ in range(4)]
        c.floor.append((t, trip, near, far))
    c.margin = []  # (target, p0, p): p0 first in docid order
    for t, p0, h0, p, h in F.margin_edges(8, 40, steps=2):
        c.margin.append((t, c.add(p0), c.add(p)))
    c.radius = []  # (target, radius)
    for t, p, h, r in F.radius_edges(9, 400):
        c.add(p)
        c.radius.append((t, r))
    c.seam = [c.add((0.0, -180.0)), c.add((0.0, 180.0)), c.add((0.0, 179.9999999)), c.add((90.0, 10.0)), c.add((90.0, -170.0)),
              c.add((-90.0, 0.0))]
    c.anti = []  # (target, [docs]): the target's exact antipode twice, the target, and a neighbour
    for cls, pairs in F.antipodes(10, 4).items():
        for t, p in pairs:
            c.anti.append((t, [c.add(p), c.add(p), c.add(t), c.add((t[0] + 1e-4, t[1]))]))
    return c.build()


def run_sorts(c, queries, strategy, max_bucket, scoring, limit=20):
    """queries [(sort list, docids of the universe)]: every query against the specification"""
    words = [bitmap(c.img.n_docs, u) for _, u in queries]
    r = (c.ix.search().query([""] * len(queries)).sort([s for s, _ in queries]).universes(words).limit(limit)
         .scoring_strategy(scoring).geo_strategy(*strategy).geo_max_bucket_size(max_bucket).execute())
    bad = []
    for q, (s, u) in enumerate(queries):
        assert r.status[q] == 0, (q, s)
        want_ids, want_sc = placeholder_search(c.dbs, c.gix, sort_rules(CRITERIA, s, c.fac.fields), sorted(u), 0, limit, scoring,
                                               strategy[0], strategy[1], max_bucket)
        if r.ids(q) != want_ids or r.scores(q) != want_sc or int(r.n_candidates[q]) != len(u):
            bad.append((s, sorted(u), r.ids(q), want_ids))
    assert not bad, (len(bad), len(queries), bad[:3])


def geo_sort(t, asc, then=()):
    return [f"_geoPoint({t[0]!r}, {t[1]!r}):{'asc' if asc else 'desc'}", *then]


@pytest.mark.parametrize("strategy", [("iterative", 1000), ("dynamic", 4)])
@pytest.mark.parametrize("asc", [True, False])
def test_floor_edges(corpus, strategy, asc):
    # {L at n + 0.5, the boundary point B, H at n - 0.5}, docids L < B < H: B's floor (n or n - 1) decides whether it comes before
    # or after H.  Under Dynamic(4) four fillers first fill the rtree part (near the target ascending, near its antipode descending),
    # so the three come in the iterative tail (mode 2).
    qs = []
    for t, trip, near, far in corpus.floor:
        u = trip + (near if asc else far) if strategy[0] == "dynamic" else trip
        qs.append((geo_sort(t, asc, ["price:asc"]), u))
    run_sorts(corpus, qs, strategy, 1, "detailed")


@pytest.mark.parametrize("strategy", [("iterative", 1000), ("rtree", 1000)])
@pytest.mark.parametrize("scoring", ["detailed", "skip"])
def test_margin_edges(corpus, strategy, scoring):
    # p's distance is within doubles of p0's + 1 m: one bucket {p0, p} (then price puts p first) or two ([p0], [p])
    qs = [(geo_sort(t, asc, ["price:asc"]), [p0, p]) for t, p0, p in corpus.margin for asc in (True, False)]
    run_sorts(corpus, qs, strategy, 1000, scoring)


def test_radius_edges(corpus):
    # radius = a point's distance (take_while keeps it) and one double below (it stops there), through b200_geo_filter_batch
    clauses = [f"_geoRadius({t[0]!r}, {t[1]!r}, {r!r})" for t, r in corpus.radius]
    out, status = corpus.ix.geo_filter(clauses)
    assert list(status) == [0] * len(clauses)
    bad = [c for i, c in enumerate(clauses) if not np.array_equal(out[i], bitmap(corpus.img.n_docs, corpus.spec.clause(0, False, mb.parse_geo_filter(c)[2])))]
    assert not bad, (len(bad), len(clauses), bad[:5])


def test_radius_edges_in_filter_trees(corpus):
    # a subset with NOT, and ANDed pairs, through b200_filter_batch
    rad = [f"_geoRadius({t[0]!r}, {t[1]!r}, {r!r})" for t, r in corpus.radius[:300]]
    filters = [("NOT " if i % 2 else "") + c for i, c in enumerate(rad)] + [f"{rad[i]} AND NOT {rad[i + 1]}" for i in range(0, 100, 2)]
    out, status, _ = corpus.ix.filter_batch(filters)
    assert list(status) == [0] * len(filters)
    sp = corpus.spec
    bad = []
    for i, f in enumerate(filters):
        if " AND " in f:
            a, b = f.split(" AND ")
            want = sp.clause(0, False, mb.parse_geo_filter(a)[2]) & sp.clause(0, True, mb.parse_geo_filter(b)[2])
        else:
            kind, neg, args = mb.parse_geo_filter(f)
            want = sp.clause(kind, neg, args)
        if not np.array_equal(out[i], bitmap(corpus.img.n_docs, want)):
            bad.append(f)
    assert not bad, (len(bad), len(filters), bad[:5])


def test_seam_and_poles(corpus):
    # (0, -180) is 1.56e-9 m from (0, 180) by the reference's formula: outside _geoRadius(0, 180, 0) and a radius of 1e-9 m, inside
    # one of 2e-9 m
    clauses = ["_geoRadius(0.0, 180.0, 0.0)", "_geoRadius(0.0, -180.0, 0.0)", "_geoRadius(0.0, 180.0, 1e-09)", "_geoRadius(0.0, 180.0, 2e-09)",
               "_geoRadius(90.0, 0.0, 0.0)", "_geoRadius(90.0, 0.0, 1e-09)", "_geoRadius(-90.0, 123.0, 0.0)"]
    out, status = corpus.ix.geo_filter(clauses)
    assert list(status) == [0] * len(clauses)
    for i, cl in enumerate(clauses):
        want = corpus.spec.clause(0, False, mb.parse_geo_filter(cl)[2])
        assert np.array_equal(out[i], bitmap(corpus.img.n_docs, want)), (cl, sorted(want))
    assert corpus.seam[0] not in corpus.spec.clause(0, False, (0.0, 180.0, 0.0, 0.0))
    u = corpus.seam
    qs = [(geo_sort(t, asc, ["price:asc"]), u) for t in ((0.0, 180.0), (0.0, -180.0), (90.0, 0.0), (-90.0, 45.0)) for asc in (True, False)]
    for strategy in (("rtree", 1000), ("iterative", 1000)):
        for mb_size in (1, 1000):
            run_sorts(corpus, qs, strategy, mb_size, "detailed")


@pytest.mark.parametrize("strategy", [("iterative", 1000), ("rtree", 1000), ("dynamic", 2)])
@pytest.mark.parametrize("max_bucket", [2, 1000])
def test_antipodes(corpus, strategy, max_bucket):
    # the antipode (twice) may be at NaN metres: first ascending in iterative order (`NaN as usize` = 0), a bucket that takes every
    # following point when it leads one (NaN > 1.0 is false), the end of a radius's take_while
    qs = []
    for t, docs in corpus.anti:
        for asc in (True, False):
            qs.append((geo_sort(t, asc, ["price:asc"]), docs))
    run_sorts(corpus, qs, strategy, max_bucket, "detailed")


def test_antipode_radius(corpus):
    clauses, filters = [], []
    for t, _ in corpus.anti:
        clauses.append(f"_geoRadius({t[0]!r}, {t[1]!r}, 21000000.0)")
        filters.append("NOT " + clauses[-1])
    out, status = corpus.ix.geo_filter(clauses)
    assert list(status) == [0] * len(clauses)
    fout, fstatus, _ = corpus.ix.filter_batch(filters)
    assert list(fstatus) == [0] * len(filters)
    for i, cl in enumerate(clauses):
        args = mb.parse_geo_filter(cl)[2]
        assert np.array_equal(out[i], bitmap(corpus.img.n_docs, corpus.spec.clause(0, False, args))), cl
        assert np.array_equal(fout[i], bitmap(corpus.img.n_docs, corpus.spec.clause(0, True, args))), filters[i]
    # at least one target's take_while stops at a NaN antipode before the whole earth
    nan_stop = [t for t, docs in corpus.anti if math.isnan(distance_between_two_points(t, corpus.points[docs[0]]))]
    assert nan_stop and any(len(corpus.spec.clause(0, False, (t[0], t[1], 2.1e7, 0.0))) < corpus.img.n_docs for t in nan_stop)
