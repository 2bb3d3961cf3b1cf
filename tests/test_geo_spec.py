"""CPU: the GeoSort specification (tests/geo_spec.py) against the reference's known answers under every strategy, the haversine
against the `_geoDistance` snapshots, the literal port against a direct evaluation of the order model, and the `_geo` extraction."""
import random

import pytest

from corpus.facets import FacetImage, geo_points
from tests.geo_fixtures import STRATEGIES, doc_images, load_geo_goldens, spec_state
from tests.geo_spec import GeoIndex, GeoSort, distance_between_two_points, order_model, placeholder_search, sort_rules


@pytest.mark.parametrize("strategy,cache", STRATEGIES)
def test_spec_goldens(strategy, cache):
    g = load_geo_goldens()
    for t in g["tests"]:
        img, fac = doc_images(t["docs"])
        dbs, gix = spec_state(fac)
        for c in t["cases"]:
            rules = sort_rules(g["criteria"], c["sort"], fac.fields)
            ids, scores = placeholder_search(dbs, gix, rules, range(len(t["docs"])), 0, 20, "detailed", strategy, cache)
            assert ids == c["ids"], (t["name"], c["sort"], strategy, cache)
            assert [list(s[0][2]) if s[0][2] is not None else None for s in scores] == c["geo_values"], (t["name"], c["sort"])


def test_spec_max_bucket_size():
    g = load_geo_goldens()
    m = g["max_bucket"]
    img, fac = doc_images(m["docs"])
    dbs, gix = spec_state(fac)
    ext = [d["id"] for d in m["docs"]]
    for strategy, cache in m["strategies"]:
        rules = sort_rules(g["criteria"], m["sort"], fac.fields)
        ids, _ = placeholder_search(dbs, gix, rules, range(len(ext)), 0, 20, "detailed", strategy, cache, m["max_bucket_size"])
        ids = [ext[d] for d in ids]
        assert len(ids) == 15
        assert all(m["first_6_ids_in"][0] <= x <= m["first_6_ids_in"][1] for x in ids[:6])
        assert all(m["next_4_ids_in"][0] <= x <= m["next_4_ids_in"][1] for x in ids[6:10])
        assert ids[10:] == m["no_geo_ids"]


def test_haversine_snapshots():
    g = load_geo_goldens()["geo_distance"]
    assert [round(distance_between_two_points(g["target"], p)) for p in g["points"]] == g["rounded_metres"]


def _random_points(rng, n):
    pts = {}
    for d in range(n):
        r = rng.random()
        if r < 0.1:
            continue  # no _geo
        if r < 0.3:
            pts[d] = (10.0, 20.0 + rng.randrange(5) * 1e-6)  # duplicates and points < 1 m apart
        elif r < 0.4:
            pts[d] = (rng.choice([-1, 1]) * 30.0, rng.choice([179.9999, -179.9999, 180.0, -180.0]))  # the seam
        else:
            pts[d] = (rng.uniform(-90, 90), rng.uniform(-180, 180))
    return pts


@pytest.mark.parametrize("strategy,cache", [("dynamic", 7), ("dynamic", 1000), ("rtree", 3), ("iterative", 5)])
@pytest.mark.parametrize("ascending", [True, False])
def test_literal_port_follows_the_order_model(strategy, cache, ascending):
    rng = random.Random(7)
    gix = GeoIndex(_random_points(rng, 300))
    for target in [(10.0, 20.0), (-10.0, -160.0), (0.0, 180.0), (rng.uniform(-90, 90), rng.uniform(-180, 180))]:
        universe = set(d for d in range(300) if rng.random() < 0.8)
        order = order_model(gix, target, ascending, universe, strategy, cache)
        g = GeoSort(gix, target, ascending, strategy, cache, max_bucket_size=10**9)
        left = set(universe)
        g.start_iteration(left)
        walked = []
        while left & set(gix.points):
            bucket, value = g.next_bucket(left)
            # a bucket is a run of the order: its documents are the next ones of the model, and its value their first point
            assert sorted(order[len(walked): len(walked) + len(bucket)]) == bucket
            assert value == gix.points[order[len(walked)]]
            walked += order[len(walked): len(walked) + len(bucket)]
            left.difference_update(bucket)
        assert walked == order


def test_geo_extraction():
    fac = FacetImage()
    fac.add_json(0, "_geo", {"lat": 1.5, "lng": "-2.25"})
    fac.add_json(1, "_geo", None)
    fac.add_json(2, "_geo", {"lat": "3", "lng": 4})
    fac.add_facet(3, "_geo.lat", 7.0)
    fac.add_facet(3, "_geo.lat", 5.0)
    fac.add_facet(3, "_geo.lng", "6.5")  # a string coordinate is parsed
    fac.build()
    pts = geo_points(fac, fac.fields["_geo.lat"], fac.fields["_geo.lng"])
    assert pts == {0: (1.5, -2.25), 2: (3.0, 4.0), 3: (5.0, 6.5)}
    fac.add_facet(4, "_geo.lat", 1.0)
    with pytest.raises(ValueError):
        geo_points(fac, fac.fields["_geo.lat"], fac.fields["_geo.lng"])
