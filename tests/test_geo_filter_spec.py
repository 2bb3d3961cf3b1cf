"""CPU: the geo filter specification (tests/geo_filter_spec.py) and the Python clause parser."""
import math

import numpy as np
import pytest

import meilisearch_b200 as mb
from tests.geo_filter_spec import EPSILON, NOT_FILTERABLE, GeoFilterError, GeoFilterIndex, rust_f64
from tests.geo_fixtures import spec_state
from tests.geo_spec import distance_between_two_points


def random_index(n, seed):
    from corpus.facets import FacetImage

    rng = np.random.default_rng(seed)
    fac = FacetImage()
    docs = np.arange(n)
    has = rng.random(n) < 0.8
    lat = np.degrees(np.arcsin(rng.uniform(-1, 1, n)))
    lng = rng.uniform(-180, 180, n)
    near = rng.random(n) < 0.5  # half of them clustered, some exact duplicates
    lat = np.where(near, 48.85 + rng.normal(0, 0.05, n), lat)
    lng = np.where(near, 2.35 + rng.normal(0, 0.05, n), lng)
    lat = np.where(rng.random(n) < 0.05, 48.85, lat)
    lng = np.where(lat == 48.85, 2.35, lng)
    fac._bulk("_geo.lat", docs[has], lat[has], numbers=True)
    fac._bulk("_geo.lng", docs[has], lng[has], numbers=True)
    fac.build()
    dbs, gix = spec_state(fac)
    return GeoFilterIndex(dbs, gix, n, fac.fields["_geo.lat"], fac.fields["_geo.lng"])


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_radius_prefix_is_the_haversine_scan(seed):
    # mathematically the chord and the haversine order the points alike, so the take_while prefix is the plain scan on these points
    ix = random_index(3000, seed)
    for base in ((48.85, 2.35), (0.0, 0.0), (-48.85, -177.65), (90.0, 0.0)):
        for r in (0.0, 1.0, 500.0, 5000.0, 2e6, 2.0001e7, -3.0):
            scan = {d for d, p in ix.gix.points.items() if distance_between_two_points(base, p) <= r + EPSILON}
            assert ix.geo_radius(*base, r) == scan, (base, r)


def test_box_and_not():
    ix = random_index(2000, 7)
    pts = ix.gix.points
    box = ix.geo_bounding_box(49.0, 2.5, 48.8, 2.2)
    assert box == {d for d, (la, ln) in pts.items() if 48.8 <= la <= 49.0 and 2.2 <= ln <= 2.5}
    wrap = ix.geo_bounding_box(10.0, -170.0, -10.0, 170.0)
    assert wrap == {d for d, (la, ln) in pts.items() if -10 <= la <= 10 and (ln >= 170 or ln <= -170)}
    assert ix.geo_bounding_box(48.85, 2.35, 48.85, 2.35) == {d for d, p in pts.items() if p == (48.85, 2.35)}
    assert ix.clause(1, True, (49.0, 2.5, 48.8, 2.2)) == ix.documents_ids - box
    assert ix.filtered_universe([(1, False, (49.0, 2.5, 48.8, 2.2)), (0, True, (48.85, 2.35, 1.0))], range(1000)) == \
        {d for d in box if d < 1000} - ix.geo_radius(48.85, 2.35, 1.0)


def test_validation_order_and_messages():
    ix = random_index(100, 1)
    cases = [
        ((math.nan, 200.0, 1.0), "Non finite floats are not supported"),  # finiteness of both coordinates first
        ((91.0, math.inf, 1.0), "Non finite floats are not supported"),
        ((91.0, 200.0, math.nan), "Bad latitude `91`. Latitude must be contained between -90 and 90 degrees."),
        ((0.0, 200.5, math.nan), "Bad longitude `200.5`. Longitude must be contained between -180 and 180 degrees. Hint: try using `-159.5` instead."),
        ((0.0, -181.0, 1.0), "Bad longitude `-181`. Longitude must be contained between -180 and 180 degrees. Hint: try using `179` instead."),
        ((0.0, 0.0, math.inf), "Non finite floats are not supported"),
    ]
    for args, msg in cases:
        with pytest.raises(GeoFilterError) as e:
            ix.geo_radius(*args)
        assert str(e.value) == msg, args
    with pytest.raises(GeoFilterError, match="The top latitude `1` is below the bottom latitude `3.5`."):
        ix.geo_bounding_box(1.0, 2.0, 3.5, 1.0)
    with pytest.raises(GeoFilterError, match="Bad latitude `-95`"):
        ix.geo_bounding_box(1.0, 2.0, -95.0, 1.0)
    ix.filterable = False
    with pytest.raises(GeoFilterError) as e:
        ix.geo_bounding_box(1.0, 2.0, 0.0, 1.0)
    assert str(e.value) == NOT_FILTERABLE + " This index does not have configured filterable attributes."
    with pytest.raises(GeoFilterError, match="Bad latitude"):  # the range checks come before the filterable check
        ix.geo_radius(-90.5, 0.0, 1.0)
    assert rust_f64(100.0) == "100" and rust_f64(0.1) == "0.1" and rust_f64(-1e-7) == "-0.0000001"


def test_parser():
    assert mb.parse_geo_filter("_geoRadius(48.85, 2.35, 2000)") == (0, False, (48.85, 2.35, 2000.0, 0.0))
    assert mb.parse_geo_filter("NOT  _geoBoundingBox([1, 2.5], [-1, -2])") == (1, True, (1.0, 2.5, -1.0, -2.0))
    assert mb.parse_geo_filter("_geoRadius(0,0,inf)")[2][2] == math.inf  # refused by the library with the reference's message
    for bad in ("_geoRadius(1, 2, 3, 125)",  # the resolution argument steers GeoJSON only
                "_geoRadius(1, 2)", "_geoPolygon([1, 2], [3, 4], [5, 6])", "NOT_geoRadius(1, 2, 3)", "_geoBoundingBox([1, 2], [3])",
                "_geoBoundingBox(1, 2, 3, 4)", "price > 3", "_geoRadius(a, 2, 3)", "_georadius(1, 2, 3)"):
        with pytest.raises(ValueError):
            mb.parse_geo_filter(bad)
