"""CPU: the geo filter specification (tests/geo_filter_spec.py) against the reference's known answers
(tests/golden/geo_filter_goldens.json, written by tests/golden/extract_geo_filter_goldens.py)."""
import pytest

import meilisearch_b200 as mb
from tests.geo_filter_fixtures import geo_images, load_geo_filter_goldens, spec_index
from tests.geo_filter_spec import GeoFilterError

def clause(f):
    return mb.parse_geo_filter(f)


def test_bounding_box_goldens():
    g = load_geo_filter_goldens()["bounding_box"]
    assert any(isinstance(v, str) for d in g["docs"] for v in d["_geo"].values())  # string coordinates are exercised
    img, fac = geo_images(g["docs"])
    spec = spec_index(img, fac)
    assert len(g["cases"]) == 8 and len(g["errors"]) == 2
    for c in g["cases"]:
        assert sorted(spec.filtered_universe([clause(c["filter"])])) == c["ids"], c["filter"]
    for e in g["errors"]:
        with pytest.raises(GeoFilterError) as err:
            spec.clause(*clause(e["filter"]))
        assert str(err.value) == e["message"]


def test_zero_radius_golden():
    g = load_geo_filter_goldens()["zero_radius"]
    img, fac = geo_images(g["docs"])
    assert sorted(spec_index(img, fac).filtered_universe([clause(g["filter"])])) == g["ids"]


def test_error_goldens():
    g = load_geo_filter_goldens()
    img, fac = geo_images(g["bounding_box"]["docs"])
    for e in g["not_filterable"]:
        spec = spec_index(img, fac, filterable=False, other_filterable=e["other_filterable"])
        with pytest.raises(GeoFilterError) as err:
            spec.clause(*clause(e["filter"]))
        assert str(err.value) == e["message"]
    spec = spec_index(img, fac)
    assert len(g["range_errors"]) == 12
    for e in g["range_errors"]:
        with pytest.raises(GeoFilterError) as err:
            spec.clause(*clause(e["filter"]))
        assert str(err.value) == e["message"], e["filter"]


def test_keyword_and_meilisearch_goldens():
    g = load_geo_filter_goldens()
    k = g["keyword"]
    img, fac = geo_images(k["docs"], k["searchable"])
    spec = spec_index(img, fac)
    ext = [d["id"] for d in k["docs"]]
    for c in k["cases"]:  # every document matches the query (expected_order keeps all 17 under Last), so the filter decides
        assert sorted(ext[d] for d in spec.filtered_universe([clause(c["filter"])])) == c["ids"], c["name"]
    m = g["meilisearch"]
    img, fac = geo_images(m["docs"])
    spec = spec_index(img, fac)
    box = m["geo_bounding_box_with_string_and_number"]
    got = sorted(m["docs"][d]["id"] for d in spec.filtered_universe([clause(box["filter"])]))
    assert got == box["ids"] and len(got) == box["estimated_total_hits"]
    spec.filtered_universe([clause(m["geo_sort_with_geo_strings"]["filter"])])  # status 200: no error
