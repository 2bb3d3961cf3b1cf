"""GPU: every geo filter golden of the reference (tests/golden/geo_filter_goldens.json) through the CUDA path: the candidate sets
through b200_search_batch and b200_geo_filter_batch, the error messages, and the keyword searches of filters.rs on the test_set
index."""
import numpy as np
import pytest

import meilisearch_b200 as mb
from tests.geo_filter_fixtures import geo_images, load_geo_filter_goldens

pytestmark = pytest.mark.gpu

LIB_NOT_FILTERABLE = "Attribute `_geo/_geojson` is not filterable."


def ids_of(bits, n_docs):
    return [int(d) for d in np.nonzero(np.unpackbits(bits.view(np.uint8), bitorder="little")[:n_docs])[0]]


def test_bounding_box_and_zero_radius_goldens():
    g = load_geo_filter_goldens()
    b = g["bounding_box"]
    img, fac = geo_images(b["docs"])
    ix = mb.Index(img, criteria=["words", "sort"], facets=fac)
    filters = [c["filter"] for c in b["cases"]]
    r = ix.search().query([""] * len(filters)).geo_filter([[f] for f in filters]).with_candidates().execute()
    out, st = ix.geo_filter(filters)
    for q, c in enumerate(b["cases"]):
        assert r.status[q] == 0 and ids_of(r.candidates[q], img.n_docs) == c["ids"] and r.ids(q) == c["ids"], c["filter"]
        assert st[q] == 0 and ids_of(out[q], img.n_docs) == c["ids"], c["filter"]
    for e in b["errors"]:
        r = ix.search().query([""]).geo_filter([e["filter"]]).execute()
        assert r.status[0] == -3 and ix.last_error() == e["message"]
    z = g["zero_radius"]
    img, fac = geo_images(z["docs"])
    ix = mb.Index(img, criteria=["words", "sort"], facets=fac)
    r = ix.search().query([""]).geo_filter([z["filter"]]).execute()
    assert r.status[0] == 0 and r.ids(0) == z["ids"]


def test_error_goldens():
    g = load_geo_filter_goldens()
    img, fac = geo_images(g["bounding_box"]["docs"])
    bare = mb.Index(img, criteria=["words", "sort"], facets=fac, geo=(0xFFFF, 0xFFFF))
    for e in g["not_filterable"]:
        r = bare.search().query([""]).geo_filter([e["filter"]]).execute()
        # the library gives the attribute part; the caller appends the index's filterable patterns
        assert r.status[0] == -3 and bare.last_error() == LIB_NOT_FILTERABLE and e["message"].startswith(LIB_NOT_FILTERABLE)
    ix = mb.Index(img, criteria=["words", "sort"], facets=fac)
    for e in g["range_errors"]:
        r = ix.search().query(["", ""]).geo_filter([[e["filter"]], ["_geoBoundingBox([90, 180], [-90, -180])"]]).execute()
        assert list(r.status) == [-3, 0] and r.n_hits[1] == img.n_docs
        out, st = ix.geo_filter([e["filter"]])
        assert st[0] == -3 and ix.last_error() == e["message"], e["filter"]


def test_keyword_goldens_on_test_set():
    k = load_geo_filter_goldens()["keyword"]
    img, fac = geo_images(k["docs"], k["searchable"])
    ix = mb.Index(img, criteria=k["criteria"], facets=fac, synonyms=k["synonyms"])
    ext = [d["id"] for d in k["docs"]]
    r = ix.search().query([k["query"]] * len(k["cases"])).terms_matching_strategy(k["terms_matching_strategy"]).limit(k["limit"]) \
        .geo_filter([[c["filter"]] for c in k["cases"]]).execute()
    for q, c in enumerate(k["cases"]):
        assert r.status[q] == 0 and sorted(ext[d] for d in r.ids(q)) == c["ids"], c["name"]


def test_meilisearch_goldens():
    m = load_geo_filter_goldens()["meilisearch"]
    img, fac = geo_images(m["docs"])
    ix = mb.Index(img, criteria=["words", "typo", "proximity", "attribute", "sort", "exactness"], facets=fac)
    box = m["geo_bounding_box_with_string_and_number"]
    r = ix.search().query([""]).geo_filter([box["filter"]]).execute()
    assert r.status[0] == 0 and [m["docs"][d]["id"] for d in r.ids(0)] == box["ids"]
    assert int(r.n_candidates[0]) == box["estimated_total_hits"]
    s = m["geo_sort_with_geo_strings"]
    r = ix.search().query([""]).geo_filter([s["filter"]]).sort(s["sort"]).execute()
    assert r.status[0] == 0 and s["status"] == 200
