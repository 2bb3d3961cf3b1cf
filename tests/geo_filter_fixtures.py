"""Index images and specification state for the geo filter goldens (tests/golden/geo_filter_goldens.json)."""
import json
import os

from corpus.facets import FacetImage
from tests.geo_filter_spec import GeoFilterIndex
from tests.geo_fixtures import spec_state
from tests.helpers import image_from_corpus

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "geo_filter_goldens.json")


def load_geo_filter_goldens():
    return json.load(open(GOLDEN))


def geo_images(docs, searchable=None):
    """documents in insertion order (docid = position), their `_geo` through milli's facet extraction (string coordinates become
    numbers); text in `searchable` fields, else none"""
    img = image_from_corpus({"searchable": searchable or ["text"], "exact_attributes": [], "stop_words": [], "docs": docs})
    fac = FacetImage()
    for d, doc in enumerate(docs):
        if "_geo" in doc:
            fac.add_json(d, "_geo", doc["_geo"])
    fac.fid("_geo.lat")
    fac.fid("_geo.lng")
    fac.build()
    return img, fac


def spec_index(img, fac, filterable=True, other_filterable=()):
    dbs, gix = spec_state(fac)
    return GeoFilterIndex(dbs, gix, img.n_docs, fac.fields["_geo.lat"], fac.fields["_geo.lng"], filterable, other_filterable)
