"""Index images with `_geo` points for the GeoSort tests."""
import json
import os

from corpus.facets import FacetImage, geo_points
from corpus.pyindexgen import IndexImage
from tests.geo_spec import GeoIndex
from tests.sort_spec import FacetDbs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "geo_sort_goldens.json")
STRATEGIES = [("iterative", 2), ("iterative", 1000), ("rtree", 2), ("rtree", 1000), ("dynamic", 1000)]


def load_geo_goldens():
    return json.load(open(GOLDEN))


def doc_images(docs):
    """the index of geo_sort.rs create_index(): empty text, `_geo` and `score` faceted; docids in insertion order"""
    img = IndexImage(1)
    fac = FacetImage()
    for d, doc in enumerate(docs):
        img.add_text(d, 0, "")
        for name in ("_geo", "score"):
            if name in doc:
                fac.add_json(d, name, doc[name])
    fac.fid("_geo.lat")
    fac.fid("_geo.lng")
    img.build()
    fac.build()
    return img, fac


def synthetic_geo_images(n_docs, vocab=2000, seed=0xB200, geo_seed=0x6E0, with_geo=0.9):
    img = IndexImage(1)
    img.add_synthetic(n_docs, vocab, seed=seed)
    img.build()
    fac = FacetImage().add_synthetic(n_docs).add_synthetic_geo(n_docs, seed=geo_seed, with_geo=with_geo)
    fac.build()
    return img, fac


def spec_state(fac):
    return FacetDbs(fac.f64_db, fac.string_db), GeoIndex(geo_points(fac, fac.fields["_geo.lat"], fac.fields["_geo.lng"]))
