"""Facet images for the facet distribution goldens (tests/golden/facet_goldens.json)."""
import json
import os

from corpus.facets import FacetImage

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "facet_goldens.json")


def load_facet_goldens():
    return json.load(open(GOLDEN))


def golden_facets(test):
    """the documents of a golden test in insertion order (docid = position), their field through milli's facet extraction"""
    fac = FacetImage()
    fac.fid(test["field"])
    for d, v in enumerate(test["docs"]):
        fac.add_json(d, test["field"], v)
    fac.build()
    return fac


def case_candidates(case):
    """the candidates a golden case passes (None: none given)"""
    c = case["candidates"]
    if c is None:
        return None
    return set(range(*c["range"])) if isinstance(c, dict) else set(c)
