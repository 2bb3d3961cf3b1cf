"""Facet images for the facet search goldens (tests/golden/facet_search_goldens.json)."""
import json
import os

from corpus.facets import FacetImage, hyper_normalize

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "facet_search_goldens.json")


def load_facet_search_goldens():
    return json.load(open(GOLDEN))["cases"]


def golden_facets(case):
    """the case's documents in insertion order (docid = position), their facet field through milli's facet extraction"""
    fac = FacetImage()
    fac.fid(case["facet"])
    for d, v in enumerate(case["genres"]):
        fac.add_json(d, case["facet"], v)
    fac.build()
    fac.build_search()
    return fac


def host_query(case):
    """the query as the route hands it on: normalize_facet_string (charabia's lossy normaliser, approximated as indexing's is)"""
    return None if case["query"] is None else hyper_normalize(case["query"])


def matches(case, hits):
    """hits [(value, count)] against what the reference's test asserts"""
    if "n_hits" in case and len(hits) != case["n_hits"]:
        return False
    if "leading_hits" in case and [list(h) for h in hits[:len(case["leading_hits"])]] != case["leading_hits"]:
        return False
    return "hits" not in case or [list(h) for h in hits] == case["hits"]
