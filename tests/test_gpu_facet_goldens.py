"""GPU: the reference's own facet answers (tests/golden/facet_goldens.json) through the library: b200_facet_distribution_batch for
the cases that pass candidates, a placeholder search batch for the cases without (documents_ids through the facet levels; only
where documents_ids holds more than 3000 documents, because a search always hands its candidates over, and with 3000 or fewer
the reference's FacetDistribution without candidates walks the levels where one with them would not)."""
import hashlib

import numpy as np
import pytest

import meilisearch_b200 as mb
from corpus.pyindexgen import IndexImage
from tests.facet_fixtures import case_candidates, golden_facets, load_facet_goldens
from tests.facet_spec import debug_string, stats_debug_string

pytestmark = pytest.mark.gpu

G = load_facet_goldens()


def index_of(test):
    img = IndexImage(1)
    for d in range(len(test["docs"])):
        img.add_text(d, 0, "")
    img.build()
    fac = golden_facets(test)
    return img, mb.Index(img, facets=fac)


def bitmap(n_docs, docs):
    bits = np.zeros(((n_docs + 63) // 64) * 64, np.uint8)
    bits[np.asarray(sorted(docs), np.int64)] = 1
    return np.packbits(bits, bitorder="little").view(np.uint64)


def digest(got, case):
    return hashlib.md5(got.encode()).hexdigest() if case["md5"] else got


@pytest.mark.parametrize("name", [t["name"] for t in G["milli"]])
def test_facet_distribution_rs(name):
    t = next(x for x in G["milli"] if x["name"] == name)
    img, ix = index_of(t)
    field, n = t["field"], len(t["docs"])
    ran = 0
    for c in t["cases"]:
        cand = case_candidates(c)
        if cand is None:
            if c["call"] == "compute_stats" or n <= 3000:
                continue  # compute_stats without candidates returns {}; see the module docstring for the rest
            r = ix.search().query([""]).facets([field]).max_values_per_facet(c["max_values"]).execute()
            assert r.status[0] == 0
            assert digest(debug_string(field, r.facet_distribution(0)[field]), c) == c["expect"]
            ran += 1
            continue
        dists, stats, status = ix.facet_distribution([bitmap(n, cand)], [field], max_values=c["max_values"], order=c["order"])
        if c["order"] == "count":
            assert list(status) == [-4]  # B200_ERR_UNSUPPORTED
            continue
        assert list(status) == [0]
        if c["call"] == "compute_stats":
            assert stats_debug_string(field, stats[0].get(field)) == c["expect"]
        else:
            assert digest(debug_string(field, dists[0][field]), c) == c["expect"]
        ran += 1
    assert ran > 0


def test_server_cases():
    mv, casing = G["server"]
    img, ix = index_of(mv)
    for c in mv["cases"]:
        r = ix.search().query([""]).facets(["number"]).max_values_per_facet(c["max_values"]).execute()
        assert r.status[0] == 0 and len(r.facet_distribution(0)["number"]) == c["len"]
    img, ix = index_of(casing)
    r = ix.search().query([""]).facets(["dog"]).execute()
    assert dict(r.facet_distribution(0)["dog"]) == casing["facet_distribution"]["dog"]
