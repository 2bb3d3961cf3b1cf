"""GPU: the reference's own facet search answers (tests/golden/facet_search_goldens.json) through b200_facet_search_batch and
through a placeholder search batch whose facet search runs over the search's candidates (every document)."""
import pytest

import meilisearch_b200 as mb
from corpus.pyindexgen import IndexImage
from tests.facet_search_fixtures import golden_facets, host_query, load_facet_search_goldens, matches

pytestmark = pytest.mark.gpu

CASES = load_facet_search_goldens()


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{c['test']}-{c['query']}" for c in CASES])
def test_library_matches_golden(i):
    case = CASES[i]
    img = IndexImage(1)
    for d in range(len(case["genres"])):
        img.add_text(d, 0, "")
    img.build()
    fac = golden_facets(case)
    ix = mb.Index(img, facets=fac, authorize_typos=case["typos"], exact_words=case["exact_words"])
    q = host_query(case)
    got, status = ix.facet_search([None], case["facet"], q, order=case["order"], max_values=case["max_values"])
    assert status[0] == 0 and matches(case, got[0]), (case, got)
    res = ix.search().query([""]).facet_search(case["facet"], q, case["order"], case["max_values"]).execute()
    assert res.status[0] == 0 and res.facet_hits(0) == got[0]
