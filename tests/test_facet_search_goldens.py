"""CPU: the facet search specification (tests/facet_search_spec.py) against the reference's own answers
(tests/golden/facet_search_goldens.json, from crates/meilisearch/tests/search/facet_search.rs)."""
import pytest

from tests.facet_search_fixtures import golden_facets, host_query, load_facet_search_goldens, matches
from tests.facet_search_spec import facet_search

CASES = load_facet_search_goldens()


def test_goldens_cover_the_cases():
    names = {c["test"] for c in CASES}
    assert {"simple_facet_search", "simple_facet_search_on_movies", "advanced_facet_search", "more_advanced_facet_search",
            "simple_facet_search_with_max_values", "simple_facet_search_by_count_with_max_values", "facet_search_dont_support_words",
            "simple_facet_search_with_sort_by_count"} <= names


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{c['test']}-{c['query']}" for c in CASES])
def test_spec_matches_golden(i):
    case = CASES[i]
    fac = golden_facets(case)
    hits = facet_search(fac, fac.fields[case["facet"]], range(len(case["genres"])), host_query(case), order=case["order"],
                        max_values=case["max_values"], authorize_typos=case["typos"], exact_words=case["exact_words"])
    assert matches(case, hits), (case, hits)
