"""CPU: the facet search specification (tests/facet_search_spec.py) on hand-checked cases, and the library's count order (cut count,
then the heap replayed over the hits at or above it) against the reference's heap over every hit."""
import json
import random

from corpus.facets import FacetImage, hyper_normalize
from tests.facet_search_spec import ValuesCollection, count_order_by_cut, decode_cbo, facet_search, osa_prefix_distance


def test_osa_prefix_distance():
    assert osa_prefix_distance("adv", "adventure") == 0
    assert osa_prefix_distance("avd", "adventure") == 1  # a transposition
    assert osa_prefix_distance("adventrue", "adventure") == 1
    assert osa_prefix_distance("xdventure", "adventure") == 1  # no first-letter rule
    assert osa_prefix_distance("", "anything") == 0
    assert osa_prefix_distance("café", "cafe") == 1  # one Unicode scalar value, two bytes
    assert osa_prefix_distance("ab", "") == 2


def test_count_order_by_cut_matches_the_heap():
    rng = random.Random(7)
    for _ in range(3000):
        n = rng.randint(0, 30)
        hits = [(rng.choice("abcdefgh") * rng.randint(1, 2), rng.randint(1, 4)) for _ in range(n)]
        for mx in (0, 1, 2, 3, 5, 100):
            vc = ValuesCollection("count", mx)
            for v, c in hits:
                vc.insert(v, c)
            assert count_order_by_cut(hits, mx) == vc.into_sorted_vec(), (hits, mx)


def test_lexicographic_keeps_the_first_hits():
    vc = ValuesCollection("alpha", 2)
    assert not vc.insert("b", 1)
    assert vc.insert("a", 5)
    assert vc.insert("c", 9)
    assert vc.into_sorted_vec() == [("b", 1), ("a", 5)]
    assert ValuesCollection("alpha", 0).insert("a", 1)


def test_json_sets_with_escapes_round_trip():
    fac = FacetImage()
    for d, v in enumerate(['Quote "q"', "back\\slash", "tab\there", "Ünïcode", "emoji 🎉", "line\nbreak"]):
        fac.add_facet(d, "f", v)
    fac.build()
    norm, _ = fac.build_search()
    seen = set()
    for i in range(norm.n_keys):
        seen.update(json.loads(norm.val(i).decode()))
    assert seen == set(fac.strings[0])


def facets_fixture():
    fac = FacetImage()
    docs = ["Adventure", "adventure", "Àdventure", "Action", "Comedy", "comédie", "Drama", "Adventure", "Horror", "Action"]
    for d, v in enumerate(docs):
        fac.add_facet(d, "genres", v)
    fac.build()
    fac.build_search()
    return fac


def test_spec_on_a_small_field():
    fac = facets_fixture()
    fid = fac.fields["genres"]
    every = range(10)
    # None: every level-0 key in key order (NFKD keys: "a\u0300dventure" after "adventure"), the original of the smallest docid
    assert facet_search(fac, fid, every) == [("Action", 2), ("Adventure", 3), ("Àdventure", 1), ("Comedy", 1), ("comédie", 1),
                                             ("Drama", 1), ("Horror", 1)]
    # "adv": the hyper-normalised "adventure" stands for "adventure" and "àdventure"
    assert facet_search(fac, fid, every, "adv") == [("Adventure", 3), ("Àdventure", 1)]
    # typos: "advnture" (8 bytes, one typo)
    assert facet_search(fac, fid, every, "advnture") == [("Adventure", 3), ("Àdventure", 1)]
    assert facet_search(fac, fid, every, "advnture", field_typos=False) == []
    # FST order: "comedie" then "comedy"; at equal counts the later hit replaces the heap's smallest
    assert facet_search(fac, fid, every, "com", order="count", max_values=1) == [("Comedy", 1)]
    assert facet_search(fac, fid, [1, 2], "adv") == [("Adventure", 1), ("Àdventure", 1)]
    assert facet_search(fac, fid, every, "", max_values=2) == [("Action", 2), ("Adventure", 3)]
    assert facet_search(fac, fid, every, "adventure", exact_words={"adventure"}) == [("Adventure", 3), ("Àdventure", 1)]
    assert facet_search(fac, fid, every, "adventur", exact_words={"adventur"}) == []
    assert facet_search(fac, fid, every, max_values=0) == []


def test_hyper_normalize():
    assert hyper_normalize("àdventure") == "adventure"
    assert hyper_normalize("comédie") == "comedie"


def test_decode_cbo_round_trip():
    from corpus.facets import cbo_encode

    for docs in ([], [3], list(range(0, 700, 7)), list(range(5000)) + [70000, 70001]):
        assert decode_cbo(cbo_encode(docs)) == docs
