"""CPU: the Sort specification (tests/sort_spec.py) against the reference's known answers, and the facet database formats."""
import numpy as np

from corpus.facets import FacetImage, cbo_encode, ordered_f64
from oracle.pyoracle import cbo_decode
from tests.sort_fixtures import golden_images, load_sort_goldens, synthetic_images
from tests.sort_spec import FacetDbs, placeholder_search, sort_buckets, sort_rules, universe_docs


def test_sort_goldens_on_spec():
    g = load_sort_goldens()
    img, fac = golden_images(g)
    dbs = FacetDbs(fac.f64_db, fac.string_db)
    for c in g["cases"]:
        rules = sort_rules(g["criteria"], c["sort"], fac.fields)
        ids, scores = placeholder_search(dbs, rules, universe_docs(len(g["docs"])), 0, g["limit"], "detailed")
        assert ids == c["ids"], c["name"]
        if c["sort_values"] is not None:
            assert [s[0][3] for s in scores] == c["sort_values"], c["name"]


def test_cbo_round_trip():
    rng = np.random.default_rng(1)
    for n in (0, 1, 7, 8, 100, 5000, 70000):
        d = np.unique(rng.integers(0, 300000, n)).astype(np.uint32)
        assert list(cbo_decode(cbo_encode(d))) == list(d)


def test_ordered_f64_orders_like_floats():
    xs = sorted([-1e9, -2.5, -0.0, 0.0, 1e-9, 1.0, 1.5, 2.0, 1e12])
    enc = [ordered_f64(x)[:8] for x in xs]
    assert enc == sorted(enc)


def test_facet_extraction_rules():
    f = FacetImage()
    f.add_json(0, "v", [1, "A ", None, "", {"x": 1}, True])
    f.add_json(1, "v", None)
    fid = f.fields["v"]
    assert f.numbers[fid] == {1.0: [0]}
    assert f.strings[fid] == {"a": [0], "true": [0]}


def test_rule_list_dedup():
    fields = {"price": 0, "brand": 1}
    rules = sort_rules(["words", "desc:price", "sort", "asc:brand"], ["price:asc", "brand:desc", "nope:asc"], fields)
    assert rules == [("price", 0, False), ("brand", 1, False), ("nope", None, True)]


def test_levels_above_zero_are_emitted():
    _, fac = synthetic_images(3000)
    levels = {fac.f64_db.key(i)[2] for i in range(fac.f64_db.n_keys)}
    assert max(levels) >= 1


def bucket_sort_loop(dbs, rules, universe, offset, limit, scoring):
    """a second, literal port of bucket_sort's loop (bucket_sort.rs:160-330, maybe_add_to_results :387-455) with a stack of rule
    universes and bucket iterators, as a cross-check of the recursive form of sort_spec.placeholder_search"""
    ids, scores, cur_offset = [], [], 0
    universes, iters, rr_scores = [set(universe)], [iter(sort_buckets(dbs, rules[0], universe))], []

    def add(bucket):
        nonlocal cur_offset
        bucket = sorted(bucket)
        if cur_offset < offset:
            if cur_offset + len(bucket) >= offset:
                take = bucket[offset - cur_offset:][: limit - len(ids)]
                ids.extend(take)
                scores.extend([list(rr_scores)] * len(take))
        else:
            take = bucket[: limit - len(ids)]
            ids.extend(take)
            scores.extend([list(rr_scores)] * len(take))
        cur_offset += len(bucket)

    def back():
        universes.pop()
        iters.pop()
        if rr_scores and len(rr_scores) >= len(universes):
            rr_scores.pop()

    while len(ids) < limit and universes:
        u = universes[-1]
        if not u or (scoring == "skip" and len(u) == 1):
            add(u)
            back()
            continue
        bucket, value = next(iters[-1])
        bucket = [d for d in bucket if d in u]
        rr_scores.append(("sort", rules[len(universes) - 1][0], rules[len(universes) - 1][2], value))
        u.difference_update(bucket)
        if len(universes) == len(rules) or (scoring == "skip" and len(bucket) <= 1) or cur_offset + len(bucket) < offset:
            add(bucket)
            rr_scores.pop()
            continue
        universes.append(set(bucket))
        iters.append(iter(sort_buckets(dbs, rules[len(universes) - 1], bucket)))
    return ids, scores


def test_spec_matches_the_bucket_sort_loop():
    img, fac = synthetic_images(40000)
    dbs = FacetDbs(fac.f64_db, fac.string_db)
    rng = np.random.default_rng(9)
    crit = ["words", "sort", "exactness"]
    for sort in (["tags:desc", "brand:asc", "price:asc"], ["price:asc"], ["brand:desc", "tags:asc"], ["missing:asc", "price:desc"]):
        rules = sort_rules(crit, sort, fac.fields)
        for universe in (list(range(40000)), [5], [3, 9], sorted(rng.choice(40000, 37, replace=False).tolist())):
            for scoring in ("skip", "detailed"):
                for offset, limit in ((0, 20), (7, 33), (0, 3)):
                    want = bucket_sort_loop(dbs, rules, universe, offset, limit, scoring)
                    assert placeholder_search(dbs, rules, universe, offset, limit, scoring) == want, (sort, len(universe), scoring, offset)


def test_skip_last_document_of_a_rule_universe():
    # bucket_sort.rs:196-204: over a 2-document universe under Skip the second document is returned with no Sort score
    img, fac = synthetic_images(3000)
    dbs = FacetDbs(fac.f64_db, fac.string_db)
    rules = sort_rules(["sort"], ["price:asc"], fac.fields)
    ids, scores = placeholder_search(dbs, rules, [10, 11], 0, 20, "skip")
    assert len(ids) == 2 and len(scores[0]) == 1 and scores[1] == []
