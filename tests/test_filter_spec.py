"""CPU: the filter specification (tests/filter_spec.py) against brute force over synthetic documents, its error-reach rules, the
presence databases' extraction rules, and the filter parser."""
import numpy as np
import pytest

from meilisearch_b200.filter import parse_filter, preorder
from tests.filter_fixtures import brute, filter_images, geo_spec, random_tree, synthetic_docs
from tests.filter_spec import FilterError, FilterSpec, Unsupported


@pytest.fixture(scope="module")
def world():
    docs = synthetic_docs(600)
    img, fac = filter_images(docs)
    return docs, fac, FilterSpec(fac, range(len(docs)), geo_spec(fac, len(docs)))


def test_spec_matches_brute_force_on_random_trees(world):
    docs, fac, spec = world
    rng = np.random.default_rng(11)
    for _ in range(400):
        tree = random_tree(rng, int(rng.integers(1, 5)))
        assert spec.evaluate(tree) == brute(docs, tree, spec.geo), tree


@pytest.mark.parametrize("expr", ["n > 1", "n >= 1", "n < 1", "n <= 1", "n 1 TO 10", "n 10 TO 1", "s > b", "s apple TO banana", "s > 10",
                                  "m = 2", "m != 2", "s IN [apple, \"zz top\", nope]", "n IN []", "n EXISTS", "n IS NULL", "n IS EMPTY",
                                  "s IS NOT EMPTY", "m NOT EXISTS", "absent = 1", "absent != 1", "flag = true", "n > nope",
                                  "n -7.5 TO nope", "NOT (n > 1 OR s = apple)", "(n > 1 AND s = apple) OR m IS NULL"])
def test_spec_matches_brute_force_on_fixed_expressions(world, expr):
    docs, fac, spec = world
    tree = parse_filter(expr)
    assert spec.evaluate(tree) == brute(docs, tree, spec.geo)


def test_presence_databases_follow_the_extraction_rules():
    docs = [{"a": None}, {"a": ""}, {"a": []}, {"a": {}}, {"a": [None, ""]}, {"a": 1}, {}, {"a": "  "}, {"a": {"b": 1}}]
    img, fac = filter_images(docs, with_geo=False)
    spec = FilterSpec(fac, range(len(docs)))
    assert spec.evaluate("a EXISTS") == {0, 1, 2, 3, 4, 5, 7, 8}
    assert spec.evaluate("a IS NULL") == {0}
    assert spec.evaluate("a IS EMPTY") == {1, 2, 3}


def test_existing_facet_bytes_do_not_change_with_presence():
    docs = synthetic_docs(200)
    _, a = filter_images(docs, with_geo=False, presence=False)
    _, b = filter_images(docs, with_geo=False, presence=True)
    for x, y in ((a.f64_db, b.f64_db), (a.string_db, b.string_db)):
        assert x.key_bytes.tobytes() == y.key_bytes.tobytes() and x.val_bytes.tobytes() == y.val_bytes.tobytes()


def test_error_reached_only_past_a_non_empty_and_prefix(world):
    docs, fac, spec = world
    denied = {("s", "comparison")}
    # the first AND child empties the running bitmap: the denied leaf is never evaluated
    assert spec.evaluate("n = 12345 AND s > a", denied) == set()
    with pytest.raises(FilterError) as e:
        spec.evaluate("n = 1 AND s > a", denied)
    assert e.value.leaf == 2
    # an OR evaluates every child
    with pytest.raises(FilterError):
        spec.evaluate("n = 12345 OR s > a", denied)
    # the first reached failing leaf in pre-order wins
    with pytest.raises(FilterError) as e:
        spec.evaluate("(n = 12345 AND s > a) OR (n = 1 AND s < b) OR s >= c", denied)
    assert e.value.leaf == 6


def test_hint_intersection_decides_reach():
    """a range leaf and a bounding box intersect with their hint, an equality does not: the same set, a different reach"""
    docs = [{"n": 150.0, "_geo": {"lat": 10.0, "lng": 10.0}}, {"s": "apple", "n": 1.0, "_geo": {"lat": 50.0, "lng": 50.0}}, {"m": "x"}]
    img, fac = filter_images(docs, with_geo=False)
    spec = FilterSpec(fac, range(len(docs)), geo_spec(fac, len(docs)))
    denied = {("m", "equality")}
    assert spec.evaluate("n >= 100") == {0} and spec.evaluate("s = apple") == {1}
    # the inner AND's hint is {0}; its first child, an equality, ignores it: the running bitmap is {1}, the denied leaf is reached
    with pytest.raises(FilterError) as e:
        spec.evaluate("n >= 100 AND (s = apple AND m = x)", denied)
    assert e.value.leaf == 4
    # a range first: its running bitmap is {1} & {0} = empty, the denied leaf is not reached
    assert spec.evaluate("n >= 100 AND (s apple TO apple AND m = x)", denied) == set()
    # a bounding box around document 1 is intersected with the hint {0} as well; a radius around it is not
    assert spec.evaluate("n >= 100 AND (_geoBoundingBox([51, 51], [49, 49]) AND m = x)", denied) == set()
    with pytest.raises(FilterError):
        spec.evaluate("n >= 100 AND (_geoRadius(50, 50, 1000) AND m = x)", denied)


def test_geo_argument_errors_are_reached_only(world):
    docs, fac, spec = world
    assert spec.evaluate("n = 12345 AND _geoRadius(91, 0, 10)") == set()
    with pytest.raises(FilterError):
        spec.evaluate("n = 1 AND _geoRadius(91, 0, 10)")
    # `_geo` not filterable (no geo fields) is raised on reach too, after the argument checks
    bare = FilterSpec(fac, range(len(docs)))
    assert bare.evaluate("n = 12345 AND _geoRadius(48, 2, 10)") == set()
    with pytest.raises(FilterError) as e:
        bare.evaluate("n = 1 AND _geoRadius(48, 2, 10)")
    assert "not filterable" in str(e.value)


def test_unsupported_anywhere(world):
    docs, fac, spec = world
    for expr in ("n = 12345 AND s CONTAINS a", "_geoPolygon([0, 0], [1, 1], [0, 1])", "_shard = a", "s STARTS WITH a"):
        with pytest.raises(Unsupported):
            spec.evaluate(expr)


def test_parser():
    assert parse_filter("a = 1 AND b = 2 AND c = 3")[0] == "and" and len(parse_filter("a = 1 AND b = 2 AND c = 3")[1]) == 3
    assert parse_filter("a NOT IN [1, 2]") == ("not", ("cond", "a", "IN", ["1", "2"]))
    assert parse_filter("a IS NOT NULL") == ("not", ("cond", "a", "NULL", []))
    assert parse_filter("'x y' = \"it's\"") == ("cond", "x y", "=", ["it's"])
    assert parse_filter("_geoRadius(1, 2, 3, 4)") == ("geo", "radius_resolution", ["1", "2", "3", "4"])
    assert len(preorder(parse_filter("NOT (a = 1 OR b = 2)"))) == 4
    for bad in ("", "a =", "a = 1 AND", "(a = 1", "a IS b", "a = 1 b = 2", "a IN [1 2]"):
        with pytest.raises(ValueError):
            parse_filter(bad)
