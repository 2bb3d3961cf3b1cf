"""CPU: the split of the facet distribution between the library and its caller (b200milli.h, b200_results::facet_*) reproduces the
reference's facet_values on both paths, including a string whose original equals a number's Display string."""
import numpy as np
import pytest

from corpus.facets import FacetImage
from meilisearch_b200 import rust_f64_display as lib_display
from tests.facet_spec import CANDIDATES_THRESHOLD, facet_stats, facet_values, rust_f64_display


def library_entries(fac, fid, cand, max_values):
    """what the library returns for one slot: (number entries, string entries), each (key, count), in order and cut to length"""
    nums = [(v, sum(d in cand for d in set(ds))) for v, ds in fac.numbers.get(fid, {}).items()]
    strs = []
    for v, ds in sorted(fac.strings.get(fid, {}).items(), key=lambda x: x[0].encode()):
        hits = sorted(d for d in set(ds) if d in cand)
        if hits:
            strs.append((fac.originals.get((fid, hits[0], v), v), len(hits)))
    nums = [(v, c) for v, c in nums if c]
    if len(cand) <= CANDIDATES_THRESHOLD:
        n = sorted(((rust_f64_display(v), c) for v, c in nums))[:max_values]
        return n, strs[: max_values - len(n)]
    n = [(rust_f64_display(v), c) for v, c in sorted(nums)]
    n = n[:max_values] if max_values else n
    return n, strs[:max_values] if len(n) < max_values else strs


def caller_merge(numbers, strings, max_values):
    out = dict(numbers)
    for k, c in strings:
        out[k] = c
        if len(out) == max_values:
            break
    return list(out.items())


def collision_image(n_docs, n_numbers):
    """numbers 0..n_numbers-1 and strings whose originals are "0", "1", ... (colliding with the numbers) and "s0", "s1", ..."""
    fac = FacetImage()
    rng = np.random.default_rng(n_docs + n_numbers)
    for d in range(n_docs):
        fac.add_facet(d, "f", int(rng.integers(n_numbers)))
        fac.add_facet(d, "f", str(int(rng.integers(n_numbers + 3))))  # "12" collides with the number 12 while 12 < n_numbers
        if d % 3 == 0:
            fac.add_facet(d, "f", f"s{int(rng.integers(40))}")
    return fac


@pytest.mark.parametrize("n_docs", [200, CANDIDATES_THRESHOLD + 1])
@pytest.mark.parametrize("n_numbers", [5, 12, 30])
@pytest.mark.parametrize("max_values", [0, 1, 2, 5, 12, 13, 50, 100])
def test_caller_merge_equals_spec(n_docs, n_numbers, max_values):
    fac = collision_image(n_docs, n_numbers)
    fid = fac.fields["f"]
    for cand in (set(range(n_docs)), set(range(0, n_docs, 2))):
        nums, strs = library_entries(fac, fid, cand, max_values)
        assert caller_merge(nums, strs, max_values) == facet_values(fac, fid, cand, max_values)


def test_levels_path_after_max_numbers():
    """once the numbers reach max the strings' walk never breaks, unless its first string collides with a number"""
    n = CANDIDATES_THRESHOLD + 1
    fac = FacetImage()
    for d in range(n):
        fac.add_facet(d, "f", d % 30)
        fac.add_facet(d, "f", f"s{d % 40}")
    got = facet_values(fac, fac.fields["f"], set(range(n)), 5)
    assert [k for k, _ in got] == [str(i) for i in range(5)] + sorted(f"s{i}" for i in range(40))
    fac.add_facet(0, "f", "0")  # the first string in byte order is now "0", the Display string of the number 0
    got = facet_values(fac, fac.fields["f"], set(range(n)), 5)
    assert [k for k, _ in got] == [str(i) for i in range(5)] and got[0][1] == 1


def test_from_documents_orders_numbers_as_strings():
    fac = FacetImage()
    for d, v in enumerate([9, 10, 100, 2.5, -0.0, 1e21, 1e-7]):
        fac.add_facet(d, "n", v)
    got = facet_values(fac, fac.fields["n"], set(range(7)), 100)
    assert [k for k, _ in got] == sorted(["9", "10", "100", "2.5", "-0", "1000000000000000000000", "0.0000001"])
    assert facet_stats(fac, fac.fields["n"], set(range(7))) == (-0.0, 1e21)
    assert facet_stats(fac, fac.fields["n"], set()) is None


@pytest.mark.parametrize("x", [0.0, -0.0, 1.0, 1.5, 0.1, 1e16, 1e21, 1.2345678901234567e25, 5e-324, 1.7976931348623157e308, -3.25e-7, 123456.789])
def test_display_port(x):
    assert rust_f64_display(x) == lib_display(x)
    assert float(rust_f64_display(x)) == x and "e" not in rust_f64_display(x)
