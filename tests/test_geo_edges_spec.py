"""CPU: the edge fixtures of tests/geo_edge_fixtures.py lie where they claim, by the host formula; the specification gives NaN
distances the reference's meanings (`as usize`, the chain's `>`, take_while's `<=`); and away from the antipode the host formula
agrees with a 200-bit evaluation within its measured error."""
import math

import pytest

from tests import geo_edge_fixtures as F
from tests.geo_filter_spec import GeoFilterIndex
from tests.geo_spec import GeoIndex, GeoSort, as_usize, distance_between_two_points, haversine_a, order_model


def ulps(a, b):
    return abs(a - b) / math.ulp(b)


def test_floor_edges_straddle_whole_metres():
    pts = F.floor_edges(1, 300)
    below = [(n, h) for _, _, n, h in pts if h < n]
    above = [(n, h) for _, _, n, h in pts if h >= n]
    assert below and above
    assert all(as_usize(h) == n - 1 for n, h in below) and all(as_usize(h) == n for n, h in above if h < n + 1)
    # a few steps of a coordinate's last bit from the crossing: within nanometres of the metre
    far = max(abs(h - n) for _, _, n, h in pts)
    print(f"\nfloor edges: {len(below)} below and {len(above)} at or above their metre, at most {far:.2e} m from it")
    assert far <= 1e-6


def test_margin_edges_straddle_one_metre():
    pts = F.margin_edges(2, 100)
    split = [abs(h0 - h) > 1.0 for _, _, h0, _, h in pts]
    assert any(split) and not all(split)
    far = max(abs(abs(h0 - h) - 1.0) for _, _, h0, _, h in pts)
    print(f"\nmargin edges: {sum(split)} split, {len(split) - sum(split)} merged, |h0 - h| within {far:.2e} m of 1 m")
    assert far <= 1e-7


def test_radius_edges_straddle_the_radius():
    pts = F.radius_edges(3, 2000)
    keep = [h <= r + F.EPSILON for _, _, h, r in pts]
    assert any(keep) and not all(keep)
    for _, _, h, r in pts:
        if r == h:
            assert h <= r + F.EPSILON
        elif r == math.nextafter(h, -math.inf) and h >= 4.0:  # below 4 m, r + EPSILON can round back up to h
            assert not h <= r + F.EPSILON


def test_seam_and_poles():
    s = {(t, p): h for t, p, h in F.seam_pairs(4, 10)}
    assert s[((0.0, 180.0), (0.0, -180.0))] == 1.5604449514735575e-09  # sin(-pi rounded) != 0
    assert all(0.0 <= h < 2e-9 for h in s.values())
    assert all(0.0 <= h < 2e-9 for _, _, h in F.pole_pairs(5, 10))
    # so _geoRadius(0, 180, 0) leaves (0, -180) out
    gix = GeoIndex({0: (0.0, -180.0), 1: (0.0, 180.0)})
    assert GeoFilterIndex(None, gix, 2, 0, 1).geo_radius(0.0, 180.0, 0.0) == {1}


def test_nan_exactly_when_a_exceeds_one():
    classes = F.antipodes(6, 200)
    assert all(len(v) == 200 for v in classes.values())
    for cls, pairs in classes.items():
        for t, p in pairs:
            a, h = haversine_a(t, p), distance_between_two_points(t, p)
            assert (a > 1.0) == math.isnan(h) == (cls == ">"), (t, p, a, h)
    assert math.isnan(distance_between_two_points((8.0, 120.0), (-8.0, -60.0)))
    assert as_usize(math.nan) == 0 and as_usize(-1.0) == 0 and as_usize(3.9) == 3 and as_usize(1e30) == 2 ** 64 - 1


def test_nan_in_the_iterative_order_the_chain_and_take_while():
    t, anti = (8.0, 120.0), (-8.0, -60.0)
    pts = {0: (8.0, 121.0), 1: (8.0, 122.0), 2: anti, 3: (8.0, 120.5), 4: (-7.0, -60.0)}
    gix = GeoIndex(pts)
    # iterative: `NaN as usize` = 0, so the antipode comes first ascending and last descending
    assert order_model(gix, t, True, pts, "iterative")[0] == 2
    assert order_model(gix, t, False, pts, "iterative")[-1] == 2
    # a descending rtree bucket led by the NaN point takes every following point (NaN > 1.0 is false), up to max_bucket_size
    for cap, want in ((1000, [[0, 1, 2, 3, 4]]), (2, [[2, 4], [1], [0], [3]])):
        g = GeoSort(gix, t, False, "rtree", 1000, cap)
        left = set(pts)
        g.start_iteration(left)
        got = []
        while left:
            b, _ = g.next_bucket(left)
            got.append(b)
            left.difference_update(b)
        assert got == want, (cap, got)
    # take_while stops at the NaN point (the last in rtree order) even with a radius past the whole earth
    assert GeoFilterIndex(None, gix, 5, 0, 1).geo_radius(t[0], t[1], 2.1e7) == {0, 1, 3, 4}


def test_host_formula_against_mpmath():
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.prec = 200
    pairs = [(t, p) for t, p, _, _ in F.radius_edges(7, 1200) if 1e-3 <= distance_between_two_points(t, p) <= 1.9e7]
    worst, differ = 0.0, 0
    for t, p in pairs:
        rad = mpmath.pi / 180
        x = mpmath.sin((mpmath.mpf(p[0]) - t[0]) * rad / 2) ** 2 + mpmath.sin((mpmath.mpf(p[1]) - t[1]) * rad / 2) ** 2 * \
            mpmath.cos(mpmath.mpf(t[0]) * rad) * mpmath.cos(mpmath.mpf(p[0]) * rad)
        true = float(2 * mpmath.atan2(mpmath.sqrt(x), mpmath.sqrt(1 - x)) * F.R)
        h = distance_between_two_points(t, p)
        differ += h != true
        worst = max(worst, ulps(h, true))
    print(f"\nhost formula against 200-bit mpmath: {differ} of {len(pairs)} differ, at most {worst:.0f} ULP")
    assert differ > 0 and worst <= 32
