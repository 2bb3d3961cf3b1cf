"""Seeded (target, point) pairs placed where the reference's geo decisions turn on the last bits of a haversine distance
(documents/geo_sort.rs:129 `distance as usize`, :177-180 `(d0 - d).abs() > 1.0`, index_filter.rs:493-500
`take_while(d <= radius + EPSILON)`).

Every pair is found with the host formula (tests/geo_spec.py's distance_between_two_points): one coordinate of the point is
bisected between two doubles whose distances lie on either side of the threshold, down to adjacent doubles, and the points a few
steps of nextafter around the crossing are kept.  Each record carries the host distance, so a test can say on which side the
reference puts it without recomputing."""
from __future__ import annotations

import math
import random

from tests.geo_spec import distance_between_two_points, haversine_a

EPSILON = 2.220446049250313e-16
R = 6371000.0


def _step(x, k):
    """x moved k doubles (k < 0: down)"""
    for _ in range(abs(k)):
        x = math.nextafter(x, math.inf if k > 0 else -math.inf)
    return x


def _bisect(f, lo, hi):
    """two adjacent doubles (a, b) between lo and hi with f(a) False and f(b) True, given f(lo) False and f(hi) True"""
    assert not f(lo) and f(hi)
    while True:
        mid = lo + (hi - lo) / 2.0
        if mid == lo or mid == hi:
            return lo, hi
        if f(mid):
            hi = mid
        else:
            lo = mid


def _wrap(lng):
    return lng - 360.0 if lng > 180.0 else lng + 360.0 if lng < -180.0 else lng


def _path(rng, kind):
    """(target, coordinate -> point, c_near, c_far): a path of points along which the distance from the target grows from about 0
    (c_near) to its end (c_far)"""
    if kind == "meridian":  # north along the target's meridian, near the equator (fine latitude ULPs) or near the poles
        t = (rng.choice([rng.uniform(-1.0, 1.0), rng.uniform(-89.5, -80.0), rng.uniform(60.0, 80.0)]), rng.uniform(-180.0, 180.0))
        return t, (lambda c: (c, t[1])), t[0], 90.0
    if kind == "parallel":  # east along the target's parallel, up to half a turn
        t = (rng.choice([rng.uniform(-1.0, 1.0), rng.uniform(-89.0, -85.0), rng.uniform(85.0, 89.9)]), rng.uniform(-180.0, 0.0))
        return t, (lambda c: (t[0], c)), t[1], t[1] + 180.0
    if kind == "diagonal":  # north along a meridian a few degrees east of the target
        t = (rng.uniform(-60.0, 30.0), rng.uniform(-170.0, 170.0))
        off = rng.uniform(1e-6, 10.0)
        return t, (lambda c: (c, _wrap(t[1] + off))), t[0], 90.0
    # over the pole: south along the opposite meridian, to within a centimetre of the antipode
    t = (rng.uniform(0.0, 60.0), rng.uniform(-180.0, 180.0))
    opp = t[1] - 180.0 if t[1] > 0.0 else t[1] + 180.0
    return t, (lambda c: (c, opp)), 90.0, -t[0] + 1e-7


PATHS = ("meridian", "parallel", "diagonal", "over_pole")


def _crossing(rng, kind, thr_of, steps):
    """one threshold crossing along a path of `kind`: (target, [(point, h)]) for the points `steps` nextafters around it, or
    None when the path does not reach the threshold; thr_of(h_far) picks the threshold given the path's largest distance"""
    t, at, near, far = _path(rng, kind)
    h_far = distance_between_two_points(t, at(far))
    thr = thr_of(h_far) if math.isfinite(h_far) else None
    if thr is None or not distance_between_two_points(t, at(near)) < thr <= h_far:
        return None
    a, _ = _bisect(lambda c: distance_between_two_points(t, at(c)) >= thr, near, far)
    pts = []
    for k in range(-steps + 1, steps + 1):
        p = at(_step(a, k))
        pts.append((p, distance_between_two_points(t, p)))
    return t, thr, pts


def floor_edges(seed, n, steps=4):
    """points within `steps` doubles of a whole metre n (1 m .. 2e7 m, log-uniform) -> [(target, point, n, h)]"""
    rng = random.Random(seed)
    out = []
    while len(out) < n * 2 * steps:
        kind = PATHS[len(out) // (2 * steps) % len(PATHS)]

        def thr_of(h_far):
            m = math.floor(math.exp(rng.uniform(0.0, math.log(min(h_far, 2e7)))))
            return float(max(m, 1))

        got = _crossing(rng, kind, thr_of, steps)
        if got:
            t, thr, pts = got
            out.extend((t, p, thr, h) for p, h in pts)
    return out


def margin_edges(seed, n, steps=4):
    """(target, first point, point) with the point's distance within `steps` doubles of the first's + 1 m or - 1 m
    -> [(target, p0, h0, p, h)]; the chain breaks between them when |h0 - h| > 1"""
    rng = random.Random(seed)
    out = []
    while len(out) < n * 2 * steps:
        kind = PATHS[len(out) // (2 * steps) % len(PATHS)]

        def thr_of(h_far):
            return None if h_far < 3.0 else math.exp(rng.uniform(0.0, math.log(h_far - 1.0))) + 1.0

        got = _crossing(rng, kind, thr_of, steps)
        if not got:
            continue
        t, thr, pts = got
        # p0: the two points of the target's meridian whose distances lie on either side of thr - 1
        lo_hi = _bisect(lambda c: distance_between_two_points(t, (c, t[1])) >= thr - 1.0, t[0], 90.0) if \
            distance_between_two_points(t, (90.0, t[1])) >= thr - 1.0 else None
        if lo_hi is None:
            continue
        for c in lo_hi:
            p0 = (c, t[1])
            h0 = distance_between_two_points(t, p0)
            out.extend((t, p0, h0, p, h) for p, h in pts)
    return out


def radius_edges(seed, n):
    """(target, point, h, radius): radius = h and radius = nextafter(h, -inf) for random pairs from 1 mm to the antipode, and
    sub-metre pairs with the radius stepped around the crossing of radius + EPSILON over h -> [(t, p, h, r)]"""
    rng = random.Random(seed)
    out = []
    for i in range(n):
        t = (rng.uniform(-89.0, 89.0), rng.uniform(-180.0, 180.0))
        if i % 4 == 3:  # sub-metre: a point a hair away
            dd = 10.0 ** rng.uniform(-12.0, -6.0)
            p = (t[0] + dd * rng.choice((-1.0, 1.0)), t[1])
            h = distance_between_two_points(t, p)
            if h == 0.0:
                continue
            a, b = _bisect(lambda r: r + EPSILON >= h, -1.0, h)  # r + EPSILON >= h from b on
            out.extend((t, p, h, r) for r in (_step(a, -1), a, b, _step(b, 1)))
            continue
        d = 10.0 ** rng.uniform(-3.0, math.log10(2e7))
        brg = rng.uniform(0.0, 2.0 * math.pi)
        ang = d / R
        lat1, lng1 = math.radians(t[0]), math.radians(t[1])
        lat2 = math.asin(max(-1.0, min(1.0, math.sin(lat1) * math.cos(ang) + math.cos(lat1) * math.sin(ang) * math.cos(brg))))
        lng2 = lng1 + math.atan2(math.sin(brg) * math.sin(ang) * math.cos(lat1), math.cos(ang) - math.sin(lat1) * math.sin(lat2))
        p = (math.degrees(lat2), _wrap(math.degrees(lng2)))
        h = distance_between_two_points(t, p)
        if math.isnan(h):
            continue
        out.append((t, p, h, h))
        out.append((t, p, h, math.nextafter(h, -math.inf)))
    return out


def seam_pairs(seed, n):
    """(lat, 180) and (lat, -180): the same place, at distance 0 or a few nanometres by the host formula -> [(t, p, h)]"""
    rng = random.Random(seed)
    lats = [0.0, 45.0, -45.0, 89.999, -89.999] + [rng.uniform(-90.0, 90.0) for _ in range(n)]
    out = []
    for lat in lats:
        for t, p in (((lat, 180.0), (lat, -180.0)), ((lat, -180.0), (lat, 180.0))):
            out.append((t, p, distance_between_two_points(t, p)))
    return out


def pole_pairs(seed, n):
    """points at a pole under different longitudes -> [(t, p, h)]"""
    rng = random.Random(seed)
    out = []
    for lat in (90.0, -90.0):
        lngs = [0.0, 180.0, -180.0, 90.0] + [rng.uniform(-180.0, 180.0) for _ in range(n)]
        for a in lngs[:4]:
            for b in lngs:
                out.append(((lat, a), (lat, b), distance_between_two_points((lat, a), (lat, b))))
    return out


def antipode(p):
    return (-p[0], p[1] - 180.0 if p[1] > 0.0 else p[1] + 180.0)


def antipodes(seed, n_each):
    """exact antipodal pairs by the sign of a - 1 on the host -> {">": [(t, p)], "==": [...], "<": [...]}; (8, 120) and its
    antipode lead the "> 1" class"""
    rng = random.Random(seed)
    out = {">": [((8.0, 120.0), (-8.0, -60.0))], "==": [], "<": []}
    for _ in range(200000):
        if all(len(v) >= n_each for v in out.values()):
            break
        t = (float(rng.randrange(-89, 90)) + rng.choice((0.0, 0.5, rng.random())), float(rng.randrange(-179, 180)) + rng.choice((0.0, 0.25, rng.random())))
        p = antipode(t)
        a = haversine_a(t, p)
        cls = ">" if a > 1.0 else "==" if a == 1.0 else "<"
        if len(out[cls]) < n_each:
            out[cls].append((t, p))
    return out
