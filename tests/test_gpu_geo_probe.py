"""GPU: the device's geo functions (geo_math.cuh) against the host formula of the reference, over random pairs and the edge sets of
tests/geo_edge_fixtures.py.  rtree keys must be identical bit for bit; the haversine may differ by a few ULP (the device's sin /
atan2 are not glibc's), and wherever that difference could change a decision (a whole metre, a radius) the device must call the
distance ambiguous, so the host decides it.  The measured error is printed (pytest -s) and bounded by GEO_TAU with a 4x margin."""
import ctypes
import math
import os
import random
import subprocess

import numpy as np
import pytest

from tests import geo_edge_fixtures as F
from tests.geo_spec import as_usize, distance_2, distance_between_two_points, lat_lng_to_xyz, opposite_of

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 6371000.0
GEO_FLOOR_MAX = (1 << 25) - 1


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    out = tmp_path_factory.mktemp("geo_probe") / "geo_probe.so"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
                           "-I", os.path.join(ROOT, "meilisearch_b200", "csrc"), os.path.join(ROOT, "tests", "cuda", "geo_probe.cu"),
                           "-o", str(out)])
    lib = ctypes.CDLL(str(out))
    lib.geo_probe_tau.restype = ctypes.c_double
    lib.geo_probe_antipode_m.restype = ctypes.c_double
    return lib


def run(lib, pairs, thr=None, rtree_targets=None):
    """pairs [(target, point)] -> dict of device arrays"""
    n = len(pairs)
    t = np.array([(a[0], a[1], math.cos(math.radians(a[0]))) for a, _ in pairs], np.float64)
    p = np.array([lat_lng_to_xyz(b) + (b[0], b[1], math.cos(math.radians(b[0]))) for _, b in pairs], np.float64)
    q = np.array([lat_lng_to_xyz(a) for a, _ in pairs] if rtree_targets is None else rtree_targets, np.float64)
    th = np.zeros(n) if thr is None else np.asarray(thr, np.float64)
    out = {"m": np.zeros(n), "c1": np.zeros(n), "floor": np.zeros(n, np.uint32), "amb_floor": np.zeros(n, np.uint8),
           "amb_thr": np.zeros(n, np.uint8), "key": np.zeros(n, np.uint64)}
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = lib.geo_probe(ctypes.c_int(n), ptr(t), ptr(p), ptr(q), ptr(th), ptr(out["m"]), ptr(out["c1"]), ptr(out["floor"]),
                       ptr(out["amb_floor"]), ptr(out["amb_thr"]), ptr(out["key"]))
    assert rc == 0
    return out


def random_pairs(seed, n):
    """pairs from 1 mm to the antipode (log-uniform distance, uniform bearing), plus uniform random pairs"""
    rng = random.Random(seed)
    out = []
    for i in range(n):
        t = (rng.uniform(-90.0, 90.0), rng.uniform(-180.0, 180.0))
        if i % 2:
            out.append((t, (rng.uniform(-90.0, 90.0), rng.uniform(-180.0, 180.0))))
            continue
        ang = 10.0 ** rng.uniform(-3.0, math.log10(math.pi * R)) / R
        brg = rng.uniform(0.0, 2.0 * math.pi)
        la1, ln1 = math.radians(t[0]), math.radians(t[1])
        la2 = math.asin(max(-1.0, min(1.0, math.sin(la1) * math.cos(ang) + math.cos(la1) * math.sin(ang) * math.cos(brg))))
        ln2 = ln1 + math.atan2(math.sin(brg) * math.sin(ang) * math.cos(la1), math.cos(ang) - math.sin(la1) * math.sin(la2))
        lng = math.degrees(ln2)
        lng = lng - 360.0 if lng > 180.0 else lng + 360.0 if lng < -180.0 else lng
        out.append((t, (math.degrees(la2), lng)))
    return out


def edge_pairs():
    out = [(t, p) for t, p, _, _ in F.floor_edges(21, 400)]
    out += [(t, p) for t, _, _, p, _ in F.margin_edges(22, 100)]
    out += [(t, p) for t, p, _, _ in F.radius_edges(23, 800)]
    out += [(t, p) for t, p, _ in F.seam_pairs(24, 50)] + [(t, p) for t, p, _ in F.pole_pairs(25, 20)]
    for v in F.antipodes(26, 300).values():
        out += v
    return out


def host_floor(h):
    return min(as_usize(h), GEO_FLOOR_MAX)


def error_units(dev, host, c1_host):
    """|device - host| over max(h, 1) + R / sqrt(1 - a), the scale of geo_ambiguous's tolerance"""
    return abs(dev - host) / (max(host, 1.0) + R / c1_host)


def test_rtree_key_is_bit_identical(probe):
    pairs = random_pairs(1, 50_000) + edge_pairs()
    rng = random.Random(2)
    # ascending targets, and descending ones (the antipode of the target by opposite_of)
    qs = [lat_lng_to_xyz(t if rng.random() < 0.5 else opposite_of(t)) for t, _ in pairs]
    got = run(probe, pairs, rtree_targets=qs)["key"]
    want = np.array([np.float64(distance_2(lat_lng_to_xyz(p), q)).view(np.uint64) for (_, p), q in zip(pairs, qs)], np.uint64)
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, [(pairs[i], int(got[i]), int(want[i])) for i in bad[:5]]


def test_haversine_error_and_ambiguity(probe):
    tau, antipode_m = probe.geo_probe_tau(), probe.geo_probe_antipode_m()
    pairs = random_pairs(3, 100_000) + edge_pairs()
    out = run(probe, pairs)
    hist, worst, worst_units = {}, 0, 0.0
    missed = []
    for i, (t, p) in enumerate(pairs):
        h, d = distance_between_two_points(t, p), float(out["m"][i])
        if math.isnan(h) or h > antipode_m:  # the device must leave these to the host
            assert out["amb_floor"][i], (t, p, h, d)
            continue
        ulps = 0 if d == h else round(abs(d - h) / math.ulp(h)) if h > 0 else -1
        hist[ulps] = hist.get(ulps, 0) + 1
        if h >= 1e-3:
            worst = max(worst, ulps)
        a = F.haversine_a(t, p)
        worst_units = max(worst_units, error_units(d, h, math.sqrt(1.0 - a)))
        if int(out["floor"][i]) != host_floor(h) and not out["amb_floor"][i]:
            missed.append((t, p, h, d))
    print(f"\nhaversine |device - host| in ULP of the host value, {len(pairs)} pairs: "
          + ", ".join(f"{k}: {v}" for k, v in sorted(hist.items())))
    print(f"largest error over (max(h, 1) + R / sqrt(1 - a)): {worst_units:.3e} = {worst_units / 2.0**-52:.2f} x 2^-52; "
          f"GEO_TAU = {tau:.3e}, margin {tau / max(worst_units, 1e-300):.1f}x")
    assert not missed, missed[:5]
    assert worst_units * 4.0 <= tau
    assert worst <= 64  # the ULP histogram above: a few ULP away from the antipode


def test_ambiguity_covers_every_floor_and_radius_edge(probe):
    # the floor of every edge point, and radii equal to a distance and one double below it: where the device's decision differs
    # from the host's, the device must flag the distance
    fe = F.floor_edges(31, 600)
    re = F.radius_edges(32, 1500)
    pairs = [(t, p) for t, p, _, _ in fe] + [(t, p) for t, p, _, _ in re]
    thr = [float(n) for _, _, n, _ in fe] + [r + F.EPSILON for _, _, _, r in re]
    out = run(probe, pairs, thr=thr)
    differ = flagged = 0
    for i, (t, p) in enumerate(pairs):
        h, d = distance_between_two_points(t, p), float(out["m"][i])
        if i < len(fe):
            if int(out["floor"][i]) != host_floor(h):
                differ += 1
                assert out["amb_floor"][i], (t, p, h, d)
        elif (d <= thr[i]) != (h <= thr[i]):
            differ += 1
            assert out["amb_thr"][i], (t, p, h, d, thr[i])
        flagged += int(out["amb_floor"][i] if i < len(fe) else out["amb_thr"][i])
    print(f"\nedge decisions the device alone would take differently: {differ} of {len(pairs)}; flagged ambiguous: {flagged}")


def test_seam_poles_antipodes_recorded(probe):
    sets = {"seam": [(t, p) for t, p, _ in F.seam_pairs(41, 20)], "poles": [(t, p) for t, p, _ in F.pole_pairs(42, 10)]}
    for k, v in F.antipodes(43, 100).items():
        sets[f"antipodes a {k} 1"] = v
    for name, pairs in sets.items():
        out = run(probe, pairs)
        host = [distance_between_two_points(t, p) for t, p in pairs]
        same = sum(1 for h, d in zip(host, out["m"]) if h == d or (math.isnan(h) and math.isnan(d)))
        print(f"\n{name}: {len(pairs)} pairs, device == host bit for bit in {same}, device NaN in {int(np.isnan(out['m']).sum())},"
              f" host NaN in {sum(map(math.isnan, host))}, floors {sorted(set(out['floor'].tolist()))[:4]}")
        for i, h in enumerate(host):
            if math.isnan(out["m"][i]):
                assert out["floor"][i] == 0  # `NaN as usize`
            if host_floor(h) != int(out["floor"][i]):
                assert out["amb_floor"][i], (pairs[i], h, out["m"][i])


def test_host_formula_against_mpmath_on_device_subset(probe):
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.prec = 200
    pairs = random_pairs(5, 400)
    out = run(probe, pairs)
    worst_dev = worst_host = 0
    for i, (t, p) in enumerate(pairs):
        h = distance_between_two_points(t, p)
        if math.isnan(h) or h < 1e-3 or h > math.pi * R - 1.0:
            continue
        rad = mpmath.pi / 180
        x = mpmath.sin((mpmath.mpf(p[0]) - t[0]) * rad / 2) ** 2 + mpmath.sin((mpmath.mpf(p[1]) - t[1]) * rad / 2) ** 2 * \
            mpmath.cos(mpmath.mpf(t[0]) * rad) * mpmath.cos(mpmath.mpf(p[0]) * rad)
        true = float(2 * mpmath.atan2(mpmath.sqrt(x), mpmath.sqrt(1 - x)) * R)
        worst_host = max(worst_host, abs(h - true) / math.ulp(true))
        worst_dev = max(worst_dev, abs(float(out["m"][i]) - true) / math.ulp(true))
    print(f"\nagainst 200-bit mpmath: host up to {worst_host:.0f} ULP, device up to {worst_dev:.0f} ULP")
    assert worst_host <= 64 and worst_dev <= 64
