"""CPU specification of the GeoSort ranking rule for placeholder searches, a literal port of the reference (v1.50.0):

* GeoSort::start_iteration / next_bucket (search/new/geo_sort.rs:77-160) over documents/geo_sort.rs: fill_cache (:66-134) with its
  rtree and iterative strategies, next_bucket (:137-228) with the cache, its refills and the put-back of the point that breaks a
  bucket, opposite_of (:280-290);
* distance_between_two_points / lat_lng_to_xyz (lib.rs:388-404), haversine as geoutils computes it (R = 6371000 m);
* composed with the field rules of sort_spec.py and bucket_sort's descent, offset / limit and Skip shortcuts.

The rtree's nearest_neighbor_iter is the points in ascending squared distance (rstar's distance_2), ties in ascending docid (rstar's
own tie order is not pinned).  It deliberately does not use the tuple-order model the device uses (DESIGN.md §3)."""
from __future__ import annotations

import math
from collections import deque

from tests.sort_spec import sort_buckets

GEO_STRATEGIES = ("dynamic", "iterative", "rtree")


def f64_sqrt(x):
    """f64::sqrt: NaN for a negative number (or NaN) instead of a domain error"""
    return math.sqrt(x) if x >= 0.0 else math.nan


def haversine_a(a, b):
    """the haversine's `a` term, as geoutils rounds it; it exceeds 1 by an ULP for some antipodal pairs"""
    d_lat = math.radians(b[0] - a[0])
    d_lon = math.radians(b[1] - a[1])
    lat1, lat2 = math.radians(a[0]), math.radians(b[0])
    return math.sin(d_lat / 2.0) * math.sin(d_lat / 2.0) + math.sin(d_lon / 2.0) * math.sin(d_lon / 2.0) * math.cos(lat1) * math.cos(lat2)


def distance_between_two_points(a, b):
    """Location::haversine_distance_to (geoutils) in metres, from a to b, with f64 semantics: a > 1 gives NaN"""
    x = haversine_a(a, b)
    return 2.0 * math.atan2(f64_sqrt(x), f64_sqrt(1.0 - x)) * 6371000.0


def as_usize(d):
    """Rust's `d as usize` on an f64: truncation, saturating at 0 (negatives, NaN) and at usize::MAX"""
    if math.isnan(d) or d <= 0.0:
        return 0
    return min(int(d), 2 ** 64 - 1)


def lat_lng_to_xyz(p):
    lat, lng = math.radians(p[0]), math.radians(p[1])
    return (math.cos(lat) * math.cos(lng), math.cos(lat) * math.sin(lng), math.sin(lat))


def opposite_of(p):
    lat, lng = p
    return (-lat, lng - 180.0 if lng > 0.0 else lng + 180.0)


def distance_2(a, b):
    """rstar PointExt::distance_2: the components' squares summed in order"""
    acc = 0.0
    for x, y in zip(a, b):
        acc = (x - y) * (x - y) + acc
    return acc


class GeoIndex:
    """what GeoSort reads from an index: geo_faceted_documents_ids and every geo document's point (and its rtree xyz)"""

    def __init__(self, points):
        self.points = dict(points)  # docid -> (lat, lng)
        self.xyz = {d: lat_lng_to_xyz(p) for d, p in self.points.items()}
        self._nn = {}

    def nearest_neighbor_iter(self, q):
        if q not in self._nn:
            self._nn[q] = sorted(self.points, key=lambda d: (distance_2(self.xyz[d], q), d))
        return self._nn[q]


class GeoSort:
    """one GeoSort rule: target point, direction, GeoSortParameter"""

    def __init__(self, gix, target, ascending, strategy="dynamic", cache_size=1000, max_bucket_size=1000, distance_error_margin=1.0):
        self.gix, self.point, self.ascending = gix, tuple(target), ascending
        self.strategy, self.cache_size = strategy, cache_size
        self.max_bucket_size, self.distance_error_margin = max_bucket_size, distance_error_margin
        self.geo_candidates = set(gix.points)
        self.cached_sorted_docids = deque()

    def use_rtree(self, candidates):
        return self.strategy == "rtree" or (self.strategy == "dynamic" and candidates >= self.cache_size)

    def fill_cache(self, geo_candidates):
        cache = self.cached_sorted_docids
        assert not cache
        if self.use_rtree(len(geo_candidates)):
            if self.ascending:
                for d in self.gix.nearest_neighbor_iter(lat_lng_to_xyz(self.point)):
                    if d in geo_candidates:
                        cache.append((d, self.gix.points[d]))
                        if len(cache) >= self.cache_size:
                            break
            else:
                for d in self.gix.nearest_neighbor_iter(lat_lng_to_xyz(opposite_of(self.point))):
                    if d in geo_candidates:
                        cache.appendleft((d, self.gix.points[d]))
                        if len(cache) >= self.cache_size:
                            break
        else:
            documents = [(d, self.gix.points[d]) for d in sorted(geo_candidates)]
            documents.sort(key=lambda x: as_usize(distance_between_two_points(self.point, x[1])))  # stable: docid order within a metre
            cache.extend(documents)

    def start_iteration(self, universe):
        self.cached_sorted_docids.clear()
        geo_candidates = self.geo_candidates & set(universe)
        if not geo_candidates:
            return
        self.fill_cache(geo_candidates)

    def next_bucket(self, universe):
        """-> (bucket docids, value): value is the bucket's first point, None for what is left without geo"""
        geo_candidates = self.geo_candidates & set(universe)
        if not geo_candidates:
            return sorted(universe), None
        cache = self.cached_sorted_docids
        nxt = cache.popleft if self.ascending else cache.pop
        put_back = cache.appendleft if self.ascending else cache.append
        current_bucket = []
        current_distance = None
        while True:
            if cache:
                docid, point = nxt()
                if docid in geo_candidates:
                    distance = distance_between_two_points(self.point, point)
                    if current_distance is not None:
                        point0, bucket_distance = current_distance
                        if abs(bucket_distance - distance) > self.distance_error_margin:
                            put_back((docid, point))
                            return sorted(current_bucket), point0
                        current_bucket.append(docid)
                        geo_candidates.discard(docid)
                        if len(current_bucket) == self.max_bucket_size:
                            return sorted(current_bucket), point0
                    else:
                        current_distance = (point, distance)
                        current_bucket.append(docid)
                        geo_candidates.discard(docid)
                        if len(current_bucket) == self.max_bucket_size:
                            return sorted(current_bucket), point
            else:
                self.fill_cache(geo_candidates)
                if not cache:
                    if current_distance is not None:
                        return sorted(current_bucket), current_distance[0]
                    return sorted(universe), None


def parse_sort_entry(s):
    """"_geoPoint(lat, lng):asc" -> ("geo", (lat, lng), True); "field:desc" -> (field, None, False)"""
    name, d = s.rsplit(":", 1)
    if name.startswith("_geoPoint("):
        lat, lng = name[len("_geoPoint("):-1].split(",")
        return ("geo", (float(lat), float(lng)), d == "asc")
    return (name, None, d == "asc")


def sort_rules(criteria, sort_list, fields):
    """search/new/mod.rs:651-716 resolve_sort_criteria: a GeoSort rule per `_geoPoint` entry (never deduplicated), field rules as in
    sort_spec.sort_rules -> [("geo", (lat, lng), asc) | (field, fid or None, asc)]"""
    rules, sorted_fields, done = [], set(), False

    def add(name, asc):
        if name not in sorted_fields:
            sorted_fields.add(name)
            rules.append((name, fields.get(name), asc))

    for c in criteria:
        if c == "sort" and not done:
            done = True
            for s in sort_list or []:
                kind, point, asc = parse_sort_entry(s)
                if kind == "geo":
                    rules.append(("geo", point, asc))
                else:
                    add(kind, asc)
        elif c.startswith("asc:"):
            add(c[4:], True)
        elif c.startswith("desc:"):
            add(c[5:], False)
    return rules


def placeholder_search(dbs, gix, rules, universe, offset=0, limit=20, scoring="skip", strategy="dynamic", cache_size=1000,
                       max_bucket_size=1000):
    """bucket_sort over the rules of a placeholder search -> (docids, scores); scores are ("geo", ascending, point | None) and
    ("sort", field, ascending, value)"""
    universe = sorted(universe)
    if not rules:
        return universe[offset: offset + limit], [[] for _ in universe[offset: offset + limit]]
    ids, scores = [], []
    cur = [0]

    def add(bucket, sc):
        if cur[0] < offset:
            if cur[0] + len(bucket) < offset:
                cur[0] += len(bucket)
                return
            take = bucket[offset - cur[0]:][: limit - len(ids)]
        else:
            take = bucket[: limit - len(ids)]
        ids.extend(take)
        scores.extend([list(sc)] * len(take))
        cur[0] += len(bucket)

    def buckets(level, univ):
        """the rule's buckets, each one asked for with the universe left after the previous ones (bucket_sort.rs:298)"""
        rule = rules[level]
        if rule[0] != "geo":
            for bucket, value in sort_buckets(dbs, rule, univ):
                yield bucket, ("sort", rule[0], rule[2], value)
            return
        g = GeoSort(gix, rule[1], rule[2], strategy, cache_size, max_bucket_size)
        left = set(univ)
        g.start_iteration(left)
        while left:
            bucket, value = g.next_bucket(left)
            left.difference_update(bucket)
            yield bucket, ("geo", rule[2], value)

    def descend(level, univ, sc):
        remaining = len(univ)
        for bucket, score in buckets(level, univ):
            if len(ids) >= limit:
                return
            if scoring == "skip" and remaining == 1:  # bucket_sort.rs:196-204
                add(bucket, sc)
                return
            remaining -= len(bucket)
            s2 = sc + [score]
            if level == len(rules) - 1 or (scoring == "skip" and len(bucket) <= 1) or cur[0] + len(bucket) < offset:
                add(bucket, s2)
            else:
                descend(level + 1, bucket, s2)

    if limit > 0:
        descend(0, universe, [])
    return ids, scores


def order_model(gix, target, ascending, universe, strategy="dynamic", cache_size=1000):
    """the order in which the rule hands out G = universe AND geo, evaluated directly (DESIGN.md §3): the first m documents in rtree
    order (ascending squared distance to the target, or to its antipode when descending; ties by docid), then the rest in
    iterative order (floor metres, docid), reversed when descending; m = n (rtree), 0 (iterative), n - n mod c when n >= c else 0"""
    g = sorted(set(universe) & set(gix.points))
    n = len(g)
    m = n if strategy == "rtree" else 0 if strategy == "iterative" else (n - n % cache_size if n >= cache_size else 0)
    q = lat_lng_to_xyz(target if ascending else opposite_of(target))
    rt = sorted(g, key=lambda d: (distance_2(gix.xyz[d], q), d))
    head, tail = rt[:m], sorted(rt[m:])
    tail.sort(key=lambda d: as_usize(distance_between_two_points(target, gix.points[d])))
    return head + (tail if ascending else tail[::-1])
