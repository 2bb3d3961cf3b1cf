"""CPU specification of the geo filters, a literal port of IndexFilter::inner_evaluate (search/facet/filter/index_filter.rs, v1.50.0):

* `_geoRadius(lat, lng, radius)` (:465-530): the coordinates and the radius must be finite, then the latitude in [-90, 90] and the
  longitude in [-180, 180] (BadGeoError::Lat / Lng), checked before the filterable check; the result is
  `rtree.nearest_neighbor_iter(lat_lng_to_xyz(base)).take_while(distance_between_two_points(base, p) <= radius + f64::EPSILON)`,
  over the rtree order of tests/geo_spec.py's GeoIndex (squared distance, ties by docid);
* `_geoBoundingBox([top, right], [bottom, left])` (:531-696): the same range checks and BoundingBoxTopIsBelowBottom, then
  `_geo.lat BETWEEN bottom AND top` AND `_geo.lng BETWEEN left AND right` over the level-0 entries of facet_id_f64_docids, the
  longitude one split into `BETWEEN left AND 180` OR `BETWEEN -180 AND right` when right < left;
* NOT (:345-360): documents_ids minus the clause;
* `_geo` not filterable (no geo fields): `Attribute _geo/_geojson is not filterable` and the index's filterable patterns.

It deliberately does not use the prefix model the device uses (DESIGN.md §3): the radius is an ordered walk with take_while."""
from __future__ import annotations

import math

import numpy as np

from tests.geo_spec import distance_between_two_points, lat_lng_to_xyz

EPSILON = 2.220446049250313e-16
NON_FINITE = "Non finite floats are not supported"
NOT_FILTERABLE = "Attribute `_geo/_geojson` is not filterable."  # what the library returns; the caller appends the patterns


def not_filterable(patterns):
    """FilterError::AttributeNotFilterable for `_geo/_geojson` (filter/mod.rs:82-98), given the index's filterable patterns"""
    if not patterns:
        return NOT_FILTERABLE + " This index does not have configured filterable attributes."
    return NOT_FILTERABLE + " Available filterable attribute patterns are: " + ", ".join(f"`{p}`" for p in sorted(patterns)) + "."


class GeoFilterError(ValueError):
    pass


def rust_f64(v):
    """f64 as Rust's Display writes it (shortest round-trip digits, no exponent)"""
    return np.format_float_positional(v, trim="-")


def _finite(*xs):
    for x in xs:
        if not math.isfinite(x):
            raise GeoFilterError(NON_FINITE)


def _check_point(lat, lng):
    if not -90.0 <= lat <= 90.0:
        raise GeoFilterError(f"Bad latitude `{rust_f64(lat)}`. Latitude must be contained between -90 and 90 degrees.")
    if not -180.0 <= lng <= 180.0:
        norm = (lng + 180.0) % 360.0 - 180.0  # rem_euclid
        raise GeoFilterError(f"Bad longitude `{rust_f64(lng)}`. Longitude must be contained between -180 and 180 degrees. "
                             f"Hint: try using `{rust_f64(norm)}` instead.")


class GeoFilterIndex:
    """what the two geo leaves read: documents_ids, the rtree (a GeoIndex), the `_geo.lat` / `_geo.lng` number facets (FacetDbs)"""

    def __init__(self, dbs, gix, n_docs, lat_fid, lng_fid, filterable=True, other_filterable=()):
        self.dbs, self.gix, self.lat_fid, self.lng_fid, self.filterable = dbs, gix, lat_fid, lng_fid, filterable
        self.other_filterable = list(other_filterable)  # the index's filterable patterns when `_geo` is not among them
        self.documents_ids = set(range(n_docs))

    def geo_radius(self, lat, lng, radius):
        _finite(lat, lng)
        _check_point(lat, lng)
        _finite(radius)
        if not self.filterable:
            raise GeoFilterError(not_filterable(self.other_filterable))
        base = (lat, lng)
        out = set()
        for d in self.gix.nearest_neighbor_iter(lat_lng_to_xyz(base)):
            if not distance_between_two_points(base, self.gix.points[d]) <= radius + EPSILON:
                break
            out.add(d)
        return out

    def _between(self, fid, lo, hi):
        out = set()
        for value, docids in self.dbs.numbers.get(fid, []):
            if lo <= value <= hi:
                out.update(int(d) for d in docids)
        return out

    def geo_bounding_box(self, top, right, bottom, left):
        _finite(top, right, bottom, left)
        _check_point(top, right)
        _check_point(bottom, left)
        if top < bottom:
            raise GeoFilterError(f"The top latitude `{rust_f64(top)}` is below the bottom latitude `{rust_f64(bottom)}`.")
        if not self.filterable:
            raise GeoFilterError(not_filterable(self.other_filterable))
        lat = self._between(self.lat_fid, bottom, top)
        if right < left:  # the box wraps the antimeridian
            lng = self._between(self.lng_fid, left, 180.0) | self._between(self.lng_fid, -180.0, right)
        else:
            lng = self._between(self.lng_fid, left, right)
        return lat & lng

    def clause(self, kind, neg, args):
        sel = self.geo_radius(*args[:3]) if kind == 0 else self.geo_bounding_box(*args)
        return self.documents_ids - sel if neg else sel

    def filtered_universe(self, clauses, universe=None):
        """documents_ids AND universe AND every (kind, neg, args) clause"""
        out = set(self.documents_ids) if universe is None else self.documents_ids & set(universe)
        for c in clauses:
            out &= self.clause(*c)
        return out


def bitmap(n_docs, docs):
    """dense little-endian u64 words of a docid set"""
    w = np.zeros((n_docs + 63) // 64, np.uint64)
    for d in docs:
        w[d >> 6] |= np.uint64(1) << np.uint64(d & 63)
    return w
