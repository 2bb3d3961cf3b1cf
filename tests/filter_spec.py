"""CPU specification of facet filters: IndexFilter::inner_evaluate (search/facet/filter/index_filter.rs:332-696, v1.50.0) restated node
by node, universe hints and the reach of errors included, and read from the facet databases' byte images:

* inner_evaluate returns an empty bitmap, evaluating nothing, when its hint is Some(empty);
* NOT: hint - x, or documents_ids - x without a hint; OR: the union, every child with the OR's hint; AND: the first child with the
  AND's hint, then each next child with Some(running bitmap), stopping as soon as the running bitmap is empty; AND of nothing: empty;
* a condition on a field absent from the fields map: empty; a DENIED feature (FilterableAttributesFeatures): the error, raised when
  evaluation reaches it (an IN over no values never calls evaluate_operator, so it never raises);
* ranges (ValueBounds::new, explore_facet_levels :287-321, find_docids_of_facet_within_bounds): the number part (Excluded / Included
  of the value and f64::MAX / f64::MIN) when the bound parses, over the 16-byte OrderedF64 keys, and the string part over the
  normalised key bytes; the inverted-interval checks compare the f64 / String values; the result is intersected with the hint;
* EQUAL / IN / NOT_EQUAL: evaluate_equal (value_bounds.rs), exact keys, no hint; EXISTS / IS NULL / IS EMPTY: the presence databases;
* geo leaves: tests/geo_filter_spec.py, whose argument errors, and `_geo` not being filterable, are raised when reached; a bounding
  box is intersected with its hint (it is evaluated as two Between conditions, index_filter.rs:586-660).

It deliberately does not use the ordinal intervals the device uses (DESIGN.md §3 "Facet filters")."""
from __future__ import annotations

import struct
import sys

from corpus.facets import normalize_facet, ordered_f64
from meilisearch_b200.filter import parse_filter, parse_finite_float
from oracle.pyoracle import cbo_decode
from tests.geo_filter_spec import GeoFilterError, GeoFilterIndex

F64_MAX = sys.float_info.max
FEATURE = {">": "comparison", ">=": "comparison", "<": "comparison", "<=": "comparison", "TO": "comparison", "=": "equality",
           "!=": "equality", "IN": "equality", "EXISTS": "exists", "NULL": "null", "EMPTY": "empty"}


class FilterError(Exception):
    """a leaf's error; leaf = its pre-order index"""

    def __init__(self, leaf, msg):
        super().__init__(msg)
        self.leaf = leaf


class Unsupported(Exception):
    """a node outside the implemented scope; leaf = its pre-order index"""

    def __init__(self, leaf, what):
        super().__init__(what)
        self.leaf = leaf


def _level0(db):
    out = {}
    for i in range(db.n_keys):
        k = db.key(i)
        fid, level = struct.unpack(">HB", k[:3])
        if level == 0:
            out.setdefault(fid, []).append((k[3:], set(cbo_decode(db.val(i)[1:]))))
    return out


def _presence(db):
    return None if db is None else {struct.unpack(">H", db.key(i))[0]: set(cbo_decode(db.val(i))) for i in range(db.n_keys)}


def _index(tree, at=0):
    """(pre-order index, node, indexed children) -> and the next index"""
    if tree[0] in ("and", "or"):
        kids, nxt = [], at + 1
        for c in tree[1]:
            k, nxt = _index(c, nxt)
            kids.append(k)
        return (at, tree, kids), nxt
    if tree[0] == "not":
        k, nxt = _index(tree[1], at + 1)
        return (at, tree, [k]), nxt
    return (at, tree, []), at + 1


def _in_bounds(key, lo, hi):
    (lk, lv), (hk, hv) = lo, hi
    if lk == "inc" and key < lv or lk == "exc" and key <= lv:
        return False
    if hk == "inc" and key > hv or hk == "exc" and key >= hv:
        return False
    return True


def _inverted(lo, hi):
    (lk, lv), (hk, hv) = lo, hi
    if lk == "unb" or hk == "unb":
        return False
    return lv > hv if (lk, hk) == ("inc", "inc") else lv >= hv


class FilterSpec:
    """facets: a FacetImage after build() (and build_presence() for EXISTS / IS NULL / IS EMPTY); geo: a GeoFilterIndex or None
    (`_geo` not filterable); documents_ids: a set of docids"""

    def __init__(self, facets, documents_ids, geo=None):
        self.fields = dict(facets.fields)
        self.numbers, self.strings = _level0(facets.f64_db), _level0(facets.string_db)
        self.presence = [_presence(getattr(facets, n, None)) for n in ("exists_db", "null_db", "empty_db")]
        self.documents_ids = set(documents_ids)
        self.geo = geo
        self.no_geo = GeoFilterIndex(None, None, 0, None, None, filterable=False)  # validates, then refuses

    def evaluate(self, tree, denied=()):
        """IndexFilter::evaluate -> the docids; raises FilterError (the reached leaf), Unsupported, or FilterError for the checks the
        caller and the library make up front (a missing presence database)"""
        if isinstance(tree, str):
            tree = parse_filter(tree)
        root, _ = _index(tree)
        self.denied = set(denied)
        self._upfront(root)
        return self._eval(root, None)

    def _upfront(self, n):
        at, t, kids = n
        if t[0] == "geo":
            if t[1] not in ("radius", "bbox"):
                raise Unsupported(at, t[1])
        elif t[0] == "cond":
            _, field, op, _ = t
            if field == "_shard" or field == "_vectors" or field.startswith("_vectors.") or op in ("CONTAINS", "STARTS_WITH"):
                raise Unsupported(at, op)
            k = {"EXISTS": 0, "NULL": 1, "EMPTY": 2}.get(op)
            if k is not None and field in self.fields and (field, FEATURE[op]) not in self.denied and self.presence[k] is None:
                raise FilterError(at, "presence database not staged")
        for c in kids:
            self._upfront(c)

    def _eval(self, n, hint):
        if hint is not None and not hint:
            return set()
        at, t, kids = n
        if t[0] == "not":
            sel = self._eval(kids[0], hint)
            return (hint if hint is not None else self.documents_ids) - sel
        if t[0] == "or":
            out = set()
            for c in kids:
                out |= self._eval(c, hint)
            return out
        if t[0] == "and":
            if not kids:
                return set()
            bm = self._eval(kids[0], hint)
            for c in kids[1:]:
                if not bm:
                    return bm
                bm = bm & self._eval(c, bm)
            return bm
        if t[0] == "geo":  # the arguments are checked before `_geo` is found not filterable, both only when reached
            args = [float(x) for x in t[2]]
            geo = self.geo or self.no_geo
            try:
                sel = geo.geo_radius(*args) if t[1] == "radius" else geo.geo_bounding_box(*args)
            except GeoFilterError as e:
                raise FilterError(at, str(e))
            # a bounding box is two Between conditions on _geo.lat / _geo.lng evaluated under the hint (index_filter.rs:586-660)
            return sel & hint if t[1] == "bbox" and hint is not None else sel
        _, field, op, vals = t
        if field not in self.fields:
            return set()
        if (field, FEATURE[op]) in self.denied:
            if op == "IN" and not vals:
                return set()
            raise FilterError(at, f"{field}: {FEATURE[op]} not allowed")
        fid = self.fields[field]
        if op in (">", ">=", "<", "<=", "TO"):
            return self._range(fid, op, vals, hint)
        if op == "=":
            return self._equal(fid, vals[0])
        if op == "!=":
            return self.documents_ids - self._equal(fid, vals[0])
        if op == "IN":
            out = set()
            for v in vals:
                out |= self._equal(fid, v)
            return out
        return set(self.presence[{"EXISTS": 0, "NULL": 1, "EMPTY": 2}[op]].get(fid, ()))

    def _equal(self, fid, raw):
        s, x = normalize_facet(raw).encode(), parse_finite_float(raw)
        out = set()
        for key, docs in self.strings.get(fid, []):
            if key == s:
                out |= docs
        if x is not None:
            for key, docs in self.numbers.get(fid, []):
                if key == ordered_f64(x):
                    out |= docs
        return out

    def _range(self, fid, op, vals, hint):
        # ValueBounds::new
        x = [parse_finite_float(v) for v in vals]
        s = [normalize_facet(v) for v in vals]
        if op == ">":
            num = (("exc", x[0]), ("inc", F64_MAX)) if x[0] is not None else None
            st = (("exc", s[0]), ("unb", None))
        elif op == ">=":
            num = (("inc", x[0]), ("inc", F64_MAX)) if x[0] is not None else None
            st = (("inc", s[0]), ("unb", None))
        elif op == "<":
            num = (("inc", -F64_MAX), ("exc", x[0])) if x[0] is not None else None
            st = (("unb", None), ("exc", s[0]))
        elif op == "<=":
            num = (("inc", -F64_MAX), ("inc", x[0])) if x[0] is not None else None
            st = (("unb", None), ("inc", s[0]))
        else:
            num = (("inc", x[0]), ("inc", x[1])) if x[0] is not None and x[1] is not None else None
            st = (("inc", s[0]), ("inc", s[1]))
        out = set()
        if num is not None and not _inverted(*num):  # explore_facet_levels compares the f64s, the search the key bytes
            lo, hi = ((k, None if v is None else ordered_f64(v)) for k, v in num)
            for key, docs in self.numbers.get(fid, []):
                if _in_bounds(key, lo, hi):
                    out |= docs
        if not _inverted(*st):
            lo, hi = ((k, None if v is None else v.encode()) for k, v in st)
            for key, docs in self.strings.get(fid, []):
                if _in_bounds(key, lo, hi):
                    out |= docs
        return out & hint if hint is not None else out
