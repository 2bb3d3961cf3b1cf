"""Synthetic documents for the filter tests: mixed number and string values, arrays, null, "", [], {} and missing fields, `_geo`
points; a random filter-tree generator; and a brute-force evaluation straight from the documents."""
import json
import os

import numpy as np

from corpus.facets import FacetImage, normalize_facet
from corpus.pyindexgen import IndexImage
from meilisearch_b200.filter import parse_finite_float
from tests.geo_filter_spec import GeoFilterIndex
from tests.geo_fixtures import spec_state

NUMS = [-7.5, -1.0, 0.5, 1.0, 2.0, 3.25, 10.0, 42.0, 100.0, 1e6]
STRS = ["apple", "Apple ", "banana", "cherry", "10", "2", "zz top", "éclair", "b"]
ODD = [None, "", [], {}]


def _value(rng):
    r = rng.random()
    if r < 0.35:
        return float(rng.choice(NUMS))
    if r < 0.65:
        return str(rng.choice(STRS))
    if r < 0.85:
        return [float(rng.choice(NUMS)) if rng.random() < 0.5 else str(rng.choice(STRS)) for _ in range(rng.integers(1, 4))]
    return ODD[rng.integers(0, len(ODD))]


def synthetic_docs(n_docs, seed=7):
    rng = np.random.default_rng(seed)
    docs = []
    for _ in range(n_docs):
        d = {}
        for f, p in (("n", 0.8), ("s", 0.7), ("m", 0.5)):
            if rng.random() < p:
                d[f] = _value(rng)
        if rng.random() < 0.6:
            d["flag"] = bool(rng.random() < 0.5)
        docs.append(d)
    return docs


def filter_images(docs, with_geo=True, presence=True, vocab=None):
    """(index image, facet image); text is empty (or synthetic over `vocab` words), the facet image has every field, its presence
    databases and `_geo`"""
    img = IndexImage(1)
    fac = FacetImage()
    if vocab:
        img.add_synthetic(len(docs), vocab, seed=0xB200)
    for d, doc in enumerate(docs):
        if not vocab:
            img.add_text(d, 0, "")
        for k, v in doc.items():
            fac.add_json(d, k, v)
    for f in ("n", "s", "m", "flag"):
        fac.fid(f)
    if with_geo:
        fac.add_synthetic_geo(len(docs))
    img = img.build()
    fac.build()
    if presence:
        fac.build_presence()
    return img, fac


def geo_spec(fac, n_docs):
    dbs, gix = spec_state(fac)
    return GeoFilterIndex(dbs, gix, n_docs, fac.fields["_geo.lat"], fac.fields["_geo.lng"])


# ---- random trees
def _raw(rng):
    r = rng.random()
    if r < 0.4:
        return repr(float(rng.choice(NUMS)))
    if r < 0.6:  # between and outside the values
        return repr(float(rng.choice([-100.0, -3.0, 0.75, 1.5, 5.0, 50.0, 1e7])))
    return str(rng.choice(STRS + ["a", "bz", "c", "zzz", "1", "99"]))


def random_leaf(rng, geo=True, fields=("n", "s", "m", "flag", "absent")):
    if geo and rng.random() < 0.1:
        if rng.random() < 0.5:
            return ("geo", "radius", [repr(float(x)) for x in (48.85 + rng.normal(0, 1), 2.35 + rng.normal(0, 1), rng.choice([1e3, 5e4, 2e5]))])
        lat, lng = 48.85 + rng.normal(0, 1), 2.35 + rng.normal(0, 1)
        return ("geo", "bbox", [repr(float(x)) for x in (lat + 1, lng + 1, lat - 1, lng - 1)])
    f = str(rng.choice(fields))
    op = str(rng.choice([">", ">=", "<", "<=", "TO", "=", "!=", "IN", "EXISTS", "NULL", "EMPTY"]))
    if op == "TO":
        return ("cond", f, op, [_raw(rng), _raw(rng)])
    if op == "IN":
        return ("cond", f, op, [_raw(rng) for _ in range(rng.integers(0, 5))])
    if op in ("EXISTS", "NULL", "EMPTY"):
        return ("cond", f, op, [])
    return ("cond", f, op, [_raw(rng)])


def random_tree(rng, depth, geo=True):
    if depth <= 0 or rng.random() < 0.3:
        return random_leaf(rng, geo)
    r = rng.random()
    if r < 0.2:
        return ("not", random_tree(rng, depth - 1, geo))
    return ("and" if r < 0.6 else "or", [random_tree(rng, depth - 1, geo) for _ in range(rng.integers(0, 4))])


# ---- brute force: set semantics straight from the documents (no hints, so no error reach)
def _facets(v, top=True):
    nums, strs = set(), set()
    if isinstance(v, list):
        for x in v:
            a, b = _facets(x, False)
            nums |= a
            strs |= b
    elif isinstance(v, bool):
        strs.add("true" if v else "false")
    elif isinstance(v, (int, float)):
        nums.add(float(v))
    elif isinstance(v, str) and normalize_facet(v):
        strs.add(normalize_facet(v))
    return nums, strs


def brute(docs, tree, geo=None):
    all_ids = set(range(len(docs)))
    t = tree[0]
    if t == "and":
        out = set(all_ids) if tree[1] else set()
        for c in tree[1]:
            out &= brute(docs, c, geo)
        return out
    if t == "or":
        out = set()
        for c in tree[1]:
            out |= brute(docs, c, geo)
        return out
    if t == "not":
        return all_ids - brute(docs, tree[1], geo)
    if t == "geo":
        args = [float(x) for x in tree[2]]
        return geo.geo_radius(*args) if tree[1] == "radius" else geo.geo_bounding_box(*args)
    _, f, op, vals = tree
    out = set()
    if not any(f in doc for doc in docs):  # not in the fields map: an empty bitmap whatever the operator
        return out
    for d, doc in enumerate(docs):
        if f not in doc:
            continue
        v = doc[f]
        nums, strs = _facets(v)
        if op == "EXISTS":
            hit = True
        elif op == "NULL":
            hit = v is None
        elif op == "EMPTY":
            hit = v in ("", [], {}) and not isinstance(v, bool)
        elif op in ("=", "!=", "IN"):
            hit = any(normalize_facet(r) in strs or (parse_finite_float(r) is not None and parse_finite_float(r) in nums) for r in vals)
        else:
            x = [parse_finite_float(r) for r in vals]
            s = [normalize_facet(r) for r in vals]
            lo, hi = {">": ((x[0], s[0], False), None), ">=": ((x[0], s[0], True), None), "<": (None, (x[0], s[0], False)),
                      "<=": (None, (x[0], s[0], True)), "TO": ((x[0], s[0], True), (x[-1], s[-1], True))}[op]
            num_ok = all(b is None or b[0] is not None for b in (lo, hi))

            def inside(val, i):
                if lo is not None and not (val > lo[i] or (lo[2] and val == lo[i])):
                    return False
                return hi is None or val < hi[i] or (hi[2] and val == hi[i])

            hit = (num_ok and any(inside(n, 0) for n in nums)) or any(inside(sv, 1) for sv in strs)
        if op == "!=":
            hit = not hit
        if hit:
            out.add(d)
    if op == "!=":
        out |= all_ids - {d for d, doc in enumerate(docs) if f in doc}
    return out


# ---- the reference's known answers (tests/golden/filter_goldens.json)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "filter_goldens.json")


def load_filter_goldens():
    return json.load(open(GOLDEN))


def golden_images(g):
    """test_set.ndjson through milli's facet extraction (nested objects included) for the filterable attributes; empty text"""
    img = IndexImage(1)
    fac = FacetImage()
    for d, doc in enumerate(g["docs"]):
        img.add_text(d, 0, "")
        fac.add_document(d, doc, g["filterable"])
    for name in g["filterable"]:
        if name != "_geo":
            fac.fid(name)
    img = img.build()
    fac.build()
    fac.build_presence()
    return img, fac


def golden_tree(filters):
    """Filter::from_array: an AND of the entries, each a filter string or an OR of filter strings"""
    from meilisearch_b200.filter import parse_filter

    parts = [("or", [parse_filter(x) for x in e]) if isinstance(e, list) else parse_filter(e) for e in filters]
    return parts[0] if len(parts) == 1 else ("and", parts)
