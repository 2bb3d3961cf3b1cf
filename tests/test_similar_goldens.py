"""CPU: the Similar::execute specification (tests/similar_spec.py) against the reference's known answers
(tests/golden/similar_goldens.json, written by tests/golden/extract_similar_goldens.py from crates/meilisearch/tests/similar/mod.rs):
hit ids in order and estimatedTotalHits exactly, `_rankingScore` within 1e-6."""
import json
import operator
import os

import numpy as np

from meilisearch_b200.filter import parse_filter
from tests import similar_spec as ss

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "similar_goldens.json")
OPS = {"=": operator.eq, "<": operator.lt, ">": operator.gt, "<=": operator.le, ">=": operator.ge}


def load():
    return json.load(open(GOLDEN))


def universe(docs, flt):
    """documents_ids AND the request's filter (the goldens filter `release_year` with one comparison)"""
    if flt is None:
        return list(range(len(docs)))
    kind, field, op, (value,) = parse_filter(flt)
    assert kind == "cond" and field == "release_year"
    return [i for i, d in enumerate(docs) if OPS[op](d[field], float(value))]


def request(g, c):
    """(target docid, universe, offset, limit, threshold) of a golden case; internal docid = insertion order"""
    docs = g["documents"]
    ext = [d["id"] for d in docs]
    rq = c["request"]
    return (ext.index(str(rq["id"])), universe(docs, rq.get("filter")), rq.get("offset", 0), rq.get("limit", 20),
            rq.get("rankingScoreThreshold"))


def test_similar_goldens_on_the_spec():
    g = load()
    assert len(g["documents"]) == 5 and len(g["cases"]) == 11
    rows = np.asarray([d["vector"] for d in g["documents"]], np.float32)
    ext = [d["id"] for d in g["documents"]]
    for c in g["cases"]:
        target, u, offset, limit, thr = request(g, c)
        hits, scores, n_cand = ss.similar(rows, np.arange(len(rows)), target, u, offset=offset, limit=limit, threshold=thr, distance=ss.f64)
        assert [ext[h] for h in hits] == c["hits"], c
        if c["scores"] is not None:
            assert np.allclose(scores, c["scores"], rtol=0, atol=1e-6), (c, scores)
        if c["estimatedTotalHits"] is not None:
            assert n_cand == c["estimatedTotalHits"], (c, n_cand)


def test_spec_per_store_rule():
    """documents with several rows: store k is every document's k-th row, searched with the target's k-th row; the merged list is
    deduplicated before the skip and the take"""
    rows = np.asarray([[1, 0], [0, 1], [1, 0.1], [0.1, 1], [1, 0.2], [0.2, 1]], np.float32)
    docids = [0, 0, 1, 1, 2, 3]  # store 0: rows 0 (doc 0), 2 (doc 1), 4 (doc 2), 5 (doc 3); store 1: rows 1 (doc 0), 3 (doc 1)
    assert ss.stores(docids) == [[0, 2, 4, 5], [1, 3]]
    hits, _, n_cand = ss.similar(rows, docids, 0, range(4), limit=3, distance=ss.f64)
    # store 0 with [1, 0]: 1, 2, 3; store 1 with [0, 1]: 1; doc 1 comes back twice and counts once
    assert hits == [1, 2, 3] and n_cand == 3
    hits, _, _ = ss.similar(rows, docids, 0, range(4), offset=1, limit=1, distance=ss.f64)
    assert hits == [2]
    hits, _, _ = ss.similar(rows, docids, 2, range(4), limit=5, distance=ss.f64)  # doc 2 has one row: store 0 only
    assert hits == [1, 0, 3]
