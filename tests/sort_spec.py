"""CPU specification of the Sort ranking rule for placeholder searches, restated from the reference (v1.50.0) and read straight
from the facet databases' byte images.  It is what the CUDA path is checked against, and deliberately does not use the
per-document key form the device works with (DESIGN.md §3):

* rule list: get_ranking_rules_for_placeholder_search + resolve_sort_criteria (search/new/mod.rs:351-416, 651-716);
* one rule: Sort::start_iteration / next_bucket (search/new/sort.rs:98-223) over ascending_facet_sort / descending_facet_sort
  (search/new/facet/facet_sort_{ascending,descending}.rs) at level 0: numbers, then strings, each bucket `&= universe`, then the
  Null bucket (what is left of the universe);
* bucket_sort (search/new/bucket_sort.rs:104-330, maybe_add_to_results :387-455): descent, offset / limit, and the two Skip
  shortcuts: a remaining universe of one document (:196-204) and a bucket of at most one document (:299-312)."""
from __future__ import annotations

import struct

import numpy as np

from oracle.pyoracle import cbo_decode


class FacetDbs:
    """level-0 entries of facet_id_f64_docids / facet_id_string_docids: per fid, [(value, docids)] in LMDB order"""

    def __init__(self, f64_db, string_db):
        self.numbers, self.strings = {}, {}
        for tab, db, is_num in ((self.numbers, f64_db, True), (self.strings, string_db, False)):
            for i in range(db.n_keys):
                k = db.key(i)
                fid, level = struct.unpack(">HB", k[:3])
                if level != 0:
                    continue
                value = struct.unpack(">d", k[11:19])[0] if is_num else k[3:].decode()
                tab.setdefault(fid, []).append((value, np.asarray(cbo_decode(db.val(i)[1:]), np.int64)))


def sort_rules(criteria, sort_list, fields):
    """criteria: names ("sort", "asc:f", "desc:f", text rules); sort_list: ["f:asc", ...] -> [(field name, fid or None, ascending)]"""
    rules, sorted_fields, sort_done = [], set(), False

    def add(name, asc):
        if name in sorted_fields:
            return
        sorted_fields.add(name)
        rules.append((name, fields.get(name), asc))

    for c in criteria:
        if c == "sort":
            if sort_done:
                continue
            sort_done = True
            for s in sort_list or []:
                f, d = s.rsplit(":", 1)
                add(f, d == "asc")
        elif c.startswith("asc:"):
            add(c[4:], True)
        elif c.startswith("desc:"):
            add(c[5:], False)
    return rules


def sort_buckets(dbs, rule, universe):
    """the buckets of one Sort rule over `universe` (a set of docids), in order: [(docids sorted, value)]"""
    name, fid, asc = rule
    left = set(universe)
    out = []
    if fid is not None:
        for tab in (dbs.numbers, dbs.strings):  # numbers before strings in both directions
            entries = tab.get(fid, [])
            for value, docids in (entries if asc else reversed(entries)):
                if not left:
                    break
                b = [int(d) for d in docids if int(d) in left]
                if b:
                    left.difference_update(b)
                    out.append((sorted(b), value))
    if left:
        out.append((sorted(left), None))
    return out


def placeholder_search(dbs, rules, universe, offset=0, limit=20, scoring="skip"):
    """bucket_sort over the sort rules of a placeholder search -> (docids, scores); scores are ("sort", field, ascending, value)"""
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

    def descend(level, univ, sc):
        remaining = len(univ)
        for bucket, value in sort_buckets(dbs, rules[level], univ):
            if len(ids) >= limit:
                return
            # top of bucket_sort's loop (:196-204): under Skip a rule whose remaining universe is one document returns it with the
            # scores of the rules above
            if scoring == "skip" and remaining == 1:
                add(bucket, sc)
                return
            remaining -= len(bucket)
            s2 = sc + [("sort", rules[level][0], rules[level][2], value)]
            if level == len(rules) - 1 or (scoring == "skip" and len(bucket) <= 1) or cur[0] + len(bucket) < offset:
                add(bucket, s2)
            else:
                descend(level + 1, bucket, s2)

    if limit > 0:
        descend(0, universe, [])
    return ids, scores


def universe_docs(n_docs, words=None):
    """docids of a dense u64 universe (None = every document below n_docs)"""
    if words is None:
        return list(range(n_docs))
    bits = np.unpackbits(np.asarray(words, np.uint64).view(np.uint8), bitorder="little")
    return [int(d) for d in np.nonzero(bits[:n_docs])[0]]
