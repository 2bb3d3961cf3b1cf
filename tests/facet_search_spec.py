"""CPU specification of facet search: a literal port of SearchForFacetValues::inner_execute and ValuesCollection
(crates/milli/src/search/facet/search.rs:119-353) over the staged byte databases (corpus/facets.py formats).  Independent of the
library: the Levenshtein prefix test is written from its definition, the minimum OSA distance between the query and a prefix of the
string, over Unicode scalar values."""
import heapq
import json
import struct


def osa_prefix_distance(q, w):
    """min over the prefixes p of w of the restricted Damerau-Levenshtein (optimal string alignment) distance OSA(q, p)"""
    m, n = len(q), len(w)
    d = [[0] * (n + 1) for _ in range(m + 1)]
    for i in range(m + 1):
        d[i][0] = i
    for j in range(n + 1):
        d[0][j] = j
    for i in range(1, m + 1):
        for j in range(1, n + 1):
            v = min(d[i - 1][j] + 1, d[i][j - 1] + 1, d[i - 1][j - 1] + (q[i - 1] != w[j - 1]))
            if i > 1 and j > 1 and q[i - 1] == w[j - 2] and q[i - 2] == w[j - 1]:
                v = min(v, d[i - 2][j - 2] + 1)
            d[i][j] = v
    return min(d[m])


def typo_budget(query, one_typo=5, two_typos=9):
    """search.rs:163-171: by the query's length in bytes"""
    n = len(query.encode())
    return 0 if n < one_typo else 1 if n < two_typos else 2


class ValuesCollection:
    """search.rs:292-353.  Hits are (value, count); Ord is (count, value as bytes)."""

    def __init__(self, order, max_values):
        self.order, self.max, self.content = order, max_values, []

    def insert(self, value, count):
        """-> True for ControlFlow::Break"""
        if self.order == "alpha":
            if len(self.content) < self.max:
                self.content.append((value, count))
                if len(self.content) < self.max:
                    return False
            return True
        item = (count, value.encode(), value)
        if len(self.content) == self.max:
            if not self.content:
                return True  # peek_mut on an empty heap
            if self.content[0][0] <= count:
                heapq.heapreplace(self.content, item)
        else:
            heapq.heappush(self.content, item)
        return False

    def into_sorted_vec(self):
        if self.order == "alpha":
            return list(self.content)
        return [(v, c) for c, _, v in sorted(self.content, reverse=True)]


def decode_cbo(b):
    """CboRoaringBitmapCodec bytes -> docids: raw u32s up to 28 bytes, else the portable roaring format without run containers"""
    if len(b) <= 28:
        return list(struct.unpack(f"<{len(b) // 4}I", b))
    cookie, n = struct.unpack("<II", b[:8])
    assert cookie == 12346
    at, out = 8 + 8 * n, []
    for c in range(n):
        key, card = struct.unpack("<HH", b[8 + 4 * c:12 + 4 * c])
        card += 1
        if card <= 4096:
            out += [key << 16 | x for x in struct.unpack(f"<{card}H", b[at:at + 2 * card])]
            at += 2 * card
        else:
            words = struct.unpack("<1024Q", b[at:at + 8192])
            out += [key << 16 | (w * 64 + i) for w, x in enumerate(words) for i in range(64) if x >> i & 1]
            at += 8192
    return out


def _level0(string_db, fid):
    """{key: sorted docids} and the keys in key order, for the field's level-0 entries of facet_id_string_docids"""
    out, order = {}, []
    for i in range(string_db.n_keys):
        k = string_db.key(i)
        f, level = struct.unpack(">HB", k[:3])
        if f == fid and level == 0:
            key = k[3:].decode()
            out[key] = sorted(decode_cbo(string_db.val(i)[1:]))
            order.append(key)
    return out, order


def _normalized(norm_db, fid):
    """[(hyper-normalised string, its JSON set)] of the field, in key (= FST) order"""
    out = []
    for i in range(norm_db.n_keys):
        k = norm_db.key(i)
        if struct.unpack(">H", k[:2])[0] == fid:
            # serde_json into a BTreeSet<String>: byte order, duplicates dropped
            out.append((k[2:].decode(), sorted(set(json.loads(norm_db.val(i).decode())), key=lambda x: x.encode())))
    return out


def _originals(orig_db):
    out = {}
    for i in range(orig_db.n_keys):
        k = orig_db.key(i)
        f, d = struct.unpack(">HI", k[:6])
        out[(f, d, k[6:].decode())] = orig_db.val(i).decode()
    return out


_CACHE = {}


def facet_search(facets, fid, candidates, query=None, order="alpha", max_values=100, field_typos=True, authorize_typos=True,
                 exact_words=(), one_typo=5, two_typos=9):
    """inner_execute for field `fid` over the candidate docid set: [(value, count), ...] in the reference's order.  facets: a
    FacetImage after build() and build_search(); query: None or the already normalised query."""
    key = (id(facets), fid)
    if key not in _CACHE:  # the decoded databases of one facet image
        _CACHE[key] = (_level0(facets.string_db, fid), _normalized(facets.norm_db, fid), _originals(facets.orig_db))
    (level0, keys), norm, orig = _CACHE[key]
    cands = set(candidates)
    results = ValuesCollection(order, max_values)
    if not norm:
        return []  # no FST for the field
    if query is None:
        for key in keys:
            docids = level0[key]
            count = sum(1 for d in docids if d in cands)
            if count:
                if results.insert(orig.get((fid, docids[0], key), key), count):
                    break
        return results.into_sorted_vec()
    fst = [h for h, _ in norm]
    mkey = (key, query, authorize_typos and field_typos, query in exact_words, one_typo, two_typos)
    if mkey not in _CACHE:  # the FST strings the automaton accepts do not depend on the candidates
        if authorize_typos and field_typos:
            if query in exact_words:
                _CACHE[mkey] = [query] if query in fst else []
            else:
                k = typo_budget(query, one_typo, two_typos)
                _CACHE[mkey] = [h for h in fst if osa_prefix_distance(query, h) <= k]
        else:
            _CACHE[mkey] = [h for h in fst if h.startswith(query)]
    matches = _CACHE[mkey]
    sets = dict(norm)
    for h in matches:
        for key in sets[h]:
            if key not in level0:
                break  # the reference logs the missing key and returns Continue
            docids = level0[key]
            count = sum(1 for d in docids if d in cands)
            if count:
                if results.insert(orig.get((fid, docids[0], key), query), count):
                    break
    return results.into_sorted_vec()


def count_order_by_cut(hits, max_values):
    """The library's count order: the cut count c (the max-th largest count), the hits at or above it in insertion order, and the
    heap replayed over those alone.  Must equal ValuesCollection('count') over all the hits."""
    if max_values == 0 or not hits:
        return []
    counts = sorted((c for _, c in hits), reverse=True)
    cut = counts[min(max_values, len(counts)) - 1]
    vc = ValuesCollection("count", max_values)
    for v, c in hits:
        if c >= cut:
            vc.insert(v, c)
    return vc.into_sorted_vec()
