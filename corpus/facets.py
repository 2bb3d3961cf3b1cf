"""Facet databases in their LMDB byte formats (test/bench infrastructure): facet_id_f64_docids and facet_id_string_docids.

Key: u16 BE fid | u8 level | bound (OrderedF64Codec, heed_codec/facet/ordered_f64_codec.rs, or the normalised string);
value: FacetGroupValueCodec = u8 size | CBO roaring (heed_codec/facet/mod.rs).  Level-0 entries hold one value each; levels >= 1
group FACET_GROUP_SIZE entries of the level below (left bound = the first one's) as the reference's incremental indexer does, so
that readers which must ignore them see them.  JSON documents go through milli's extraction rules: arrays are flattened, `null`,
objects and the empty string get no facet, booleans become the strings "true" / "false", strings are normalised (lib.rs:442).
`_geo` objects become the number facets `_geo.lat` / `_geo.lng` (update/new/extract/faceted/facet_document.rs:82-99).
build_presence() adds facet_id_{exists,is_null,is_empty}_docids (key u16 BE fid, value CBO) as extract_facets.rs writes them: a field
exists in a document for any value, `null`, `[]`, `{}` and non-empty objects included; it is null for a top-level `null` and empty for
a top-level `""`, `[]` or `{}`.  add_document walks a whole document as milli does, nested objects included (dotted field names)."""
from __future__ import annotations

import struct
import unicodedata

import numpy as np

from .pyindexgen import DbImage

FACET_GROUP_SIZE = 4


def normalize_facet(s: str) -> str:
    """lib.rs normalize_facet: NFKD (compatibility decomposition) of the trimmed string, lower-cased"""
    return unicodedata.normalize("NFKD", s.strip()).lower()


def hyper_normalize(s: str) -> str:
    """The facet-search key of an already normalize_facet'd value: NFKD, combining marks dropped, lower-cased.  This only
    approximates charabia's lossy normaliser, which indexing uses (update/new/facet_search_builder.rs); the library never
    recomputes it and reads whatever facet_id_normalized_string_strings holds."""
    return "".join(c for c in unicodedata.normalize("NFKD", s) if not unicodedata.combining(c)).lower()


def ordered_f64(f: float) -> bytes:
    """OrderedF64Codec: globally ordered bytes (facet/value_encoding.rs f64_into_bytes), then the f64 big-endian"""
    f = float(f)
    be = bytearray(struct.pack(">d", 0.0 if f == 0.0 else f))
    if f < 0:
        be = bytearray(b ^ 0xFF for b in be)
    else:
        be[0] ^= 0x80
    return bytes(be) + struct.pack(">d", f)


def cbo_encode(docids) -> bytes:
    """CboRoaringBitmapCodec: <= 7 docids as raw native-endian u32, otherwise the portable roaring format without run containers"""
    d = np.unique(np.asarray(docids, np.uint32))
    if len(d) <= 7:
        return d.astype("<u4").tobytes()
    hi = d >> 16
    keys, starts = np.unique(hi, return_index=True)
    ends = list(starts[1:]) + [len(d)]
    desc, bodies = [], []
    for k, a, b in zip(keys, starts, ends):
        lo = (d[a:b] & 0xFFFF).astype(np.uint16)
        desc.append(struct.pack("<HH", int(k), len(lo) - 1))
        if len(lo) <= 4096:
            bodies.append(lo.astype("<u2").tobytes())
        else:
            words = np.zeros(1024, np.uint64)
            np.bitwise_or.at(words, lo >> 6, np.left_shift(np.uint64(1), (lo & 63).astype(np.uint64)))
            bodies.append(words.astype("<u8").tobytes())
    n = len(keys)
    head = struct.pack("<II", 12346, n) + b"".join(desc)
    offs, at = [], len(head) + 4 * n
    for body in bodies:
        offs.append(struct.pack("<I", at))
        at += len(body)
    return head + b"".join(offs) + b"".join(bodies)


def _db(entries):
    """entries: sorted list of (key bytes, value bytes)"""
    kb = b"".join(k for k, _ in entries)
    vb = b"".join(v for _, v in entries)
    ko = np.zeros(len(entries) + 1, np.uint64)
    vo = np.zeros(len(entries) + 1, np.uint64)
    ko[1:] = np.cumsum([len(k) for k, _ in entries]) if entries else []
    vo[1:] = np.cumsum([len(v) for _, v in entries]) if entries else []
    return DbImage(np.frombuffer(kb, np.uint8).copy(), ko, np.frombuffer(vb, np.uint8).copy(), vo)


class FacetImage:
    """Faceted fields of an index: field name -> fid, and per field the documents of every number / string value."""

    def __init__(self):
        self.fields = {}  # name -> fid
        self.numbers = {}  # fid -> {float: [docids]}
        self.strings = {}  # fid -> {normalised str: [docids]}
        # (fid, docid, normalised str) -> original string, what field_id_docid_facet_strings holds.  A document can give one normalised
        # value several originals ("Blue" and "blue " in one array); the first one it gives is kept.
        self.originals = {}
        # fid -> docids: documents holding the field with a value that gives no number or string facet (exists), and with a
        # top-level null / "" [] {} (is_null / is_empty); documents with a facet value exist without being listed here
        self.present, self.null, self.empty = {}, {}, {}

    def fid(self, name):
        if name not in self.fields:
            self.fields[name] = len(self.fields)
        return self.fields[name]

    def add_facet(self, docid, name, value):
        """one already-extracted facet value: a number (int/float) or a string (normalised here)"""
        f = self.fid(name)
        if isinstance(value, str):
            v = normalize_facet(value)
            if v:
                self.strings.setdefault(f, {}).setdefault(v, []).append(docid)
                self.originals.setdefault((f, docid, v), value)
        else:
            self.numbers.setdefault(f, {}).setdefault(float(value), []).append(docid)

    def add_json(self, docid, name, value, top=True):
        """a JSON field value through milli's facet extraction: arrays flattened; null / objects / "" give nothing; `_geo`
        ({"lat": .., "lng": ..}, numbers or numeric strings) gives the number facets `_geo.lat` / `_geo.lng`.  A top-level null, "",
        [] or {} is recorded for build_presence, and so is a document holding the field at all."""
        if name == "_geo":
            if value is None:
                return
            lat, lng = (float(value[k]) for k in ("lat", "lng"))  # extract_geo_coordinates: both, as f64 (else the document is refused)
            self.add_facet(docid, "_geo.lat", lat)
            self.add_facet(docid, "_geo.lng", lng)
            return
        f = self.fid(name)
        if top:  # extract_facets.rs:309-313: every value the field holds, objects and arrays included, makes it exist
            self.present.setdefault(f, set()).add(docid)
            if value is None:
                self.null.setdefault(f, set()).add(docid)
            elif value in ("", [], {}):
                self.empty.setdefault(f, set()).add(docid)
        if isinstance(value, list):
            for v in value:
                self.add_json(docid, name, v, top=False)
        elif isinstance(value, bool):
            self.add_facet(docid, name, "true" if value else "false")
        elif isinstance(value, (int, float)):
            self.add_facet(docid, name, value)
        elif isinstance(value, str):
            self.add_facet(docid, name, value)

    def _extract_field(self, docid, name, on_base, value):
        """extract_facets.rs facet_fn_with_options (:300-410) for one value the walk reaches"""
        f = self.fid(name)
        self.present.setdefault(f, set()).add(docid)
        if isinstance(value, bool):
            v = "true" if value else "false"
            self.strings.setdefault(f, {}).setdefault(v, []).append(docid)
            self.originals.setdefault((f, docid, v), v)
        elif isinstance(value, (int, float)):
            self.numbers.setdefault(f, {}).setdefault(float(value), []).append(docid)
        elif isinstance(value, str) and value:
            v = normalize_facet(value)
            self.strings.setdefault(f, {}).setdefault(v, []).append(docid)
            self.originals.setdefault((f, docid, v), value)
        elif on_base and value is None:
            self.null.setdefault(f, set()).add(docid)
        elif on_base and value in ("", [], {}):
            self.empty.setdefault(f, set()).add(docid)

    def _seek_object(self, docid, obj, base, on_base, keep):
        """perm_json_p::seek_leaf_values_in_object (update/new/extract/mod.rs:34-66)"""
        if not obj:
            self._visit(docid, base, on_base, {}, keep)
        for k, v in obj.items():
            key = f"{base}.{k}" if base else k
            self._visit(docid, key, True, v, keep)
            if isinstance(v, dict):
                self._seek_object(docid, v, key, True, keep)
            elif isinstance(v, list):
                self._seek_array(docid, v, key, True, keep)

    def _seek_array(self, docid, arr, base, on_base, keep):
        """perm_json_p::seek_leaf_values_in_array (update/new/extract/mod.rs:68-91)"""
        if not arr:
            self._visit(docid, base, on_base, [], keep)
        for v in arr:
            if isinstance(v, dict):
                self._seek_object(docid, v, base, False, keep)
            elif isinstance(v, list):
                self._seek_array(docid, v, base, False, keep)
            else:
                self._visit(docid, base, False, v, keep)

    def _visit(self, docid, name, on_base, value, keep):
        if keep(name):
            self._extract_field(docid, name, on_base, value)

    def add_document(self, docid, doc, filterable):
        """a whole JSON document through milli's facet extraction (facet_document.rs:20-99): every field matching a name in
        `filterable`, or nested under one (`opt1.opt2` under `opt1`), is extracted at every value the walk reaches; an object or
        array field is first walked, then extracted itself; `_geo` becomes `_geo.lat` / `_geo.lng`"""
        keep = lambda name: any(name == p or name.startswith(p + ".") for p in filterable)  # noqa: E731
        for name, value in doc.items():
            if name == "_geo":
                if "_geo" in filterable:
                    self.add_json(docid, "_geo", value)
                continue
            if isinstance(value, dict):
                self._seek_object(docid, value, name, True, keep)
            elif isinstance(value, list):
                self._seek_array(docid, value, name, True, keep)
            self._visit(docid, name, True, value, keep)

    def add_synthetic(self, n_docs, seed=0x50A7):
        """seeded facet fields: `price` (numbers with many duplicates, ~10 % missing), `brand` (Zipf-distributed strings), `tags`
        (arrays of 1-3 mixed numbers and strings)"""
        rng = np.random.default_rng(seed)
        docs = np.arange(n_docs, dtype=np.uint32)
        price = np.round(rng.gamma(2.0, 40.0, n_docs), 1)
        has_price = rng.random(n_docs) >= 0.10
        self._bulk("price", docs[has_price], price[has_price], numbers=True)
        n_brands = 500
        w = 1.0 / np.arange(1, n_brands + 1) ** 1.1
        brand = rng.choice(n_brands, n_docs, p=w / w.sum())
        has_brand = rng.random(n_docs) >= 0.05
        names = np.array([f"brand{b:03d}" for b in range(n_brands)])
        self._bulk("brand", docs[has_brand], names[brand[has_brand]], numbers=False)
        n_tags = rng.integers(1, 4, n_docs)
        for k in range(3):
            sel = docs[n_tags > k]
            is_num = rng.random(len(sel)) < 0.4
            nums = rng.integers(0, 200, len(sel))
            strs = np.array([f"tag{t:02d}" for t in range(60)])[rng.integers(0, 60, len(sel))]
            self._bulk("tags", sel[is_num], nums[is_num].astype(np.float64), numbers=True)
            self._bulk("tags", sel[~is_num], strs[~is_num], numbers=False)
        return self

    def add_synthetic_geo(self, n_docs, seed=0x6E0, with_geo=0.9):
        """seeded `_geo` points for the GeoSort tests: clusters around a few cities, exact duplicates, runs of points less than 1 m
        apart (chains of the 1 m error margin), points at distances sharing a floor metre, antipodes, the +/-180 degree seam, and
        documents without `_geo` (1 - with_geo of them)"""
        rng = np.random.default_rng(seed)
        docs = np.arange(n_docs)
        has = rng.random(n_docs) < with_geo
        kind = rng.integers(0, 6, n_docs)
        centers = np.array([[48.85, 2.35], [40.71, -74.0], [-33.86, 151.21], [35.68, 139.69], [0.0, 179.99], [-48.85, -177.65]])
        c = centers[rng.integers(0, len(centers), n_docs)]
        lat = np.clip(c[:, 0] + rng.normal(0, 0.5, n_docs), -90, 90)
        lng = c[:, 1] + rng.normal(0, 0.5, n_docs)
        lng = (lng + 180.0) % 360.0 - 180.0
        # kind 1: exact duplicates of a handful of points; 2: chains of points ~0.4 m apart; 3: uniform over the sphere;
        # 4: round coordinates (many equal floor metres); 5: cluster (kept)
        dup = rng.integers(0, 40, n_docs)
        lat = np.where(kind == 1, 10.0 + dup * 0.001, lat)
        lng = np.where(kind == 1, 20.0, lng)
        step = docs * 3.6e-6  # about 0.4 m of latitude per document
        lat = np.where(kind == 2, 45.0 + (step % 0.01), lat)
        lng = np.where(kind == 2, 7.0, lng)
        u = rng.random(n_docs)
        lat = np.where(kind == 3, np.degrees(np.arcsin(2 * u - 1)), lat)
        lng = np.where(kind == 3, rng.uniform(-180, 180, n_docs), lng)
        lat = np.where(kind == 4, np.round(lat, 1), lat)
        lng = np.where(kind == 4, np.round(lng, 1), lng)
        self._bulk("_geo.lat", docs[has], lat[has], numbers=True)
        self._bulk("_geo.lng", docs[has], lng[has], numbers=True)
        return self

    def _bulk(self, name, docids, values, numbers):
        f = self.fid(name)
        tab = (self.numbers if numbers else self.strings).setdefault(f, {})
        order = np.argsort(values, kind="stable")
        vals, starts = np.unique(values[order], return_index=True)
        ends = list(starts[1:]) + [len(order)]
        for v, a, b in zip(vals, starts, ends):
            key = float(v) if numbers else normalize_facet(str(v))
            tab.setdefault(key, []).extend(int(x) for x in docids[order[a:b]])
            if not numbers:
                for x in docids[order[a:b]]:
                    self.originals.setdefault((f, int(x), key), str(v))

    def build(self):
        """-> (facet_id_f64_docids, facet_id_string_docids) as DbImage, keys in LMDB (bytewise) order"""
        self.f64_db = _db(self._entries(self.numbers, lambda v: ordered_f64(v)))
        self.string_db = _db(self._entries(self.strings, lambda v: v.encode()))
        return self.f64_db, self.string_db

    def build_presence(self):
        """-> (facet_id_exists_docids, facet_id_is_null_docids, facet_id_is_empty_docids) as DbImage, keys in LMDB order; also kept as
        self.exists_db / self.null_db / self.empty_db, which Index.stage stages when present"""
        exists = {f: set(d) for f, d in self.present.items()}
        for tab in (self.numbers, self.strings):
            for f, vals in tab.items():
                for docs in vals.values():
                    exists.setdefault(f, set()).update(int(x) for x in docs)
        dbs = [_db(sorted((struct.pack(">H", f), cbo_encode(sorted(d))) for f, d in tab.items() if d)) for tab in (exists, self.null, self.empty)]
        self.exists_db, self.null_db, self.empty_db = dbs
        return tuple(dbs)

    def build_search(self):
        """-> (facet_id_normalized_string_strings, field_id_docid_facet_strings) as DbImage, keys in LMDB order: per string field
        every hyper-normalised string with the JSON set of the level-0 keys it stands for, and every (fid, docid, normalised key)
        with its original string.  Also kept as self.norm_db / self.orig_db, which Index.stage stages when present."""
        import json

        norm = []
        for fid, vals in self.strings.items():
            groups = {}
            for v in vals:
                groups.setdefault(hyper_normalize(v), []).append(v)
            for h, keys in groups.items():
                keys = sorted(keys, key=lambda s: s.encode())  # BTreeSet<String> order
                norm.append((struct.pack(">H", fid) + h.encode(), json.dumps(keys, ensure_ascii=False, separators=(",", ":")).encode()))
        norm.sort(key=lambda e: e[0])
        orig = sorted((struct.pack(">HI", f, d) + v.encode(), o.encode()) for (f, d, v), o in self.originals.items())
        self.norm_db, self.orig_db = _db(norm), _db(orig)
        return self.norm_db, self.orig_db

    def add_synthetic_search(self, n_docs, n_values=100_000, seed=0x5EA7):
        """seeded `model`: a high-cardinality string field (n_values distinct values, one per document, the rest drawn uniformly) of
        lower-case letter-and-digit words, for facet search at scale"""
        rng = np.random.default_rng(seed)
        letters = np.array(list("abcdefghijklmnopqrstuvwxyz"))
        lens = rng.integers(4, 11, n_values)
        words = np.array(["".join(rng.choice(letters, n)) + str(i) for i, n in enumerate(lens)])
        pick = np.concatenate([np.arange(min(n_values, n_docs)), rng.integers(0, n_values, max(0, n_docs - n_values))])
        self._bulk("model", np.arange(n_docs, dtype=np.uint32), words[pick[:n_docs]], numbers=False)
        return self

    @staticmethod
    def _entries(tab, enc):
        out = []
        for fid, vals in tab.items():
            level = sorted((enc(v), np.unique(np.asarray(d, np.uint32))) for v, d in vals.items())
            lv = 0
            while level:
                for bound, d in level:
                    out.append((struct.pack(">HB", fid, lv) + bound, bytes([1 if lv == 0 else FACET_GROUP_SIZE]) + cbo_encode(d)))
                if len(level) <= FACET_GROUP_SIZE:
                    break
                level = [(level[i][0], np.unique(np.concatenate([d for _, d in level[i:i + FACET_GROUP_SIZE]])))
                         for i in range(0, len(level), FACET_GROUP_SIZE)]
                lv += 1
        out.sort(key=lambda e: e[0])
        return out


def geo_points(facets, lat_fid, lng_fid):
    """docid -> (lat, lng) as geo_value reads it (documents/geo_sort.rs:252-277): per coordinate the smallest number value, else the
    bytewise-smallest string value parsed as f64; documents with neither coordinate are left out"""
    out = [{}, {}]
    for c, fid in enumerate((lat_fid, lng_fid)):
        for v in sorted(facets.numbers.get(fid, {})):
            for d in facets.numbers[fid][v]:
                out[c].setdefault(d, v)
        for v in sorted(facets.strings.get(fid, {}), key=lambda x: x.encode()):
            for d in facets.strings[fid][v]:
                out[c].setdefault(d, float(v))
    if set(out[0]) != set(out[1]):
        raise ValueError("a document has one geo coordinate without the other")
    return {d: (out[0][d], out[1][d]) for d in out[0]}
