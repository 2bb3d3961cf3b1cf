"""meilisearch_b200 — H100-native (sm_90a) implementation of milli's query-time scoring path.

Python host-side mirror of the reference interface for this path (crates/milli/src/search/mod.rs:58-86,280-415,526-535):
`Index` (the staged, HBM-resident copy of what `milli::Index` exposes to search), the `Search` builder with
`execute()` / `execute_hybrid()`, and `SearchResult`.  Everything goes through the C ABI of include/b200milli.h
(libb200milli.so, built in-tree by meilisearch_b200/csrc/build.sh).  There is no CPU fallback: without the CUDA
library or without a device, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .filter import parse_filter, preorder  # noqa: F401
from .tokenizer import TokenBatch, tokenize  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200milli.so")
MAX_SCORES = 12
CRITERIA = {"words": 0, "typo": 1, "proximity": 2, "attribute": 3, "attributeRank": 4, "wordPosition": 5, "sort": 6, "exactness": 7}
DEFAULT_CRITERIA = ["words", "typo", "proximity", "attributeRank", "sort", "wordPosition", "exactness"]  # criterion.rs:121-131
TMS = {"last": 0, "all": 1, "frequency": 2}
SCORE_KINDS = ["words", "typo", "proximity", "fid", "position", "exactAttribute", "exactWords", "vector", "skipped", "sort", "geo"]
GEO_STRATEGIES = {"dynamic": 0, "iterative": 1, "rtree": 2}  # GeoSortStrategy::Dynamic / AlwaysIterative / AlwaysRtree
DB_FACET_F64, DB_FACET_STRING = 10, 11
DB_FACET_NORMALIZED, DB_FACET_ORIGINALS = 12, 13  # facet_id_normalized_string_strings, field_id_docid_facet_strings
DB_FACET_EXISTS, DB_FACET_IS_NULL, DB_FACET_IS_EMPTY = 14, 15, 16  # facet_id_{exists,is_null,is_empty}_docids
NO_FIELD = 0xFFFF  # a sort field absent from the fields map
ERRORS = {-1: "NO_DEVICE", -2: "CUDA", -3: "INVALID", -4: "UNSUPPORTED", -5: "CAPACITY", -6: "STATE"}


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200milli error {ERRORS.get(code, code)}: {msg}")
        self.code = code


class _Settings(C.Structure):
    _fields_ = [("n_fields", C.c_uint32), ("weights", C.c_void_p), ("criteria", C.c_void_p), ("n_criteria", C.c_uint32),
                ("authorize_typos", C.c_int32), ("min_word_len_one_typo", C.c_uint32), ("min_word_len_two_typos", C.c_uint32),
                ("prefix_search", C.c_int32), ("exact_words", C.c_char_p)]


class _Batch(C.Structure):
    _fields_ = [("n_queries", C.c_uint32), ("token_begin", C.c_void_p), ("token_kind", C.c_void_p), ("lemma_off", C.c_void_p),
                ("lemma_bytes", C.c_void_p), ("terms_matching_strategy", C.c_int32), ("scoring_strategy", C.c_int32),
                ("offset", C.c_uint32), ("limit", C.c_uint32), ("words_limit", C.c_uint32), ("vectors", C.c_void_p),
                ("mode", C.c_int32), ("semantic_ratio", C.c_float), ("universes", C.c_void_p), ("n_universe_words", C.c_uint64),
                ("time_budget_ns", C.c_uint64), ("stop_after", C.c_int64), ("has_ranking_score_threshold", C.c_int32),
                ("ranking_score_threshold", C.c_double), ("sort_begin", C.c_void_p), ("sort_fid", C.c_void_p), ("sort_asc", C.c_void_p),
                ("sort_geo", C.c_void_p), ("sort_geo_point", C.c_void_p), ("geo_strategy", C.c_int32), ("geo_cache_size", C.c_uint32),
                ("geo_max_bucket_size", C.c_uint64), ("geo_filter_begin", C.c_void_p), ("geo_filter_kind", C.c_void_p),
                ("geo_filter_not", C.c_void_p), ("geo_filter_args", C.c_void_p), ("facet_begin", C.c_void_p), ("facet_fid", C.c_void_p),
                ("facet_order", C.c_void_p), ("facet_max_values", C.c_uint32), ("facet_cap", C.c_uint32), ("facet_search_fid", C.c_void_p),
                ("facet_query_kind", C.c_void_p), ("facet_query_off", C.c_void_p), ("facet_query_bytes", C.c_void_p),
                ("facet_search_flags", C.c_void_p), ("facet_search_max", C.c_uint32), ("filter", C.c_void_p)]


class _Results(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("docids", "n_hits", "n_scores", "score_kind", "score_rank", "score_max", "score_sim",
                                          "n_candidates", "semantic_hits", "status", "degraded", "used_negative_operator", "candidates")] + \
               [("candidates_words", C.c_uint64)] + \
               [(n, C.c_void_p) for n in ("facet_n_num", "facet_n_str", "facet_key", "facet_count", "facet_docid", "facet_has_stats", "facet_min",
                                          "facet_max")] + \
               [(n, C.c_void_p) for n in ("fs_n", "fs_key", "fs_count", "fs_docid", "fs_fallback", "filter_error_leaf")]


class _FilterPrograms(C.Structure):
    _fields_ = [("n", C.c_uint32), ("begin", C.c_void_p), ("nodes", C.c_void_p), ("n_values", C.c_uint32), ("value_off", C.c_void_p),
                ("value_bytes", C.c_void_p), ("value_num", C.c_void_p)]


class _SimilarRequest(C.Structure):
    _fields_ = [("n_queries", C.c_uint32), ("docids", C.c_void_p), ("offset", C.c_uint32), ("limit", C.c_uint32), ("universes", C.c_void_p),
                ("n_universe_words", C.c_uint64), ("filter", C.c_void_p), ("has_ranking_score_threshold", C.c_int32),
                ("ranking_score_threshold", C.c_double)]


class _Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("device_steps", C.c_uint64), ("posting_bytes", C.c_uint64), ("matrix_bytes", C.c_uint64),
                ("dictionary_bytes", C.c_uint64), ("vector_bytes", C.c_uint64), ("kernel_ms", C.c_double * 16),
                ("kernel_count", C.c_uint64 * 16), ("kernel_bytes", C.c_uint64 * 16), ("device_ms", C.c_double), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("host_ms", C.c_double * 8),
                ("hbm_bytes_staged", C.c_uint64), ("deferred", C.c_uint64), ("arena_peak_bytes", C.c_uint64),
                ("eval_class_launches", C.c_uint64 * 9), ("eval_class_tiles", C.c_uint64 * 9),
                ("lev_terms", C.c_uint64), ("lev_items", C.c_uint64), ("lev_pairs", C.c_uint64)]


KERNELS = ["lev_match", "act_compact", "pair_probe", "scatter", "eval_paths", "emit", "vec_dist", "topk_select", "vec_gemm_topk", "vec_merge", "sort", "geo", "geo_filter", "facet", "facet_search", "filter"]


def build_library(force=False):
    """Compile the CUDA extension in-tree for sm_90a (works without a GPU)."""
    csrc = os.path.join(_HERE, "csrc")
    srcs = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cu", ".cpp", ".h"))] + [os.path.join(_HERE, "..", "include", "b200milli.h")]
    if force or not os.path.exists(LIB_PATH) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs):
        subprocess.check_call(["sh", os.path.join(csrc, "build.sh")])
    return LIB_PATH


_lib = None


def load_library():
    """Load libb200milli.so.  Fails loudly when the extension has not been built — there is no fallback path."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)")
        l = C.CDLL(LIB_PATH)
        l.b200_open.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        l.b200_close.argtypes = [C.c_void_p]
        l.b200_last_error.restype = C.c_char_p
        l.b200_last_error.argtypes = [C.c_void_p]
        l.b200_open_error.restype = C.c_char_p
        l.b200_stage_dictionary.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
        l.b200_stage_db.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        l.b200_stage_documents_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        l.b200_stage_settings.argtypes = [C.c_void_p, C.POINTER(_Settings)]
        l.b200_stage_synonyms.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p)]
        l.b200_stage_finish.argtypes = [C.c_void_p]
        l.b200_stage_geo_fields.argtypes = [C.c_void_p, C.c_uint16, C.c_uint16]
        l.b200_stage_embeddings.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p]
        l.b200_stage_embeddings_f16.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p]
        l.b200_stage_distribution.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float]
        l.b200_derive_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_void_p] * 4
        l.b200_union_postings.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
        l.b200_nns_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        l.b200_nns_batch_sharded.argtypes = l.b200_nns_batch.argtypes
        l.b200_comm_unique_id.argtypes = [C.c_void_p, C.c_void_p]
        l.b200_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        l.b200_search_batch.argtypes = [C.c_void_p, C.POINTER(_Batch), C.POINTER(_Results)]
        l.b200_geo_filter_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        l.b200_filter_batch.argtypes = [C.c_void_p, C.POINTER(_FilterPrograms), C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        l.b200_facet_distribution_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                                    C.c_uint32] + [C.c_void_p] * 9
        l.b200_facet_search_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64] + [C.c_void_p] * 5 + [C.c_uint32, C.c_uint32] + \
            [C.c_void_p] * 6
        l.b200_similar_batch.argtypes = [C.c_void_p, C.POINTER(_SimilarRequest), C.POINTER(_Results)]
        l.b200_proximity_pairs.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
        l.b200_graph_from_tokens.argtypes = [C.c_void_p, C.POINTER(_Batch), C.POINTER(C.c_void_p)]
        l.b200_graph_free.argtypes = [C.c_void_p]
        l.b200_rule_start.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]
        l.b200_rule_next.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_void_p)]
        l.b200_rule_end.argtypes = [C.c_void_p]
        l.b200_get_stats.argtypes = [C.c_void_p, C.POINTER(_Stats)]
        l.b200_reset_stats.argtypes = [C.c_void_p]
        _lib = l
    return _lib


SYMBOLS = ["b200_open", "b200_close", "b200_last_error", "b200_open_error", "b200_stage_dictionary", "b200_stage_db",
           "b200_stage_documents_ids", "b200_stage_settings", "b200_stage_synonyms", "b200_stage_geo_fields", "b200_stage_finish", "b200_stage_embeddings", "b200_stage_embeddings_f16", "b200_stage_distribution",
           "b200_derive_batch", "b200_union_postings", "b200_proximity_pairs", "b200_nns_batch", "b200_nns_batch_sharded", "b200_comm_unique_id", "b200_comm_init", "b200_search_batch", "b200_geo_filter_batch", "b200_filter_batch", "b200_facet_distribution_batch", "b200_facet_search_batch", "b200_similar_batch", "b200_graph_from_tokens",
           "b200_graph_free", "b200_rule_start", "b200_rule_next", "b200_rule_end", "b200_get_stats", "b200_reset_stats"]


def parse_geo_point(name):
    """(lat, lng) of a `_geoPoint(lat, lng)` sort entry's name, None for a field name (AscDesc parsing, asc_desc.rs)"""
    import re

    m = re.fullmatch(r"_geoPoint\(\s*([^,\s]+)\s*,\s*([^)\s]+)\s*\)", name)
    return (float(m.group(1)), float(m.group(2))) if m else None


# a number as Rust's f64::from_str reads the filter's tokens: sign, digits with an optional fraction and exponent, or inf / infinity /
# nan in any case (non-finite values are refused by the library with the reference's message)
_NUM = r"\s*([+-]?(?:(?:\d+\.?\d*|\.\d+)(?:[eE][+-]?\d+)?|(?i:inf|infinity|nan)))\s*"
_GEO_RADIUS = r"_geoRadius\(" + _NUM + "," + _NUM + "," + _NUM + r"(,.*)?\)"
_GEO_BOX = r"_geoBoundingBox\(\s*\[" + _NUM + "," + _NUM + r"\]\s*,\s*\[" + _NUM + "," + _NUM + r"\]\s*\)"
GEO_RADIUS, GEO_BOUNDING_BOX = 0, 1


def parse_geo_filter(clause):
    """(kind, negated, four args) of a geo filter clause: `_geoRadius(lat, lng, radius)` or `_geoBoundingBox([top, right], [bottom,
    left])`, optionally prefixed by `NOT `, with numbers in Rust's f64 syntax.  Anything else raises ValueError, and so does the `resolution` argument of _geoRadius,
    which only steers the GeoJSON index (not built here).  Non-finite numbers pass: the library refuses them with the reference's
    message."""
    import re

    s = clause.strip()
    neg = re.match(r"NOT\s+", s)
    if neg:
        s = s[neg.end():]
    m = re.fullmatch(_GEO_RADIUS, s)
    if m:
        if m.group(4) is not None:
            raise ValueError(f"{clause!r}: the resolution argument of _geoRadius is out of scope (GeoJSON filtering is not built)")
        return GEO_RADIUS, bool(neg), (float(m.group(1)), float(m.group(2)), float(m.group(3)), 0.0)
    m = re.fullmatch(_GEO_BOX, s)
    if m:
        return GEO_BOUNDING_BOX, bool(neg), tuple(float(m.group(i)) for i in range(1, 5))
    raise ValueError(f"{clause!r} is not a geo filter clause (`[NOT ]_geoRadius(lat, lng, radius)` or `[NOT ]_geoBoundingBox([top, right], [bottom, left])`)")


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


F_AND, F_OR, F_NOT, F_RANGE, F_EQUAL, F_NOT_EQUAL, F_IN, F_EXISTS, F_IS_NULL, F_IS_EMPTY, F_GEO_RADIUS, F_GEO_BBOX, F_EMPTY, F_DENIED, \
    F_UNSUPPORTED = range(15)
B_INCLUDED, B_EXCLUDED, B_UNBOUNDED = 0, 1, 2
FILTER_NODE = np.dtype({"names": ["op", "lo", "hi", "has_number", "fid", "pad", "n", "value", "args"],
                        "formats": ["u1", "u1", "u1", "u1", "<u2", "<u2", "<u4", "<u4", ("<f8", 4)],
                        "offsets": [0, 1, 2, 3, 4, 6, 8, 12, 16], "itemsize": 48})
# the FilterableAttributesFeatures check each operator makes (index_filter.rs:94-125)
OP_FEATURE = {">": "comparison", ">=": "comparison", "<": "comparison", "<=": "comparison", "TO": "comparison", "=": "equality",
              "!=": "equality", "IN": "equality", "EXISTS": "exists", "NULL": "null", "EMPTY": "empty"}
_RANGE = {">": (B_EXCLUDED, B_UNBOUNDED), ">=": (B_INCLUDED, B_UNBOUNDED), "<": (B_UNBOUNDED, B_EXCLUDED), "<=": (B_UNBOUNDED, B_INCLUDED),
          "TO": (B_INCLUDED, B_INCLUDED)}


class _Programs:
    """the arrays of a b200_filter_programs and the struct pointing at them"""

    def __init__(self, nodes, begin, values):
        from corpus.facets import normalize_facet
        from .filter import parse_finite_float

        self.nodes = np.asarray(nodes if nodes else [np.zeros((), FILTER_NODE)], FILTER_NODE)
        self.begin = np.asarray(begin, np.uint32)
        enc = [normalize_facet(v).encode() for v in values]
        self.off = np.zeros(len(values) + 1, np.uint32)
        self.off[1:] = np.cumsum([len(e) for e in enc]) if enc else []
        self.bytes = np.frombuffer(b"".join(enc) + b"\0", np.uint8).copy()
        nums = [parse_finite_float(v) for v in values]
        self.num = np.asarray([np.nan if x is None else x for x in nums] or [0.0], np.float64)
        self.struct = _FilterPrograms(len(begin) - 1, _p(self.begin), _p(self.nodes), len(values), _p(self.off), _p(self.bytes), _p(self.num))


def encode_filters(index, filters, denied=()):
    """b200_filter_programs of filters (strings for parse_filter, trees, or None for no filter), lowered as a Rust shim lowers
    FilterCondition: a field absent from the index's fields map is an EMPTY leaf; `denied` holds (field, feature) pairs whose
    FilterableAttributesFeatures forbid the feature (comparison, equality, exists, null, empty), which become DENIED leaves;
    CONTAINS, STARTS WITH, _geoPolygon, the resolution argument, _vectors and _shard become UNSUPPORTED leaves"""
    from .filter import parse_filter

    denied = set(denied)
    nodes, begin, values = [], [0], []

    def node(op, **kw):
        x = np.zeros((), FILTER_NODE)
        x["op"] = op
        for k, v in kw.items():
            x[k] = v
        nodes.append(x)
        return x

    def emit(t):
        kind = t[0]
        if kind in ("and", "or"):
            node(F_AND if kind == "and" else F_OR, n=len(t[1]))
            for c in t[1]:
                emit(c)
        elif kind == "not":
            node(F_NOT)
            emit(t[1])
        elif kind == "geo":
            if t[1] in ("radius", "bbox"):
                args = [float(x) for x in t[2]] + ([0.0] if t[1] == "radius" else [])
                node(F_GEO_RADIUS if t[1] == "radius" else F_GEO_BBOX, args=args)
            else:
                node(F_UNSUPPORTED)
        else:
            _, field, op, vals = t
            if field == "_shard" or field == "_vectors" or field.startswith("_vectors.") or op in ("CONTAINS", "STARTS_WITH"):
                node(F_UNSUPPORTED)
            elif field not in index._fields:
                node(F_EMPTY)
            elif (field, OP_FEATURE[op]) in denied and not (op == "IN" and not vals):
                node(F_DENIED, fid=index._fields[field])
            else:
                fid = index._fields[field]
                at = len(values)
                if op in _RANGE:
                    from .filter import parse_finite_float

                    lo, hi = _RANGE[op]
                    pair = vals if op == "TO" else vals * 2
                    has = all(parse_finite_float(v) is not None for v in (vals if op == "TO" else vals[:1]))
                    values.extend(pair)
                    node(F_RANGE, fid=fid, lo=lo, hi=hi, has_number=int(has), value=at)
                elif op in ("=", "!=", "IN"):
                    values.extend(vals)
                    node({"=": F_EQUAL, "!=": F_NOT_EQUAL, "IN": F_IN}[op], fid=fid, value=at, n=len(vals))
                else:
                    node({"EXISTS": F_EXISTS, "NULL": F_IS_NULL, "EMPTY": F_IS_EMPTY}[op], fid=fid)

    for f in filters:
        if f is not None:
            emit(parse_filter(f) if isinstance(f, str) else f)
        begin.append(len(nodes))
    return _Programs(nodes, begin, values)


FACET_ORDERS = {"alpha": 0, "count": 1}  # OrderBy::Lexicographic / OrderBy::Count (sortFacetValuesBy)
DEFAULT_VALUES_PER_FACET = 100  # facet_distribution.rs DEFAULT_VALUES_PER_FACET
DEFAULT_MAX_FACET_SEARCH_VALUES = 100  # search/facet/search.rs DEFAULT_MAX_NUMBER_OF_VALUES_PER_FACET


def rust_f64_display(x):
    """Rust's `impl Display for f64`: the shortest digits that read back as the same value, never an exponent ("-0" for -0.0)"""
    import decimal

    if x != x:
        return "NaN"
    if x in (float("inf"), float("-inf")):
        return "inf" if x > 0 else "-inf"
    s = format(decimal.Decimal(repr(float(x))), "f")  # repr: the shortest round-trip digits
    return s.rstrip("0").rstrip(".") if "." in s else s


class _FacetOutputs:
    """The slots of a facet request and their b200_results::facet_* outputs: per_set holds one list of field names per query (or
    candidate set); begin / fid / orders are the request's arrays, with `cap` entries per slot"""

    def __init__(self, index, per_set, order, max_values, cap=None):
        self.begin = np.zeros(len(per_set) + 1, np.uint32)
        self.begin[1:] = np.cumsum([len(x) for x in per_set])
        n_slots = int(self.begin[-1])
        self.fid = np.asarray([index.field_id(x) for p in per_set for x in p] or [0], np.uint16)
        self.fids = [int(x) for x in self.fid]
        self.orders = np.full(max(n_slots, 1), FACET_ORDERS[order], np.uint8)
        cap = index.facet_cap({x for p in per_set for x in p}, max_values) if cap is None else cap
        n = max(n_slots, 1)
        self.cap = cap
        self.n_num = np.zeros(n, np.uint32)
        self.n_str = np.zeros(n, np.uint32)
        self.key = np.zeros(max(n * cap, 1), np.uint32)
        self.count = np.zeros(max(n * cap, 1), np.uint64)
        self.docid = np.zeros(max(n * cap, 1), np.uint32)
        self.has_stats = np.zeros(n, np.uint8)
        self.min = np.zeros(n, np.float64)
        self.max = np.zeros(n, np.float64)

    def pointers(self):
        return [_p(a) for a in (self.n_num, self.n_str, self.key, self.count, self.docid, self.has_stats, self.min, self.max)]

    def distribution(self, index, k, max_values):
        """the reference's IndexMap for slot k, built with the caller's merge rule (b200milli.h): the numbers, keyed by their f64
        Display string, then the strings one by one, keyed by their original, until an insert leaves the map at max_values entries"""
        fid = self.fids[k]
        out = {}
        at, nn, ns = k * self.cap, int(self.n_num[k]), int(self.n_str[k])
        for e in range(at, at + nn):
            out[rust_f64_display(index.sort_value(fid, 0, int(self.key[e]))[1])] = int(self.count[e])
        for e in range(at + nn, at + nn + ns):
            out[index.facet_original(fid, int(self.docid[e]), index.sort_value(fid, 1, int(self.key[e]))[1])] = int(self.count[e])
            if len(out) == max_values:
                break
        return list(out.items())

    def stats(self, k):
        return (float(self.min[k]), float(self.max[k])) if self.has_stats[k] else None


class SearchResult:
    """milli::SearchResult (search/mod.rs:526-535) for a batch of queries."""

    def __init__(self, n, limit, sort_value=None, geo_point=None):
        self._sort_value = sort_value  # (fid, is_string, key index) -> (field name, value)
        self._geo_point = geo_point  # docid -> its (lat, lng)
        self.sort_names = None  # per query: the field name of each sort rule, in rule order
        self.limit = max(limit, 1)
        L = self.limit
        self.documents_ids = np.zeros((n, L), np.uint32)
        self.n_hits = np.zeros(n, np.uint32)
        self.n_scores = np.zeros((n, L), np.uint8)
        self.score_kind = np.zeros((n, L, MAX_SCORES), np.uint8)
        self.score_rank = np.zeros((n, L, MAX_SCORES), np.uint32)
        self.score_max = np.zeros((n, L, MAX_SCORES), np.uint32)
        self.score_sim = np.zeros((n, L, MAX_SCORES), np.float32)
        self.n_candidates = np.zeros(n, np.uint64)
        self.semantic_hit_count = np.zeros(n, np.uint32)
        self.status = np.zeros(n, np.int32)
        self.filter_error_leaf = None  # with Search.filter: per query the failing filter leaf, -1 for none
        self.degraded = np.zeros(n, np.uint8)
        self.used_negative_operator = np.zeros(n, np.uint8)
        self.candidates = None  # (n, words) uint64 when requested with Search.with_candidates()
        self._facets = None  # (index, per query its field names, begin, _FacetOutputs, max values) with Search.facets()
        self._facet_search = None  # (index, per query (fid, query or None), outputs) with Search.facet_search()

    def facet_hits(self, q):
        """facetHits of query q's facet search: [(value, count), ...] in the reference's order"""
        ix, per_q, (n_out, key, count, docid, fallback, mx) = self._facet_search
        fid, query = per_q[q]
        return ix._facet_hits(fid, query, key[q * mx:q * mx + int(n_out[q])], count[q * mx:], docid[q * mx:], fallback[q * mx:])

    def facet_distribution(self, q):
        """facetDistribution of query q: {field name: [(key, count), ...]} in the reference's order"""
        ix, names, begin, out, mx = self._facets
        return {name: out.distribution(ix, int(begin[q]) + j, mx) for j, name in enumerate(names[q])}

    def facet_stats(self, q):
        """facetStats of query q: {field name: (min, max)} over its number values, fields without one left out"""
        ix, names, begin, out, _ = self._facets
        st = {name: out.stats(int(begin[q]) + j) for j, name in enumerate(names[q])}
        return {k: v for k, v in st.items() if v is not None}

    def ids(self, q):
        return [int(x) for x in self.documents_ids[q, : self.n_hits[q]]]

    def scores(self, q):
        out = []
        for i in range(int(self.n_hits[q])):
            row = []
            for s in range(int(self.n_scores[q, i])):
                k = SCORE_KINDS[self.score_kind[q, i, s]]
                if k == "vector":
                    sim = float(self.score_sim[q, i, s])
                    row.append(("vector", None if sim < 0 else sim))
                elif k == "sort":
                    m, key = int(self.score_max[q, i, s]), int(self.score_rank[q, i, s])
                    field, value = self._sort_value(m >> 2, m & 1, key)
                    if self.sort_names is not None and s < len(self.sort_names[q]):
                        field = self.sort_names[q][s]  # the rule's field name (also for a field absent from the fields map)
                    row.append(("sort", field, bool(m & 2), value))
                elif k == "geo":  # ScoreDetails::GeoSort: the bucket's first point, None for the Null bucket
                    d = int(self.score_rank[q, i, s])
                    row.append(("geo", bool(self.score_max[q, i, s] & 2), None if d == 0xFFFFFFFF else self._geo_point(d)))
                else:
                    row.append((k, int(self.score_rank[q, i, s]), int(self.score_max[q, i, s])))
            out.append(row)
        return out


class Index:
    """The staged index: what milli reads from LMDB at query time, resident in HBM."""

    def __init__(self, image=None, *, device=0, criteria=None, authorize_typos=True, one_typo=5, two_typos=9, prefix_search=True,
                 weights=None, exact_words=(), synonyms=None, facets=None, geo=None):
        self._l = load_library()
        h = C.c_void_p()
        rc = self._l.b200_open(device, C.byref(h))
        if rc != 0:
            raise B200Error(rc, self._l.b200_open_error().decode())
        self._h = h
        self.dim = 0
        if image is not None:
            self.stage(image, criteria=criteria, authorize_typos=authorize_typos, one_typo=one_typo, two_typos=two_typos,
                       prefix_search=prefix_search, weights=weights, exact_words=exact_words, synonyms=synonyms, facets=facets,
                       geo=geo)

    def _ck(self, rc):
        if rc != 0:
            raise B200Error(rc, self._l.b200_last_error(self._h).decode())

    def stage(self, image, *, criteria=None, authorize_typos=True, one_typo=5, two_typos=9, prefix_search=True, weights=None, exact_words=(),
              synonyms=None, facets=None, geo=None):
        """image: anything with dict_bytes/dict_offsets/n_words, dbs[i].{key_bytes,key_offsets,val_bytes,val_offsets,n_keys},
        documents_ids_cbo, n_fields — i.e. the LMDB databases in their on-disk formats.  facets: a corpus.facets.FacetImage (or
        anything with `fields` (name -> fid) and built `f64_db` / `string_db`); criteria may name custom rules "asc:<field>" /
        "desc:<field>" (Criterion::Asc / Desc).  geo: the (lat fid, lng fid) of `_geo.lat` / `_geo.lng` for the GeoSort rule; by default
        those of the facet image's `_geo.lat` / `_geo.lng` fields when it has them."""
        l = self._l
        self._facets = facets
        self._fields = dict(facets.fields) if facets is not None else {}
        self._level0 = {}  # (is_string) -> list of level-0 keys in staged order, for decoding Sort scores
        if facets is not None:
            for is_string, (dbid, db) in enumerate(((DB_FACET_F64, facets.f64_db), (DB_FACET_STRING, facets.string_db))):
                self._ck(l.b200_stage_db(self._h, dbid, db.n_keys, _p(db.key_bytes), _p(db.key_offsets), _p(db.val_bytes), _p(db.val_offsets)))
                self._level0[is_string] = [db.key(i) for i in range(db.n_keys) if db.key(i)[2] == 0]
            for dbid, db in ((DB_FACET_NORMALIZED, getattr(facets, "norm_db", None)), (DB_FACET_ORIGINALS, getattr(facets, "orig_db", None)),
                             (DB_FACET_EXISTS, getattr(facets, "exists_db", None)), (DB_FACET_IS_NULL, getattr(facets, "null_db", None)),
                             (DB_FACET_IS_EMPTY, getattr(facets, "empty_db", None))):
                if db is not None:
                    self._ck(l.b200_stage_db(self._h, dbid, db.n_keys, _p(db.key_bytes), _p(db.key_offsets), _p(db.val_bytes), _p(db.val_offsets)))
        self._n_docs = int(image.n_docs)
        self._ck(l.b200_stage_dictionary(self._h, _p(image.dict_bytes), _p(image.dict_offsets), image.n_words))
        for i, db in enumerate(image.dbs):
            self._ck(l.b200_stage_db(self._h, i, db.n_keys, _p(db.key_bytes), _p(db.key_offsets), _p(db.val_bytes), _p(db.val_offsets)))
        self._ck(l.b200_stage_documents_ids(self._h, _p(image.documents_ids_cbo), len(image.documents_ids_cbo)))
        w = np.asarray(weights if weights is not None else list(range(image.n_fields)), np.uint16)
        self._criteria_names = list(DEFAULT_CRITERIA if criteria is None else criteria)
        c = np.asarray([self._criterion(x) for x in self._criteria_names], np.int32)
        s = _Settings(image.n_fields, _p(w), _p(c), len(c), int(authorize_typos), one_typo, two_typos, int(prefix_search),
                      "\n".join(exact_words).encode() if exact_words else None)
        self._ck(l.b200_stage_settings(self._h, C.byref(s)))
        if synonyms:
            pairs = [(k, v) for k, vs in synonyms.items() for v in vs]
            fr = (C.c_char_p * len(pairs))(*[k.encode() for k, _ in pairs])
            to = (C.c_char_p * len(pairs))(*[v.encode() for _, v in pairs])
            self._ck(l.b200_stage_synonyms(self._h, len(pairs), fr, to))
        if geo is None and facets is not None and "_geo.lat" in facets.fields and "_geo.lng" in facets.fields:
            geo = (facets.fields["_geo.lat"], facets.fields["_geo.lng"])
        self._geo = geo
        if geo is not None:
            self._ck(l.b200_stage_geo_fields(self._h, geo[0], geo[1]))
        self._ck(l.b200_stage_finish(self._h))
        self.n_fields = image.n_fields

    def geo_point(self, docid):
        """the document's (lat, lng) as the GeoSort rule reads it (documents/geo_sort.rs:252-277): the smallest number value of each
        coordinate field, else its smallest string value parsed as f64"""
        if not hasattr(self, "_geo_points"):
            from corpus.facets import geo_points
            self._geo_points = geo_points(self._facets, *self._geo) if self._geo is not None else {}
        return self._geo_points[docid]

    def _criterion(self, name):
        if name.startswith(("asc:", "desc:")):
            d, field = name.split(":", 1)
            return (0x10000 if d == "asc" else 0x20000) | self.field_id(field)
        return CRITERIA[name]

    def sort_rule_names(self, sort_list):
        """field names of the sort rules of a search, in rule order (search/new/mod.rs:351-416, 651-716: the `sort` criterion expands
        to the list once, Asc/Desc criteria add one rule each, a name already sorted is skipped) -> (names, the list's survivors)"""
        names, kept, done = [], [], False
        for c in self._criteria_names:
            if c == "sort" and not done:
                done = True
                for item in sort_list:
                    f = item.rsplit(":", 1)[0]
                    if parse_geo_point(f) is not None:  # every `_geoPoint` entry is a rule of its own
                        names.append(f)
                        kept.append(item)
                    elif f not in names:
                        names.append(f)
                        kept.append(item)
            elif c.startswith(("asc:", "desc:")):
                f = c.split(":", 1)[1]
                if f not in names:
                    names.append(f)
        return names, kept

    def field_id(self, name):
        """the field's id in the facet databases, NO_FIELD when the fields map lacks it"""
        return self._fields.get(name, NO_FIELD)

    def sort_value(self, fid, is_string, key_index):
        """(field name, value) of a Sort score: the staged level-0 key's bound as a float or str, None for the Null bucket"""
        import struct

        name = next((n for n, f in self._fields.items() if f == fid), None)
        if key_index == 0xFFFFFFFF:
            return name, None
        k = self._level0[is_string][key_index]
        return name, (k[3:].decode() if is_string else struct.unpack(">d", k[11:19])[0])

    def set_embeddings(self, matrix, docids=None, distribution=None):
        """f32 rows (converted to fp16 on the device), or a float16 matrix staged as it is."""
        ids = None if docids is None else np.ascontiguousarray(docids, np.uint32)
        if getattr(matrix, "dtype", None) == np.float16:
            m = np.ascontiguousarray(matrix)
            self._ck(self._l.b200_stage_embeddings_f16(self._h, _p(m), m.shape[0], m.shape[1], _p(ids)))
        else:
            m = np.ascontiguousarray(matrix, np.float32)
            self._ck(self._l.b200_stage_embeddings(self._h, _p(m), m.shape[0], m.shape[1], _p(ids)))
        self.dim = m.shape[1]
        if distribution:
            self._ck(self._l.b200_stage_distribution(self._h, 1, distribution[0], distribution[1]))

    # S3 — compute_fully_if_needed (compute_derivations.rs:21-37)
    def derive(self, words, max_typo, is_prefix):
        enc = [w.encode() for w in words]
        off = np.zeros(len(enc) + 1, np.uint32)
        off[1:] = np.cumsum([len(b) for b in enc])
        buf = np.frombuffer(b"".join(enc) + b"\0", np.uint8).copy()
        mt = np.asarray(max_typo, np.uint8)
        ip = np.asarray(is_prefix, np.uint8)
        n = len(enc)
        one = np.zeros((n, 150), np.uint32)
        two = np.zeros((n, 50), np.uint32)
        n1 = np.zeros(n, np.uint32)
        n2 = np.zeros(n, np.uint32)
        self._ck(self._l.b200_derive_batch(self._h, n, _p(buf), _p(off), _p(mt), _p(ip), _p(one), _p(n1), _p(two), _p(n2)))
        return [(one[i, : n1[i]].copy(), two[i, : n2[i]].copy()) for i in range(n)]

    # S4 — VectorStore::nns_by_vector (vector/store.rs:638-675)
    def union_postings(self, db, key_indices, universe=None):
        """S2: (OR of the posting lists of database `db` at the given key positions) AND universe, as dense u64 words."""
        keys = np.ascontiguousarray(key_indices, np.uint32)
        n_words = (self._n_docs + 63) // 64
        out = np.zeros(n_words, np.uint64)
        uni = None if universe is None else np.ascontiguousarray(universe, np.uint64)
        self._ck(self._l.b200_union_postings(self._h, int(db), _p(keys), len(keys), _p(uni), 0 if uni is None else len(uni), _p(out)))
        return out

    def proximity_pairs(self, left, right, fwd_prox, bwd_prox, universe=None):
        """S2 for proximity conditions: universe AND the union of word_pair_proximity_docids[(fwd, l, r)] and [(bwd, r, l)]"""
        lw, rw = np.ascontiguousarray(left, np.uint32), np.ascontiguousarray(right, np.uint32)
        n_words = (self._n_docs + 63) // 64
        out = np.zeros(n_words, np.uint64)
        uni = None if universe is None else np.ascontiguousarray(universe, np.uint64)
        self._ck(self._l.b200_proximity_pairs(self._h, _p(lw), len(lw), _p(rw), len(rw), int(fwd_prox), int(bwd_prox), _p(uni),
                                              0 if uni is None else len(uni), _p(out)))
        return out

    def query_graph(self, query, stop_words=frozenset(), terms_matching_strategy="last", words_limit=10):
        """S1: QueryGraph::from_query for one query, as an opaque QueryGraph handle"""
        tokens = query if isinstance(query, TokenBatch) else TokenBatch([query], stop_words)
        b = _Batch(1, _p(tokens.token_begin), _p(tokens.token_kind), _p(tokens.lemma_off), _p(tokens.lemma_bytes), TMS[terms_matching_strategy], 0, 0, 1,
                   words_limit, None, 0, 0.0)
        b.stop_after = -1
        g = C.c_void_p()
        self._ck(self._l.b200_graph_from_tokens(self._h, C.byref(b), C.byref(g)))
        return QueryGraph(self, g)

    def nns_by_vector(self, queries, limit, candidates=None):
        q = np.ascontiguousarray(np.atleast_2d(queries), np.float32)
        n = q.shape[0]
        ids = np.zeros((n, limit), np.uint32)
        dist = np.zeros((n, limit), np.float32)
        cnt = np.zeros(n, np.uint32)
        cw = None if candidates is None else np.ascontiguousarray(candidates, np.uint64)
        self._ck(self._l.b200_nns_batch(self._h, _p(q), n, q.shape[1], limit, _p(cw), 0 if cw is None else len(cw), _p(ids), _p(dist), _p(cnt)))
        return ids, dist, cnt

    def comm_unique_id(self):
        out = np.zeros(128, np.uint8)
        self._ck(self._l.b200_comm_unique_id(self._h, _p(out)))
        return out

    def comm_init(self, rank, world, unique_id):
        """join the NCCL communicator of a corpus partitioned across GPUs (unique_id: 128 bytes drawn by rank 0)"""
        uid = np.ascontiguousarray(unique_id, np.uint8)
        self._ck(self._l.b200_comm_init(self._h, int(rank), int(world), _p(uid)))

    def nns_by_vector_sharded(self, queries, limit, candidates=None):
        """every rank: the same queries; returns the merged global top-k (per-shard scan + ncclAllGather + device merge)"""
        q = np.ascontiguousarray(np.atleast_2d(queries), np.float32)
        n = q.shape[0]
        ids = np.zeros((n, limit), np.uint32)
        dist = np.zeros((n, limit), np.float32)
        cnt = np.zeros(n, np.uint32)
        cw = None if candidates is None else np.ascontiguousarray(candidates, np.uint64)
        self._ck(self._l.b200_nns_batch_sharded(self._h, _p(q), n, q.shape[1], limit, _p(cw), 0 if cw is None else len(cw), _p(ids), _p(dist), _p(cnt)))
        return ids, dist, cnt

    def similar(self, ids, *, offset=0, limit=20, filter=None, universes=None, ranking_score_threshold=None, denied=()):
        """Similar::execute (search/similar.rs:66-152) for a batch of target documents (internal docids), as the `/similar` route
        runs it (b200_similar_batch): the nearest documents to each target's stored vector, the target left out.  filter: one filter
        (a string for parse_filter, or a tree it returns) for every target, or a list with one per target (None: no filter), see
        encode_filters for `denied`; universes: as Search.universes.  Returns a SearchResult (one Vector score per hit,
        n_candidates = estimatedTotalHits)."""
        targets = np.ascontiguousarray(np.atleast_1d(ids), np.uint32)
        n = len(targets)
        res = SearchResult(n, limit)
        rq = _SimilarRequest(n, _p(targets), offset, limit)
        keep = []
        if universes is not None:
            us = [universes] * n if isinstance(universes, np.ndarray) and universes.ndim == 1 else universes
            ptrs = (C.c_void_p * max(n, 1))()
            cache = {}
            for i, u in enumerate(us):
                if u is not None:
                    a = cache.setdefault(id(u), np.ascontiguousarray(u, np.uint64))
                    ptrs[i] = a.ctypes.data
                    rq.n_universe_words = len(a)
            keep += [cache, ptrs]
            rq.universes = C.cast(ptrs, C.c_void_p)
        r = _Results(_p(res.documents_ids), _p(res.n_hits), _p(res.n_scores), _p(res.score_kind), _p(res.score_rank), _p(res.score_max),
                     _p(res.score_sim), _p(res.n_candidates), None, _p(res.status))
        if filter is not None:
            prog = encode_filters(self, list(filter) if isinstance(filter, list) else [filter] * n, denied)
            keep.append(prog)
            rq.filter = C.cast(C.pointer(prog.struct), C.c_void_p)
            res.filter_error_leaf = np.full(max(n, 1), -1, np.int32)
            r.filter_error_leaf = _p(res.filter_error_leaf)
        rq.has_ranking_score_threshold = int(ranking_score_threshold is not None)
        rq.ranking_score_threshold = float(ranking_score_threshold or 0.0)
        self._ck(self._l.b200_similar_batch(self._h, C.byref(rq), C.byref(r)))
        return res

    def search(self):
        return Search(self)

    def geo_filter(self, clauses):
        """the geo leaves of a filter tree, one bitmap each (b200_geo_filter_batch): clause strings as Search.geo_filter takes them,
        without `NOT ` -> (uint64 bitmaps [n, words], statuses [n]); a clause with a non-zero status has an empty bitmap"""
        parsed = [parse_geo_filter(c) for c in clauses]
        if any(neg for _, neg, _ in parsed):
            raise ValueError("Index.geo_filter takes clauses without NOT: complement the bitmap against documents_ids")
        n = len(parsed)
        kind = np.asarray([k for k, _, _ in parsed] or [0], np.uint8)
        args = np.asarray([a for _, _, a in parsed] or [(0.0,) * 4], np.float64).reshape(-1)
        words = (self._n_docs + 63) // 64
        out = np.zeros((n, words), np.uint64)
        status = np.zeros(max(n, 1), np.int32)
        self._ck(self._l.b200_geo_filter_batch(self._h, n, _p(kind), _p(args), _p(out), words, _p(status)))
        return out, status[:n]

    def filter_batch(self, filters, denied=()):
        """IndexFilter::evaluate over documents_ids (b200_filter_batch): one filter per entry (a string for parse_filter, or a tree it
        returns; None = no filter) -> (uint64 bitmaps [n, words], statuses [n], failing leaves [n]); see encode_filters for `denied`"""
        prog = encode_filters(self, list(filters), denied)
        n = len(filters)
        words = (self._n_docs + 63) // 64
        out = np.zeros((n, words), np.uint64)
        status = np.zeros(max(n, 1), np.int32)
        leaf = np.zeros(max(n, 1), np.int32)
        self._ck(self._l.b200_filter_batch(self._h, C.byref(prog.struct), _p(out), words, _p(status), _p(leaf)))
        return out, status[:n], leaf[:n]

    def last_error(self):
        return self._l.b200_last_error(self._h).decode()

    def facet_original(self, fid, docid, normalized):
        """the original string of a string facet value (field_id_docid_facet_strings at (fid, docid, normalised)), the normalised
        value when the facet image did not record one (the reference logs an error and does the same)"""
        orig = getattr(self._facets, "originals", {}) if self._facets is not None else {}
        return orig.get((fid, docid, normalized), normalized)

    def facet_cap(self, names, max_values):
        """entries per slot that always suffice: max_values + the field's string values, or all its values when max_values is 0"""
        f = self._facets
        cap = 1
        for name in names:
            fid = self.field_id(name)
            n_num, n_str = len(f.numbers.get(fid, {})) if f else 0, len(f.strings.get(fid, {})) if f else 0
            cap = max(cap, n_num + n_str if max_values == 0 else max_values + n_str)
        return cap

    def facet_distribution(self, candidates, names, max_values=DEFAULT_VALUES_PER_FACET, order="alpha", cap=None):
        """FacetDistribution::execute + compute_stats for candidate bitmaps the caller holds (b200_facet_distribution_batch):
        candidates: a list of uint64 word arrays; names: one list of field names for all, or one per bitmap ->
        (per bitmap {name: [(key, count), ...]}, per bitmap {name: (min, max)}, statuses)"""
        n = len(candidates)
        per = names if (names and isinstance(names[0], (list, tuple))) else [names] * n
        out = _FacetOutputs(self, per, order, max_values, cap)
        begin = out.begin
        cache = {}
        arrs = [cache.setdefault(id(c), np.ascontiguousarray(c, np.uint64)) for c in candidates]
        ptrs = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in arrs])
        words = len(arrs[0]) if arrs else 0
        status = np.zeros(max(n, 1), np.int32)
        self._ck(self._l.b200_facet_distribution_batch(self._h, n, C.cast(ptrs, C.c_void_p), words, _p(begin), _p(out.fid), _p(out.orders), max_values,
                                                       out.cap, *out.pointers(), _p(status)))
        dists, stats = [], []
        for i in range(n):
            ks = range(int(begin[i]), int(begin[i + 1]))
            dists.append({name: out.distribution(self, k, max_values) for name, k in zip(per[i], ks)})
            stats.append({name: out.stats(k) for name, k in zip(per[i], ks) if out.stats(k) is not None})
        return dists, stats, status[:n]

    def facet_search(self, candidates, name, query=None, order="alpha", max_values=DEFAULT_MAX_FACET_SEARCH_VALUES, typos=True, cap=None):
        """SearchForFacetValues::execute for candidate bitmaps the caller holds (b200_facet_search_batch): candidates: a list of
        uint64 word arrays (None entries: documents_ids); name: the field; query: None, or the already normalised query, or one such
        value per bitmap; typos: the field is not an exact attribute -> (per bitmap [(value, count), ...] in the reference's order,
        statuses)"""
        n = len(candidates)
        qs = list(query) if isinstance(query, (list, tuple)) else [query] * n
        fid = np.full(max(n, 1), self.field_id(name), np.uint16)
        kind = np.asarray([0 if q is None else 1 for q in qs] or [0], np.uint8)
        enc = [b"" if q is None else q.encode() for q in qs]
        off = np.zeros(n + 1, np.uint32)
        off[1:] = np.cumsum([len(b) for b in enc]) if n else []
        qb = np.frombuffer(b"".join(enc) + b"\0", np.uint8).copy()
        flags = np.full(max(n, 1), (FACET_ORDERS[order]) | (2 if typos else 0), np.uint8)
        cap = max(1, max_values) if cap is None else cap
        cache = {}
        arrs = [None if c is None else cache.setdefault(id(c), np.ascontiguousarray(c, np.uint64)) for c in candidates]
        ptrs = (C.c_void_p * max(n, 1))(*[None if a is None else a.ctypes.data for a in arrs])
        words = next((len(a) for a in arrs if a is not None), (self._n_docs + 63) // 64)
        n_out = np.zeros(max(n, 1), np.uint32)
        key = np.zeros(max(n * cap, 1), np.uint32)
        count = np.zeros(max(n * cap, 1), np.uint64)
        docid = np.zeros(max(n * cap, 1), np.uint32)
        fallback = np.zeros(max(n * cap, 1), np.uint8)
        status = np.zeros(max(n, 1), np.int32)
        self._ck(self._l.b200_facet_search_batch(self._h, n, C.cast(ptrs, C.c_void_p), words, _p(fid), _p(kind), _p(off), _p(qb), _p(flags),
                                                 max_values, cap, _p(n_out), _p(key), _p(count), _p(docid), _p(fallback), _p(status)))
        out = [self._facet_hits(int(fid[i]), qs[i], key[i * cap:i * cap + int(n_out[i])], count[i * cap:], docid[i * cap:], fallback[i * cap:])
               for i in range(n)]
        return out, status[:n]

    def _facet_hits(self, fid, query, key, count, docid, fallback):
        """FacetValueHit { value, count } of each returned hit: the original string of (fid, docid, level-0 key), or the query (the key
        itself without a query) when fallback is set"""
        hits = []
        for e in range(len(key)):
            k = self._level0[1][int(key[e])][3:].decode()
            value = (query if query is not None else k) if fallback[e] else self.facet_original(fid, int(docid[e]), k)
            hits.append((value, int(count[e])))
        return hits

    def stats(self):
        s = _Stats()
        self._l.b200_get_stats(self._h, C.byref(s))
        d = {n: getattr(s, n) for n, _ in _Stats._fields_ if not n.startswith("kernel_") and not n.startswith("eval_class") and n != "host_ms"}
        d["eval_class_launches"] = list(s.eval_class_launches)
        d["eval_class_tiles"] = list(s.eval_class_tiles)
        d["host_ms"] = dict(zip(["parse", "derive", "terms", "pack", "device_wait", "advance", "results", "total"], list(s.host_ms)))
        d["kernel_launches"] = s.kernel_launches
        d["kernels"] = {KERNELS[i]: {"ms": s.kernel_ms[i], "count": s.kernel_count[i], "bytes": s.kernel_bytes[i]} for i in range(len(KERNELS))}
        return d

    def reset_stats(self):
        self._l.b200_reset_stats(self._h)

    def close(self):
        if getattr(self, "_h", None):
            self._l.b200_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class QueryGraph:
    """S1: an opaque query graph of the library (QueryGraph + its terms).  `rule()` is RankingRule::start_iteration .. next_bucket ..
    end_iteration for one ranking rule (ranking_rules.rs:26-83)."""

    def __init__(self, index, handle):
        self.index, self._g = index, handle

    def rule(self, kind, universe=None, terms_matching_strategy="last"):
        """yields (candidates bitmap, rank, max_rank, child QueryGraph or None) per bucket in ascending cost order"""
        ix = self.index
        uni = None if universe is None else np.ascontiguousarray(universe, np.uint64)
        r = C.c_void_p()
        ix._ck(ix._l.b200_rule_start(ix._h, SCORE_KINDS.index(kind), TMS[terms_matching_strategy], self._g, _p(uni), 0 if uni is None else len(uni), C.byref(r)))
        try:
            n_words = (ix._n_docs + 63) // 64
            while True:
                out = np.zeros(n_words, np.uint64)
                rank, mx, child = C.c_uint32(), C.c_uint32(), C.c_void_p()
                rc = ix._l.b200_rule_next(r, None, _p(out), n_words, C.byref(rank), C.byref(mx), C.byref(child))
                if rc == 1:
                    return
                if rc != 0:
                    raise B200Error(rc, "b200_rule_next")
                yield out, rank.value, mx.value, (QueryGraph(ix, child) if child.value else None)
        finally:
            ix._l.b200_rule_end(r)

    def close(self):
        if self._g is not None and self._g.value:
            self.index._l.b200_graph_free(self._g)
            self._g = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Search:
    """milli::Search builder (search/mod.rs:58-278) for a *batch* of queries sharing the same parameters."""

    def __init__(self, index):
        self.index = index
        self._tokens = None
        self._vectors = None
        self._tms = "last"
        self._scoring = "skip"
        self._offset, self._limit, self._words_limit = 0, 20, 10
        self._universes, self._budget_ms, self._stop_after, self._threshold, self._want_candidates = None, None, None, None, False
        self._sort = None
        self._geo_strategy, self._geo_max_bucket = (0, 1000), 1000
        self._geo_filter = None
        self._filter = None
        self._facet_names, self._max_values, self._facet_order, self._facet_cap = None, DEFAULT_VALUES_PER_FACET, "alpha", None
        self._fsearch = None

    def query(self, queries, stop_words=frozenset()):
        self._tokens = queries if isinstance(queries, TokenBatch) else TokenBatch([queries] if isinstance(queries, str) else list(queries), stop_words)
        return self

    def semantic(self, vectors):
        self._vectors = np.ascontiguousarray(np.atleast_2d(vectors), np.float32)
        return self

    def terms_matching_strategy(self, s):
        self._tms = s
        return self

    def scoring_strategy(self, s):
        self._scoring = s
        return self

    def offset(self, n):
        self._offset = n
        return self

    def limit(self, n):
        self._limit = n
        return self

    def words_limit(self, n):
        self._words_limit = n
        return self

    def universes(self, bitmaps):
        """filtered_universe per query: a list of uint64 word arrays (None = all documents), or one array shared by the batch"""
        self._universes = bitmaps
        return self

    def deadline(self, budget_ms=None, stop_after=None):
        """Search::deadline: a time budget in ms, or the reference's poll-count hook Deadline::never().with_stop_after(n)"""
        self._budget_ms, self._stop_after = budget_ms, stop_after
        return self

    def ranking_score_threshold(self, t):
        self._threshold = t
        return self

    def sort(self, criteria):
        """Search::sort_criteria: ["price:asc", "_geoPoint(48.85, 2.35):desc", ...] for every query of the batch, or one such list
        per query"""
        self._sort = criteria
        return self

    def geo_strategy(self, strategy, cache_size=1000):
        """Search::geo_sort_strategy: "dynamic" (the default), "iterative" or "rtree", with its cache size"""
        self._geo_strategy = (GEO_STRATEGIES[strategy], cache_size)
        return self

    def geo_max_bucket_size(self, n):
        """Search::geo_max_bucket_size (default 1000)"""
        self._geo_max_bucket = n
        return self

    def geo_filter(self, clauses):
        """geo leaves at the top of the filter, ANDed with the universe: ["_geoRadius(48.85, 2.35, 2000)", "NOT _geoBoundingBox([1, 2],
        [0, 1])"] for every query of the batch, or one such list per query (see parse_geo_filter)"""
        self._geo_filter = clauses
        return self

    def filter(self, trees, denied=()):
        """the `filter` search parameter: one filter (a string for parse_filter, or a tree it returns) for every query of the batch,
        or a list with one per query (None: no filter); see encode_filters for `denied`"""
        self._filter = (trees, denied)
        return self

    def facet_search(self, name, query=None, order="alpha", max_values=DEFAULT_MAX_FACET_SEARCH_VALUES, typos=True):
        """a facet search over each query's candidates (the facet-search route): field `name` (None: no facet search for that query),
        the already normalised query (None or a string), sortFacetValuesBy, maxValuesPerFacet, and whether the field allows typos (it
        is not an exact attribute).  name and query may be lists, one entry per query."""
        self._fsearch = (name, query, order, max_values, typos)
        return self

    def facets(self, names):
        """the `facets` search parameter: field names for every query of the batch, or one such list per query"""
        self._facet_names = names
        return self

    def max_values_per_facet(self, n):
        """maxValuesPerFacet (default 100)"""
        self._max_values = n
        return self

    def facet_order(self, order):
        """sortFacetValuesBy for every field: "alpha" (the default) or "count" (refused by the library)"""
        self._facet_order = order
        return self

    def facet_cap(self, cap):
        """entries per (query, field) in the facet outputs (default: Index.facet_cap, always enough)"""
        self._facet_cap = cap
        return self

    def with_candidates(self):
        self._want_candidates = True
        return self

    def _run(self, mode, ratio=0.0):
        ix = self.index
        tokens = self._tokens
        if tokens is None:
            n = self._vectors.shape[0] if self._vectors is not None else 1
            tokens = TokenBatch([""] * n)
        n = tokens.n_queries
        res = SearchResult(n, self._limit, ix.sort_value, ix.geo_point)
        b = _Batch(n, _p(tokens.token_begin), _p(tokens.token_kind), _p(tokens.lemma_off), _p(tokens.lemma_bytes), TMS[self._tms],
                   1 if self._scoring == "detailed" else 0, self._offset, self._limit, self._words_limit,
                   _p(self._vectors) if self._vectors is not None else None, mode, ratio)
        keep = []
        if self._universes is not None:
            us = self._universes
            if isinstance(us, np.ndarray) and us.ndim == 1:
                us = [us] * n
            ptrs = (C.c_void_p * n)()
            cache = {}
            for i, u in enumerate(us):
                if u is None:
                    continue
                if id(u) not in cache:
                    a = np.ascontiguousarray(u, np.uint64)
                    keep.append(a)
                    cache[id(u)] = a
                a = cache[id(u)]
                ptrs[i] = a.ctypes.data
                b.n_universe_words = len(a)
            keep.append(ptrs)
            b.universes = C.cast(ptrs, C.c_void_p)
        if self._sort is not None:
            per_q = self._sort if (self._sort and isinstance(self._sort[0], (list, tuple))) else [self._sort] * n
            rules = [ix.sort_rule_names(list(x)) for x in per_q]
            res.sort_names = [r_[0] for r_ in rules]
            # the library deduplicates by field id; a repeated name of a field absent from the fields map is dropped here
            if "sort" in ix._criteria_names:  # (without it the list is SortRankingRuleMissing: sent as it is)
                per_q = [kept if any(ix.field_id(i.rsplit(":", 1)[0]) == NO_FIELD for i in x) else list(x) for x, (_, kept) in zip(per_q, rules)]
            begin = np.zeros(n + 1, np.uint32)
            begin[1:] = np.cumsum([len(x) for x in per_q])
            items = [c.rsplit(":", 1) for x in per_q for c in x]
            geo = [parse_geo_point(f) for f, _ in items]
            fid = np.asarray([NO_FIELD if g is not None else ix.field_id(f) for (f, _), g in zip(items, geo)] or [0], np.uint16)
            asc = np.asarray([1 if d == "asc" else 0 for _, d in items] or [0], np.uint8)
            is_geo = np.asarray([g is not None for g in geo] or [0], np.uint8)
            point = np.asarray([g if g is not None else (0.0, 0.0) for g in geo] or [(0.0, 0.0)], np.float64).reshape(-1)
            keep += [begin, fid, asc, is_geo, point]
            b.sort_begin, b.sort_fid, b.sort_asc = _p(begin), _p(fid), _p(asc)
            b.sort_geo, b.sort_geo_point = _p(is_geo), _p(point)
        if self._geo_filter is not None:
            gf = self._geo_filter
            per_q = gf if (gf and isinstance(gf[0], (list, tuple))) else [gf] * n
            parsed = [[parse_geo_filter(c) for c in x] for x in per_q]
            begin = np.zeros(n + 1, np.uint32)
            begin[1:] = np.cumsum([len(x) for x in parsed])
            flat = [c for x in parsed for c in x]
            kind = np.asarray([k for k, _, _ in flat] or [0], np.uint8)
            neg = np.asarray([int(g) for _, g, _ in flat] or [0], np.uint8)
            args = np.asarray([a for _, _, a in flat] or [(0.0,) * 4], np.float64).reshape(-1)
            keep += [begin, kind, neg, args]
            b.geo_filter_begin, b.geo_filter_kind, b.geo_filter_not, b.geo_filter_args = _p(begin), _p(kind), _p(neg), _p(args)
        if self._filter is not None:
            trees, denied = self._filter
            per_q = list(trees) if isinstance(trees, list) else [trees] * n
            prog = encode_filters(ix, per_q, denied)
            keep.append(prog)
            b.filter = C.cast(C.pointer(prog.struct), C.c_void_p)
            res.filter_error_leaf = np.full(max(n, 1), -1, np.int32)
        b.geo_strategy, b.geo_cache_size = self._geo_strategy
        b.geo_max_bucket_size = self._geo_max_bucket
        b.time_budget_ns = 0 if self._budget_ms is None else max(1, int(self._budget_ms * 1e6))
        b.stop_after = -1 if self._stop_after is None else int(self._stop_after)
        b.has_ranking_score_threshold = int(self._threshold is not None)
        b.ranking_score_threshold = float(self._threshold or 0.0)
        r = _Results(_p(res.documents_ids), _p(res.n_hits), _p(res.n_scores), _p(res.score_kind), _p(res.score_rank), _p(res.score_max),
                     _p(res.score_sim), _p(res.n_candidates), _p(res.semantic_hit_count), _p(res.status), _p(res.degraded),
                     _p(res.used_negative_operator), None, 0)
        if self._facet_names is not None:
            fn = self._facet_names
            per_q = [list(x) for x in fn] if (fn and isinstance(fn[0], (list, tuple))) else [list(fn)] * n
            out = _FacetOutputs(ix, per_q, self._facet_order, self._max_values, self._facet_cap)
            keep.append(out)
            b.facet_begin, b.facet_fid, b.facet_order = _p(out.begin), _p(out.fid), _p(out.orders)
            b.facet_max_values, b.facet_cap = self._max_values, out.cap
            (r.facet_n_num, r.facet_n_str, r.facet_key, r.facet_count, r.facet_docid, r.facet_has_stats, r.facet_min,
             r.facet_max) = out.pointers()
            res._facets = (ix, per_q, out.begin, out, self._max_values)
        if self._fsearch is not None:
            name, query, order, mx, typos = self._fsearch
            names = list(name) if isinstance(name, (list, tuple)) else [name] * n
            qs = list(query) if isinstance(query, (list, tuple)) else [query] * n
            fid = np.asarray([NO_FIELD if nm is None else ix.field_id(nm) for nm in names] or [NO_FIELD], np.uint16)
            kind = np.asarray([0 if q is None else 1 for q in qs] or [0], np.uint8)
            enc = [b"" if q is None else q.encode() for q in qs]
            off = np.zeros(n + 1, np.uint32)
            off[1:] = np.cumsum([len(x) for x in enc]) if n else []
            qb = np.frombuffer(b"".join(enc) + b"\0", np.uint8).copy()
            flags = np.full(max(n, 1), FACET_ORDERS[order] | (2 if typos else 0), np.uint8)
            outs = (np.zeros(max(n, 1), np.uint32), np.zeros(max(n * mx, 1), np.uint32), np.zeros(max(n * mx, 1), np.uint64),
                    np.zeros(max(n * mx, 1), np.uint32), np.zeros(max(n * mx, 1), np.uint8))
            keep += [fid, kind, off, qb, flags]
            b.facet_search_fid, b.facet_query_kind, b.facet_query_off, b.facet_query_bytes = _p(fid), _p(kind), _p(off), _p(qb)
            b.facet_search_flags, b.facet_search_max = _p(flags), mx
            r.fs_n, r.fs_key, r.fs_count, r.fs_docid, r.fs_fallback = (_p(a) for a in outs)
            res._facet_search = (ix, [(int(fid[q]), qs[q]) for q in range(n)], outs + (mx,))
        if self._filter is not None:
            r.filter_error_leaf = _p(res.filter_error_leaf)
        if self._want_candidates:
            words = (ix._n_docs + 63) // 64
            res.candidates = np.zeros((n, words), np.uint64)
            r.candidates, r.candidates_words = _p(res.candidates), words
        ix._ck(ix._l.b200_search_batch(ix._h, C.byref(b), C.byref(r)))
        return res

    def execute(self):
        """Search::execute (search/mod.rs:280): keyword search, or semantic search when a vector was given and no query."""
        return self._run(1 if (self._vectors is not None and self._tokens is None) else 0)

    def execute_hybrid(self, semantic_ratio):
        """Search::execute_hybrid (search/hybrid.rs:264)."""
        return self._run(2, float(semantic_ratio))
