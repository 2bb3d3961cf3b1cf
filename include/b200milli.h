/* b200milli — H100-native (sm_90a) implementation of milli's query-time scoring path.
 *
 * C ABI of the drop-in boundary (SURVEY.md §8(b)).  The reference has no FFI for this path; its
 * seams are Rust-internal.  Each entry point names the reference interface a Rust shim would
 * replace with a call to it (paths relative to the meilisearch checkout, v1.50.0 @ 5cb2f2e).
 * Conventions: caller allocates every output; the library never frees caller memory; handles are
 * opaque; every function returns 0 on success or a negative B200_ERR_* code, with a message
 * available from b200_last_error(); no exceptions/panics cross the boundary; one handle may be
 * used from many threads (calls are serialised per handle; each call runs on the handle's stream).
 * There is NO CPU fallback: without a CUDA device b200_open fails with B200_ERR_NO_DEVICE.
 */
#ifndef B200MILLI_H
#define B200MILLI_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ERR_NO_DEVICE (-1)   /* no CUDA device / driver (the product never falls back to the CPU) */
#define B200_ERR_CUDA (-2)        /* a CUDA call failed; see b200_last_error */
#define B200_ERR_INVALID (-3)     /* bad argument */
#define B200_ERR_UNSUPPORTED (-4) /* query feature outside the implemented scope (distinct, more than 12 terms, ...) */
#define B200_ERR_CAPACITY (-5)    /* a device work queue / arena overflowed */
#define B200_ERR_STATE (-6)       /* call order (e.g. search before b200_stage_finish) */

typedef struct b200_index b200_index;

/* ---- lifecycle ------------------------------------------------------------------------- */
/* Replaces: opening the LMDB env for search (crates/milli/src/index.rs:129-…) — here a device-resident copy. */
int b200_open(int device_ordinal, b200_index **out);
void b200_close(b200_index *);
const char *b200_last_error(const b200_index *); /* valid until the next call on the handle */
/* message of the last failure of b200_open itself */
const char *b200_open_error(void);

/* ---- staging: done once, copies everything (LMDB pages are only borrowed for a RoTxn) --- */
/* database ids, in the key/value formats of crates/milli/src/index.rs:97-124 and
 * heed_codec/{str_beu32_codec.rs (StrBEU16Codec), str_str_u8_codec.rs (U8StrStrCodec)};
 * values are CboRoaringBitmapCodec bytes (heed_codec/roaring_bitmap/cbo_roaring_bitmap_codec.rs:15-85). */
enum b200_db {
    B200_DB_WORD_DOCIDS = 0,               /* key: word */
    B200_DB_EXACT_WORD_DOCIDS = 1,         /* key: word */
    B200_DB_WORD_PREFIX_DOCIDS = 2,        /* key: prefix */
    B200_DB_EXACT_WORD_PREFIX_DOCIDS = 3,  /* key: prefix */
    B200_DB_WORD_PAIR_PROXIMITY_DOCIDS = 4,/* key: u8 prox | w1 | 0x00 | w2 */
    B200_DB_WORD_POSITION_DOCIDS = 5,      /* key: word | 0x00 | u16 BE bucketed position */
    B200_DB_WORD_FID_DOCIDS = 6,           /* key: word | 0x00 | u16 BE field id */
    B200_DB_WORD_PREFIX_POSITION_DOCIDS = 7,
    B200_DB_WORD_PREFIX_FID_DOCIDS = 8,
    B200_DB_FIELD_ID_WORD_COUNT_DOCIDS = 9,/* key: u16 BE fid | u8 count */
    /* facet databases read by the Sort rule (search/new/sort.rs:98-195).  Key: u16 BE fid | u8 level | left bound, where the bound
     * is the 16-byte OrderedF64Codec (heed_codec/facet/ordered_f64_codec.rs: globally ordered f64 bytes, then the f64 big-endian)
     * or the normalised string bytes (lib.rs normalize_facet; booleans are "true" / "false").  Value: FacetGroupValueCodec =
     * u8 size | CBO bytes (heed_codec/facet/mod.rs).  Only level-0 entries are read; higher levels are accepted and ignored. */
    B200_DB_FACET_ID_F64_DOCIDS = 10,
    B200_DB_FACET_ID_STRING_DOCIDS = 11,
    /* facet databases read by facet search (search/facet/search.rs:119-265).  facet_id_normalized_string_strings: key u16 BE fid |
     * hyper-normalised string, value the serde_json bytes of the BTreeSet<String> of level-0 keys of facet_id_string_docids it
     * stands for (index.rs facet_id_normalized_string_strings).  A field's facet-string FST (facet_id_string_fst) holds exactly
     * the keys of its entries here: indexing registers every key it writes or deletes in this database with the FST merger
     * (update/new/facet_search_builder.rs:148-213), so a shim may stage the keys from either source.  A value that is not a JSON
     * array of strings makes b200_stage_finish fail with B200_ERR_INVALID.
     * field_id_docid_facet_strings: key u16 BE fid | u32 BE docid | normalised string, value the original string
     * (heed_codec/facet/field_doc_id_facet_codec.rs, index.rs:181-188). */
    B200_DB_FACET_ID_NORMALIZED_STRING_STRINGS = 12,
    B200_DB_FIELD_ID_DOCID_FACET_STRINGS = 13,
    /* facet databases read by the EXISTS / IS NULL / IS EMPTY filters (Index::{exists,null,empty}_faceted_documents_ids).  Key: u16
     * BE fid; value: CBO bytes.  An index staged without one of them searches as before; a filter program with a leaf that reads a
     * database that was not staged fails its query with B200_ERR_INVALID. */
    B200_DB_FACET_ID_EXISTS_DOCIDS = 14,
    B200_DB_FACET_ID_IS_NULL_DOCIDS = 15,
    B200_DB_FACET_ID_IS_EMPTY_DOCIDS = 16,
    B200_DB_COUNT = 17
};
/* Replaces Index::words_fst (index.rs:1238): the FST enumerated once on the host into its sorted word list. */
int b200_stage_dictionary(b200_index *, const uint8_t *word_bytes, const uint64_t *word_offsets, uint64_t n_words);
/* Replaces the typed `Database<..., CboRoaringBitmapCodec>` handles read by search/new/db_cache.rs:183-719.
 * Keys must be in LMDB (bytewise) order. */
int b200_stage_db(b200_index *, int db, uint64_t n_keys, const uint8_t *key_bytes, const uint64_t *key_offsets,
                  const uint8_t *val_bytes, const uint64_t *val_offsets);
/* Replaces Index::documents_ids (index.rs, main["documents-ids"]); CBO bytes. */
int b200_stage_documents_ids(b200_index *, const uint8_t *cbo, uint64_t len);

/* criteria (crates/milli/src/criterion.rs:121-131) */
enum b200_criterion { B200_C_WORDS = 0, B200_C_TYPO = 1, B200_C_PROXIMITY = 2, B200_C_ATTRIBUTE = 3, B200_C_ATTRIBUTE_RANK = 4,
                      B200_C_WORD_POSITION = 5, B200_C_SORT = 6, B200_C_EXACTNESS = 7 };
/* custom criteria Criterion::Asc(field) / Desc(field) (criterion.rs:32-35), fid = the field's id in the facet databases */
#define B200_C_ASC(fid) (0x10000 | (int32_t)(fid))
#define B200_C_DESC(fid) (0x20000 | (int32_t)(fid))
typedef struct {
    uint32_t n_fields;              /* searchable fields; fid = 0..n_fields-1 */
    const uint16_t *weights;        /* fieldids_weights_map: fid -> weight */
    const int32_t *criteria;        /* index `criteria` setting */
    uint32_t n_criteria;
    int32_t authorize_typos;        /* index.rs authorize-typos */
    uint32_t min_word_len_one_typo; /* index.rs:46 (5) */
    uint32_t min_word_len_two_typos;/* index.rs:47 (9) */
    int32_t prefix_search;          /* PrefixSearch::IndexingTime (1) / Disabled (0) */
    const char *exact_words;        /* '\n'-joined exact_words set (may be NULL) */
} b200_settings;
int b200_stage_settings(b200_index *, const b200_settings *);
/* The index `synonyms` database (crates/milli/src/index.rs synonyms; read by compute_derivations.rs:221-239 and
 * parse_query.rs:277-285): entry i maps the word sequence from_words[i] to the word sequence to_words[i], both already
 * tokenised and joined by single spaces.  Several entries may share the same `from`.  Replaces any previous set. */
int b200_stage_synonyms(b200_index *, uint32_t n, const char *const *from_words, const char *const *to_words);
/* The GeoSort rule's fields (search/new/geo_sort.rs): the fids of `_geo.lat` and `_geo.lng` in the facet databases.  Indexing writes
 * them as number facets (update/new/extract/faceted/facet_document.rs:82-99); b200_stage_finish reads each document's point from
 * their level-0 entries in facet_id_f64_docids (the smallest value when there are several, as geo_value's prefix iteration takes,
 * documents/geo_sort.rs:252-277), else from facet_id_string_docids parsed as f64.  The geo documents (geo_faceted_documents_ids)
 * are those with a point.  A document with only one of the two coordinates, or an unparsable string one, makes
 * b200_stage_finish fail with B200_ERR_INVALID (the reference panics).  Without this call no document is geo: every GeoSort rule
 * returns one Null bucket.  Must precede b200_stage_finish. */
int b200_stage_geo_fields(b200_index *, uint16_t lat_fid, uint16_t lng_fid);
/* Uploads everything to HBM and builds the device directories.  Must follow the stage_* calls. */
int b200_stage_finish(b200_index *);
/* Replaces the arroy/hannoy item nodes read by VectorStore (crates/milli/src/vector/store.rs:1427-1434):
 * one f32[d] vector per row + its docid.  Stored on device as fp16 rows + f32 inverse norms. */
int b200_stage_embeddings(b200_index *, const float *vectors, uint64_t n, uint32_t d, const uint32_t *docids);
/* Same store from rows that are already IEEE binary16 (a quantised store, or a corpus generated as fp16): no f32 round trip;
 * the inverse norms are those of the fp16 values. */
int b200_stage_embeddings_f16(b200_index *, const uint16_t *rows_fp16, uint64_t n, uint32_t d, const uint32_t *docids);
/* Embedder `distribution` (crates/milli/src/vector/distribution.rs): enabled=0 disables the shift. */
int b200_stage_distribution(b200_index *, int enabled, float mean, float sigma);

/* ---- S3: term derivation --------------------------------------------------------------- */
/* Replaces Interned<QueryTerm>::compute_fully_if_needed -> find_one_typo_derivations /
 * find_one_two_typo_derivations (crates/milli/src/search/new/query_term/compute_derivations.rs:21-168),
 * i.e. `fst.search_with_state(Intersection/Union(StartsWith, LevenshteinDFA))`.
 * For word i (bytes words[word_off[i]..word_off[i+1]]), max_typo[i] in {1,2}, is_prefix[i] in {0,1}:
 * one_out[i*150..] gets up to 150 dictionary ranks at distance 1, two_out[i*50..] up to 50 at distance 2
 * (ascending rank order, caps and first-letter rule exactly as the reference). */
#define B200_MAX_ONE_TYPO 150
#define B200_MAX_TWO_TYPOS 50
int b200_derive_batch(b200_index *, uint32_t n_words, const char *words, const uint32_t *word_off, const uint8_t *max_typo,
                      const uint8_t *is_prefix, uint32_t *one_out, uint32_t *n_one, uint32_t *two_out, uint32_t *n_two);

/* ---- S2: condition resolver (union-shaped conditions) ---------------------------------- */
/* Replaces the posting-list part of G::resolve_condition as called by ConditionDocIdsCache::get_computed_condition
 * (crates/milli/src/search/new/ranking_rule_graph/condition_docids_cache.rs:34-57; the unions are
 * compute_query_term_subset_docids, crates/milli/src/search/new/resolve_query_graph.rs:33-59): out = (OR of the posting lists of
 * `db` at key indices key_index[0..n_keys)) AND universe.  db: the b200_stage_db id; a key index is the position of the key in the
 * database as staged (LMDB order).  universe: dense little-endian u64 words over docids, NULL = all documents; out: the same
 * shape, ceil((max docid + 1) / 64) words. */
int b200_union_postings(b200_index *, int db, const uint32_t *key_index, uint32_t n_keys, const uint64_t *universe, uint64_t n_universe_words,
                        uint64_t *out);

/* Replaces ProximityGraph::resolve_condition for one edge (crates/milli/src/search/new/ranking_rule_graph/proximity/compute_docids.rs:15-108,
 * the non-prefix lookups :172-211): out = universe AND the union, over every l in `left` and r in `right` (dictionary ranks, i.e.
 * positions in the staged dictionary), of word_pair_proximity_docids[(fwd_prox, l, r)] and word_pair_proximity_docids[(bwd_prox, r, l)];
 * a proximity of 0 disables that direction.  universe / out as in b200_union_postings. */
int b200_proximity_pairs(b200_index *, const uint32_t *left, uint32_t n_left, const uint32_t *right, uint32_t n_right, uint32_t fwd_prox,
                         uint32_t bwd_prox, const uint64_t *universe, uint64_t n_universe_words, uint64_t *out);

/* ---- S4: vector store ------------------------------------------------------------------ */
/* Replaces VectorStore::nns_by_vector (crates/milli/src/vector/store.rs:638-675) for a batch of queries:
 * exact scan, ascending distance (1 - cos)/2, ties by ascending docid.
 * queries: n_q x d f32 (host).  cand_bitmap: optional dense little-endian u64 words over docids (filter),
 * shared by the batch (NULL = all).  ids_out/dist_out: n_q x limit; n_out: n_q. */
int b200_nns_batch(b200_index *, const float *queries, uint32_t n_q, uint32_t d, uint32_t limit, const uint64_t *cand_bitmap,
                   uint64_t n_cand_words, uint32_t *ids_out, float *dist_out, uint32_t *n_out);

/* ---- corpus partitioned across GPUs (SURVEY §8(e), cfg 5) --------------------------------- */
/* One process per GPU, each with the rows of its docid range staged (b200_stage_embeddings with global docids).  The library
 * binds NCCL at run time (libnccl.so.2).  Rank 0 draws a unique id, the host application carries its 128 bytes to the other
 * ranks, every rank calls b200_comm_init. */
int b200_comm_unique_id(b200_index *, uint8_t *out128);
int b200_comm_init(b200_index *, int rank, int world, const uint8_t *unique_id128);
/* b200_nns_batch over the partitioned store: every rank passes the SAME queries (and candidate bitmap over global docids); each
 * scans its shard, the per-shard top-`limit` lists are exchanged with one ncclAllGather on the library's vector stream and merged
 * on the device by (distance, docid); every rank receives the global result. */
int b200_nns_batch_sharded(b200_index *, const float *queries, uint32_t n_q, uint32_t d, uint32_t limit, const uint64_t *cand_bitmap,
                           uint64_t n_cand_words, uint32_t *ids_out, float *dist_out, uint32_t *n_out);

/* ---- S0: whole search ------------------------------------------------------------------ */
/* Replaces milli::Search::execute / execute_hybrid (crates/milli/src/search/mod.rs:280-415,
 * search/hybrid.rs:264-366) for a batch of queries against one index, as called from
 * search_from_kind (crates/meilisearch/src/search/mod.rs:2126-2148) / SearchByIndex::execute
 * (crates/meilisearch/src/search/federated/perform.rs:1544).
 * Queries arrive tokenised (charabia stays on the host): tokens of query i are
 * [token_begin[i], token_begin[i+1]); kind: 0 Word, 1 StopWord, 2 Separator(Soft), 3 Separator(Hard). */
enum b200_tms { B200_TMS_LAST = 0, B200_TMS_ALL = 1, B200_TMS_FREQUENCY = 2 };

/* Filter programs: the parsed FilterCondition tree of IndexFilter::inner_evaluate (search/facet/filter/index_filter.rs:332-696),
 * as a Rust shim gets it from filter-parser, after the caller's not-filterable check of `evaluate` (:43-73).  Program i is the nodes
 * [begin[i], begin[i + 1]) in pre-order (an empty range: no filter).  AND / OR take the next `n` subtrees as their children, in
 * order; NOT the next one.  Value strings arrive normalize_facet'd; a value's number is what parse_finite_float gives, NaN when it
 * does not parse.  Semantics (bitmaps, `docs` = documents_ids):
 *   RANGE(fid, lo, hi, values [value, value + 2)): the level-0 keys of facet_id_f64_docids between the numbers of the two values
 *     (only when has_number: for `TO` both ends parse, for `>`, `>=`, `<`, `<=` the one given), in OrderedF64 key order, plus the
 *     keys of facet_id_string_docids between the two strings in byte order (ValueBounds::new); lo / hi are b200_bound kinds, the
 *     same for both; an inverted interval is empty.
 *   EQUAL(fid, value): the string key's docids OR the number key's docids when the number parses (evaluate_equal).  NOT_EQUAL:
 *     docs - EQUAL.  IN(fid, values [value, value + n)): the union of the EQUALs.
 *   EXISTS / IS_NULL / IS_EMPTY(fid): the field's entry in B200_DB_FACET_ID_{EXISTS,IS_NULL,IS_EMPTY}_DOCIDS.
 *   GEO_RADIUS / GEO_BBOX: args as b200_query_batch::geo_filter_args; a GEO_BBOX is the range conditions on `_geo.lat` /
 *     `_geo.lng` it stands for, so it intersects with its hint like RANGE.  EMPTY: nothing (a field absent from the fields map or
 *     matching no filterable rule).  DENIED(fid): the field's FilterableAttributesFeatures forbid the operator (the caller keeps the
 *     message).  AND of zero children: nothing.  NOT x: docs - x.
 * A value leaf on a fid without facet values matches nothing.  The reference raises a leaf's error only when evaluation reaches it:
 * AND stops at an empty running bitmap and passes it as the universe hint of its next child; RANGE, GEO_BBOX and NOT intersect with
 * their hint, the other leaves ignore it; a node whose hint is empty is not evaluated.  The library reproduces that reach exactly: a
 * DENIED leaf, or a geo leaf with bad arguments or on an index without b200_stage_geo_fields (`_geo` not filterable), fails its
 * query with B200_ERR_INVALID and the reference's message only when reached, the first in pre-order winning.  Per query, whatever is
 * reached: an UNSUPPORTED node (CONTAINS, STARTS WITH, _geoPolygon, _geojson, the `resolution` argument, _vectors, the `_shard`
 * field) or nesting deeper than B200_MAX_FILTER_DEPTH nodes (milli's MAX_FILTER_DEPTH, search/facet/filter/mod.rs, the bound
 * IndexFilter::evaluate walks the tree with) is B200_ERR_UNSUPPORTED; EXISTS / IS_NULL / IS_EMPTY without their staged database, an
 * unknown op or a tree that does not fit its node range is B200_ERR_INVALID. */
#define B200_MAX_FILTER_DEPTH 2000
enum b200_filter_op { B200_F_AND = 0, B200_F_OR = 1, B200_F_NOT = 2, B200_F_RANGE = 3, B200_F_EQUAL = 4, B200_F_NOT_EQUAL = 5, B200_F_IN = 6,
                      B200_F_EXISTS = 7, B200_F_IS_NULL = 8, B200_F_IS_EMPTY = 9, B200_F_GEO_RADIUS = 10, B200_F_GEO_BBOX = 11,
                      B200_F_EMPTY = 12, B200_F_DENIED = 13, B200_F_UNSUPPORTED = 14 };
enum b200_bound { B200_B_INCLUDED = 0, B200_B_EXCLUDED = 1, B200_B_UNBOUNDED = 2 };
typedef struct {
    uint8_t op;          /* b200_filter_op */
    uint8_t lo, hi;      /* RANGE: b200_bound of each end */
    uint8_t has_number;  /* RANGE: the number bounds exist */
    uint16_t fid;        /* the field's id in the facet databases */
    uint16_t pad;
    uint32_t n;          /* AND / OR: children; IN: values */
    uint32_t value;      /* RANGE, EQUAL, NOT_EQUAL, IN: the first value */
    double args[4];      /* GEO_RADIUS / GEO_BBOX */
} b200_filter_node;
typedef struct {
    uint32_t n;                      /* programs */
    const uint32_t *begin;           /* n + 1 node offsets */
    const b200_filter_node *nodes;
    uint32_t n_values;
    const uint32_t *value_off;       /* n_values + 1: value v is value_bytes[value_off[v] .. value_off[v + 1]) */
    const char *value_bytes;
    const double *value_num;         /* value v's number, NaN = none */
} b200_filter_programs;

typedef struct {
    uint32_t n_queries;
    const uint32_t *token_begin;  /* n_queries + 1 */
    const uint8_t *token_kind;
    const uint32_t *lemma_off;    /* n_tokens + 1 */
    const char *lemma_bytes;
    int32_t terms_matching_strategy; /* b200_tms */
    int32_t scoring_strategy;        /* 0 Skip, 1 Detailed (score_details.rs:431-438) */
    uint32_t offset, limit;          /* Search::offset / limit */
    uint32_t words_limit;            /* Search::words_limit (default 10) */
    const float *vectors;            /* n_queries x d, or NULL: the `semantic` vector per query */
    int32_t mode;                    /* 0 keyword (execute), 1 semantic (execute with vector), 2 hybrid (execute_hybrid) */
    float semantic_ratio;            /* hybrid only */
    /* filtered_universe (search/new/mod.rs:719: documents_ids & filter), what Search::filter / candidates produce on the host:
     * n_queries pointers to dense little-endian u64 words over docids (n_universe_words each), NULL entry = all documents,
     * NULL array = no filter anywhere.  Queries may share a bitmap (equal pointers are uploaded once). */
    const uint64_t *const *universes;
    uint64_t n_universe_words;
    /* Search::deadline (crates/milli/src/lib.rs:154-226).  time_budget_ns > 0: Deadline::from_budget, counted from the start of
     * the call; 0: Deadline::never.  stop_after >= 0: the reference's poll-count hook (Deadline::with_stop_after(n): exceeded from
     * the n-th poll on, the clock is then ignored); -1: unused.  When the deadline is exceeded the remaining universe of every
     * rule is returned unsorted with a Skipped score and the result is marked degraded (bucket_sort.rs:206-264). */
    uint64_t time_budget_ns;
    int64_t stop_after;
    /* Search::ranking_score_threshold (bucket_sort.rs:188,221-224,293-296) */
    int32_t has_ranking_score_threshold;
    double ranking_score_threshold;
    /* Search::sort_criteria (search/mod.rs:160): the `sort` list of query i is entries [sort_begin[i], sort_begin[i+1]) of
     * sort_fid / sort_asc / sort_geo; sort_begin NULL = no `sort` anywhere.  sort_fid: the field's id in the facet databases, 0xFFFF
     * for a field absent from the fields map (it sorts nothing: every document lands in the Null bucket).  Rules on a field already
     * sorted earlier in the rule list are skipped by fid; 0xFFFF entries are never skipped, so the caller, which sees the names,
     * leaves out an absent field whose name is already sorted (milli deduplicates by name); sort_asc: 1 Asc, 0 Desc.
     * sort_geo (NULL = none): 1 marks a `_geoPoint(lat, lng)` entry, whose point is sort_geo_point[2 k], [2 k + 1] and whose sort_fid
     * is ignored.  Each one adds a GeoSort rule; geo entries are never deduplicated (resolve_sort_criteria, search/new/mod.rs:651-716).
     * The sortable-attributes check stays with the caller.  A non-empty list while the criteria lack `sort`
     * (SortRankingRuleMissing, search/new/mod.rs:998-1040) is B200_ERR_INVALID for that query, in every mode.  Sort rules are
     * implemented for placeholder searches of mode 0 only (no positive or negative query term: the rule stack is the sort rules
     * alone, search/new/mod.rs:353-416), and a GeoSort rule only as the first rule of that stack.  B200_ERR_UNSUPPORTED for that
     * query, never an answer without its sort rules: a sort rule (from the list or from Asc/Desc criteria) in a search with query
     * terms or with negative terms only, in a semantic or hybrid search, more than B200_MAX_SCORES sort rules, `stop_after`
     * together with a sort rule, a GeoSort rule after the first rule. */
    const uint32_t *sort_begin;
    const uint16_t *sort_fid;
    const uint8_t *sort_asc;
    const uint8_t *sort_geo;
    const double *sort_geo_point;
    /* Search::geo_sort_strategy / geo_max_bucket_size (search/mod.rs:190-198, documents/geo_sort.rs:12-63): geo_strategy 0
     * Dynamic(geo_cache_size), 1 AlwaysIterative(geo_cache_size), 2 AlwaysRtree(geo_cache_size); geo_cache_size 0 = 1000;
     * geo_max_bucket_size 0 = 1000.  The distance error margin is the reference's 1.0 m. */
    int32_t geo_strategy;
    uint32_t geo_cache_size;
    uint64_t geo_max_bucket_size;
    /* Geo filters (IndexFilter::evaluate, search/facet/filter/index_filter.rs:345-360,465-696): the geo leaves at the top of a
     * query's filter, pushed down.  Query i has clauses [geo_filter_begin[i], geo_filter_begin[i+1]); geo_filter_begin NULL = no geo
     * filter anywhere.  geo_filter_kind: 0 `_geoRadius(lat, lng, radius)`, 1 `_geoBoundingBox([top, right], [bottom, left])`;
     * geo_filter_not (NULL = none): 1 = `NOT clause`; geo_filter_args: four doubles per clause, (lat, lng, radius in metres, unused)
     * or (top, right, bottom, left).  The query's filtered universe is documents_ids AND universes[i] AND every clause, a NOT clause
     * counting as documents_ids minus the clause.  _geoRadius is the prefix of the rtree order (squared chord distance, ties by
     * docid) that take_while keeps (haversine <= radius + f64::EPSILON); _geoBoundingBox is the inclusive latitude and longitude
     * ranges over the staged points, the longitude one wrapping the antimeridian when right < left.  Per query, with the reference's
     * message: a non-finite argument, a latitude outside [-90, 90], a longitude outside [-180, 180], or top < bottom is
     * B200_ERR_INVALID, and so is a geo clause when b200_stage_geo_fields was not called (`_geo` not filterable: the message is
     * `Attribute `_geo/_geojson` is not filterable.`, to which the caller appends the index's filterable patterns as
     * FilterError::AttributeNotFilterable does).  Every mode takes
     * the filtered universe exactly as if it had been passed through `universes`.  Queries with the same universe pointer and the
     * same clause list share one device bitmap; B200_ERR_CAPACITY for the call when the batch's bitmaps do not fit.  GeoJSON
     * (`_geojson`, `_geoPolygon`, the `resolution` argument) is not implemented. */
    const uint32_t *geo_filter_begin;
    const uint8_t *geo_filter_kind;
    const uint8_t *geo_filter_not;
    const double *geo_filter_args;
    /* The `facets` search parameter (crates/meilisearch/src/search/mod.rs:1945-1952,2041-2124): FacetDistribution::execute and
     * compute_stats (search/facet/facet_distribution.rs:110-337, facet_distribution_iter.rs:26-232) over the query's
     * SearchResult::candidates, on the device.  Query i asks for slots [facet_begin[i], facet_begin[i+1]), slot k for the field
     * facet_fid[k] (its id in the facet databases; the caller resolves the names against the filterable rules, as
     * compute_facet_distribution_stats does, and a fid without facet values gives an empty distribution and no stats); facet_begin
     * NULL = no facets anywhere.  facet_order (NULL = all alpha): 0 OrderBy::Lexicographic, 1 OrderBy::Count (B200_ERR_UNSUPPORTED for
     * that query).  facet_max_values: maxValuesPerFacet (0 is legal and keeps the reference's meaning).  facet_cap: entries per slot
     * in the b200_results::facet_* outputs; a slot that needs more fails its query alone with B200_ERR_CAPACITY (max_values + the
     * field's number of string values always suffices when max_values > 0, the field's number of values when it is 0).
     * Per query: facets in mode 1 or 2 (use b200_facet_distribution_batch) or with a ranking-score threshold are B200_ERR_UNSUPPORTED;
     * a facet_begin without facet_fid or without the facet_* outputs is B200_ERR_INVALID. */
    const uint32_t *facet_begin;
    const uint16_t *facet_fid;
    const uint8_t *facet_order;
    uint32_t facet_max_values;
    uint32_t facet_cap;
    /* Facet search over each query's candidates (perform_facet_search, crates/meilisearch/src/search/mod.rs:2514-2574, with
     * execute_for_candidates, search/mod.rs:254-278), as b200_facet_search_batch answers it: query i searches field
     * facet_search_fid[i] (0xFFFF: no facet search for that query; facet_search_fid NULL: none anywhere) with facet_query_kind[i]
     * (0 None, 1 Some), the query bytes facet_query_bytes[facet_query_off[i] .. facet_query_off[i + 1]) and facet_search_flags[i]
     * (bit 0 order by count, bit 1 the field is not an exact attribute), keeping at most facet_search_max hits, which is also the
     * stride of the b200_results::fs_* outputs.  The candidates are, in mode 0, exactly the bitmap `candidates` holds
     * (SearchResult::candidates, degraded results included), copied on the device where the search hands it over, and in modes 1
     * and 2 the query's filtered universe (documents_ids AND universes[i] AND its geo clauses); they never cross PCIe.  Per query: a
     * facet search with a ranking-score threshold is B200_ERR_UNSUPPORTED; facet_search_fid without facet_query_kind,
     * facet_search_flags or the fs_* outputs (or without facet_query_off / facet_query_bytes when a kind is 1) is B200_ERR_INVALID;
     * the errors of b200_facet_search_batch apply to the query alone (its search results are then dropped as well). */
    const uint16_t *facet_search_fid;
    const uint8_t *facet_query_kind;
    const uint32_t *facet_query_off;
    const char *facet_query_bytes;
    const uint8_t *facet_search_flags;
    uint32_t facet_search_max;
    /* The `filter` search parameter (NULL = none): program i filters query i (filter->n == n_queries).  The query's filtered universe
     * is documents_ids AND universes[i] AND its geo_filter_* clauses AND its program; every mode and the facet outputs take it as
     * they take `universes`.  Queries with the same universe pointer, geo clauses and program bytes share one device bitmap.  Errors
     * (see b200_filter_programs) fail the query alone; b200_results::filter_error_leaf names the failing leaf. */
    const b200_filter_programs *filter;
} b200_query_batch;
#define B200_MAX_SCORES 12
/* score kinds: ScoreDetails variants (score_details.rs:9-32) */
enum b200_score_kind { B200_S_WORDS = 0, B200_S_TYPO = 1, B200_S_PROXIMITY = 2, B200_S_FID = 3, B200_S_POSITION = 4,
                       B200_S_EXACT_ATTRIBUTE = 5, B200_S_EXACT_WORDS = 6, B200_S_VECTOR = 7, B200_S_SKIPPED = 8, B200_S_SORT = 9,
                       B200_S_GEO_SORT = 10 };
/* B200_S_SORT (ScoreDetails::Sort, score_details.rs): score_max = fid << 2 | ascending << 1 | is_string; score_rank = position of
 * the bucket's value among the staged level-0 keys of its database (facet_id_f64_docids when is_string = 0, else
 * facet_id_string_docids), 0xFFFFFFFF for the Null bucket (no value).  Sort has no Rank: global scores ignore it.
 * B200_S_GEO_SORT (ScoreDetails::GeoSort): score_rank = docid of the bucket's first point (its `value` is that document's point),
 * 0xFFFFFFFF for the Null bucket (None); score_max = ascending << 1; the target point is the query's.  No Rank either. */
typedef struct {                  /* SearchResult (search/mod.rs:526-535), flattened; all caller-allocated */
    uint32_t *docids;             /* n_queries x limit      documents_ids */
    uint32_t *n_hits;             /* n_queries */
    uint8_t *n_scores;            /* n_queries x limit      len of document_scores[i] (Detailed only) */
    uint8_t *score_kind;          /* n_queries x limit x B200_MAX_SCORES */
    uint32_t *score_rank;         /* idem: Rank.rank  (score_details.rs:512-522) */
    uint32_t *score_max;          /* idem: Rank.max_rank */
    float *score_sim;             /* idem: Vector.similarity, -1 when None */
    uint64_t *n_candidates;       /* n_queries: candidates.len() */
    uint32_t *semantic_hits;      /* n_queries: execute_hybrid's semantic_hit_count (may be NULL) */
    int32_t *status;              /* n_queries: 0 or a B200_ERR_* for that query (e.g. UNSUPPORTED) */
    uint8_t *degraded;            /* n_queries: SearchResult::degraded (may be NULL) */
    uint8_t *used_negative_operator; /* n_queries: SearchResult::used_negative_operator (may be NULL) */
    uint64_t *candidates;         /* optional (may be NULL): n_queries x candidates_words dense u64 words, SearchResult::candidates
                                     for keyword searches without a ranking-score threshold (others: B200_ERR_UNSUPPORTED) */
    uint64_t candidates_words;    /* words per query in `candidates` (>= ceil((max docid + 1) / 64)) */
    /* Facets of slot k (b200_query_batch::facet_*), over exactly the bitmap `candidates` holds for the query.  The distribution
     * comes as facet_n_num[k] number entries then facet_n_str[k] string entries at [k * facet_cap, ..), each already in the
     * reference's order and cut to the reference's length (facet_values, facet_distribution.rs:258-294):
     *   |candidates| <= 3000 (from documents, :110-177): up to max_values numbers in the order of their f64 Display strings, then up
     *     to max_values - n_num strings in byte order of their normalised value;
     *   |candidates| > 3000 (facet levels, :181-253): numbers ascending, up to max_values of them (all when max_values is 0), then
     *     strings in byte order, up to max_values of them when n_num < max_values, all of them otherwise.
     * The caller builds the IndexMap<String, u64>: insert the numbers (key: the value's f64 Display string), then the strings one by one
     * (key: the original string of (fid, facet_docid, normalised value) in field_id_docid_facet_strings), stopping right after an
     * insert that leaves the map's length at max_values.  That reproduces both paths including a string whose original equals a
     * number's Display string (it overwrites that entry in place).
     * facet_key: the value's position among the staged level-0 keys of its database (facet_id_f64_docids for the first n_num
     * entries, facet_id_string_docids after them), as B200_S_SORT's score_rank; facet_count: |candidates AND docids(value)|;
     * facet_docid: the smallest candidate holding the value (any_docid).  facet_has_stats / facet_min / facet_max: compute_stats
     * (:298-337, facet/mod.rs:39-59), the smallest and largest number value of the field over the candidates (has_stats 0: none). */
    uint32_t *facet_n_num;
    uint32_t *facet_n_str;
    uint32_t *facet_key;
    uint64_t *facet_count;
    uint32_t *facet_docid;
    uint8_t *facet_has_stats;
    double *facet_min;
    double *facet_max;
    /* Facet search of query i (b200_query_batch::facet_search_*): fs_n[i] hits at [i * facet_search_max, ..), each as in
     * b200_facet_search_batch (key, count, docid, fallback). */
    uint32_t *fs_n;
    uint32_t *fs_key;
    uint64_t *fs_count;
    uint32_t *fs_docid;
    uint8_t *fs_fallback;
    /* n_queries (may be NULL): the node index, relative to the query's first node, of the filter node whose error failed the query
     * (a reached failing leaf, an unsupported node, a leaf without its staged database), -1 when no node's error did */
    int32_t *filter_error_leaf;
} b200_results;
int b200_search_batch(b200_index *, const b200_query_batch *, b200_results *);

/* Replaces the geo leaves of IndexFilter::evaluate (index_filter.rs:465-696) inside filter trees the caller combines itself (OR,
 * nested NOT): clause i (kind[i], args[4 i .. 4 i + 4), as in b200_query_batch::geo_filter_*) becomes the dense bitmap
 * out[i * out_words ..] (out_words >= ceil((max docid + 1) / 64); words past the document range are zero).  status[i]: 0 or
 * B200_ERR_INVALID with the reference's message (its bitmap is then empty).  The same kernels as the search batch. */
int b200_geo_filter_batch(b200_index *, uint32_t n, const uint8_t *kind, const double *args, uint64_t *out, uint64_t out_words, int32_t *status);

/* Replaces IndexFilter::evaluate after its not-filterable check (index_filter.rs:43-73) for callers that filter outside a search
 * (facet distribution with a filter, document fetch or delete by filter): program i (b200_query_batch::filter semantics) becomes the
 * dense bitmap out[i * out_words ..] (out_words >= ceil((max docid + 1) / 64); words past the document range are zero).  status[i]:
 * 0 or the program's error (its bitmap is then empty); error_leaf[i] (may be NULL) as b200_results::filter_error_leaf.  The same
 * kernels as the search batch. */
int b200_filter_batch(b200_index *, const b200_filter_programs *programs, uint64_t *out, uint64_t out_words, int32_t *status, int32_t *error_leaf);

/* Replaces FacetDistribution::execute and compute_stats (search/facet/facet_distribution.rs:110-337) for callers that hold the
 * candidates themselves (semantic and hybrid searches, the S1 seam, federated search): candidate set i is the host bitmap
 * candidates[i] (dense little-endian u64 words, n_words >= ceil((max docid + 1) / 64); only docids below max docid + 1 are read;
 * equal pointers are uploaded once) and asks for slots [facet_begin[i], facet_begin[i+1]) of facet_fid / facet_order, as in
 * b200_query_batch.  The outputs are b200_results::facet_* with stride `cap`; status[i]: 0, B200_ERR_UNSUPPORTED (count order) or
 * B200_ERR_CAPACITY (a slot needs more than `cap` entries), for that set alone.  The same kernels as the search batch. */
int b200_facet_distribution_batch(b200_index *, uint32_t n, const uint64_t *const *candidates, uint64_t n_words, const uint32_t *facet_begin,
                                  const uint16_t *facet_fid, const uint8_t *facet_order, uint32_t max_values, uint32_t cap, uint32_t *n_num,
                                  uint32_t *n_str, uint32_t *key, uint64_t *count, uint32_t *docid, uint8_t *has_stats, double *min,
                                  double *max, int32_t *status);

/* Replaces SearchForFacetValues::execute after its facet-searchable check and field resolution (search/facet/search.rs:74-265), as
 * called by perform_facet_search (crates/meilisearch/src/search/mod.rs:2514-2574) with the candidates of execute_for_candidates
 * (search/mod.rs:254-278), for callers that hold the candidates themselves.  Request i searches field fid[i] (its id in the facet
 * databases; 0xFFFF or a field without facet_id_normalized_string_strings entries: no FST, an empty answer) over the host bitmap
 * candidates[i] (dense little-endian u64 words, n_words >= ceil((max docid + 1) / 64), NULL entry = documents_ids; equal pointers
 * are uploaded once).
 *   kind[i] 0 (query None): every level-0 key of facet_id_string_docids for the field, in key order (:224-240).
 *   kind[i] 1 (Some(q)): q = query_bytes[off[i] .. off[i + 1]) (off has n + 1 entries), already normalize_facet_string'd by the
 *     caller.  With typos allowed (flags bit 1 set, meaning the field is not an exact attribute, and the staged authorize_typos):
 *     when q is in the staged exact_words, the one string q if the FST holds it; otherwise the FST strings accepted by
 *     build_dfa(q, k, prefix = true) (search/mod.rs:565-577): the minimum restricted Damerau-Levenshtein (OSA) distance between q and a
 *     prefix of the string, over Unicode scalar values, is at most k = 0 / 1 / 2 as q's byte length is below min_word_len_one_typo
 *     / below min_word_len_two_typos / neither, with no first-letter rule.  Without typos: the FST strings that start with q.
 *     Matches are walked in byte order; each one's level-0 keys in its JSON set order, stopping at a key that facet_id_string_docids
 *     lacks (:242-289).  q longer than B200_FACET_QUERY_MAX Unicode scalar values is B200_ERR_UNSUPPORTED for that request.
 * Every walked key whose docids meet the candidates is a hit: count = |docids AND candidates|.  flags bit 0 clear: the first `max`
 * hits (OrderBy::Lexicographic); set: OrderBy::Count, the BinaryHeap<Reverse<FacetValueHit>> replay of ValuesCollection::insert
 * (:292-353) ordered by (count, value bytes), output in descending order.  A hit's value is the original string at (fid, docid,
 * key) in field_id_docid_facet_strings, where docid is the smallest of all the key's docids, or, without that entry, q (kind 1) or
 * the key (kind 0).
 * Outputs, stride `cap` per request: n_out[i] hits; key[i * cap + j] the hit's position among the staged level-0 keys of
 * facet_id_string_docids (as B200_S_SORT's score_rank), count, docid (the smallest docid of the key) and fallback (1: no original,
 * the value is q or the key).  status[i]: 0; B200_ERR_UNSUPPORTED (query too long); B200_ERR_INVALID (kind > 1, or off not
 * ascending); B200_ERR_CAPACITY (min(max, hits) > cap), for that request alone, with n_out[i] = 0.  max = 0 answers nothing. */
#define B200_FACET_QUERY_MAX 64
int b200_facet_search_batch(b200_index *, uint32_t n, const uint64_t *const *candidates, uint64_t n_words, const uint16_t *fid,
                            const uint8_t *kind, const uint32_t *off, const char *query_bytes, const uint8_t *flags, uint32_t max,
                            uint32_t cap, uint32_t *n_out, uint32_t *key, uint64_t *count, uint32_t *docid, uint8_t *fallback,
                            int32_t *status);

/* Replaces Similar::execute (crates/milli/src/search/similar.rs:66-152), as called by perform_similar
 * (crates/meilisearch/src/search/mod.rs:2577-2735), with VectorStore::nns_by_item (vector/store.rs:615-637,980-1034) answered by an
 * exact scan of the staged store.  For query i, target `id` = docids[i] and U = documents_ids AND universes[i] AND program i of
 * `filter` (b200_query_batch semantics for both; filter->n == n_queries):
 *   1. the universe is U \ {id};
 *   2. the query is the target's staged row; the candidate list is the nearest offset + limit + 1 rows of U \ {id}, ascending by
 *      (distance, docid), distance (1 - cos) / 2 with the norm rule of b200_nns_batch;
 *   3. the list is walked in order: `seen` starts as {id}, a docid already in it is dropped, otherwise added (before the skip and the
 *      take); the first `offset` survivors are skipped (still added to `seen`); at most `limit` are taken, each with score
 *      1 - distance, shifted by the staged distribution if there is one.  With a threshold, a taken document whose score is below it
 *      ends the walk and sets candidates = (candidates \ {doc}) AND seen; skipped documents are never tested;
 *   4. outputs: the hits in b200_results::docids (stride `limit`) and n_hits, one B200_S_VECTOR score per hit (n_scores = 1,
 *      score_sim = the score, which is also the global score), n_candidates = |candidates|, candidates starting as U \ {id} (the
 *      route's estimatedTotalHits).  Unembedded documents are never returned (unlike VectorSort's last bucket in searches);
 *   5. a target without an embedding, outside documents_ids or beyond the document range has no hits, n_candidates = |U \ {id}| and
 *      status 0, as nns_by_item answers for an absent item.
 * The reference scans once per store, store k holding each document's k-th vector and searched with the target's k-th vector; the
 * staged store is flat, so on a store where a document has more than one row every query fails alone with B200_ERR_UNSUPPORTED.
 * Per query, as in searches: filter errors (filter_error_leaf names the node).  For the call: B200_ERR_INVALID for NULL docids or
 * universes shorter than the document range, B200_ERR_STATE before b200_stage_finish or without staged embeddings,
 * B200_ERR_UNSUPPORTED for a non-NULL b200_results::candidates (the route reads only its length).  The target's vector never crosses
 * PCIe: the scan gathers it from HBM. */
typedef struct {
    uint32_t n_queries;
    const uint32_t *docids;          /* n_queries internal docids of the target documents */
    uint32_t offset, limit;
    const uint64_t *const *universes; /* as b200_query_batch::universes (NULL array / entry: documents_ids) */
    uint64_t n_universe_words;
    const b200_filter_programs *filter; /* as b200_query_batch::filter (NULL = none) */
    int32_t has_ranking_score_threshold;
    double ranking_score_threshold;
} b200_similar_request;
int b200_similar_batch(b200_index *, const b200_similar_request *, b200_results *);

/* ---- S1: the RankingRule seam ---------------------------------------------------------- */
/* Replaces `dyn RankingRule` as driven by bucket_sort (crates/milli/src/search/new/ranking_rules.rs:26-83, bucket_sort.rs:123,266,323)
 * for the graph-based rules and ExactAttribute.  Query graphs are opaque library objects (a QueryGraph plus the terms it refers
 * to): the first one comes from b200_graph_from_tokens (QueryGraph::from_query, query_graph.rs:96-187, with every term's
 * derivations computed), the next ones from b200_rule_next (RankingRuleOutput::query: the graph rebuilt from the paths that
 * produced the bucket, graph_based_ranking_rule.rs:340-353).  Every graph handed out must be released with b200_graph_free. */
typedef struct b200_graph b200_graph;
typedef struct b200_rule b200_rule;
/* one_query: a b200_query_batch with n_queries == 1 (tokens, words_limit, terms_matching_strategy) */
int b200_graph_from_tokens(b200_index *, const b200_query_batch *one_query, b200_graph **out);
void b200_graph_free(b200_graph *);
/* RankingRule::start_iteration(universe, query).  rule_kind: B200_S_WORDS, _TYPO, _PROXIMITY, _FID, _POSITION, _EXACT_ATTRIBUTE,
 * _EXACT_WORDS (= Exactness); terms_matching_strategy matters for B200_S_WORDS only.  universe: dense u64 words, NULL = all
 * documents.  All buckets of the rule are evaluated here, in one device step. */
int b200_rule_start(b200_index *, int rule_kind, int terms_matching_strategy, const b200_graph *query, const uint64_t *universe,
                    uint64_t n_universe_words, b200_rule **out);
/* RankingRule::next_bucket(universe): returns 0 and the next bucket in ascending cost order (empty ones included, like the
 * reference, graph_based_ranking_rule.rs:231-236), or 1 when the rule is exhausted (None).  out_bitmap (n_words words) =
 * RankingRuleOutput::candidates = bucket AND universe (NULL = the start universe); rank / max_rank = the bucket's score
 * (score_details.rs Rank); out_query = RankingRuleOutput::query (NULL for an empty bucket; caller frees). */
int b200_rule_next(b200_rule *, const uint64_t *universe, uint64_t *out_bitmap, uint64_t n_words, uint32_t *rank, uint32_t *max_rank,
                   b200_graph **out_query);
/* RankingRule::end_iteration */
void b200_rule_end(b200_rule *);

/* ---- introspection for measurement ----------------------------------------------------- */
/* kernel classes for the per-kernel accounting below */
enum b200_kernel { B200_K_LEV = 0, B200_K_COMPACT = 1, B200_K_PAIR_PROBE = 2, B200_K_SCATTER = 3, B200_K_EVAL_PATHS = 4, B200_K_EMIT = 5,
                   B200_K_VEC_DIST = 6, B200_K_TOPK = 7, B200_K_VEC_GEMM = 8, B200_K_VEC_MERGE = 9, B200_K_SORT = 10, B200_K_GEO = 11,
                   B200_K_GEO_FILTER = 12, B200_K_FACET = 13, B200_K_FACET_SEARCH = 14, B200_K_FILTER = 15, B200_K_COUNT = 16 };
typedef struct {
    uint64_t kernel_launches;     /* kernels launched by the library since the last reset */
    uint64_t device_steps;        /* host<->device round trips since the last reset */
    uint64_t posting_bytes;       /* algorithmic bytes: stored bytes of posting lists read (SURVEY §8(d)) */
    uint64_t matrix_bytes;        /* algorithmic bytes: condition/bucket matrix words read+written */
    uint64_t dictionary_bytes;    /* algorithmic bytes of the term-derivation sweeps */
    uint64_t vector_bytes;        /* algorithmic bytes of the distance scans */
    double kernel_ms[B200_K_COUNT];      /* CUDA-event time accumulated per kernel class (events on the library's stream) */
    uint64_t kernel_count[B200_K_COUNT]; /* launches per kernel class */
    uint64_t kernel_bytes[B200_K_COUNT]; /* algorithmic bytes attributed to each kernel class */
    double device_ms;             /* CUDA-event time from the first to the last kernel of every step */
    uint64_t h2d_bytes, d2h_bytes; /* bytes copied across PCIe/NVLink-C2C by search/derive/nns calls */
    double host_ms[8];            /* wall time of the host phases of b200_search_batch: 0 parse, 1 derive (incl. device), 2 term finalisation,
                                     3 step packing, 4 step device wait, 5 bucket-sort advance, 6 result copy, 7 total */
    uint64_t hbm_bytes_staged;
    uint64_t deferred;            /* ranking-rule activations that had to wait for a later device step (scratch / arena full) */
    uint64_t arena_peak_bytes;    /* high-water mark of the per-batch level storage (universes + bucket columns) */
    uint64_t eval_class_launches[9]; /* eval_dp launches per DP-table class: <= 16 / 24 / 40 / 56 / 80 / 112 / 160 / 216 slots in shared memory, [8] = global matrices */
    uint64_t eval_class_tiles[9];    /* 128-row tiles evaluated per class */
    uint64_t lev_terms;           /* term derivation: distinct terms derived */
    uint64_t lev_items;           /* term derivation: lev_match work items (one CTA each) */
    uint64_t lev_pairs;           /* term derivation: (term, dictionary word) pairs the work items cover */
} b200_stats;
int b200_get_stats(b200_index *, b200_stats *out);
int b200_reset_stats(b200_index *);

#ifdef __cplusplus
}
#endif
#endif
