// POD structures shared by the host engine and the CUDA kernels.
#pragma once
#include <cstdint>

namespace b200 {

struct DListRef {  // mirrors host ListRef
    unsigned long long off;
    uint32_t card;
    uint32_t dense;
};

// ---- term derivation (lev kernel) ----
constexpr int LEV_MAX_Q = 64;        // longest query word handled on device (bytes)
constexpr int LEV_TERMS_PER_CTA = 32;
constexpr int LEV_REC_CAP = 2048;    // match records (32 words each) per term
// Record slots per term.  A term's work items scan at most LEV_MAX_RANGES disjoint word ranges (first bytes q[0] and q[1], the
// 2-byte prefixes (c, q[1]) and (c, q[0]) for c outside {q[0], q[1]}); two ranges can share one 32-word group, so the records of a
// term exceed its distinct groups by fewer than LEV_MAX_RANGES and finalize, which merges them, still sees every group up to the cap.
constexpr int LEV_MAX_RANGES = 2 + 2 * 254;
constexpr int LEV_REC_SLOTS = LEV_REC_CAP + LEV_MAX_RANGES;
struct LevTerm {
    uint8_t q[LEV_MAX_Q];
    uint8_t len;
    int8_t k_same;    // budget when first chars are equal
    int8_t k_diff;    // budget when they differ (-1: excluded)
    uint8_t prefix;   // prefix automaton
};
struct LevRec {
    uint32_t base;              // first word id of the 32-word group
    uint32_t pad;
    unsigned long long codes;   // 2 bits per lane: 0 none, 1 same-first d=1, 2 same-first d=2, 3 different-first (d=1)
};
// Which (term, word) pairs a term's slot in a work item owns.  Every pair the filter of lev_match_kernel can accept is owned by
// exactly one family, and each family only scans dictionary ranges where it can own pairs (DESIGN.md §3 "Term derivation").
enum LevFamily : uint32_t {
    LEV_F1 = 0,   // first-byte range q[0], every typo-tolerant term:              w[0] == q[0]
    LEV_F2A = 1,  // first-byte range q[1], 2-typo terms:                          w[0] == q[1] != q[0]
    LEV_F2B = 2,  // 2-byte ranges (c, q[1]), 2-typo terms:                        w[1] == q[1], w[0] not in {q[0], q[1]}
    LEV_F3 = 3,   // 2-byte ranges (c, q[0]), 2-typo terms with q[0] != q[1]:      w[1] == q[0], w[0] not in {q[0], q[1]}
    LEV_F0 = 4,   // whole dictionary, 2-typo terms with m < 2 or a zero q[0]/q[1]: w[0] != q[0]
};
constexpr int LEV_FAMILY_SHIFT = 29;  // term permutation entry: term index | family << LEV_FAMILY_SHIFT
// A work item: the words [lo, lo + n) of one 256-aligned dictionary tile against the term slots perm[t_off, t_off + t_cnt)
struct LevItem {
    uint32_t lo;
    uint32_t t_off;
    uint16_t n;      // <= 256
    uint16_t t_cnt;  // <= LEV_TERMS_PER_CTA
};

// ---- rule activations ----
constexpr uint32_t MAX_COSTS = 128;
constexpr uint32_t JOB_CHUNK = 2048;  // elements (sparse) or rows (dense) per scatter job

// An activation evaluates a small DAG ("state graph") over the activation's universe, 64 documents per thread:
//   S[state][r] = documents that can go from `state` to END spending exactly r        (backward min-plus DP, bit-sliced)
//   bucket[ci]  = S[ROOT][cost_vals[ci]] minus the cheaper buckets                    (= the rule's buckets, all at once)
//   walk        = per document the first START->END path in edge order among its cheapest ones; distinct paths are
//                 reported to the host, which rebuilds the next query graph from them (graph_based_ranking_rule.rs:340-353)
struct DpState {
    uint32_t edge_begin;  // into DpEdge[], edges in visiting (DFS) order
    uint32_t pair_off;    // first S column of this state
    uint16_t n_edges;
    uint16_t rmin, rcount;  // S columns cover costs [rmin, rmin + rcount)
    uint16_t pad;
};
struct DpEdge {
    uint16_t dst;   // state index (always greater than the source: states are in topological order)
    uint16_t cost;
    uint16_t col;   // condition column, 0xffff = unconditional
    uint16_t pad;
};
constexpr uint32_t MAX_WALK = 14;  // edges on a START->END path (10 words + END, with slack)
struct PathOut {     // one distinct first-match path
    uint32_t act;
    uint16_t cost_idx;
    uint16_t len;
    uint16_t edges[MAX_WALK];  // activation-local DpEdge indices
};

struct ActDesc {
    // parent universe: rows (p_uw,p_ub); child = rows where OR(p_out[col_lo..col_hi)) != 0. p_out==0: take p_ub as is.
    const uint32_t *p_uw;            // nullptr => identity (row j is word j)
    const unsigned long long *p_ub;
    const unsigned long long *p_out; // column-major, leading dimension p_ld
    uint32_t p_rows, p_ld, p_col_lo, p_col_hi;
    // this activation
    uint32_t *uw;
    unsigned long long *ub;
    unsigned long long *C;    // column-major [n_cols][ld], scratch for this step
    unsigned long long *S;    // column-major [n_pairs][ld], scratch
    unsigned long long *out;  // column-major [n_costs+1][ld]; last column = matched by no path
    unsigned long long *tab;  // path dedup table (tab_size slots, zeroed), scratch
    uint32_t ld, n_cols, n_costs, n_states;
    uint32_t state_off, edge_off, cost_off;  // into DpState[], DpEdge[], u16 cost_vals[]
    uint32_t colprog_off, colprog_len;
    uint32_t prog_off, prog_len;  // DP program, u32 ops in the step's program pool; prog_len is a multiple of 4
    uint32_t n_pairs;             // (state, cost) pairs of the DP table; START's pairs come first, END's single pair last
    uint32_t root_rmin, root_rcount;  // START's cost range
    uint32_t need;                // documents bucket_sort can still use from this activation (hits left + offset left), saturating
    uint32_t tab_size, want_paths;
    uint32_t res_off;         // into results u32[]: [0] rows, [1..n_costs+1] counts, then: path-table saturation flag, last walked bucket
    uint32_t all_conditional; // every START->END path has at least one condition: rows whose columns are all zero match nothing
    // per-query lookup table word index -> (tag << 20 | row), written by act_compact, read by scatter instead of a binary search in
    // uw; nullptr = not available (then uw is searched).  Entries of other activations carry other tags.
    uint32_t *row_tab;
    uint32_t row_tag, pad_;
};

struct ColOp {  // executed per row before the paths
    uint16_t op;  // 0 AND dst=a&b, 1 OR dst=a|b, 2 ANDNOT dst=a&~b, 3 COPY dst=a
    uint16_t dst, a, b;
};

struct Job {  // scatter one chunk of one posting list into column `col` of activation `act`
    uint32_t act, col, list, chunk;
};

struct PairSet {  // expanded on device into Jobs: all (l, r) pairs of two word sets
    uint32_t act, col;
    uint32_t left_off, n_left, right_off, n_right;  // into the step's u32 word pool
    uint8_t fwd_prox, bwd_prox;  // 0 = no lookup in that direction
    uint8_t right_is_range;      // right entries are [lo,hi) dictionary ranges (prefix db): n_right pairs of u32
    uint8_t pad;
    uint32_t probe_base;         // first global probe index of this set
};

struct EmitDesc {  // append the first docids of OR(out[col_lo..col_hi)) to a result buffer
    const uint32_t *uw;
    const unsigned long long *ub;
    const unsigned long long *out;  // nullptr: emit ub itself
    uint32_t rows, ld, col_lo, col_hi;
    uint32_t skip, take;
    uint32_t *dst;
};

struct TileDesc {
    uint32_t act, row_begin;
    uint32_t rows_per_thread, pad;  // the tile covers 128 * rows_per_thread rows
};
// eval_dp_kernel keeps a row's condition words and DP table in thread-private shared-memory slots ([slot][128 rows] u64 = 1 KB per
// slot and CTA); a step's tiles are binned by the slot count (n_cols + n_pairs) of their activation, one launch per class; wider
// activations use the global-memory variant.
constexpr uint32_t EVAL_CLASSES = 8;
constexpr uint32_t EVAL_CLASS_SLOTS[EVAL_CLASSES] = {16, 24, 40, 56, 80, 112, 160, 216};
inline uint32_t eval_class(uint32_t slots) {
    for (uint32_t c = 0; c < EVAL_CLASSES; c++)
        if (slots <= EVAL_CLASS_SLOTS[c]) return c;
    return EVAL_CLASSES;
}
// DP program ops (built by the host, emit_activation_work): src slot | last-of-pair << 15 | condition slot << 16.  Slots of a row:
// [0, n_cols) condition columns, [n_cols, n_cols + n_pairs) DP table, then the constants ZERO and ONES.
constexpr uint32_t EVAL_EXTRA_SLOTS = 2;

// one segment of COMPACT_SEG parent rows of an activation's compaction (act_count_kernel / act_compact_kernel)
constexpr uint32_t COMPACT_SEG = 8192;
struct CompactTile {
    uint32_t act, seg;
    uint32_t first_tile;  // index of the activation's segment 0 in the tile list (segment counts are stored per tile)
    uint32_t n_seg;
};

// one window of a sort activation (sort.cu): the documents of ranks [lo, hi) of the universe ordered by (key_0, ..., key_{L-1}, docid)
constexpr uint32_t SORT_MAX_LEVELS = 12;  // B200_MAX_SCORES
constexpr uint32_t SORT_WINDOW = 2048;    // rows one CTA produces
struct SortDesc {
    const unsigned long long *ub;          // dense universe bitmap, n_words words
    const unsigned long long *exclude;     // nullptr, or documents left out of ub (n_words words)
    const uint32_t *ids;                   // non-null: the universe is this docid list instead of ub
    uint32_t n_ids;
    const uint32_t *keys[SORT_MAX_LEVELS]; // per level: u32[n_docs] sort keys, nullptr = every key 0 (a field without values)
    uint32_t bits[SORT_MAX_LEVELS + 1];    // significant bits of each tuple word ([n_levels]: the docid)
    uint32_t n_words, n_levels;
    uint32_t lo, hi;                       // hi - lo <= SORT_WINDOW, hi <= |universe|
    uint32_t *dst;                         // hi - lo docids
    uint32_t *dst_keys;                    // (hi - lo) x n_levels keys
    uint32_t *info;                        // out: universe passes, documents collected for the window
};

// one document of the GeoSort rule (geo.cu): lat_lng_to_xyz of its point (lib.rs:397-404, what the rtree holds), its point in
// degrees and cos(lat) (the haversine's per-point factor), all computed on the host with the platform libm at staging
struct GeoPoint {
    double x, y, z, lat, lng, cos_lat;
};
// one window of the order of a GeoSort rule over (universe AND geo documents) (geo.cu), tuple (part, key_hi, key_lo, rdoc, docid):
//   rtree order:     part 0, key = bits of the f64 squared chord distance to `q`, rdoc 0;
//   iterative order: part 1 (0 when the whole order is iterative), key = floor(haversine metres) (ascending) or GEO_FLOOR_MAX minus
//                    it (descending), rdoc = 0 (ascending) or GEO_DOC_MAX minus the docid (descending);
//   mode 0: every document in rtree order; 1: every document in iterative order; 2: rtree order for the documents whose rtree tuple
//   (key, docid) is at most `split`, iterative order after them (the Dynamic strategy's tail).
constexpr uint32_t GEO_FLOOR_BITS = 25;  // floor(haversine) <= pi * 6371000 < 2^25
constexpr uint32_t GEO_FLOOR_MAX = (1u << GEO_FLOOR_BITS) - 1;
struct GeoDesc {
    const unsigned long long *ub;   // universe, n_words words
    const unsigned long long *geo;  // geo documents, n_words words
    const GeoPoint *pts;            // per docid
    double q[3];                    // rtree target: lat_lng_to_xyz(target), or of opposite_of(target) when descending
    double t_lat, t_lng, t_cos_lat; // haversine target
    unsigned long long split_key;   // mode 2
    uint32_t split_doc;
    uint32_t mode, asc, doc_max;
    uint32_t n_words;
    uint32_t bits[5];
    uint32_t lo, hi;                // hi - lo <= SORT_WINDOW
    uint32_t *dst;                  // hi - lo docids
    unsigned long long *dst_key;    // their rtree key
    uint32_t *info;                 // out: passes, documents collected
    // iterative keys decided on the host (geo_math.cuh, geo_ambiguous): (docid << 32 | floor metres), ascending
    const unsigned long long *patch;
    uint32_t n_patch;
    // geo_ambiguous_kernel: the documents of universe AND geo whose floor is ambiguous, the first amb_cap of them into amb, their
    // number into *amb_count
    uint32_t amb_cap;
    uint32_t *amb, *amb_count;
};
// geo_count_kernel: |universe AND geo| per query
struct GeoCount {
    const unsigned long long *ub, *geo;
    uint32_t n_words;
    uint32_t *out;
};

// ---- geo filters (geo_filter.cu): _geoRadius / _geoBoundingBox clauses over the staged points
constexpr uint32_t GEO_FILTER_TILE_WORDS = 16;  // 64-document words one CTA stages in shared memory
constexpr uint32_t GEO_FILTER_SLOT_CHUNK = 1024; // slots whose counts one CTA accumulates in shared memory at a time
struct GeoClause {
    uint32_t kind;        // 0 _geoRadius, 1 _geoBoundingBox
    uint32_t neg;         // NOT clause
    // radius: the rtree target lat_lng_to_xyz(base), the haversine target, radius + f64::EPSILON, and squared-chord bounds: a point
    // with d2 < lo is within the radius, one with d2 > hi beyond it, the haversine decides in between (geo_filter.cu)
    double q[3];
    double t_lat, t_lng, t_cos_lat;
    double r_eps, lo, hi;
    double top, right, bottom, left;  // bounding box, degrees
};
// the first point of the rtree order whose haversine exceeds the radius: (squared distance bits, docid); all ones = none
struct __align__(16) GeoFirst {
    unsigned long long key, doc;
};
// a band point whose haversine is ambiguous against its clause's radius (geo_math.cuh), left to the host: clause, docid, rtree key
struct GeoAmb {
    uint32_t clause, doc;
    unsigned long long key;
};
// one filtered universe: ub AND the clauses slot_clauses[c_begin, c_end) (NOT clauses complemented), written to dst, its popcount
// added to *count
struct GeoSlot {
    const unsigned long long *ub;
    unsigned long long *dst;
    unsigned long long *count;
    uint32_t c_begin, c_end;
};

// ---- filter programs (filter.cu): the tree of a filter as a straight-line program over one-bit registers per document
constexpr uint16_t FILTER_NO_REG = 0xffff;  // hint register of a node evaluated without a universe hint
constexpr uint32_t FILTER_REG_WORDS = 63;   // 2016 registers: a program of depth B200_MAX_FILTER_DEPTH needs depth + 1
enum : uint16_t {
    FOP_ZERO = 0,    // dst = 0
    FOP_VALUE = 1,   // dst = the document has an ordinal in intervals [a, b) of iv (doc_off / doc_ord: the field's CSR; nullptr: none);
                     // neg: docs AND NOT that; hint != FILTER_NO_REG: AND hint
    FOP_BITMAP = 2,  // dst = bit of bm (nullptr: 0); hint != FILTER_NO_REG: AND hint
    FOP_AND = 3,     // dst &= src
    FOP_OR = 4,      // dst |= src
    FOP_NOT = 5,     // dst = (hint, or docs when FILTER_NO_REG) AND NOT dst
    FOP_FLAG = 6,    // flag a of the slot = 1 when dst is set for any document
};
struct FilterOp {
    uint16_t code, dst, src, hint;
    uint32_t a, b;
    uint32_t neg, pad;
    const uint32_t *doc_off, *doc_ord;
    const unsigned long long *bm;
};
// one filtered universe: ub AND the program ops[op_begin, op_end) (result in register 0), written to dst, its popcount added to
// *count; the program's flags live at flags[0 ..); all: every document is evaluated (the flags need the whole document range)
struct FilterSlot {
    const unsigned long long *ub;
    unsigned long long *dst;
    unsigned long long *count;
    uint32_t *flags;
    uint32_t op_begin, op_end;
    uint32_t all, pad;
};

// ---- facet distribution (facet.cu): one slot = one (candidate bitmap, faceted field)
constexpr uint32_t FACET_CANDIDATES_THRESHOLD = 3000;  // facet_distribution.rs:32 CANDIDATES_THRESHOLD
constexpr uint32_t FACET_SHARED_VALUES = 2048;         // fields with at most this many values count in shared memory
constexpr uint32_t FACET_ALL = 0xffffffffu;            // "no limit" for the number of entries taken
// per slot in scratch, zero at launch: |candidates|; the smallest number ordinal met as ~ordinal (atomicMax; 0 = none); the largest
// plus one (0 = none)
struct FacetHead {
    unsigned long long n_cand;
    uint32_t min_inv, max_p1;
};
struct FacetSlot {
    const unsigned long long *cand;  // candidates: n_words words
    const uint32_t *doc_off;         // the field's document-major ordinals (SortField), nullptr for a field without values
    const uint32_t *doc_ord;
    const uint32_t *disp;            // number ordinals in f64 Display-string order
    uint32_t n_num, n_str;
    uint32_t *cnt, *first;           // scratch, zero at launch: per ordinal |candidates AND docids| and ~(smallest such docid)
    FacetHead *head;
    uint32_t max_values, cap;
    uint32_t *out_ord, *out_doc;     // cap entries: numbers first, then strings
    unsigned long long *out_cnt;
    uint32_t *out_sum;               // 4 u32: numbers taken, strings taken, FacetHead::min_inv, FacetHead::max_p1
};

// ---- facet search (facet_search.cu): one request = one (candidate bitmap, field, query)
constexpr uint32_t FS_MAX_Q = 64;  // B200_FACET_QUERY_MAX: query length in Unicode scalar values
enum : uint8_t { FS_ALL = 0, FS_PREFIX = 1, FS_EXACT = 2 };
struct FsTables {  // the staged tables (host_index.h FacetSearchIndex)
    const uint32_t *chars, *char_off, *csr_off, *csr_key;
    const uint32_t *pool;
    const DListRef *lists;
};
struct FsReq {
    const unsigned long long *cand;  // candidates: n_words64 words
    uint32_t q_off, q_len;           // the query's chars in the batch's query table
    uint32_t h0, h1;                 // FS_PREFIX / FS_EXACT: the field's hyper-normalised strings
    uint32_t k0, n_str;              // FS_ALL: the field's level-0 string keys
    uint32_t max;                    // maxValuesPerFacet (> 0)
    uint32_t list_base;              // the posting list of level-0 key k is list_base + k (mod 2^32)
    uint8_t mode, by_count;
    int8_t k;                        // FS_PREFIX: the OSA budget (0: plain prefix)
    uint8_t pad;
    uint32_t *items, *cnt;           // scratch: the walked keys in insertion order and their counts
    uint32_t *sum;                   // 4 u32: keys walked, hits kept, cut count, offset of the kept hits in the packed outputs
};

}  // namespace b200

