// Host-side view of the staged index: key directories (which lists exist, how long they are) and
// the layout of the HBM posting store.  List *contents* live only on the device after staging.
//
// HBM layout (DESIGN.md §2):
//   pool      u32[]   every posting list back to back; a list is either `card` ascending docids (sparse)
//                     or, when card > n_docs/32, a dense bitmap of n_words64 little-endian u64 words
//   lists     ListRef[]  (offset into pool, cardinality, dense flag) indexed by list id
//   pair_keys u64[]   sorted packed keys prox<<42 | w1<<21 | w2 of word_pair_proximity_docids; the i-th key's
//                     list id is pair_list_base + i (so a prefix range of w2 is a contiguous run of lists)
//   dict      bytes + u32 offsets of the sorted dictionary (word id = rank)
//   base_ub   u64[]   documents_ids as a dense bitmap (the initial universe)
#pragma once
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

namespace b200 {

struct ListRef {
    uint64_t off;    // u32 index into the pool (even when dense)
    uint32_t card;   // number of docids
    uint32_t dense;  // 1: bitmap words at off
};

struct RawDb {
    bool staged = false;  // b200_stage_db was called for it
    uint64_t n = 0;
    std::vector<uint8_t> keys, vals;
    std::vector<uint64_t> koff, voff;
};

struct Settings {
    uint32_t n_fields = 1;
    std::vector<uint16_t> weights{0};
    std::vector<int> criteria{0, 1, 2, 4, 6, 5, 7};
    bool authorize_typos = true;
    uint32_t one_typo = 5, two_typos = 9;
    bool prefix_search = true;
    std::unordered_map<std::string, int> exact_words;
    std::map<std::vector<std::string>, std::vector<std::vector<std::string>>> synonyms;  // pre-tokenised (index `synonyms` db)
    uint16_t max_weight() const {
        uint16_t m = 0;
        for (auto w : weights) m = m > w ? m : w;
        return m;
    }
};

constexpr uint32_t NO_LIST = 0xffffffffu;

// One faceted field as the Sort rule sees it (search/new/sort.rs:98-195 over the level-0 entries of facet_id_f64_docids and
// facet_id_string_docids).  Its values are numbered in the order a sort walks them: ascending = numbers ascending, then strings
// ascending; descending = numbers descending, then strings descending (numbers still first).  key[dir][doc] is the smallest
// ordinal among the document's values, n_values() when it has none: the Sort buckets of any universe are the groups of equal key
// in ascending key order (DESIGN.md §3).
struct SortField {
    uint32_t n_num = 0, n_str = 0;
    std::vector<uint32_t> num_key, str_key;  // value i -> position among the staged level-0 keys of its database
    std::vector<uint32_t> key[2];            // [0] ascending, [1] descending: u32[n_docs], released after upload
    uint32_t *d_key[2] = {nullptr, nullptr}; // the same in HBM
    // Facet distribution (facet.cu): every document's ascending ordinals, sorted (CSR: doc_off u32[n_docs + 1] into doc_ord), the
    // number ordinals in the order of their f64 Display strings (disp), released after upload; the f64 of each number ordinal
    std::vector<uint32_t> doc_off, doc_ord, disp;
    uint32_t *d_doc_off = nullptr, *d_doc_ord = nullptr, *d_disp = nullptr;
    std::vector<double> num_val;
    std::vector<std::string> str_val;  // the string ordinals' normalised keys (filters bound them in byte order)
    uint64_t n_ord = 0;                // doc_ord's length (kept after upload)
    uint32_t n_values() const { return n_num + n_str; }
    // ordinal of direction `asc` -> (is_string, position among the level-0 keys of its database)
    void decode(bool asc, uint32_t o, bool &is_string, uint32_t &key_index) const {
        is_string = o >= n_num;
        if (!is_string)
            key_index = num_key[asc ? o : n_num - 1 - o];
        else
            key_index = str_key[asc ? o - n_num : n_str - 1 - (o - n_num)];
    }
};

// The GeoSort rule's view of the index (documents/geo_sort.rs:252-277): per document its point, from the level-0 entries of the
// `_geo.lat` / `_geo.lng` fields (number facets first, then strings parsed as f64, the smallest value of each), and the set of
// documents that have one (geo_faceted_documents_ids).
struct GeoField {
    uint16_t lat_fid = 0xFFFF, lng_fid = 0xFFFF;  // 0xFFFF: not staged (no document is geo)
    std::vector<double> lat, lng;                 // per docid (meaningful where `ub` is set)
    std::vector<uint64_t> ub;                     // n_words64 words
    uint64_t n_geo = 0;
};

// Facet search (facet_search.cu) over every field with facet_id_normalized_string_strings entries.  The hyper-normalised strings of
// all fields are one table in byte order per field, decoded to Unicode scalar values (chars / char_off, one u32 per char); string h
// walks the level-0 string keys csr_key[csr_off[h] .. csr_off[h + 1]) (positions among the staged level-0 keys of
// facet_id_string_docids, cut at the first key that database lacks; a set is read as the BTreeSet it is: sorted, deduplicated).
// Only the fields with such strings get their keys' posting lists (FacetSearchField::list0), smallest docids and originals in
// field_id_docid_facet_strings (has_orig 0: none).
struct FacetSearchField {
    uint32_t h0 = 0, h1 = 0;  // its hyper-normalised strings
    uint32_t k0 = 0, n_str = 0;  // its level-0 string keys [k0, k0 + n_str)
    uint32_t n_entries = 0;  // csr_off[h1] - csr_off[h0]
    uint32_t list0 = 0;      // the posting list of key k0 + i is list0 + i
};
struct FacetSearchIndex {
    std::map<uint16_t, FacetSearchField> fields;
    std::vector<uint32_t> chars, char_off{0}, csr_off{0}, csr_key;  // released after upload
    std::vector<uint32_t> min_doc;      // per level-0 string key
    std::vector<uint8_t> has_orig;
    std::vector<std::string> orig, key; // per level-0 string key: its original (when has_orig) and the key itself
};

struct HostIndex {
    // dictionary
    std::vector<uint8_t> dict_bytes;
    std::vector<uint64_t> dict_off;
    uint64_t n_words = 0;
    // prefix tables of the bytewise ascending dictionary (term derivation's work list): first_lo[c] = first word id >= "c" and
    // pair_lo[c << 8 | g] = first word id >= "cg", so [first_lo[c], first_lo[c + 1]) holds the words starting with byte c and
    // [pair_lo[k], pair_lo[k + 1]) (for g < 255) those starting with "cg"; the 1-byte word "c" lies in no 2-byte range
    std::vector<uint32_t> first_lo;  // 257
    std::vector<uint32_t> pair_lo;   // 65537
    uint32_t pair_hi(uint32_t c, uint32_t g) const { return g < 255 ? pair_lo[(c << 8 | g) + 1] : first_lo[c + 1]; }
    // universe
    uint32_t n_docs = 0;    // max docid + 1
    uint32_t n_words64 = 0; // ceil(n_docs / 64)
    std::vector<uint64_t> base_ub;
    uint64_t n_documents = 0;
    // posting store
    std::vector<ListRef> lists;
    std::vector<uint32_t> pool;  // host staging copy, released after upload
    // directories
    std::vector<uint32_t> wd_list, ewd_list;  // per word id
    std::vector<uint32_t> wf_off, wf_list, wp_off, wp_list;  // CSR per word id
    std::vector<uint16_t> wf_fid, wp_pos;
    std::vector<std::string> prefixes;  // sorted
    std::vector<uint32_t> pd_list, epd_list;
    std::vector<uint32_t> pf_off, pf_list, pp_off, pp_list;
    std::vector<uint16_t> pf_fid, pp_pos;
    std::vector<uint64_t> pair_keys;
    uint32_t pair_list_base = 0;
    std::map<uint32_t, uint32_t> fwc_list;  // fid<<8|count -> list
    std::map<uint16_t, SortField> sort_fields;  // faceted fields (fid -> SortField)
    GeoField geo;
    FacetSearchIndex fsearch;
    // facet_id_{exists,is_null,is_empty}_docids: fid -> dense bitmap of n_words64 words (released after upload)
    std::map<uint16_t, std::vector<uint64_t>> presence[3];
    // list id of key i of database db = db_first[db] + i (keys in LMDB order); db_keys[db] = number of staged keys.
    // (word_pair_proximity keys naming unknown words are dropped at staging: for that db the mapping only holds when none was.)
    uint32_t db_first[10] = {0}, db_keys[10] = {0};

    Settings settings;

    const uint8_t *word_ptr(uint64_t i) const { return dict_bytes.data() + dict_off[i]; }
    size_t word_len(uint64_t i) const { return dict_off[i + 1] - dict_off[i]; }
    std::string word(uint64_t i) const { return std::string((const char *)word_ptr(i), word_len(i)); }
    int cmp_word(uint64_t i, const uint8_t *k, size_t kn) const {
        size_t n_i = word_len(i);
        int c = memcmp(word_ptr(i), k, n_i < kn ? n_i : kn);
        if (c) return c;
        return n_i < kn ? -1 : (n_i > kn ? 1 : 0);
    }
    uint64_t lower_bound(const uint8_t *k, size_t kn) const {
        uint64_t lo = 0, hi = n_words;
        while (lo < hi) {
            uint64_t mid = (lo + hi) / 2;
            if (cmp_word(mid, k, kn) < 0)
                lo = mid + 1;
            else
                hi = mid;
        }
        return lo;
    }
    // rank of a word, or -1
    int64_t find_word(const uint8_t *k, size_t kn) const {
        uint64_t i = lower_bound(k, kn);
        return (i < n_words && cmp_word(i, k, kn) == 0) ? (int64_t)i : -1;
    }
    int64_t find_word(const std::string &s) const { return find_word((const uint8_t *)s.data(), s.size()); }
    // [lo, hi) of dictionary words having `p` as a prefix
    void prefix_range(const std::string &p, uint64_t &lo, uint64_t &hi) const {
        lo = lower_bound((const uint8_t *)p.data(), p.size());
        uint64_t a = lo, b = n_words;
        while (a < b) {
            uint64_t mid = (a + b) / 2;
            bool has = word_len(mid) >= p.size() && memcmp(word_ptr(mid), p.data(), p.size()) == 0;
            if (has)
                a = mid + 1;
            else
                b = mid;
        }
        hi = a;
    }
    int32_t find_prefix(const std::string &p) const {
        size_t lo = 0, hi = prefixes.size();
        while (lo < hi) {
            size_t mid = (lo + hi) / 2;
            if (prefixes[mid] < p)
                lo = mid + 1;
            else
                hi = mid;
        }
        return (lo < prefixes.size() && prefixes[lo] == p) ? (int32_t)lo : -1;
    }
    static uint64_t pair_key(uint32_t prox, uint32_t w1, uint32_t w2) { return ((uint64_t)prox << 42) | ((uint64_t)w1 << 21) | w2; }
    // list id of (prox, w1, w2) or NO_LIST
    uint32_t find_pair(uint32_t prox, uint32_t w1, uint32_t w2) const {
        uint64_t k = pair_key(prox, w1, w2);
        size_t lo = 0, hi = pair_keys.size();
        while (lo < hi) {
            size_t mid = (lo + hi) / 2;
            if (pair_keys[mid] < k)
                lo = mid + 1;
            else
                hi = mid;
        }
        return (lo < pair_keys.size() && pair_keys[lo] == k) ? pair_list_base + (uint32_t)lo : NO_LIST;
    }
    uint32_t word_fid_list(uint32_t w, uint16_t fid) const {
        for (uint32_t i = wf_off[w]; i < wf_off[w + 1]; i++)
            if (wf_fid[i] == fid) return wf_list[i];
        return NO_LIST;
    }
    uint32_t word_pos_list(uint32_t w, uint16_t pos) const {
        for (uint32_t i = wp_off[w]; i < wp_off[w + 1]; i++)
            if (wp_pos[i] == pos) return wp_list[i];
        return NO_LIST;
    }
    uint32_t prefix_fid_list(uint32_t p, uint16_t fid) const {
        for (uint32_t i = pf_off[p]; i < pf_off[p + 1]; i++)
            if (pf_fid[i] == fid) return pf_list[i];
        return NO_LIST;
    }
    uint32_t prefix_pos_list(uint32_t p, uint16_t pos) const {
        for (uint32_t i = pp_off[p]; i < pp_off[p + 1]; i++)
            if (pp_pos[i] == pos) return pp_list[i];
        return NO_LIST;
    }
};

// Decode the staged LMDB-format databases into `out` (directories + pool). Throws std::runtime_error.
void build_host_index(const std::vector<uint8_t> &dict_bytes, const std::vector<uint64_t> &dict_off, const RawDb *dbs /*[10]*/,
                      const std::vector<uint8_t> &docids_cbo, HostIndex &out);
// Decode the level-0 entries of facet_id_f64_docids / facet_id_string_docids into out.sort_fields (after build_host_index: needs
// n_docs).  Throws std::runtime_error on a malformed key or value.
void build_sort_fields(const RawDb &f64_db, const RawDb &string_db, HostIndex &out);
// Decode facet_id_exists_docids / facet_id_is_null_docids / facet_id_is_empty_docids (key u16 BE fid, value CBO) into
// out.presence[which] (after build_host_index: needs n_words64).  Throws std::runtime_error on a malformed key.
void build_presence(const RawDb &db, int which, HostIndex &out);
// Rust's `impl Display for f64`: the shortest digits that read back as the same value, never an exponent ("-0" for -0.0)
std::string rust_f64_display(double v);
// Read every document's point into out.geo (after build_host_index; out.geo.lat_fid / lng_fid set, or nothing to do).  Throws
// std::runtime_error for a document with one coordinate only or a string coordinate that does not parse as f64.
void build_geo_field(const RawDb &f64_db, const RawDb &string_db, HostIndex &out);
// Build out.fsearch from facet_id_string_docids, facet_id_normalized_string_strings and field_id_docid_facet_strings, appending the
// level-0 string keys' posting lists to the pool (after build_host_index, before the pool is uploaded).  Throws std::runtime_error
// on a malformed key or a value that is not a JSON array of strings.
void build_facet_search(const RawDb &string_db, const RawDb &norm_db, const RawDb &orig_db, HostIndex &out);
// The JSON array of strings `s` (serde_json's output for a BTreeSet<String>, escapes included), false when it is not one
bool parse_json_string_array(const uint8_t *s, size_t n, std::vector<std::string> &out);
// The Unicode scalar values of UTF-8 bytes; false when they are not UTF-8 (overlong forms and surrogates included)
bool utf8_decode(const uint8_t *s, size_t n, std::vector<uint32_t> &out);

}  // namespace b200
