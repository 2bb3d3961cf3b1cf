// C ABI (include/b200milli.h) over the engine; hybrid merge (search/hybrid.rs) lives here because it is pure host logic
// over two result lists.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <new>
#include <unordered_set>

#include "engine.h"
#include "kernels.h"

using namespace b200;

struct b200_index {
    Engine e;
};
struct b200_rule {
    Engine::RuleRun *run;
    uint64_t n_words;
};
namespace b200 {
int rule_next_impl(Engine::RuleRun *run, uint64_t n_words64, const uint64_t *universe, uint64_t *out_bitmap, uint64_t n_words, uint32_t *rank,
                   uint32_t *max_rank, GraphObj **out_query);
void rule_end_impl(Engine::RuleRun *run);
}  // namespace b200

static thread_local std::string g_open_error;

// no exception crosses the C boundary: every entry point runs its body through this
template <class F>
static int guarded(b200_index *h, F body) {
    if (!h) return B200_ERR_INVALID;
    try {
        return body();
    } catch (const std::bad_alloc &) {
        return h->e.fail(B200_ERR_CAPACITY, "out of host memory");
    } catch (const std::exception &ex) {
        return h->e.fail(B200_ERR_INVALID, ex.what());
    } catch (...) {
        return h->e.fail(B200_ERR_INVALID, "unexpected exception");
    }
}

extern "C" {

const char *b200_open_error(void) { return g_open_error.c_str(); }

int b200_open(int device_ordinal, b200_index **out) {
    *out = nullptr;
    int n = 0;
    cudaError_t err = cudaGetDeviceCount(&n);
    if (err != cudaSuccess || n == 0) {
        g_open_error = std::string("no CUDA device: ") + (err != cudaSuccess ? cudaGetErrorString(err) : "device count is 0") +
                       " (b200milli has no CPU fallback)";
        return B200_ERR_NO_DEVICE;
    }
    if (device_ordinal < 0 || device_ordinal >= n) {
        g_open_error = "device ordinal out of range";
        return B200_ERR_INVALID;
    }
    b200_index *h = new (std::nothrow) b200_index();
    if (!h) return B200_ERR_INVALID;
    h->e.device = device_ordinal;
    if ((err = cudaSetDevice(device_ordinal)) != cudaSuccess || (err = cudaStreamCreateWithFlags(&h->e.stream, cudaStreamNonBlocking)) != cudaSuccess ||
        (err = cudaStreamCreateWithFlags(&h->e.vt.stream, cudaStreamNonBlocking)) != cudaSuccess) {
        g_open_error = std::string("CUDA init failed: ") + cudaGetErrorString(err);
        delete h;
        return B200_ERR_CUDA;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device_ordinal) == cudaSuccess) h->e.sm_count = prop.multiProcessorCount;
    h->e.affinity.detect(device_ordinal);
    *out = h;
    return B200_OK;
}
void b200_close(b200_index *h) { delete h; }
const char *b200_last_error(const b200_index *h) { return h ? h->e.last_error.c_str() : "null handle"; }

int b200_stage_dictionary(b200_index *h, const uint8_t *bytes, const uint64_t *offsets, uint64_t n) {
    return guarded(h, [&]() -> int {
        std::lock_guard<std::mutex> g(h->e.mu);
        if (h->e.staged) return h->e.fail(B200_ERR_STATE, "staging after b200_stage_finish: open a new handle");
        if (!offsets || (!bytes && n && offsets[n])) return h->e.fail(B200_ERR_INVALID, "stage_dictionary: null argument");
        for (uint64_t i = 0; i < n; i++)
            if (offsets[i + 1] < offsets[i]) return h->e.fail(B200_ERR_INVALID, "stage_dictionary: offsets must not decrease");
        h->e.raw_dict_off.assign(offsets, offsets + n + 1);
        h->e.raw_dict_bytes.assign(bytes, bytes + offsets[n]);
        return B200_OK;
    });
}
int b200_stage_db(b200_index *h, int db, uint64_t n, const uint8_t *kb, const uint64_t *ko, const uint8_t *vb, const uint64_t *vo) {
    return guarded(h, [&]() -> int {
        std::lock_guard<std::mutex> g(h->e.mu);
        if (h->e.staged) return h->e.fail(B200_ERR_STATE, "staging after b200_stage_finish: open a new handle");
        if (db < 0 || db >= B200_DB_COUNT) return h->e.fail(B200_ERR_INVALID, "unknown database id");
        if (!ko || !vo || (n && (!kb || !vb))) return h->e.fail(B200_ERR_INVALID, "stage_db: null argument");
        for (uint64_t i = 0; i < n; i++)
            if (ko[i + 1] < ko[i] || vo[i + 1] < vo[i]) return h->e.fail(B200_ERR_INVALID, "stage_db: offsets must not decrease");
        RawDb &d = h->e.raw_dbs[db];
        d.staged = true;
        d.n = n;
        d.koff.assign(ko, ko + n + 1);
        d.voff.assign(vo, vo + n + 1);
        d.keys.assign(kb, kb + ko[n]);
        d.vals.assign(vb, vb + vo[n]);
        return B200_OK;
    });
}
int b200_stage_documents_ids(b200_index *h, const uint8_t *cbo, uint64_t len) {
    return guarded(h, [&]() -> int {
        std::lock_guard<std::mutex> g(h->e.mu);
        if (h->e.staged) return h->e.fail(B200_ERR_STATE, "staging after b200_stage_finish: open a new handle");
        if (!cbo && len) return h->e.fail(B200_ERR_INVALID, "stage_documents_ids: null argument");
        h->e.raw_docids.assign(cbo, cbo + len);
        return B200_OK;
    });
}
int b200_stage_settings(b200_index *h, const b200_settings *s) {
    if (!h || !s) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> g(h->e.mu);
    Settings &t = h->e.hix.settings;
    if (s->n_fields == 0 || s->n_fields > 1024) return h->e.fail(B200_ERR_INVALID, "n_fields out of range");
    if (!s->weights || (s->n_criteria && !s->criteria)) return h->e.fail(B200_ERR_INVALID, "stage_settings: null weights / criteria");
    t.n_fields = s->n_fields;
    t.weights.assign(s->weights, s->weights + s->n_fields);
    t.criteria.assign(s->criteria, s->criteria + s->n_criteria);
    t.authorize_typos = s->authorize_typos != 0;
    t.one_typo = s->min_word_len_one_typo;
    t.two_typos = s->min_word_len_two_typos;
    t.prefix_search = s->prefix_search != 0;
    t.exact_words.clear();
    if (s->exact_words) {
        std::string cur;
        for (const char *p = s->exact_words;; p++) {
            if (*p == '\n' || *p == 0) {
                if (!cur.empty()) t.exact_words[cur] = 1;
                cur.clear();
                if (!*p) break;
            } else
                cur.push_back(*p);
        }
    }
    return B200_OK;
}
static std::vector<std::string> split_ws(const char *s) {
    std::vector<std::string> out;
    std::string cur;
    for (const char *p = s;; p++) {
        if (*p == ' ' || *p == 0) {
            if (!cur.empty()) out.push_back(cur);
            cur.clear();
            if (!*p) break;
        } else
            cur.push_back(*p);
    }
    return out;
}
int b200_stage_synonyms(b200_index *h, uint32_t n, const char *const *from_words, const char *const *to_words) {
    std::lock_guard<std::mutex> g(h->e.mu);
    auto &syn = h->e.hix.settings.synonyms;
    syn.clear();
    for (uint32_t i = 0; i < n; i++) syn[split_ws(from_words[i])].push_back(split_ws(to_words[i]));
    return B200_OK;
}
int b200_stage_geo_fields(b200_index *h, uint16_t lat_fid, uint16_t lng_fid) {
    std::lock_guard<std::mutex> g(h->e.mu);
    if (h->e.staged) return h->e.fail(B200_ERR_STATE, "staging after b200_stage_finish: open a new handle");
    h->e.hix.geo.lat_fid = lat_fid;
    h->e.hix.geo.lng_fid = lng_fid;
    return B200_OK;
}
int b200_stage_finish(b200_index *h) {
    return guarded(h, [&]() -> int {
        std::lock_guard<std::mutex> g(h->e.mu);
        if (h->e.staged) return h->e.fail(B200_ERR_STATE, "b200_stage_finish was already called on this handle");
        Settings keep = h->e.hix.settings;
        int rc = h->e.stage_finish();
        h->e.hix.settings = keep;
        return rc;
    });
}
int b200_stage_embeddings(b200_index *h, const float *v, uint64_t n, uint32_t d, const uint32_t *docids) {
    std::lock_guard<std::mutex> g(h->e.mu);
    return h->e.stage_embeddings(v, nullptr, n, d, docids);
}
int b200_stage_embeddings_f16(b200_index *h, const uint16_t *rows, uint64_t n, uint32_t d, const uint32_t *docids) {
    std::lock_guard<std::mutex> g(h->e.mu);
    return h->e.stage_embeddings(nullptr, rows, n, d, docids);
}
int b200_stage_distribution(b200_index *h, int enabled, float mean, float sigma) {
    std::lock_guard<std::mutex> g(h->e.mu);
    h->e.has_distribution = enabled != 0 && sigma > 0.f;
    h->e.dist_mean = mean;
    h->e.dist_sigma = sigma;
    return B200_OK;
}
int b200_derive_batch(b200_index *h, uint32_t n, const char *words, const uint32_t *off, const uint8_t *mt, const uint8_t *ip, uint32_t *one,
                      uint32_t *n_one, uint32_t *two, uint32_t *n_two) {
    std::lock_guard<std::mutex> g(h->e.mu);
    return h->e.derive_batch(n, words, off, mt, ip, one, n_one, two, n_two);
}
int b200_nns_batch(b200_index *h, const float *q, uint32_t n_q, uint32_t d, uint32_t limit, const uint64_t *cand, uint64_t ncw, uint32_t *ids,
                   float *dist, uint32_t *n_out) {
    std::lock_guard<std::mutex> g(h->e.mu);
    int rc = h->e.nns_batch(q, n_q, d, limit, cand, ncw, ids, dist, n_out);
    h->e.fold_vector_stats();
    return rc;
}
int b200_comm_unique_id(b200_index *h, uint8_t *out128) {
    std::lock_guard<std::mutex> g(h->e.mu);
    int rc = h->e.comm_load();
    if (rc != B200_OK) return rc;
    int e = h->e.sc.get_unique_id(out128);
    return e == 0 ? B200_OK : h->e.fail(B200_ERR_CUDA, "ncclGetUniqueId failed");
}
int b200_comm_init(b200_index *h, int rank, int world, const uint8_t *unique_id128) {
    std::lock_guard<std::mutex> g(h->e.mu);
    return h->e.comm_init(rank, world, unique_id128);
}
int b200_nns_batch_sharded(b200_index *h, const float *q, uint32_t n_q, uint32_t d, uint32_t limit, const uint64_t *cand, uint64_t ncw, uint32_t *ids,
                           float *dist, uint32_t *n_out) {
    std::lock_guard<std::mutex> g(h->e.mu);
    int rc = h->e.nns_batch(q, n_q, d, limit, cand, ncw, ids, dist, n_out, true);
    h->e.fold_vector_stats();
    return rc;
}
int b200_union_postings(b200_index *h, int db, const uint32_t *key_index, uint32_t n_keys, const uint64_t *universe, uint64_t n_universe_words,
                        uint64_t *out) {
    std::lock_guard<std::mutex> g(h->e.mu);
    return h->e.union_postings(db, key_index, n_keys, universe, n_universe_words, out);
}
int b200_proximity_pairs(b200_index *h, const uint32_t *left, uint32_t n_left, const uint32_t *right, uint32_t n_right, uint32_t fwd_prox,
                         uint32_t bwd_prox, const uint64_t *universe, uint64_t n_universe_words, uint64_t *out) {
    std::lock_guard<std::mutex> g(h->e.mu);
    return h->e.proximity_pairs(left, n_left, right, n_right, fwd_prox, bwd_prox, universe, n_universe_words, out);
}
int b200_graph_from_tokens(b200_index *h, const b200_query_batch *one_query, b200_graph **out) {
    std::lock_guard<std::mutex> g(h->e.mu);
    if (!h->e.staged) return h->e.fail(B200_ERR_STATE, "graph_from_tokens before b200_stage_finish");
    GraphObj *go = nullptr;
    int rc = h->e.graph_from_tokens(one_query, &go);
    *out = reinterpret_cast<b200_graph *>(go);
    return rc;
}
void b200_graph_free(b200_graph *g) { free_graph(reinterpret_cast<GraphObj *>(g)); }
int b200_rule_start(b200_index *h, int rule_kind, int terms_matching_strategy, const b200_graph *query, const uint64_t *universe,
                    uint64_t n_universe_words, b200_rule **out) {
    std::lock_guard<std::mutex> g(h->e.mu);
    *out = nullptr;
    if (!h->e.staged) return h->e.fail(B200_ERR_STATE, "rule_start before b200_stage_finish");
    Engine::RuleRun *run = nullptr;
    int rc = h->e.rule_start(rule_kind, terms_matching_strategy, reinterpret_cast<const GraphObj *>(query), universe, n_universe_words, &run);
    if (rc != B200_OK) return rc;
    b200_rule *r = new b200_rule{run, h->e.hix.n_words64};
    *out = r;
    return B200_OK;
}
int b200_rule_next(b200_rule *r, const uint64_t *universe, uint64_t *out_bitmap, uint64_t n_words, uint32_t *rank, uint32_t *max_rank,
                   b200_graph **out_query) {
    if (!r) return B200_ERR_INVALID;
    GraphObj *child = nullptr;
    int rc = rule_next_impl(r->run, r->n_words, universe, out_bitmap, n_words, rank, max_rank, out_query ? &child : nullptr);
    if (out_query) *out_query = reinterpret_cast<b200_graph *>(child);
    return rc;
}
void b200_rule_end(b200_rule *r) {
    if (!r) return;
    rule_end_impl(r->run);
    delete r;
}
int b200_search_batch(b200_index *h, const b200_query_batch *b, b200_results *r) {
    return guarded(h, [&]() -> int {
        std::lock_guard<std::mutex> g(h->e.mu);
        if (!h->e.staged) return h->e.fail(B200_ERR_STATE, "search before b200_stage_finish");
        if (!b || !r || !r->docids || !r->n_hits) return h->e.fail(B200_ERR_INVALID, "search: null batch / results / docids / n_hits");
        if (b->n_queries && (!b->token_begin || !b->lemma_off)) return h->e.fail(B200_ERR_INVALID, "search: null token arrays");
        // every query starts with a definite status and no hits, whatever happens later
        for (uint32_t i = 0; i < b->n_queries; i++) {
            r->n_hits[i] = 0;
            if (r->status) r->status[i] = 0;
            if (r->filter_error_leaf) r->filter_error_leaf[i] = -1;
        }
        return h->e.search_batch(b, r);
    });
}
int b200_geo_filter_batch(b200_index *h, uint32_t n, const uint8_t *kind, const double *args, uint64_t *out, uint64_t out_words, int32_t *status) {
    return guarded(h, [&]() -> int {
        std::lock_guard<std::mutex> g(h->e.mu);
        if (!h->e.staged) return h->e.fail(B200_ERR_STATE, "geo filter before b200_stage_finish");
        return h->e.geo_filter_batch(n, kind, args, out, out_words, status);
    });
}
int b200_filter_batch(b200_index *h, const b200_filter_programs *programs, uint64_t *out, uint64_t out_words, int32_t *status, int32_t *error_leaf) {
    return guarded(h, [&]() -> int {
        std::lock_guard<std::mutex> g(h->e.mu);
        if (!h->e.staged) return h->e.fail(B200_ERR_STATE, "filter before b200_stage_finish");
        return h->e.filter_batch(programs, out, out_words, status, error_leaf);
    });
}
int b200_facet_distribution_batch(b200_index *h, uint32_t n, const uint64_t *const *candidates, uint64_t n_words, const uint32_t *facet_begin,
                                  const uint16_t *facet_fid, const uint8_t *facet_order, uint32_t max_values, uint32_t cap, uint32_t *n_num,
                                  uint32_t *n_str, uint32_t *key, uint64_t *count, uint32_t *docid, uint8_t *has_stats, double *min,
                                  double *max, int32_t *status) {
    return guarded(h, [&]() -> int {
        std::lock_guard<std::mutex> g(h->e.mu);
        if (!h->e.staged) return h->e.fail(B200_ERR_STATE, "facet distribution before b200_stage_finish");
        b200_results dst{};
        dst.facet_n_num = n_num;
        dst.facet_n_str = n_str;
        dst.facet_key = key;
        dst.facet_count = count;
        dst.facet_docid = docid;
        dst.facet_has_stats = has_stats;
        dst.facet_min = min;
        dst.facet_max = max;
        return h->e.facet_distribution_batch(n, candidates, n_words, facet_begin, facet_fid, facet_order, max_values, cap, dst, status);
    });
}
int b200_facet_search_batch(b200_index *h, uint32_t n, const uint64_t *const *candidates, uint64_t n_words, const uint16_t *fid,
                            const uint8_t *kind, const uint32_t *off, const char *query_bytes, const uint8_t *flags, uint32_t max,
                            uint32_t cap, uint32_t *n_out, uint32_t *key, uint64_t *count, uint32_t *docid, uint8_t *fallback,
                            int32_t *status) {
    return guarded(h, [&]() -> int {
        std::lock_guard<std::mutex> g(h->e.mu);
        if (!h->e.staged) return h->e.fail(B200_ERR_STATE, "facet search before b200_stage_finish");
        return h->e.facet_search_batch(n, candidates, n_words, fid, kind, off, query_bytes, flags, max, cap, n_out, key, count, docid,
                                       fallback, status);
    });
}
int b200_similar_batch(b200_index *h, const b200_similar_request *rq, b200_results *r) {
    return guarded(h, [&]() -> int {
        std::lock_guard<std::mutex> g(h->e.mu);
        if (!rq || !r || !r->n_hits || (rq->n_queries && rq->limit && !r->docids)) return h->e.fail(B200_ERR_INVALID, "similar: null request / results / docids / n_hits");
        if (!h->e.staged) return h->e.fail(B200_ERR_STATE, "similar before b200_stage_finish");
        for (uint32_t i = 0; i < rq->n_queries; i++) {
            r->n_hits[i] = 0;
            if (r->status) r->status[i] = 0;
            if (r->filter_error_leaf) r->filter_error_leaf[i] = -1;
        }
        int rc = h->e.similar_batch(rq, r);
        h->e.fold_vector_stats();
        return rc;
    });
}
int b200_get_stats(b200_index *h, b200_stats *out) {
    std::lock_guard<std::mutex> g(h->e.mu);
    *out = h->e.stats;
    return B200_OK;
}
int b200_reset_stats(b200_index *h) {
    std::lock_guard<std::mutex> g(h->e.mu);
    uint64_t staged = h->e.stats.hbm_bytes_staged;
    h->e.stats = b200_stats{};
    h->e.stats.hbm_bytes_staged = staged;
    return B200_OK;
}
}

// ================================================================================= semantic + hybrid
namespace b200 {

static float distribution_shift(float mean, float sigma, float score) {  // vector/distribution.rs:103-130
    float factor = 0.4f / sigma, offset = 0.5f - factor * mean;
    float s = factor * score + offset;
    if (s <= 0.f) s = 1.1920929e-7f;
    if (s > 1.f) s = 1.f;
    return s;
}

std::vector<Engine::UniverseGroup> Engine::group_by_universe(uint32_t n_queries, const uint64_t *const *universes, const GeoFiltered *gf) const {
    std::map<std::pair<const uint64_t *, const unsigned long long *>, std::vector<uint32_t>> groups;
    for (uint32_t q = 0; q < n_queries; q++) {
        if (gf && gf->status[q]) continue;
        if (gf && gf->d_univ[q])
            groups[{nullptr, gf->d_univ[q]}].push_back(q);
        else
            groups[{universes ? universes[q] : nullptr, nullptr}].push_back(q);
    }
    std::vector<UniverseGroup> out;
    for (auto &g : groups) {
        UniverseGroup u{g.first.first, g.first.second, hix.n_documents, std::move(g.second)};
        if (u.dev) {
            u.count = gf->count[u.queries[0]];
        } else if (u.host) {
            u.count = 0;
            for (uint64_t w = 0; w < hix.n_words64; w++) u.count += (uint64_t)__builtin_popcountll(u.host[w] & hix.base_ub[w]);
        }
        out.push_back(std::move(u));
    }
    return out;
}

// execute_vector_search (search/new/mod.rs:744-808): one VectorSort rule over documents_ids; buckets = runs of equal
// distance in ascending docid order (vector_sort.rs:80-95), which the (distance, docid) ordering of nns_batch reproduces.
int Engine::semantic_batch(const b200_query_batch *b, b200_results *r, uint32_t offset, uint32_t limit) {
    if (!b->vectors) return fail(B200_ERR_INVALID, "semantic search without vectors");
    uint32_t k = offset + limit;
    if (k == 0) k = 1;
    std::vector<uint32_t> ids((size_t)b->n_queries * k), n(b->n_queries);
    std::vector<float> dist((size_t)b->n_queries * k);
    std::vector<uint64_t> n_cand(b->n_queries, hix.n_documents);
    const GeoFiltered *gf = geo_filtered;  // queries with geo clauses scan their device bitmap; refused ones are answered below
    if (!b->universes && !gf) {
        int rc = nns_batch(b->vectors, b->n_queries, emb_d_user, k, nullptr, 0, ids.data(), dist.data(), n.data());
        if (rc != B200_OK) return rc;
    } else {
        // filtered_universe restricts the vector candidates (vector_sort.rs:58-78: `vector_candidates & universe`): the queries
        // are grouped by bitmap (the caller's, or a geo-filtered one on the device) and every group is one scan with that filter
        if (b->universes && b->n_universe_words < hix.n_words64) return fail(B200_ERR_INVALID, "universe bitmaps shorter than the document range");
        const uint32_t d = emb_d_user;
        for (const UniverseGroup &g : group_by_universe(b->n_queries, b->universes, gf)) {
            const uint32_t m = (uint32_t)g.queries.size();
            std::vector<float> vq((size_t)m * d);
            for (uint32_t i = 0; i < m; i++) memcpy(vq.data() + (size_t)i * d, b->vectors + (size_t)g.queries[i] * d, (size_t)d * 4);
            std::vector<uint32_t> gi((size_t)m * k), gn(m);
            std::vector<float> gd((size_t)m * k);
            int rc = nns_batch(vq.data(), m, d, k, g.host, g.host || g.dev ? hix.n_words64 : 0, gi.data(), gd.data(), gn.data(), false, g.dev);
            if (rc != B200_OK) return rc;
            for (uint32_t i = 0; i < m; i++) {
                const uint32_t q = g.queries[i];
                n[q] = gn[i];
                n_cand[q] = g.count;
                memcpy(ids.data() + (size_t)q * k, gi.data() + (size_t)i * k, (size_t)gn[i] * 4);
                memcpy(dist.data() + (size_t)q * k, gd.data() + (size_t)i * k, (size_t)gn[i] * 4);
            }
        }
    }
    // VectorSort's last bucket (vector_sort.rs:128-160): once the embedded candidates are exhausted, the rest of the universe
    // follows in docid order with `similarity: None`
    // a geo-filtered universe comes back to the host only when a query's embedded candidates run out, once per slot
    std::map<const unsigned long long *, std::vector<uint64_t>> geo_u;
    for (uint32_t q = 0; q < b->n_queries; q++) {
        if (n[q] >= k || (gf && gf->status[q])) continue;
        const uint64_t *u = b->universes ? b->universes[q] : nullptr;
        if (gf && gf->d_univ[q]) {
            std::vector<uint64_t> &h = geo_u[gf->d_univ[q]];
            if (h.empty()) {
                h.resize(hix.n_words64);
                cudaError_t e = cudaMemcpyAsync(h.data(), gf->d_univ[q], hix.n_words64 * 8, cudaMemcpyDeviceToHost, vt.stream);
                if (e == cudaSuccess) e = cudaStreamSynchronize(vt.stream);
                if (e != cudaSuccess) return cuda_fail(e, "D2H geo universe");
                vstats.d2h_bytes += hix.n_words64 * 8;
            }
            u = h.data();
        }
        for (uint64_t w = 0; w < hix.n_words64 && n[q] < k; w++) {
            uint64_t bits = hix.base_ub[w] & (u ? u[w] : ~0ull) & ~(w < emb_bitmap.size() ? emb_bitmap[w] : 0ull);
            while (bits && n[q] < k) {
                ids[(size_t)q * k + n[q]] = (uint32_t)(w * 64 + (uint64_t)__builtin_ctzll(bits));
                dist[(size_t)q * k + n[q]] = 2.0f;  // marks "no similarity"
                n[q]++;
                bits &= bits - 1;
            }
        }
    }
    for (uint32_t q = 0; q < b->n_queries; q++) {
        uint32_t hits = n[q] > offset ? std::min(limit, n[q] - offset) : 0;
        r->n_hits[q] = hits;
        if (r->status) r->status[q] = 0;
        if (r->degraded) r->degraded[q] = 0;
        if (r->used_negative_operator) r->used_negative_operator[q] = 0;
        if (r->n_candidates) r->n_candidates[q] = n_cand[q];
        for (uint32_t i = 0; i < hits; i++) {
            size_t src = (size_t)q * k + offset + i, at = (size_t)q * limit + i;
            r->docids[at] = ids[src];
            float sim = 1.0f - dist[src];
            if (dist[src] > 1.5f)
                sim = -1.f;  // Vector { similarity: None }
            else if (has_distribution)
                sim = distribution_shift(dist_mean, dist_sigma, sim);
            if (r->n_scores) {
                r->n_scores[at] = 1;
                r->score_kind[at * B200_MAX_SCORES] = B200_S_VECTOR;
                r->score_rank[at * B200_MAX_SCORES] = 0;
                r->score_max[at * B200_MAX_SCORES] = 1;
                r->score_sim[at * B200_MAX_SCORES] = sim;
            }
        }
    }
    return B200_OK;
}

// Similar::execute (search/similar.rs:66-152); semantics in include/b200milli.h (b200_similar_batch)
int Engine::similar_batch(const b200_similar_request *rq, b200_results *r) {
    const uint32_t NQ = rq->n_queries;
    const uint64_t W = hix.n_words64;
    if (!rq->docids) return fail(B200_ERR_INVALID, "similar: null docids");
    if (rq->universes && rq->n_universe_words < W) return fail(B200_ERR_INVALID, "universe bitmaps shorter than the document range");
    if (r->candidates) return fail(B200_ERR_UNSUPPORTED, "similar: the candidates bitmap is not returned (the route reads only its length)");
    if (!dix.emb) return fail(B200_ERR_STATE, "similar before b200_stage_embeddings");
    if (cudaError_t e = cudaSetDevice(device)) return cuda_fail(e, "cudaSetDevice");
    // filtered_universe: the filter programs run exactly as in searches (filter_universes), so their errors fail their query alone
    GeoFiltered gf;
    const GeoFiltered *gfp = nullptr;
    if (rq->filter) {
        b200_query_batch qb{};
        qb.n_queries = NQ;
        qb.universes = rq->universes;
        qb.n_universe_words = rq->n_universe_words;
        qb.filter = rq->filter;
        int rc = filter_universes(&qb, gf);
        if (rc != B200_OK) return rc;
        gfp = &gf;
        if (r->filter_error_leaf && !gf.error_leaf.empty())
            for (uint32_t q = 0; q < NQ; q++) r->filter_error_leaf[q] = gf.status[q] ? gf.error_leaf[q] : -1;
    }
    for (uint32_t q = 0; q < NQ; q++) {
        r->n_hits[q] = 0;
        if (r->n_candidates) r->n_candidates[q] = 0;
        if (r->degraded) r->degraded[q] = 0;
        if (r->used_negative_operator) r->used_negative_operator[q] = 0;
        if (r->semantic_hits) r->semantic_hits[q] = 0;
        int32_t st = gfp ? gf.status[q] : 0;
        if (st) last_error = gf.error[q];
        else if (emb_multi_row) {
            st = B200_ERR_UNSUPPORTED;
            last_error = "similar: a document has several embeddings (the reference searches each of its stores with the target's vector of that store)";
        }
        if (r->status) r->status[q] = st;
    }
    if (emb_multi_row) return B200_OK;
    const auto in = [](const uint64_t *bm, uint32_t doc) { return ((bm[doc >> 6] >> (doc & 63)) & 1) != 0; };
    const uint32_t offset = rq->offset, limit = rq->limit, keep = offset + limit + 1, k = keep + 1;
    for (const UniverseGroup &g : group_by_universe(NQ, rq->universes, gfp)) {
        // |U \ {id}| needs to know whether the target is in U: on the host for the caller's bitmaps, one batched read of the target
        // words for a device bitmap
        const uint32_t m = (uint32_t)g.queries.size();
        std::vector<uint8_t> member(m, 0);
        std::vector<uint32_t> probe;  // indices into g.queries whose target word is read from the device
        for (uint32_t i = 0; i < m; i++) {
            const uint32_t id = rq->docids[g.queries[i]];
            if (id >= W * 64 || !in(hix.base_ub.data(), id)) continue;  // outside documents_ids, or beyond the document range
            if (g.dev)
                probe.push_back(i);
            else
                member[i] = !g.host || in(g.host, id);
        }
        if (!probe.empty()) {
            const uint32_t np = (uint32_t)probe.size();
            std::vector<unsigned long long> addr(np), words(np);
            for (uint32_t j = 0; j < np; j++) addr[j] = (unsigned long long)(uintptr_t)(g.dev + (rq->docids[g.queries[probe[j]]] >> 6));
            cudaError_t e = d_sim_addr.reserve(np);
            if (e == cudaSuccess) e = d_sim_word.reserve(np);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d_sim_addr.p, addr.data(), (size_t)np * 8, cudaMemcpyHostToDevice, vt.stream);
            if (e == cudaSuccess) e = launch_gather_words(vt.stream, d_sim_addr.p, np, d_sim_word.p);
            if (e == cudaSuccess) e = cudaMemcpyAsync(words.data(), d_sim_word.p, (size_t)np * 8, cudaMemcpyDeviceToHost, vt.stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(vt.stream);
            if (e != cudaSuccess) return cuda_fail(e, "similar: target words");
            vstats.h2d_bytes += (size_t)np * 8;
            vstats.d2h_bytes += (size_t)np * 8;
            vstats.kernel_launches++;
            for (uint32_t j = 0; j < np; j++) member[probe[j]] = (words[j] >> (rq->docids[g.queries[probe[j]]] & 63)) & 1;
        }
        // the scan: every embedded target in documents_ids, over the group's universe with the target still in it
        std::vector<uint32_t> rows, at;
        for (uint32_t i = 0; i < m; i++) {
            const uint32_t q = g.queries[i], id = rq->docids[q];
            if (r->n_candidates) r->n_candidates[q] = g.count - member[i];
            if (id < W * 64 && in(hix.base_ub.data(), id) && id < emb_row.size() && emb_row[id] != UINT32_MAX) {
                rows.push_back(emb_row[id]);
                at.push_back(i);
            }
        }
        if (rows.empty()) continue;
        // U is always within documents_ids: a caller's bitmap is intersected with it, and without one documents_ids is the filter
        std::vector<uint64_t> hu;
        if (g.host) {
            hu.resize(W);
            for (uint64_t w = 0; w < W; w++) hu[w] = g.host[w] & hix.base_ub[w];
        }
        const unsigned long long *du = g.dev ? g.dev : (g.host ? nullptr : dix.base_ub);
        const uint32_t nr = (uint32_t)rows.size();
        std::vector<uint32_t> gi((size_t)nr * k), gn(nr);
        std::vector<float> gd((size_t)nr * k);
        int rc = nns_batch(nullptr, nr, dix.emb_d, k, g.host ? hu.data() : nullptr, W, gi.data(), gd.data(), gn.data(), false, du, rows.data());
        if (rc != B200_OK) return rc;
        for (uint32_t j = 0; j < nr; j++) {
            const uint32_t i = at[j], q = g.queries[i], id = rq->docids[q];
            // U \ {id}: the target leaves the list wherever it is (with zero vectors or ties it need not come first)
            std::vector<std::pair<uint32_t, float>> list;
            for (uint32_t e = 0; e < gn[j] && list.size() < keep; e++)
                if (gi[(size_t)j * k + e] != id) list.push_back({gi[(size_t)j * k + e], gd[(size_t)j * k + e]});
            std::unordered_set<uint32_t> seen{id};
            uint32_t skipped = 0, hits = 0;
            for (const auto &c : list) {
                if (hits == limit) break;
                if (!seen.insert(c.first).second) continue;
                if (skipped < offset) {
                    skipped++;
                    continue;
                }
                float sim = 1.0f - c.second;
                if (has_distribution) sim = distribution_shift(dist_mean, dist_sigma, sim);
                if (rq->has_ranking_score_threshold && (double)sim < rq->ranking_score_threshold) {
                    // candidates = (candidates \ {doc}) AND seen: the documents walked before this one
                    if (r->n_candidates) r->n_candidates[q] = seen.size() - 2;
                    break;
                }
                const size_t o = (size_t)q * limit + hits++;
                r->docids[o] = c.first;
                if (r->n_scores) {
                    r->n_scores[o] = 1;
                    r->score_kind[o * B200_MAX_SCORES] = B200_S_VECTOR;
                    r->score_rank[o * B200_MAX_SCORES] = 0;
                    r->score_max[o * B200_MAX_SCORES] = 1;
                    r->score_sim[o * B200_MAX_SCORES] = sim;
                }
            }
            r->n_hits[q] = hits;
        }
    }
    return B200_OK;
}

namespace {
struct Hit {
    uint32_t doc;
    std::vector<double> values;  // ScoreDetails::score_values (score_details.rs:156-175)
    uint8_t n_scores;
    uint8_t kind[B200_MAX_SCORES];
    uint32_t rank[B200_MAX_SCORES], maxr[B200_MAX_SCORES];
    float sim[B200_MAX_SCORES];
};
void rank_merge(uint64_t &orank, uint64_t &omax, uint64_t irank, uint64_t imax) {
    orank = orank > 0 ? orank - 1 : 0;
    orank *= imax;
    omax *= imax;
    orank += irank;
}
void fill_values(Hit &h) {
    bool in_rank = false;
    uint64_t rk = 0, mx = 1;
    for (int s = 0; s < h.n_scores; s++) {
        if (h.kind[s] == B200_S_VECTOR) {
            if (in_rank) {
                h.values.push_back((double)rk / (double)mx);
                in_rank = false;
            }
            h.values.push_back(h.sim[s] < 0 ? 0.0 : (double)h.sim[s]);
        } else if (!in_rank) {
            rk = h.rank[s];
            mx = h.maxr[s];
            in_rank = true;
        } else
            rank_merge(rk, mx, h.rank[s], h.maxr[s]);
    }
    if (in_rank) h.values.push_back((double)rk / (double)mx);
}
double global_score(const Hit &h) {
    uint64_t rk = 1, mx = 1;
    bool sem = false;
    double sv = 0;
    for (int s = 0; s < h.n_scores; s++) {
        if (h.kind[s] == B200_S_VECTOR) {
            sem = true;
            sv = h.sim[s] < 0 ? 0.0 : (double)h.sim[s];
        } else
            rank_merge(rk, mx, h.rank[s], h.maxr[s]);
    }
    return sem ? sv : (double)rk / (double)mx;
}
int compare_scores(const Hit &l, float lr, const Hit &r, float rr) {  // hybrid.rs:32-80
    for (size_t i = 0;; i++) {
        bool hl = i < l.values.size(), hr = i < r.values.size();
        if (!hl && !hr) return 0;
        if (!hl) return -1;
        if (!hr) return 1;
        double a = l.values[i] * (double)lr, b = r.values[i] * (double)rr;
        if (std::fabs(a - b) <= 2.220446049250313e-16) continue;
        return a < b ? -1 : 1;
    }
}
}  // namespace

// Search::execute_hybrid (search/hybrid.rs:264-366)
int Engine::search_batch(const b200_query_batch *b, b200_results *r) {
    if (!b->geo_filter_begin && !b->filter) return search_batch_filtered(b, r);
    // geo filters and filter programs: every query's filtered universe is computed once, before the modes split (hybrid runs both
    // stages on it)
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) return cuda_fail(e, "cudaSetDevice");
    GeoFiltered gf;
    int rc = b->geo_filter_begin ? geo_filter_universes(b, gf) : B200_OK;
    if (rc == B200_OK && b->filter) rc = filter_universes(b, gf);
    if (rc != B200_OK) return rc;
    struct Scope {
        const GeoFiltered *&p;
        ~Scope() { p = nullptr; }
    } scope{geo_filtered};
    geo_filtered = &gf;
    rc = search_batch_filtered(b, r);
    if (r->filter_error_leaf && !gf.error_leaf.empty())
        for (uint32_t q = 0; q < b->n_queries; q++) r->filter_error_leaf[q] = gf.status[q] ? gf.error_leaf[q] : -1;
    return rc;
}

int Engine::search_batch_filtered(const b200_query_batch *b, b200_results *r) {
    if (b->mode == 0) {
        int rc = keyword_batch(b, r, b->offset, b->limit, b->scoring_strategy);
        if (rc != B200_OK || !b->facet_search_fid) return rc;
        // each query's candidates, copied on the device where the search handed them over (KeywordBatch::setup_facet_search)
        std::vector<const unsigned long long *> dcand(b->n_queries, nullptr);
        for (uint32_t q = 0; q < b->n_queries; q++)
            if (q < fs_slot.size() && fs_slot[q] >= 0) dcand[q] = d_fs_qcand.p + (size_t)fs_slot[q] * hix.n_words64;
        return search_facet_search(b, r, dcand);
    }
    if (b->has_ranking_score_threshold || b->time_budget_ns || b->stop_after >= 0 || r->candidates)
        return fail(B200_ERR_UNSUPPORTED, "ranking-score threshold, deadlines and the candidates bitmap are implemented for keyword searches (mode 0) only");
    if (b->mode == 1) {
        int rc1 = semantic_batch(b, r, b->offset, b->limit);
        fold_vector_stats();
        // Sort rules in a semantic search (get_ranking_rules_for_vector, search/new/mod.rs:419-508: Asc/Desc criteria and the `sort`
        // list) are not built: such queries are refused one by one rather than answered in plain vector order.  A `sort` list while
        // the criteria lack `sort` is SortRankingRuleMissing (check_sort_criteria, :998-1016), as in keyword searches.
        if (rc1 == B200_OK)
            for (uint32_t q = 0; q < b->n_queries; q++) {
                if (geo_filtered && geo_filtered->status[q]) {  // a bad geo clause (the vector stage skipped the query)
                    last_error = geo_filtered->error[q];
                    r->n_hits[q] = 0;
                    if (r->status) r->status[q] = geo_filtered->status[q];
                    if (r->n_candidates) r->n_candidates[q] = 0;
                    continue;
                }
                if (b->facet_begin && b->facet_begin[q + 1] > b->facet_begin[q]) {
                    last_error = "facets in a semantic or hybrid search (use b200_facet_distribution_batch over its candidates)";
                    r->n_hits[q] = 0;
                    if (r->status) r->status[q] = B200_ERR_UNSUPPORTED;
                    if (r->n_candidates) r->n_candidates[q] = 0;
                    continue;
                }
                std::vector<SortRule> unused;
                const char *why = nullptr;
                const int code = sort_rules(b, q, true, false, unused, why);
                if (!code) continue;
                last_error = why;
                r->n_hits[q] = 0;
                if (r->status) r->status[q] = code;
                if (r->n_candidates) r->n_candidates[q] = 0;
            }
        if (rc1 == B200_OK && b->facet_search_fid) {  // execute_for_candidates: the filtered universe (search/mod.rs:254-278)
            std::vector<const unsigned long long *> dcand;
            rc1 = filtered_universes(b, dcand);
            if (rc1 == B200_OK) rc1 = search_facet_search(b, r, dcand);
        }
        return rc1;
    }
    if (b->mode != 2) return fail(B200_ERR_INVALID, "unknown search mode");
    const uint32_t NQ = b->n_queries, L = b->limit + b->offset, lim = std::max(1u, L);
    struct Side {
        std::vector<uint32_t> docids, n_hits, rank, maxr;
        std::vector<uint8_t> n_scores, kind;
        std::vector<float> sim;
        std::vector<uint64_t> n_cand;
        std::vector<int32_t> status;
        std::vector<uint8_t> neg;
        b200_results view;
        Side(uint32_t nq, uint32_t l)
            : docids((size_t)nq * l), n_hits(nq), rank((size_t)nq * l * B200_MAX_SCORES), maxr((size_t)nq * l * B200_MAX_SCORES),
              n_scores((size_t)nq * l), kind((size_t)nq * l * B200_MAX_SCORES), sim((size_t)nq * l * B200_MAX_SCORES), n_cand(nq), status(nq), neg(nq) {
            view = b200_results{docids.data(), n_hits.data(), n_scores.data(), kind.data(), rank.data(), maxr.data(), sim.data(), n_cand.data(), nullptr, status.data(),
                                nullptr, neg.data(), nullptr, 0};
        }
    };
    Side kw(NQ, lim), vec(NQ, lim);
    // the vector stage runs beside the keyword stage: its own host thread, stream and timers (the two share nothing mutable)
    bool have_vec = b->vectors != nullptr;
    int rc_vec = B200_OK;
    // It starts once the keyword stage has derived its terms (kw_derived counts the derivation waves done; B200_VEC_START picks the
    // wave, 0 = at once): the term sweep is a short, SM-filling kernel that the persistent GEMM would otherwise hold up for its whole
    // run time, while the step loop that follows leaves part of the GPU idle.
    // B200_HYBRID_SERIAL=1 runs the two stages one after the other (bench.py's device-time pass: kernel intervals must not overlap).
    std::thread sem;
    const bool serial = getenv("B200_HYBRID_SERIAL") != nullptr;
    const int vec_start = getenv("B200_VEC_START") ? atoi(getenv("B200_VEC_START")) : VEC_START_DEFAULT;
    kw_derived.store(0);
    if (have_vec && !serial)
        sem = std::thread([&]() {
            while (kw_derived.load(std::memory_order_acquire) < vec_start) std::this_thread::yield();
            rc_vec = semantic_batch(b, &vec.view, 0, lim);
        });
    int rc = keyword_batch(b, &kw.view, 0, lim, 1);
    kw_derived.store(KW_DERIVED_ALL, std::memory_order_release);  // (also when the keyword stage returned early)
    if (sem.joinable()) sem.join();
    if (have_vec && serial) rc_vec = semantic_batch(b, &vec.view, 0, lim);
    fold_vector_stats();
    if (rc != B200_OK) return rc;
    if (rc_vec != B200_OK) return rc_vec;
    float kr = 1.0f - b->semantic_ratio, vr = b->semantic_ratio;
    auto load = [&](const Side &s, uint32_t q, uint32_t i) {
        Hit h;
        size_t at = (size_t)q * lim + i;
        h.doc = s.docids[at];
        h.n_scores = s.n_scores[at];
        for (int k = 0; k < h.n_scores; k++) {
            h.kind[k] = s.kind[at * B200_MAX_SCORES + k];
            h.rank[k] = s.rank[at * B200_MAX_SCORES + k];
            h.maxr[k] = s.maxr[at * B200_MAX_SCORES + k];
            h.sim[k] = s.sim[at * B200_MAX_SCORES + k];
        }
        fill_values(h);
        return h;
    };
    auto merge_one = [&](size_t qi) {
        const uint32_t q = (uint32_t)qi;
        if (r->status) r->status[q] = kw.status[q];
        if (r->degraded) r->degraded[q] = 0;
        if (r->used_negative_operator) r->used_negative_operator[q] = kw.neg[q];
        if (kw.status[q] != 0) {
            r->n_hits[q] = 0;
            return;
        }
        std::vector<Hit> K, V;
        for (uint32_t i = 0; i < kw.n_hits[q]; i++) K.push_back(load(kw, q, i));
        // results_good_enough (:368-386)
        bool good = K.size() >= L;
        if (good)
            for (auto &h : K)
                if (global_score(h) * (double)kr < 0.45) {
                    good = false;
                    break;
                }
        std::vector<const Hit *> merged;
        uint32_t sem = 0;
        bool semantic_used = false;
        if (good || !have_vec) {
            for (auto &h : K) merged.push_back(&h);
            if (merged.size() > b->offset)
                merged.erase(merged.begin(), merged.begin() + b->offset);
            else
                merged.clear();
            if (merged.size() > b->limit) merged.resize(b->limit);
        } else {
            semantic_used = true;
            for (uint32_t i = 0; i < vec.n_hits[q]; i++) V.push_back(load(vec, q, i));
            size_t vi = 0, ki = 0, skipped = 0;
            std::vector<uint32_t> seen;
            while ((vi < V.size() || ki < K.size()) && merged.size() < b->limit) {
                bool take_vec = vi >= V.size() ? false : (ki >= K.size() ? true : compare_scores(V[vi], vr, K[ki], kr) >= 0);
                const Hit *h = take_vec ? &V[vi++] : &K[ki++];
                if (std::find(seen.begin(), seen.end(), h->doc) != seen.end()) continue;
                seen.push_back(h->doc);
                if (skipped < b->offset) {
                    skipped++;
                    continue;
                }
                if (take_vec) sem++;
                merged.push_back(h);
            }
        }
        r->n_hits[q] = (uint32_t)merged.size();
        if (r->semantic_hits) r->semantic_hits[q] = semantic_used ? sem : 0;
        if (r->n_candidates) r->n_candidates[q] = semantic_used ? std::max<uint64_t>(kw.n_cand[q], vec.n_cand[q]) : kw.n_cand[q];
        for (size_t i = 0; i < merged.size(); i++) {
            size_t at = (size_t)q * b->limit + i;
            const Hit &h = *merged[i];
            r->docids[at] = h.doc;
            if (r->n_scores) {
                r->n_scores[at] = h.n_scores;
                for (int k = 0; k < h.n_scores; k++) {
                    r->score_kind[at * B200_MAX_SCORES + k] = h.kind[k];
                    r->score_rank[at * B200_MAX_SCORES + k] = h.rank[k];
                    r->score_max[at * B200_MAX_SCORES + k] = h.maxr[k];
                    r->score_sim[at * B200_MAX_SCORES + k] = h.sim[k];
                }
            }
        }
    };
    // the merges of different queries are independent: spread them over the worker pool
    if (pool)
        pool->run(NQ, merge_one);
    else
        for (uint32_t q = 0; q < NQ; q++) merge_one(q);
    if (b->facet_search_fid) {  // execute_for_candidates: a hybrid search's candidates are its filtered universe (search/mod.rs:254-278)
        std::vector<const unsigned long long *> dcand;
        rc = filtered_universes(b, dcand);
        if (rc == B200_OK) rc = search_facet_search(b, r, dcand);
        return rc;
    }
    return B200_OK;
}

}  // namespace b200
