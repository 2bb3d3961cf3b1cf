// Facet search (facet_search.cu) for b200_facet_search_batch: request validation, the query's automaton choice, chunking by scratch,
// and the decoding of the kept hits, including the replay of the reference's count-ordered heap over the hits at the cut count.
#include <algorithm>
#include <cstring>
#include <map>

#include "engine.h"
#include "kernels.h"

namespace b200 {

#define CU(call, what)                                     \
    do {                                                   \
        cudaError_t e_ = (call);                           \
        if (e_ != cudaSuccess) return cuda_fail(e_, what); \
    } while (0)

namespace {

struct Hit {
    uint64_t count;
    const std::string *value;
    uint32_t key;
};
// FacetValueHit's Ord: count, then the value's bytes (search.rs:276-286)
bool hit_less(const Hit &a, const Hit &b) { return a.count != b.count ? a.count < b.count : *a.value < *b.value; }

}  // namespace

int Engine::facet_search_batch(uint32_t n, const uint64_t *const *candidates, uint64_t n_words, const uint16_t *fid, const uint8_t *kind,
                               const uint32_t *off, const char *query_bytes, const uint8_t *flags, uint32_t max, uint32_t cap, uint32_t *n_out,
                               uint32_t *key, uint64_t *count, uint32_t *docid, uint8_t *fallback, int32_t *status) {
    if (!n) return B200_OK;
    if (!candidates || !fid || !kind || !off || !flags || !n_out || !status || (cap && (!key || !count || !docid || !fallback)))
        return fail(B200_ERR_INVALID, "facet_search_batch: null candidates / fid / kind / off / flags / output array");
    const uint64_t W = hix.n_words64;
    if (n_words < W) return fail(B200_ERR_INVALID, "facet_search_batch: n_words smaller than the document range");
    CU(cudaSetDevice(device), "cudaSetDevice");
    // the distinct host candidate bitmaps, uploaded once each
    std::map<const uint64_t *, uint32_t> at;
    for (uint32_t i = 0; i < n; i++)
        if (candidates[i]) at.emplace(candidates[i], 0);
    uint32_t n_bitmaps = 0;
    for (auto &kv : at) kv.second = n_bitmaps++;
    if (d_fs_cand.reserve(std::max<size_t>(1, (size_t)n_bitmaps * W)) != cudaSuccess) {
        cudaGetLastError();
        return fail(B200_ERR_CAPACITY, "facet_search_batch: the candidate bitmaps do not fit in device memory");
    }
    for (auto &kv : at) {
        CU(cudaMemcpyAsync(d_fs_cand.p + (size_t)kv.second * W, kv.first, W * 8, cudaMemcpyHostToDevice, stream), "H2D facet search candidates");
        stats.h2d_bytes += W * 8;
    }
    std::vector<const unsigned long long *> dcand(n, nullptr);
    for (uint32_t i = 0; i < n; i++) {
        if (candidates[i]) dcand[i] = d_fs_cand.p + (size_t)at[candidates[i]] * W;
        status[i] = B200_OK;
    }
    return facet_search_run(n, dcand.data(), fid, kind, off, query_bytes, flags, max, cap, n_out, key, count, docid, fallback, status);
}

int Engine::facet_search_run(uint32_t n, const unsigned long long *const *dcand, const uint16_t *fid, const uint8_t *kind, const uint32_t *off,
                             const char *query_bytes, const uint8_t *flags, uint32_t max, uint32_t cap, uint32_t *n_out, uint32_t *key,
                             uint64_t *count, uint32_t *docid, uint8_t *fallback, int32_t *status) {
    const uint64_t W = hix.n_words64;
    const FacetSearchIndex &fs = hix.fsearch;
    const Settings &set = hix.settings;
    // the requests that run, each with its query's chars
    std::vector<FsReq> reqs;
    std::vector<uint32_t> req_of, q_chars, qc;
    std::vector<std::string> queries(n);
    std::vector<size_t> scratch_of;
    for (uint32_t i = 0; i < n; i++) {
        n_out[i] = 0;
        if (status[i] != B200_OK || fid[i] == 0xFFFF) continue;
        if (kind[i] > 1 || (kind[i] == 1 && (!off || off[i + 1] < off[i] || (off[i + 1] > off[i] && !query_bytes)))) {
            status[i] = B200_ERR_INVALID;
            last_error = "facet search: kind is not 0 (no query) or 1 (a query), or its query bytes are missing or not ascending";
            continue;
        }
        FsReq r{};
        if (kind[i] == 1) {
            queries[i].assign(query_bytes ? query_bytes + off[i] : "", off[i + 1] - off[i]);
            if (!utf8_decode((const uint8_t *)queries[i].data(), queries[i].size(), qc)) {
                status[i] = B200_ERR_INVALID;
                last_error = "facet search: the query is not valid UTF-8";
                continue;
            }
        }
        auto f = fs.fields.find(fid[i]);
        if (max == 0 || f == fs.fields.end()) continue;  // nothing to answer (no FST for the field), whatever the query
        if (kind[i] == 1 && qc.size() > FS_MAX_Q) {
            status[i] = B200_ERR_UNSUPPORTED;
            last_error = "facet search: a query longer than " + std::to_string(FS_MAX_Q) + " characters";
            continue;
        }
        r.cand = dcand[i] ? dcand[i] : dix.base_ub;
        r.max = max;
        r.list_base = f->second.list0 - f->second.k0;
        r.by_count = flags[i] & 1;
        r.k0 = f->second.k0;
        r.n_str = f->second.n_str;
        r.h0 = f->second.h0;
        r.h1 = f->second.h1;
        if (kind[i] == 0) {
            r.mode = FS_ALL;
        } else {
            r.q_off = (uint32_t)q_chars.size();
            r.q_len = (uint32_t)qc.size();
            q_chars.insert(q_chars.end(), qc.begin(), qc.end());
            const size_t len = queries[i].size();  // search.rs:147-186: the typo budget follows the byte length
            if ((flags[i] & 2) && set.authorize_typos) {
                if (set.exact_words.count(queries[i])) {
                    r.mode = FS_EXACT;
                } else {
                    r.mode = FS_PREFIX;
                    r.k = len < set.one_typo ? 0 : len < set.two_typos ? 1 : 2;
                }
            } else {
                r.mode = FS_PREFIX;
                r.k = 0;
            }
        }
        const size_t items = r.mode == FS_ALL ? r.n_str : f->second.n_entries;
        if (!items) continue;
        reqs.push_back(r);
        req_of.push_back(i);
        scratch_of.push_back(items);
    }
    if (reqs.empty()) return B200_OK;
    const FsTables tab{d_fs_chars, d_fs_char_off, d_fs_csr_off, d_fs_csr_key, dix.pool, dix.lists};
    // chunks of requests whose scratch (items, counts, packed keys and counts: 16 bytes per walked key) fits in 256 MB
    const size_t budget = (size_t)64 << 20;  // u32 entries
    std::vector<uint32_t> sums, okey, ocnt;
    std::vector<Hit> heap, hits;
    for (size_t j0 = 0; j0 < reqs.size();) {
        size_t j1 = j0, entries = 0, largest = 0;
        while (j1 < reqs.size() && j1 - j0 < 65535 && (j1 == j0 || entries + scratch_of[j1] <= budget / 4)) {
            entries += scratch_of[j1];
            largest = std::max(largest, scratch_of[j1]);
            j1++;
        }
        const uint32_t nr = (uint32_t)(j1 - j0);
        const size_t q_words = std::max<size_t>(1, q_chars.size());
        if (d_fs_u32.reserve(entries * 4 + (size_t)nr * 4 + 1 + q_words) != cudaSuccess || d_fs_reqs.reserve(nr) != cudaSuccess) {
            cudaGetLastError();
            return fail(B200_ERR_CAPACITY, "facet_search_batch: the scratch of a request (16 bytes per key it walks) does not fit in device memory");
        }
        uint32_t *items = d_fs_u32.p, *cnts = items + entries, *out_key = cnts + entries, *out_cnt = out_key + entries,
                 *d_sums = out_cnt + entries, *cursor = d_sums + (size_t)nr * 4, *d_q = cursor + 1;
        size_t used = 0;
        uint64_t bytes = 0;
        for (size_t j = j0; j < j1; j++) {
            reqs[j].items = items + used;
            reqs[j].cnt = cnts + used;
            reqs[j].sum = d_sums + (j - j0) * 4;
            used += scratch_of[j];
            // algorithmic bytes: the swept strings' offsets and chars (the walked keys' items and counts are added below, once known)
            bytes += reqs[j].mode == FS_ALL ? 0 : (uint64_t)(reqs[j].h1 - reqs[j].h0) * 8;
        }
        CU(cudaMemcpyAsync(d_fs_reqs.p, reqs.data() + j0, nr * sizeof(FsReq), cudaMemcpyHostToDevice, stream), "H2D facet search requests");
        if (!q_chars.empty())
            CU(cudaMemcpyAsync(d_q, q_chars.data(), q_chars.size() * 4, cudaMemcpyHostToDevice, stream), "H2D facet search queries");
        CU(cudaMemsetAsync(cursor, 0, 4, stream), "zero facet search cursor");
        stats.h2d_bytes += nr * sizeof(FsReq) + q_chars.size() * 4;
        const size_t m0 = mark();
        CU(launch_facet_search_match(stream, tab, d_fs_reqs.p, nr, d_q), "facet search match");
        CU(launch_facet_search_count(stream, tab, d_fs_reqs.p, nr, (uint32_t)largest, (uint32_t)W), "facet search count");
        CU(launch_facet_search_select(stream, d_fs_reqs.p, nr, out_key, out_cnt, cursor), "facet search select");
        const size_t m1 = mark();
        time_kernel(B200_K_FACET_SEARCH, m0, m1, bytes);
        stats.kernel_launches += 2;
        stats.kernel_count[B200_K_FACET_SEARCH] += 2;
        sums.resize((size_t)nr * 4 + 1);
        CU(cudaMemcpyAsync(sums.data(), d_sums, sums.size() * 4, cudaMemcpyDeviceToHost, stream), "D2H facet search sums");
        CU(cudaStreamSynchronize(stream), "sync facet search");
        const uint32_t packed = sums[(size_t)nr * 4];
        for (uint32_t j = 0; j < nr; j++) stats.kernel_bytes[B200_K_FACET_SEARCH] += (uint64_t)sums[(size_t)j * 4] * 16;  // items, counts
        okey.resize(packed);
        ocnt.resize(packed);
        if (packed) {
            CU(cudaMemcpyAsync(okey.data(), out_key, packed * 4, cudaMemcpyDeviceToHost, stream), "D2H facet search hits");
            CU(cudaMemcpyAsync(ocnt.data(), out_cnt, packed * 4, cudaMemcpyDeviceToHost, stream), "D2H facet search hits");
            CU(cudaStreamSynchronize(stream), "sync facet search");
        }
        stats.d2h_bytes += sums.size() * 4 + (size_t)packed * 8;
        resolve_timers();
        for (size_t j = j0; j < j1; j++) {
            const uint32_t i = req_of[j];
            const uint32_t *s = sums.data() + (j - j0) * 4;
            const FsReq &r = reqs[j];
            hits.clear();
            for (uint32_t e = 0; e < s[1]; e++) {
                const uint32_t k = okey[s[3] + e];
                const std::string *value = fs.has_orig[k] ? &fs.orig[k] : kind[i] == 1 ? &queries[i] : &fs.key[k];
                hits.push_back(Hit{ocnt[s[3] + e], value, k});
            }
            if (r.by_count) {
                // ValuesCollection::Count (search.rs:292-353): a min-heap of at most `max` hits; once full, the smallest hit is
                // replaced by any hit whose count is at least its count.  The device kept every hit at or above the cut count; the
                // ones below it can never be in the final heap, and leaving them out does not change which others are evicted
                // (DESIGN.md §3).
                heap.clear();
                auto greater = [](const Hit &a, const Hit &b) { return hit_less(b, a); };
                for (const Hit &h : hits) {
                    if (heap.size() < max) {
                        heap.push_back(h);
                        std::push_heap(heap.begin(), heap.end(), greater);
                    } else if (heap.front().count <= h.count) {
                        std::pop_heap(heap.begin(), heap.end(), greater);
                        heap.back() = h;
                        std::push_heap(heap.begin(), heap.end(), greater);
                    }
                }
                std::sort(heap.begin(), heap.end(), greater);  // descending (count, value)
                hits.swap(heap);
            }
            if (hits.size() > cap) {
                status[i] = B200_ERR_CAPACITY;
                last_error = "facet search: cap " + std::to_string(cap) + " is too small: the request has " + std::to_string(hits.size()) + " hits";
                continue;
            }
            n_out[i] = (uint32_t)hits.size();
            for (size_t e = 0; e < hits.size(); e++) {
                const size_t o = (size_t)i * cap + e;
                key[o] = hits[e].key;
                count[o] = hits[e].count;
                docid[o] = fs.min_doc[hits[e].key];
                fallback[o] = fs.has_orig[hits[e].key] ? 0 : 1;
            }
        }
        j0 = j1;
    }
    return B200_OK;
}

}  // namespace b200

namespace b200 {

int Engine::search_facet_search(const b200_query_batch *b, b200_results *r, const std::vector<const unsigned long long *> &dcand) {
    const uint32_t NQ = b->n_queries;
    if (!b->facet_search_fid || !NQ) return B200_OK;
    const uint16_t *fid = b->facet_search_fid;
    const bool outputs = b->facet_query_kind && b->facet_search_flags && r->fs_n && r->fs_key && r->fs_count && r->fs_docid && r->fs_fallback;
    const int32_t SKIP = 1;  // not a B200_ERR_*: no facet search for the query, or its search already failed
    auto fail_query = [&](uint32_t q, int32_t code, const std::string &why) {
        last_error = why;
        r->n_hits[q] = 0;
        if (r->status) r->status[q] = code;
        if (r->n_candidates) r->n_candidates[q] = 0;
    };
    std::vector<int32_t> st(NQ, SKIP);
    bool any = false;
    for (uint32_t q = 0; q < NQ; q++) {
        if (r->fs_n) r->fs_n[q] = 0;
        if (fid[q] == 0xFFFF || (r->status && r->status[q] != B200_OK)) continue;
        if (!outputs)
            fail_query(q, B200_ERR_INVALID, "facet_search_fid without facet_query_kind, facet_search_flags or the fs_* outputs");
        else if (b->has_ranking_score_threshold)
            fail_query(q, B200_ERR_UNSUPPORTED, "a facet search together with a ranking-score threshold");
        else {
            st[q] = B200_OK;
            any = true;
        }
    }
    if (!any) return B200_OK;
    const int rc = facet_search_run(NQ, dcand.data(), fid, b->facet_query_kind, b->facet_query_off, b->facet_query_bytes, b->facet_search_flags,
                                    b->facet_search_max, b->facet_search_max, r->fs_n, r->fs_key, r->fs_count, r->fs_docid, r->fs_fallback,
                                    st.data());
    if (rc != B200_OK) return rc;
    const std::string why = last_error;
    for (uint32_t q = 0; q < NQ; q++)
        if (st[q] != B200_OK && st[q] != SKIP) fail_query(q, st[q], why);
    return B200_OK;
}

int Engine::filtered_universes(const b200_query_batch *b, std::vector<const unsigned long long *> &dcand) {
    const uint32_t NQ = b->n_queries;
    const uint64_t W = hix.n_words64;
    dcand.assign(NQ, nullptr);
    std::map<const uint64_t *, uint32_t> at;
    for (uint32_t q = 0; q < NQ; q++) {
        if (geo_filtered && geo_filtered->d_univ[q]) {
            dcand[q] = geo_filtered->d_univ[q];  // documents_ids AND universes[q] AND the geo clauses, already on the device
        } else if (b->universes && b->universes[q] && b->facet_search_fid[q] != 0xFFFF) {
            if (b->n_universe_words < W) return fail(B200_ERR_INVALID, "universe bitmaps shorter than the document range");
            at.emplace(b->universes[q], 0);
        }
    }
    if (at.empty()) return B200_OK;
    uint32_t n = 0;
    for (auto &kv : at) kv.second = n++;
    if (d_fs_cand.reserve((size_t)n * W) != cudaSuccess) {
        cudaGetLastError();
        return fail(B200_ERR_CAPACITY, "facet search: the filtered universes do not fit in device memory");
    }
    std::vector<unsigned long long> tmp(W);
    for (auto &kv : at) {
        for (uint64_t w = 0; w < W; w++) tmp[w] = kv.first[w] & hix.base_ub[w];  // filtered_universe: documents_ids & filter
        CU(cudaMemcpy(d_fs_cand.p + (size_t)kv.second * W, tmp.data(), W * 8, cudaMemcpyHostToDevice), "H2D facet search universes");
        stats.h2d_bytes += W * 8;
    }
    for (uint32_t q = 0; q < NQ; q++)
        if (!dcand[q] && b->universes && b->universes[q] && at.count(b->universes[q])) dcand[q] = d_fs_cand.p + (size_t)at[b->universes[q]] * W;
    return B200_OK;
}

}  // namespace b200
