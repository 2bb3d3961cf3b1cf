// Staging to HBM, term derivation (S3) and the vector store (S4).
#include <cuda_fp16.h>
#include <dlfcn.h>

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>

#include "engine.h"
#include "kernels.h"

namespace b200 {

void HostAffinity::detect(int device) {
    valid = false;
    if (const char *env = getenv("B200_PIN"))
        if (atoi(env) == 0) return;
    char bus[32] = {};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) return;
    for (char *c = bus; *c; c++) *c = (char)tolower((unsigned char)*c);
    int node = -1;
    {
        std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
        FILE *f = fopen(path.c_str(), "r");
        if (!f) return;
        if (fscanf(f, "%d", &node) != 1) node = -1;
        fclose(f);
    }
    if (node < 0) return;
    char list[4096] = {};
    {
        std::string path = "/sys/devices/system/node/node" + std::to_string(node) + "/cpulist";
        FILE *f = fopen(path.c_str(), "r");
        if (!f) return;
        if (!fgets(list, sizeof list, f)) list[0] = 0;
        fclose(f);
    }
    cpu_set_t allowed, want;
    if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return;
    CPU_ZERO(&want);
    int n = 0, n_allowed = CPU_COUNT(&allowed);
    for (const char *c = list; *c;) {  // "0-31,64-95"
        if (*c < '0' || *c > '9') {
            c++;
            continue;
        }
        char *end;
        long a = strtol(c, &end, 10), b2 = a;
        if (*end == '-') b2 = strtol(end + 1, &end, 10);
        for (long k = a; k <= b2 && k < CPU_SETSIZE; k++)
            if (CPU_ISSET((int)k, &allowed)) {
                CPU_SET((int)k, &want);
                n++;
            }
        c = end;
    }
    if (n < 4 || n == n_allowed) return;  // nothing to narrow, or too little left to work with
    cpus = want;
    valid = true;
}


#define CU(call, what)                         \
    do {                                       \
        cudaError_t e_ = (call);               \
        if (e_ != cudaSuccess) return cuda_fail(e_, what); \
    } while (0)

template <class T>
static cudaError_t upload(T **dst, const T *src, size_t n) {
    *dst = nullptr;
    if (n == 0) n = 1;
    cudaError_t e = cudaMalloc((void **)dst, n * sizeof(T));
    if (e != cudaSuccess) return e;
    if (src) return cudaMemcpy(*dst, src, n * sizeof(T), cudaMemcpyHostToDevice);
    return cudaMemset(*dst, 0, n * sizeof(T));
}

Engine::~Engine() {
    for (auto &t : reapers)
        if (t.joinable()) t.join();
    reapers.clear();
    cudaSetDevice(device);
    for (void *p : {(void *)dix.dict_bytes, (void *)dix.dict_off, (void *)dix.pool, (void *)dix.lists, (void *)dix.pair_keys, (void *)dix.base_ub,
                    (void *)dix.emb, (void *)dix.emb_inv_norm, (void *)dix.emb_docids, (void *)arena, (void *)scratch})
        if (p) cudaFree(p);
    for (auto &kv : hix.sort_fields)
        for (auto p : {kv.second.d_key[0], kv.second.d_key[1], kv.second.d_doc_off, kv.second.d_doc_ord, kv.second.d_disp})
            if (p) cudaFree(p);
    for (auto p : {d_fs_chars, d_fs_char_off, d_fs_csr_off, d_fs_csr_key})
        if (p) cudaFree(p);
    d_fs_reqs.release();
    d_fs_u32.release();
    d_fs_cand.release();
    d_fs_qcand.release();
    d_facet_scratch.release();
    d_facet_slots.release();
    d_facet_out.release();
    d_facet_cand.release();
    if (d_geo_pts) cudaFree(d_geo_pts);
    if (d_geo_ub) cudaFree(d_geo_ub);
    d_geo_count.release();
    d_geo_desc.release();
    d_geo_u32.release();
    d_geo_patch.release();
    d_geo_key.release();
    d_gf_clause.release();
    d_gf_first.release();
    d_gf_amb.release();
    d_gf_u32.release();
    d_gf_slot.release();
    d_gf_count.release();
    d_gf_caller.release();
    d_gf_univ.release();
    for (auto &m : d_presence)
        for (auto &kv : m) cudaFree(kv.second);
    d_ft_op.release();
    d_ft_iv.release();
    d_ft_slot.release();
    d_ft_flag.release();
    d_ft_count.release();
    d_ft_caller.release();
    d_ft_univ.release();
    d_ft_geo.release();
    for (auto &ln : lanes) ln.release();
    d_docids_out.release();
    d_sort_desc.release();
    d_sort_keys.release();
    d_sort_info.release();
    d_lev_terms.release();
    d_lev_recs.release();
    d_lev_items.release();
    d_lev_perm.release();
    d_lev_u32.release();
    d_vq.release();
    d_vdist.release();
    d_vsel_dist.release();
    d_vsel_ids.release();
    d_vsel_n.release();
    d_cand.release();
    for (auto e : ev_pool) cudaEventDestroy(e);
    if (sc.comm && sc.comm_destroy) sc.comm_destroy(sc.comm);
    d_gather_ids.release();
    d_gather_dist.release();
    d_gather_n.release();
    for (auto e : vt.ev_pool) cudaEventDestroy(e);
    if (vt.stream) cudaStreamDestroy(vt.stream);
    if (stream) cudaStreamDestroy(stream);
}

size_t Engine::mark() {
    if (ev_used == ev_pool.size()) {
        cudaEvent_t e;
        cudaEventCreate(&e);
        ev_pool.push_back(e);
    }
    cudaEventRecord(ev_pool[ev_used], stream);
    return ev_used++;
}
void Engine::resolve_timers() {
    for (auto &t : timed) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, ev_pool[t.a], ev_pool[t.b]) == cudaSuccess) stats.kernel_ms[t.cls] += ms;
    }
    timed.clear();
    ev_used = 0;
}

// HostIndex::first_lo / pair_lo.  Term derivation scans the word ranges they delimit, which only holds the words of a prefix
// when the dictionary is bytewise ascending (FST order), so anything else is refused here.
static void build_prefix_tables(HostIndex &ix) {
    if (ix.n_words >= (1ull << 32)) throw std::runtime_error("dictionary: more than 2^32 - 1 words");
    for (uint64_t i = 1; i < ix.n_words; i++)
        if (ix.cmp_word(i - 1, ix.word_ptr(i), ix.word_len(i)) >= 0)
            throw std::runtime_error("dictionary: words are not in strictly ascending bytewise order at word " + std::to_string(i));
    ix.first_lo.resize(257);
    ix.pair_lo.resize(65537);
    for (uint32_t c = 0; c < 256; c++) {
        const uint8_t k[1] = {(uint8_t)c};
        ix.first_lo[c] = (uint32_t)ix.lower_bound(k, 1);
    }
    ix.first_lo[256] = (uint32_t)ix.n_words;
    for (uint32_t p = 0; p < 65536; p++) {
        const uint8_t k[2] = {(uint8_t)(p >> 8), (uint8_t)p};
        ix.pair_lo[p] = (uint32_t)ix.lower_bound(k, 2);
    }
    ix.pair_lo[65536] = (uint32_t)ix.n_words;
}

int Engine::stage_finish() {
    CU(cudaSetDevice(device), "cudaSetDevice");
    try {
        build_host_index(raw_dict_bytes, raw_dict_off, raw_dbs, raw_docids, hix);
        build_prefix_tables(hix);
        build_sort_fields(raw_dbs[B200_DB_FACET_ID_F64_DOCIDS], raw_dbs[B200_DB_FACET_ID_STRING_DOCIDS], hix);
        build_geo_field(raw_dbs[B200_DB_FACET_ID_F64_DOCIDS], raw_dbs[B200_DB_FACET_ID_STRING_DOCIDS], hix);
        build_facet_search(raw_dbs[B200_DB_FACET_ID_STRING_DOCIDS], raw_dbs[B200_DB_FACET_ID_NORMALIZED_STRING_STRINGS],
                           raw_dbs[B200_DB_FIELD_ID_DOCID_FACET_STRINGS], hix);
        for (int p = 0; p < 3; p++) build_presence(raw_dbs[B200_DB_FACET_ID_EXISTS_DOCIDS + p], p, hix);
    } catch (const std::exception &e) {
        return fail(B200_ERR_INVALID, e.what());
    }
    Settings keep = hix.settings;
    (void)keep;
    // dictionary
    std::vector<uint32_t> off32(hix.dict_off.size());
    for (size_t i = 0; i < off32.size(); i++) off32[i] = (uint32_t)hix.dict_off[i];
    if (off32.empty()) off32.push_back(0);
    CU(upload(&dix.dict_bytes, hix.dict_bytes.data(), hix.dict_bytes.size()), "upload dictionary");
    CU(upload(&dix.dict_off, off32.data(), off32.size()), "upload dictionary offsets");
    // posting store
    CU(upload(&dix.pool, hix.pool.data(), hix.pool.size()), "upload posting pool");
    static_assert(sizeof(ListRef) == sizeof(DListRef), "ListRef layout");
    CU(upload(&dix.lists, reinterpret_cast<const DListRef *>(hix.lists.data()), hix.lists.size()), "upload list table");
    CU(upload(&dix.pair_keys, reinterpret_cast<const unsigned long long *>(hix.pair_keys.data()), hix.pair_keys.size()), "upload pair keys");
    CU(upload(&dix.base_ub, reinterpret_cast<const unsigned long long *>(hix.base_ub.data()), hix.base_ub.size()), "upload universe");
    stats.hbm_bytes_staged = hix.dict_bytes.size() + off32.size() * 4 + hix.pool.size() * 4 + hix.lists.size() * sizeof(ListRef) +
                             hix.pair_keys.size() * 8 + hix.base_ub.size() * 8;
    std::vector<uint32_t>().swap(hix.pool);
    // Sort keys: two u32[n_docs] per faceted field (ascending, descending)
    for (auto &kv : hix.sort_fields)
        for (int dir = 0; dir < 2; dir++) {
            std::vector<uint32_t> &k = kv.second.key[dir];
            CU(upload(&kv.second.d_key[dir], k.data(), k.size()), "upload sort keys");
            stats.hbm_bytes_staged += k.size() * 4;
            std::vector<uint32_t>().swap(k);
        }
    // facet distribution: per faceted field its document-major ordinals and the Display order of its numbers
    for (auto &kv : hix.sort_fields) {
        SortField &f = kv.second;
        auto src = [](const std::vector<uint32_t> &v) { return v.empty() ? nullptr : v.data(); };  // upload() allocates one element for none
        CU(upload(&f.d_doc_off, src(f.doc_off), f.doc_off.size()), "upload facet ordinals");
        CU(upload(&f.d_doc_ord, src(f.doc_ord), f.doc_ord.size()), "upload facet ordinals");
        CU(upload(&f.d_disp, src(f.disp), f.disp.size()), "upload facet display order");
        stats.hbm_bytes_staged += (f.doc_off.size() + f.doc_ord.size() + f.disp.size()) * 4;
        f.n_ord = f.doc_ord.size();
        std::vector<uint32_t>().swap(f.doc_off);
        std::vector<uint32_t>().swap(f.doc_ord);
        std::vector<uint32_t>().swap(f.disp);
    }
    // filters: the EXISTS / IS NULL / IS EMPTY bitmaps of every field
    for (int p = 0; p < 3; p++)
        for (auto &kv : hix.presence[p]) {
            CU(upload(&d_presence[p][kv.first], reinterpret_cast<const unsigned long long *>(kv.second.data()), kv.second.size()),
               "upload facet presence");
            stats.hbm_bytes_staged += kv.second.size() * 8;
            std::vector<uint64_t>().swap(kv.second);
        }
    // facet search: the hyper-normalised strings as chars and the keys each one walks (the keys' posting lists are in the pool,
    // counted above)
    {
        FacetSearchIndex &fs = hix.fsearch;
        auto src = [](const std::vector<uint32_t> &v) { return v.empty() ? nullptr : v.data(); };  // upload() allocates one element for none
        CU(upload(&d_fs_chars, src(fs.chars), fs.chars.size()), "upload facet search strings");
        CU(upload(&d_fs_char_off, src(fs.char_off), fs.char_off.size()), "upload facet search strings");
        CU(upload(&d_fs_csr_off, src(fs.csr_off), fs.csr_off.size()), "upload facet search keys");
        CU(upload(&d_fs_csr_key, src(fs.csr_key), fs.csr_key.size()), "upload facet search keys");
        stats.hbm_bytes_staged += (fs.chars.size() + fs.char_off.size() + fs.csr_off.size() + fs.csr_key.size()) * 4;
        std::vector<uint32_t>().swap(fs.chars);
        std::vector<uint32_t>().swap(fs.char_off);
        std::vector<uint32_t>().swap(fs.csr_off);
        std::vector<uint32_t>().swap(fs.csr_key);
    }
    // GeoSort points: lat_lng_to_xyz (lib.rs:397-404) and cos(lat) with the host's libm, as the reference computes them
    {
        GeoField &g = hix.geo;
        std::vector<GeoPoint> pts(hix.n_docs, GeoPoint{0, 0, 0, 0, 0, 0});
        const double to_rad = M_PI / 180.0;
        for (uint32_t d = 0; d < hix.n_docs; d++) {
            if (!(g.ub[d >> 6] >> (d & 63) & 1)) continue;
            const double la = g.lat[d] * to_rad, ln = g.lng[d] * to_rad;
            pts[d] = GeoPoint{std::cos(la) * std::cos(ln), std::cos(la) * std::sin(ln), std::sin(la), g.lat[d], g.lng[d], std::cos(la)};
        }
        CU(upload(&d_geo_pts, pts.data(), pts.size()), "upload geo points");
        CU(upload(&d_geo_ub, reinterpret_cast<const unsigned long long *>(g.ub.data()), g.ub.size()), "upload geo bitmap");
        stats.hbm_bytes_staged += pts.size() * sizeof(GeoPoint) + g.ub.size() * 8;
        // lat / lng stay on the host: the decisions the device leaves ambiguous, and the distances of the GeoSort chain, are taken
        // there with libm (geo_distance_host)
    }
    // release the raw staging copies
    for (auto &db : raw_dbs) {
        std::vector<uint8_t>().swap(db.keys);
        std::vector<uint8_t>().swap(db.vals);
        std::vector<uint64_t>().swap(db.koff);
        std::vector<uint64_t>().swap(db.voff);
    }
    // work pools
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b), "cudaMemGetInfo");
    auto env_mb = [](const char *name, size_t dflt) {
        const char *v = getenv(name);
        return v ? (size_t)atoll(v) << 20 : dflt;
    };
    // a sixth of what is free each (capped; two handles can coexist): about 13 GB each on an 80 GB card, and the rest stays for the
    // embeddings staged afterwards (15.4 GB at 10 M x 768 fp16) and the row lookup tables
    arena_bytes = env_mb("B200_ARENA_MB", std::min<size_t>(free_b / 6, (size_t)32 << 30));
    scratch_bytes = env_mb("B200_SCRATCH_MB", std::min<size_t>(free_b / 6, (size_t)40 << 30));
    CU(cudaMalloc((void **)&arena, arena_bytes), "alloc arena");
    CU(cudaMalloc((void **)&scratch, scratch_bytes), "alloc scratch");
    staged = true;
    return B200_OK;
}

// The vector store: fp16 rows + f32 inverse norms + docids.  f32 input (what arroy/hannoy item nodes hold) is converted on the
// device, chunk by chunk; `half_rows` non-null = the caller already holds IEEE binary16 rows.
int Engine::stage_embeddings(const float *vectors, const uint16_t *half_rows, uint64_t n, uint32_t d, const uint32_t *docids) {
    CU(cudaSetDevice(device), "cudaSetDevice");
    if (d == 0) return fail(B200_ERR_INVALID, "embedding dimension must be positive");
    if (!vectors && !half_rows && n) return fail(B200_ERR_INVALID, "embeddings: null matrix");
    if (d % 8 != 0) {
        // the kernels read rows in 128-bit pieces: pad every row with zeros up to a multiple of 8 (cosine does not change)
        const uint32_t dp = (d + 7) & ~7u;
        std::vector<float> padded((size_t)n * dp, 0.f);
        for (uint64_t r = 0; r < n; r++)
            for (uint32_t i = 0; i < d; i++)
                padded[r * dp + i] = vectors ? vectors[r * d + i] : __half2float(reinterpret_cast<const __half *>(half_rows)[r * d + i]);
        int rc = stage_embeddings(padded.data(), nullptr, n, dp, docids);
        if (rc == B200_OK) emb_d_user = d;
        return rc;
    }
    emb_d_user = d;
    for (void *p : {(void *)dix.emb, (void *)dix.emb_inv_norm, (void *)dix.emb_docids})
        if (p) cudaFree(p);
    dix.emb = nullptr;
    dix.emb_inv_norm = nullptr;
    dix.emb_docids = nullptr;
    dix.emb_n = 0;
    const size_t rows_alloc = std::max<uint64_t>(n, 1);
    CU(cudaMalloc(&dix.emb, rows_alloc * d * 2), "alloc embeddings");
    CU(cudaMalloc((void **)&dix.emb_inv_norm, rows_alloc * 4), "alloc norms");
    CU(cudaMalloc((void **)&dix.emb_docids, rows_alloc * 4), "alloc embedding docids");
    uint8_t *dm = reinterpret_cast<uint8_t *>(dix.emb);
    const uint64_t chunk = std::max<uint64_t>(1, ((uint64_t)256 << 20) / ((uint64_t)d * 4));  // rows per 256 MB of f32
    if (half_rows) {
        for (uint64_t r0 = 0; r0 < n; r0 += chunk * 2) {
            const uint64_t nr = std::min<uint64_t>(chunk * 2, n - r0);
            CU(cudaMemcpyAsync(dm + r0 * d * 2, half_rows + r0 * d, nr * d * 2, cudaMemcpyHostToDevice, stream), "H2D embeddings");
        }
        CU(launch_emb_norm_f16(stream, dix.emb, dix.emb_inv_norm, n, d), "embedding norms");
    } else {
        float *stage = nullptr;
        CU(cudaMalloc((void **)&stage, std::min<uint64_t>(chunk, rows_alloc) * d * 4), "alloc embedding staging");
        for (uint64_t r0 = 0; r0 < n; r0 += chunk) {
            const uint64_t nr = std::min<uint64_t>(chunk, n - r0);
            cudaError_t e = cudaMemcpyAsync(stage, vectors + r0 * d, nr * d * 4, cudaMemcpyHostToDevice, stream);
            if (e == cudaSuccess) e = launch_emb_from_f32(stream, stage, dm + r0 * d * 2, dix.emb_inv_norm + r0, nr, d);
            if (e != cudaSuccess) {
                cudaFree(stage);
                return cuda_fail(e, "convert embeddings");
            }
        }
        cudaStreamSynchronize(stream);
        cudaFree(stage);
    }
    if (docids)
        CU(cudaMemcpyAsync(dix.emb_docids, docids, n * 4, cudaMemcpyHostToDevice, stream), "H2D embedding docids");
    else {
        std::vector<uint32_t> ids(n);
        for (uint64_t r = 0; r < n; r++) ids[r] = (uint32_t)r;
        CU(cudaMemcpy(dix.emb_docids, ids.data(), n * 4, cudaMemcpyHostToDevice), "H2D embedding docids");
    }
    CU(cudaStreamSynchronize(stream), "sync");
    // which documents own an embedding (VectorSort returns the others as its last bucket, vector_sort.rs:128-160)
    emb_bitmap.assign(hix.n_words64, 0);
    emb_row.assign(hix.n_words64 * 64, UINT32_MAX);
    emb_multi_row = false;
    for (uint64_t r = 0; r < n; r++) {
        const uint32_t doc = docids ? docids[r] : (uint32_t)r;
        if ((doc >> 6) < emb_bitmap.size()) emb_bitmap[doc >> 6] |= 1ull << (doc & 63);
        // rows of documents beyond the document range are scanned but never a similar query's target
        if (doc < emb_row.size()) {
            if (emb_row[doc] != UINT32_MAX) emb_multi_row = true;
            emb_row[doc] = (uint32_t)r;
        }
    }
    dix.emb_n = n;
    dix.emb_d = d;
    stats.hbm_bytes_staged += n * d * 2 + n * 8;
    return B200_OK;
}

int Engine::derive_batch(uint32_t n, const char *words, const uint32_t *off, const uint8_t *max_typo, const uint8_t *is_prefix,
                         uint32_t *one_out, uint32_t *n_one, uint32_t *two_out, uint32_t *n_two) {
    if (!staged) return fail(B200_ERR_STATE, "derive before b200_stage_finish");
    CU(cudaSetDevice(device), "cudaSetDevice");
    if (n == 0) return B200_OK;
    if (n >= (1u << LEV_FAMILY_SHIFT)) return fail(B200_ERR_UNSUPPORTED, "derive: too many terms in one batch");
    std::vector<LevTerm> terms(n);
    for (uint32_t i = 0; i < n; i++) {
        uint32_t len = off[i + 1] - off[i];
        if (len == 0 || len > LEV_MAX_Q) return fail(B200_ERR_UNSUPPORTED, "derive: word longer than 64 bytes (or empty)");
        LevTerm &t = terms[i];
        memset(&t, 0, sizeof t);
        memcpy(t.q, words + off[i], len);
        t.len = (uint8_t)len;
        t.k_same = max_typo[i] >= 2 ? 2 : 1;
        t.k_diff = max_typo[i] >= 2 ? 1 : -1;
        t.prefix = is_prefix[i] ? 1 : 0;
        if (max_typo[i] == 0) t.k_same = -1;
    }
    // Work list (DESIGN.md §3 "Term derivation"): each term joins the groups of the dictionary ranges where its filter can accept a
    // word, with the family that owns those pairs; a group's terms sweep each of its ranges in chunks of LEV_TERMS_PER_CTA.
    std::vector<uint32_t> by_first[256], by_second[256], whole;
    for (uint32_t i = 0; i < n; i++) {
        const LevTerm &t = terms[i];
        if (t.k_same < 0) continue;  // no typo budget: no derivations
        by_first[t.q[0]].push_back(i | LEV_F1 << LEV_FAMILY_SHIFT);
        if (t.k_diff < 0) continue;  // 1-typo terms keep their first byte
        if (t.len < 2 || t.q[0] == 0 || t.q[1] == 0) {  // the filter reads w[1] = 0 for 1-byte words: sweep everything
            whole.push_back(i | LEV_F0 << LEV_FAMILY_SHIFT);
            continue;
        }
        by_second[t.q[1]].push_back(i | LEV_F2B << LEV_FAMILY_SHIFT);
        if (t.q[1] != t.q[0]) {
            by_first[t.q[1]].push_back(i | LEV_F2A << LEV_FAMILY_SHIFT);
            by_second[t.q[0]].push_back(i | LEV_F3 << LEV_FAMILY_SHIFT);
        }
    }
    lev_perm.clear();
    lev_items.clear();
    uint64_t lev_bytes = 0, lev_pairs = 0;
    // the items of one group's term slots perm[p0, p0 + cnt) over the words [lo, hi), one per 256-word tile and term chunk
    auto emit = [&](uint32_t p0, uint32_t cnt, uint32_t lo, uint32_t hi) {
        for (uint32_t a = lo; a < hi;) {
            const uint32_t b = std::min(hi, (a & ~255u) + 256);
            for (uint32_t c = 0; c < cnt; c += LEV_TERMS_PER_CTA) {
                const uint32_t tc = std::min(cnt - c, (uint32_t)LEV_TERMS_PER_CTA);
                lev_items.push_back(LevItem{a, p0 + c, (uint16_t)(b - a), (uint16_t)tc});
                lev_pairs += (uint64_t)(b - a) * tc;
            }
            lev_bytes += (uint64_t)((cnt + LEV_TERMS_PER_CTA - 1) / LEV_TERMS_PER_CTA) * (hix.dict_off[b] - hix.dict_off[a] + 4ull * (b - a));
            a = b;
        }
    };
    auto slots = [&](const std::vector<uint32_t> &v) {
        lev_perm.insert(lev_perm.end(), v.begin(), v.end());
        return (uint32_t)(lev_perm.size() - v.size());
    };
    for (uint32_t g = 0; g < 256; g++) {
        if (!by_first[g].empty()) emit(slots(by_first[g]), (uint32_t)by_first[g].size(), hix.first_lo[g], hix.first_lo[g + 1]);
        if (by_second[g].empty()) continue;
        const uint32_t p0 = slots(by_second[g]), cnt = (uint32_t)by_second[g].size();
        for (uint32_t c = 0; c < 256; c++)  // (g, g) holds words whose first byte is q[1] (F2B) or q[0] (F3): owned elsewhere
            if (c != g) emit(p0, cnt, hix.pair_lo[c << 8 | g], hix.pair_hi(c, g));
    }
    if (!whole.empty()) emit(slots(whole), (uint32_t)whole.size(), 0, (uint32_t)hix.n_words);
    const uint32_t n_items = (uint32_t)lev_items.size();
    CU(d_lev_terms.reserve(n), "alloc lev terms");
    CU(d_lev_items.reserve(n_items), "alloc lev work items");
    CU(d_lev_perm.reserve(lev_perm.size()), "alloc lev term slots");
    CU(d_lev_recs.reserve((size_t)n * LEV_REC_SLOTS), "alloc lev records");
    size_t per = 1 + 150 + 1 + 50 + 1 + 1;
    CU(d_lev_u32.reserve((size_t)n * per), "alloc lev outputs");
    uint32_t *rec_count = d_lev_u32.p, *d_one = rec_count + n, *d_n_one = d_one + (size_t)n * 150, *d_two = d_n_one + n,
             *d_n_two = d_two + (size_t)n * 50;
    int32_t *d_status = reinterpret_cast<int32_t *>(d_n_two + n);
    CU(cudaMemcpyAsync(d_lev_terms.p, terms.data(), n * sizeof(LevTerm), cudaMemcpyHostToDevice, stream), "H2D lev terms");
    if (n_items) {
        CU(cudaMemcpyAsync(d_lev_items.p, lev_items.data(), n_items * sizeof(LevItem), cudaMemcpyHostToDevice, stream), "H2D lev items");
        CU(cudaMemcpyAsync(d_lev_perm.p, lev_perm.data(), lev_perm.size() * 4, cudaMemcpyHostToDevice, stream), "H2D lev term slots");
    }
    stats.h2d_bytes += n * sizeof(LevTerm) + n_items * sizeof(LevItem) + lev_perm.size() * 4;
    stats.d2h_bytes += (size_t)n * (150 + 50 + 3) * 4;
    stats.lev_terms += n;
    stats.lev_items += n_items;
    stats.lev_pairs += lev_pairs;
    size_t m0 = mark();
    CU(launch_lev(stream, dix.dict_bytes, dix.dict_off, d_lev_items.p, n_items, d_lev_perm.p, d_lev_terms.p, n, d_lev_recs.p, rec_count, d_one,
                  d_n_one, d_two, d_n_two, d_status),
       "lev kernels");
    size_t m1 = mark();
    time_kernel(B200_K_LEV, m0, m1, lev_bytes);
    stats.kernel_launches += 1;
    stats.dictionary_bytes += lev_bytes;
    std::vector<int32_t> status(n);
    CU(cudaMemcpyAsync(one_out, d_one, (size_t)n * 150 * 4, cudaMemcpyDeviceToHost, stream), "D2H");
    CU(cudaMemcpyAsync(n_one, d_n_one, (size_t)n * 4, cudaMemcpyDeviceToHost, stream), "D2H");
    CU(cudaMemcpyAsync(two_out, d_two, (size_t)n * 50 * 4, cudaMemcpyDeviceToHost, stream), "D2H");
    CU(cudaMemcpyAsync(n_two, d_n_two, (size_t)n * 4, cudaMemcpyDeviceToHost, stream), "D2H");
    CU(cudaMemcpyAsync(status.data(), d_status, (size_t)n * 4, cudaMemcpyDeviceToHost, stream), "D2H");
    CU(cudaStreamSynchronize(stream), "sync");
    resolve_timers();
    for (uint32_t i = 0; i < n; i++)
        if (status[i] != 0) return fail(B200_ERR_CAPACITY, "derive: match-record capacity exceeded for a term");
    return B200_OK;
}

int Engine::comm_load() {
    if (sc.lib) return B200_OK;
    void *lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);  // the copy this process already has (torch's), if any
    if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW);
    if (!lib) return fail(B200_ERR_STATE, std::string("cannot load libnccl.so.2: ") + dlerror());
    sc.get_unique_id = reinterpret_cast<int (*)(void *)>(dlsym(lib, "ncclGetUniqueId"));
    sc.comm_init_rank = reinterpret_cast<int (*)(void **, int, NcclId, int)>(dlsym(lib, "ncclCommInitRank"));
    sc.all_gather = reinterpret_cast<int (*)(const void *, void *, size_t, int, void *, cudaStream_t)>(dlsym(lib, "ncclAllGather"));
    sc.group_start = reinterpret_cast<int (*)()>(dlsym(lib, "ncclGroupStart"));
    sc.group_end = reinterpret_cast<int (*)()>(dlsym(lib, "ncclGroupEnd"));
    sc.comm_destroy = reinterpret_cast<int (*)(void *)>(dlsym(lib, "ncclCommDestroy"));
    sc.get_error_string = reinterpret_cast<const char *(*)(int)>(dlsym(lib, "ncclGetErrorString"));
    if (!sc.get_unique_id || !sc.comm_init_rank || !sc.all_gather || !sc.group_start || !sc.group_end || !sc.comm_destroy)
        return fail(B200_ERR_STATE, "libnccl.so.2 lacks an expected symbol");
    sc.lib = lib;
    return B200_OK;
}
int Engine::comm_init(int rank, int world, const uint8_t *unique_id) {
    int rc = comm_load();
    if (rc != B200_OK) return rc;
    if (world < 1 || rank < 0 || rank >= world) return fail(B200_ERR_INVALID, "comm_init: bad rank / world");
    CU(cudaSetDevice(device), "cudaSetDevice");
    if (sc.comm) {
        sc.comm_destroy(sc.comm);
        sc.comm = nullptr;
    }
    NcclId id;
    memcpy(id.internal, unique_id, 128);
    int e = sc.comm_init_rank(&sc.comm, world, id, rank);
    if (e != 0) return fail(B200_ERR_CUDA, std::string("ncclCommInitRank: ") + (sc.get_error_string ? sc.get_error_string(e) : "error"));
    sc.rank = rank;
    sc.world = world;
    return B200_OK;
}

int Engine::nns_batch(const float *queries, uint32_t n_q, uint32_t d, uint32_t limit, const uint64_t *cand, uint64_t n_cand_words,
                      uint32_t *ids_out, float *dist_out, uint32_t *n_out, bool sharded, const unsigned long long *dev_cand, const uint32_t *rows) {
    if (sharded && (!sc.comm || sc.world < 1)) return fail(B200_ERR_STATE, "sharded nns before b200_comm_init");
    CU(cudaSetDevice(device), "cudaSetDevice");
    if (!dix.emb) return fail(B200_ERR_STATE, "nns before b200_stage_embeddings");
    if (d != emb_d_user && d != dix.emb_d) return fail(B200_ERR_INVALID, "nns: query dimension differs from the staged embeddings");
    if (rows && d != dix.emb_d) return fail(B200_ERR_INVALID, "nns: row queries take the staged dimension");
    // the f32 queries of [q0, q0 + nq) into d_vq: copied from the host, or gathered from their staged rows (then with their inverse
    // norms into `inv` when it is given; only the row indices cross PCIe)
    auto load_queries = [&](uint32_t q0, uint32_t nq, float *inv) -> int {
        if (!rows) {
            CU(cudaMemcpyAsync(d_vq.p, queries + (size_t)q0 * d, (size_t)nq * d * 4, cudaMemcpyHostToDevice, vt.stream), "H2D queries");
            vstats.h2d_bytes += (size_t)nq * d * 4;
            return B200_OK;
        }
        CU(d_vrows.reserve(nq), "alloc query rows");
        CU(cudaMemcpyAsync(d_vrows.p, rows + q0, (size_t)nq * 4, cudaMemcpyHostToDevice, vt.stream), "H2D query rows");
        vstats.h2d_bytes += (size_t)nq * 4;
        CU(launch_vec_gather_rows(vt.stream, dix.emb, d, d_vrows.p, nq, d_vq.p, inv), "vec_gather_rows");
        vstats.kernel_launches++;
        vstats.vector_bytes += (uint64_t)nq * d * 2;
        return B200_OK;
    };
    if (d != dix.emb_d) {  // rows were zero-padded at staging: pad the queries the same way
        std::vector<float> padded((size_t)n_q * dix.emb_d, 0.f);
        for (uint32_t q = 0; q < n_q; q++) memcpy(padded.data() + (size_t)q * dix.emb_d, queries + (size_t)q * d, (size_t)d * 4);
        return nns_batch(padded.data(), n_q, dix.emb_d, limit, cand, n_cand_words, ids_out, dist_out, n_out, sharded, dev_cand);
    }
    if (n_q == 0) return B200_OK;
    const uint64_t N = dix.emb_n;
    if (N == 0 && !sharded) {  // an empty store: no hits (the batched path could not even describe a matrix of 0 rows to TMA)
        memset(n_out, 0, (size_t)n_q * 4);
        return B200_OK;
    }
    const uint32_t tie_cap = 1024;
    const uint32_t QT = 8;  // queries per scan pass
    uint32_t chunk = std::min<uint32_t>(n_q, 64);  // queries whose distance rows are resident at once
    CU(d_vq.reserve((size_t)chunk * d + chunk), "alloc queries");
    CU(d_vdist.reserve((size_t)chunk * N), "alloc distances");
    CU(d_vsel_dist.reserve((size_t)chunk * (limit + tie_cap)), "alloc selection");
    CU(d_vsel_ids.reserve((size_t)chunk * (limit + tie_cap)), "alloc selection");
    CU(d_vsel_n.reserve((size_t)chunk * 2), "alloc selection");
    const unsigned long long *d_c = dev_cand;
    if (!d_c && cand) {
        CU(d_cand.reserve(n_cand_words), "alloc candidates");
        CU(cudaMemcpyAsync(d_cand.p, cand, n_cand_words * 8, cudaMemcpyHostToDevice, vt.stream), "H2D candidates");
        d_c = d_cand.p;
    }
    // ---- batched path: wgmma GEMM with the top-k fused into its epilogue (vec_gemm.cu)
    {
        const char *force = getenv("B200_VEC_GEMM");
        bool want = force ? atoi(force) != 0 : n_q >= 16;
        if (sharded) {
            want = true;  // the exchange works on the device-resident top-k lists of the batched path
            if (!vec_gemm_supported(d, limit)) return fail(B200_ERR_UNSUPPORTED, "sharded nns: dimension / limit outside the batched kernel's range");
        }
        if (want && vec_gemm_supported(d, limit)) {
            const uint32_t vec_sms = getenv("B200_VEC_SMS") ? (uint32_t)std::max(8, std::min(sm_count, atoi(getenv("B200_VEC_SMS")))) : (uint32_t)sm_count;
            const uint32_t tiles_per_pass = vec_sms;  // query tiles resident in one launch
            std::vector<uint32_t> h_ids, h_n;
            std::vector<float> h_dist;
            constexpr uint32_t TQ = VEC_GEMM_QTILE;  // queries per tile of the kernel
            for (uint32_t q0 = 0; q0 < n_q; q0 += tiles_per_pass * TQ) {
                uint32_t nq = std::min<uint32_t>(n_q - q0, tiles_per_pass * TQ);
                uint32_t n_qtiles = (nq + TQ - 1) / TQ, n_pad = n_qtiles * TQ;
                uint64_t n_row_tiles = (N + 63) / 64;
                uint32_t n_groups = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)vec_sms / n_qtiles, n_row_tiles));
                CU(d_vq.reserve((size_t)nq * d + n_pad), "alloc queries");
                CU(d_vq16.reserve((size_t)n_pad * d), "alloc fp16 queries");
                CU(d_vruns.reserve((size_t)n_qtiles * n_groups * TQ * VEC_GEMM_CAND_CAP + (size_t)n_pad * n_groups), "alloc candidate runs");
                CU(d_vpartial.reserve((size_t)n_pad * n_groups * VEC_GEMM_KMAX), "alloc partial top-k");
                CU(d_vsel_dist.reserve((size_t)n_pad * limit), "alloc selection");
                CU(d_vsel_ids.reserve((size_t)n_pad * limit), "alloc selection");
                CU(d_vsel_n.reserve(n_pad), "alloc selection");
                float *d_qinv = d_vq.p + (size_t)nq * d;
                if (int rc = load_queries(q0, nq, nullptr)) return rc;
                CU(launch_vec_prep_queries(vt.stream, d_vq.p, nq, n_pad, d, d_vq16.p, d_qinv), "vec_prep_queries");
                vstats.kernel_launches++;
                size_t m0 = vt.mark();
                CU(launch_vec_gemm_topk(vt.stream, vec_sms, dix.emb, dix.emb_inv_norm, dix.emb_docids, N, d, d_vq16.p, d_qinv, n_qtiles, n_groups,
                                        d_c, n_cand_words, limit, d_vruns.p + (size_t)n_qtiles * n_groups * TQ * VEC_GEMM_CAND_CAP, d_vruns.p, d_vpartial.p, d_vsel_ids.p, d_vsel_dist.p, d_vsel_n.p, nq),
                   "vec_gemm_topk");
                if (sharded && sc.world > 1) {
                    // one all-gather of the per-shard top-k (ids, distances, counts) on the vector stream, then the merge: the lists
                    // never leave the device between the scan and the merged result
                    const uint32_t Wd = (uint32_t)sc.world;
                    CU(d_gather_ids.reserve((size_t)Wd * nq * limit), "alloc gather");
                    CU(d_gather_dist.reserve((size_t)Wd * nq * limit), "alloc gather");
                    CU(d_gather_n.reserve((size_t)Wd * nq), "alloc gather");
                    int e = sc.group_start();
                    if (!e) e = sc.all_gather(d_vsel_ids.p, d_gather_ids.p, (size_t)nq * limit * 4, 1 /* ncclUint8 */, sc.comm, vt.stream);
                    if (!e) e = sc.all_gather(d_vsel_dist.p, d_gather_dist.p, (size_t)nq * limit * 4, 1, sc.comm, vt.stream);
                    if (!e) e = sc.all_gather(d_vsel_n.p, d_gather_n.p, (size_t)nq * 4, 1, sc.comm, vt.stream);
                    int e2 = sc.group_end();
                    if (e || e2) return fail(B200_ERR_CUDA, std::string("ncclAllGather: ") + (sc.get_error_string ? sc.get_error_string(e ? e : e2) : "error"));
                    CU(launch_shard_merge(vt.stream, d_gather_ids.p, d_gather_dist.p, d_gather_n.p, Wd, nq, limit, d_vsel_ids.p, d_vsel_dist.p, d_vsel_n.p),
                       "shard merge");
                    vstats.kernel_launches++;
                }
                size_t m1 = vt.mark();
                // algorithmic bytes: every query tile streams the matrix once (L2 absorbs the re-reads across tiles of the same rows)
                vt.time_kernel(vstats, B200_K_VEC_GEMM, m0, m1, (uint64_t)N * d * 2 + N * 8 + (uint64_t)n_pad * d * 2);
                vstats.kernel_launches++;  // merge kernel
                vstats.vector_bytes += (uint64_t)N * d * 2;
                h_ids.resize((size_t)nq * limit);
                h_dist.resize((size_t)nq * limit);
                h_n.resize(nq);
                CU(cudaMemcpyAsync(h_ids.data(), d_vsel_ids.p, (size_t)nq * limit * 4, cudaMemcpyDeviceToHost, vt.stream), "D2H");
                CU(cudaMemcpyAsync(h_dist.data(), d_vsel_dist.p, (size_t)nq * limit * 4, cudaMemcpyDeviceToHost, vt.stream), "D2H");
                CU(cudaMemcpyAsync(h_n.data(), d_vsel_n.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, vt.stream), "D2H");
                vstats.d2h_bytes += (size_t)nq * limit * 8 + nq * 4;
                CU(cudaStreamSynchronize(vt.stream), "sync");
                vt.resolve(vstats);
                for (uint32_t q = 0; q < nq; q++) {
                    uint32_t n = std::min(h_n[q], limit);
                    n_out[q0 + q] = n;
                    memcpy(ids_out + (size_t)(q0 + q) * limit, h_ids.data() + (size_t)q * limit, (size_t)n * 4);
                    memcpy(dist_out + (size_t)(q0 + q) * limit, h_dist.data() + (size_t)q * limit, (size_t)n * 4);
                }
            }
            return B200_OK;
        }
    }
    std::vector<float> qinv(chunk);
    std::vector<float> sel_d((size_t)chunk * (limit + tie_cap));
    std::vector<uint32_t> sel_i((size_t)chunk * (limit + tie_cap)), sel_n((size_t)chunk * 2);
    for (uint32_t q0 = 0; q0 < n_q; q0 += chunk) {
        uint32_t nq = std::min(chunk, n_q - q0);
        float *d_qinv = d_vq.p + (size_t)chunk * d;
        if (int rc = load_queries(q0, nq, rows ? d_qinv : nullptr)) return rc;
        if (!rows) {
            for (uint32_t q = 0; q < nq; q++) {
                double s = 0;
                const float *v = queries + (size_t)(q0 + q) * d;
                for (uint32_t i = 0; i < d; i++) s += (double)v[i] * v[i];
                float nrm = (float)std::sqrt(s);
                qinv[q] = nrm > 0.f ? 1.0f / nrm : 0.f;
            }
            vstats.h2d_bytes += nq * 4;
            CU(cudaMemcpyAsync(d_qinv, qinv.data(), nq * 4, cudaMemcpyHostToDevice, vt.stream), "H2D query norms");
        }
        vstats.d2h_bytes += (size_t)nq * (limit + tie_cap) * 8 + nq * 8;
        for (uint32_t t = 0; t < nq;) {
            uint32_t left = nq - t;
            int qt = left >= 8 ? 8 : (left >= 4 ? 4 : (left >= 2 ? 2 : 1));
            (void)QT;
            size_t m0 = vt.mark();
            CU(launch_vec_dist(vt.stream, sm_count * 6, qt, dix.emb, dix.emb_inv_norm, dix.emb_docids, N, d, d_vq.p + (size_t)t * d, d_qinv + t, d_c,
                               n_cand_words, d_vdist.p + (size_t)t * N),
               "vec_dist");
            size_t m1 = vt.mark();
            uint64_t vb = N * d * 2 + N * 4 + (d_c ? N / 8 : 0) + (uint64_t)qt * d * 4 + (uint64_t)qt * N * 4;
            vt.time_kernel(vstats, B200_K_VEC_DIST, m0, m1, vb);
            vstats.vector_bytes += vb;
            t += qt;
        }
        size_t k0 = vt.mark();
        // long rows are selected in pieces side by side (one CTA per >= 16 k distances, about two waves of CTAs per query batch)
        const uint32_t n_slices = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(std::min<uint64_t>(128, (uint64_t)sm_count * 4 / std::max(1u, nq)), N / 16384));
        if (n_slices > 1) {
            CU(d_vpart_dist.reserve((size_t)nq * n_slices * (limit + tie_cap)), "alloc partial selection");
            CU(d_vpart_ids.reserve((size_t)nq * n_slices * (limit + tie_cap)), "alloc partial selection");
            CU(d_vpart_n.reserve((size_t)nq * n_slices * 2), "alloc partial selection");
        }
        CU(launch_topk(vt.stream, nq, d_vdist.p, dix.emb_docids, N, limit, tie_cap, n_slices, d_vpart_dist.p, d_vpart_ids.p, d_vpart_n.p, d_vsel_dist.p,
                       d_vsel_ids.p, d_vsel_n.p),
           "topk");
        size_t k1 = vt.mark();
        vt.time_kernel(vstats, B200_K_TOPK, k0, k1, (uint64_t)nq * N * 4 * 4);
        CU(cudaMemcpyAsync(sel_d.data(), d_vsel_dist.p, (size_t)nq * (limit + tie_cap) * 4, cudaMemcpyDeviceToHost, vt.stream), "D2H");
        CU(cudaMemcpyAsync(sel_i.data(), d_vsel_ids.p, (size_t)nq * (limit + tie_cap) * 4, cudaMemcpyDeviceToHost, vt.stream), "D2H");
        CU(cudaMemcpyAsync(sel_n.data(), d_vsel_n.p, (size_t)nq * 2 * 4, cudaMemcpyDeviceToHost, vt.stream), "D2H");
        CU(cudaStreamSynchronize(vt.stream), "sync");
        vt.resolve(vstats);
        for (uint32_t q = 0; q < nq; q++) {
            std::vector<std::pair<float, uint32_t>> c;
            const float *sd = sel_d.data() + (size_t)q * (limit + tie_cap);
            const uint32_t *si = sel_i.data() + (size_t)q * (limit + tie_cap);
            for (uint32_t i = 0; i < sel_n[2 * q]; i++) c.push_back({sd[i], si[i]});
            for (uint32_t i = 0; i < sel_n[2 * q + 1]; i++) c.push_back({sd[limit + i], si[limit + i]});
            std::sort(c.begin(), c.end());
            uint32_t n = (uint32_t)std::min<size_t>(c.size(), limit);
            n_out[q0 + q] = n;
            for (uint32_t i = 0; i < n; i++) {
                ids_out[(size_t)(q0 + q) * limit + i] = c[i].second;
                dist_out[(size_t)(q0 + q) * limit + i] = c[i].first;
            }
        }
    }
    return B200_OK;
}

// S2: OR of posting lists, restricted to a universe — what ConditionDocIdsCache::get_computed_condition
// (crates/milli/src/search/new/ranking_rule_graph/condition_docids_cache.rs:34-57) obtains from G::resolve_condition for the
// union-shaped conditions (compute_query_term_subset_docids, resolve_query_graph.rs:33-59: `docids |= list` for every derivation,
// then `& universe`).  One scatter_kernel launch over the dense universe.
int Engine::union_postings(int db, const uint32_t *key_index, uint32_t n_keys, const uint64_t *universe, uint64_t n_universe_words, uint64_t *out) {
    if (!staged) return fail(B200_ERR_STATE, "union_postings before b200_stage_finish");
    if (db < 0 || db >= 10) return fail(B200_ERR_INVALID, "union_postings: unknown database id");
    if (db == 4 && hix.pair_keys.size() != hix.db_keys[4])
        return fail(B200_ERR_UNSUPPORTED, "union_postings: word_pair_proximity keys were dropped at staging, key indices are not stable");
    CU(cudaSetDevice(device), "cudaSetDevice");
    const uint64_t W = hix.n_words64;
    if (universe && n_universe_words < W) return fail(B200_ERR_INVALID, "union_postings: universe bitmap shorter than the document range");
    std::vector<Job> jobs;
    for (uint32_t i = 0; i < n_keys; i++) {
        if (key_index[i] >= hix.db_keys[db]) return fail(B200_ERR_INVALID, "union_postings: key index out of range");
        const uint32_t list = hix.db_first[db] + key_index[i];
        const ListRef &lr = hix.lists[list];
        if (!lr.card) continue;
        const uint64_t units = lr.dense ? W : lr.card;
        for (uint32_t k = 0; k < (units + JOB_CHUNK - 1) / JOB_CHUNK; k++) jobs.push_back(Job{0, 0, list, k});
    }
    const size_t o_ub = 0, o_col = o_ub + W * 8, o_act = (o_col + W * 8 + 255) & ~(size_t)255, o_res = o_act + ((sizeof(ActDesc) + 255) & ~(size_t)255),
                 o_jobs = o_res + 256, o_bigq = (o_jobs + std::max<size_t>(1, jobs.size()) * sizeof(Job) + 255) & ~(size_t)255,
                 total = o_bigq + std::max<size_t>(1, jobs.size()) * 4;
    CU(d_s2.reserve(total), "alloc S2 scratch");
    uint8_t *base = d_s2.p;
    if (universe)
        CU(cudaMemcpyAsync(base + o_ub, universe, W * 8, cudaMemcpyHostToDevice, stream), "H2D universe");
    else
        CU(cudaMemcpyAsync(base + o_ub, dix.base_ub, W * 8, cudaMemcpyDeviceToDevice, stream), "universe");
    CU(cudaMemsetAsync(base + o_col, 0, W * 8, stream), "zero column");
    ActDesc a;
    memset(&a, 0, sizeof a);
    a.ub = reinterpret_cast<unsigned long long *>(base + o_ub);
    a.C = reinterpret_cast<unsigned long long *>(base + o_col);
    a.ld = (uint32_t)W;
    a.n_cols = 1;
    a.res_off = 0;
    uint32_t counters[4] = {(uint32_t)W, 0, 0, 0};      // results[0] = rows
    uint32_t qcount[8] = {(uint32_t)jobs.size(), 0, 0, 0, 0, 0, 0, 0};
    CU(cudaMemcpyAsync(base + o_act, &a, sizeof a, cudaMemcpyHostToDevice, stream), "H2D activation");
    CU(cudaMemcpyAsync(base + o_res, counters, sizeof counters, cudaMemcpyHostToDevice, stream), "H2D rows");
    CU(cudaMemcpyAsync(base + o_res + 64, qcount, sizeof qcount, cudaMemcpyHostToDevice, stream), "H2D job count");
    if (!jobs.empty()) {
        CU(cudaMemcpyAsync(base + o_jobs, jobs.data(), jobs.size() * sizeof(Job), cudaMemcpyHostToDevice, stream), "H2D jobs");
        size_t m0 = mark();
        CU(launch_scatter(stream, (uint32_t)sm_count * 5, reinterpret_cast<const Job *>(base + o_jobs), reinterpret_cast<uint32_t *>(base + o_res + 64),
                          (uint32_t)jobs.size(), reinterpret_cast<const ActDesc *>(base + o_act), reinterpret_cast<const uint32_t *>(base + o_res),
                          dix.lists, dix.pool, reinterpret_cast<uint32_t *>(base + o_bigq)),
           "scatter");
        uint64_t bytes = 0;
        for (auto &j : jobs) bytes += hix.lists[j.list].dense ? (uint64_t)JOB_CHUNK * 8 : (uint64_t)std::min<uint32_t>(JOB_CHUNK, hix.lists[j.list].card) * 4;
        time_kernel(B200_K_SCATTER, m0, mark(), bytes);
    }
    CU(cudaMemcpyAsync(out, base + o_col, W * 8, cudaMemcpyDeviceToHost, stream), "D2H column");
    CU(cudaStreamSynchronize(stream), "sync");
    resolve_timers();
    // scatter_kernel does not consult the universe for sparse lists (inside the engine the DP masks with it): apply it here
    for (uint64_t w = 0; w < W; w++) out[w] &= universe ? universe[w] : hix.base_ub[w];
    stats.h2d_bytes += (universe ? W * 8 : 0) + jobs.size() * sizeof(Job) + sizeof a;
    stats.d2h_bytes += W * 8;
    return B200_OK;
}

// S2 for proximity conditions: what ProximityGraph::resolve_condition (ranking_rule_graph/proximity/compute_docids.rs:15-108)
// unions for one edge — every (l, r) of two word sets looked up forwards at proximity `fwd_prox` and backwards (r, l) at
// `bwd_prox` (0 = no lookup in that direction) in word_pair_proximity_docids — restricted to a universe.  pair_probe_kernel
// resolves the key probes against the staged key directory, scatter_kernel ORs the lists it found.
int Engine::proximity_pairs(const uint32_t *left, uint32_t n_left, const uint32_t *right, uint32_t n_right, uint32_t fwd_prox, uint32_t bwd_prox,
                            const uint64_t *universe, uint64_t n_universe_words, uint64_t *out) {
    if (!staged) return fail(B200_ERR_STATE, "proximity_pairs before b200_stage_finish");
    if (fwd_prox > 3 || bwd_prox > 3) return fail(B200_ERR_INVALID, "proximity_pairs: proximities are 0 (none) .. 3");
    CU(cudaSetDevice(device), "cudaSetDevice");
    const uint64_t W = hix.n_words64;
    if (universe && n_universe_words < W) return fail(B200_ERR_INVALID, "proximity_pairs: universe bitmap shorter than the document range");
    for (uint32_t i = 0; i < n_left; i++)
        if (left[i] >= hix.n_words) return fail(B200_ERR_INVALID, "proximity_pairs: word id out of range");
    for (uint32_t i = 0; i < n_right; i++)
        if (right[i] >= hix.n_words) return fail(B200_ERR_INVALID, "proximity_pairs: word id out of range");
    const uint64_t n_probes = (uint64_t)n_left * n_right;
    if (n_probes == 0 || (fwd_prox == 0 && bwd_prox == 0)) {
        memset(out, 0, W * 8);
        return B200_OK;
    }
    if (n_probes > (1u << 26)) return fail(B200_ERR_CAPACITY, "proximity_pairs: more than 2^26 word pairs in one call");
    const size_t qcap = std::max<size_t>((size_t)1 << 16, (size_t)n_probes * 4);
    const size_t o_ub = 0, o_col = o_ub + W * 8, o_act = (o_col + W * 8 + 255) & ~(size_t)255, o_res = o_act + ((sizeof(ActDesc) + 255) & ~(size_t)255),
                 o_set = o_res + 256, o_words = o_set + 256, o_queue = (o_words + ((size_t)n_left + n_right) * 4 + 255) & ~(size_t)255,
                 o_bigq = o_queue + qcap * sizeof(Job), total = o_bigq + qcap * 4;
    CU(d_s2.reserve(total), "alloc S2 scratch");
    uint8_t *base = d_s2.p;
    if (universe)
        CU(cudaMemcpyAsync(base + o_ub, universe, W * 8, cudaMemcpyHostToDevice, stream), "H2D universe");
    else
        CU(cudaMemcpyAsync(base + o_ub, dix.base_ub, W * 8, cudaMemcpyDeviceToDevice, stream), "universe");
    CU(cudaMemsetAsync(base + o_col, 0, W * 8, stream), "zero column");
    ActDesc a;
    memset(&a, 0, sizeof a);
    a.ub = reinterpret_cast<unsigned long long *>(base + o_ub);
    a.C = reinterpret_cast<unsigned long long *>(base + o_col);
    a.ld = (uint32_t)W;
    a.n_cols = 1;
    uint32_t counters[16] = {(uint32_t)W};  // results[0] = rows | qcount at +16: [0] jobs, [2] scatter cursor
    PairSet ps{};
    ps.left_off = 0;
    ps.n_left = n_left;
    ps.right_off = n_left;
    ps.n_right = n_right;
    ps.fwd_prox = (uint8_t)fwd_prox;
    ps.bwd_prox = (uint8_t)bwd_prox;
    CU(cudaMemcpyAsync(base + o_act, &a, sizeof a, cudaMemcpyHostToDevice, stream), "H2D activation");
    CU(cudaMemcpyAsync(base + o_res, counters, sizeof counters, cudaMemcpyHostToDevice, stream), "H2D counters");
    CU(cudaMemcpyAsync(base + o_set, &ps, sizeof ps, cudaMemcpyHostToDevice, stream), "H2D pair set");
    CU(cudaMemcpyAsync(base + o_words, left, (size_t)n_left * 4, cudaMemcpyHostToDevice, stream), "H2D words");
    CU(cudaMemcpyAsync(base + o_words + (size_t)n_left * 4, right, (size_t)n_right * 4, cudaMemcpyHostToDevice, stream), "H2D words");
    uint32_t *d_res = reinterpret_cast<uint32_t *>(base + o_res), *d_qcount = d_res + 4;
    size_t m0 = mark();
    CU(launch_pair_probe(stream, reinterpret_cast<const PairSet *>(base + o_set), 1, (uint32_t)n_probes, reinterpret_cast<const uint32_t *>(base + o_words),
                         dix.pair_keys, hix.pair_keys.size(), hix.pair_list_base, dix.lists, reinterpret_cast<const ActDesc *>(base + o_act), d_res,
                         reinterpret_cast<Job *>(base + o_queue), d_qcount, (uint32_t)qcap),
       "pair probe");
    size_t m1 = mark();
    time_kernel(B200_K_PAIR_PROBE, m0, m1, n_probes * 8 * 23);
    CU(launch_scatter(stream, (uint32_t)sm_count * 5, reinterpret_cast<const Job *>(base + o_queue), d_qcount, (uint32_t)qcap,
                      reinterpret_cast<const ActDesc *>(base + o_act), d_res, dix.lists, dix.pool, reinterpret_cast<uint32_t *>(base + o_bigq)),
       "scatter");
    time_kernel(B200_K_SCATTER, m1, mark(), 0);
    uint32_t h_counts[8];
    CU(cudaMemcpyAsync(h_counts, d_res, sizeof h_counts, cudaMemcpyDeviceToHost, stream), "D2H counters");
    CU(cudaMemcpyAsync(out, base + o_col, W * 8, cudaMemcpyDeviceToHost, stream), "D2H column");
    CU(cudaStreamSynchronize(stream), "sync");
    resolve_timers();
    if (h_counts[4] > qcap) return fail(B200_ERR_CAPACITY, "proximity_pairs: job queue overflow");
    for (uint64_t w = 0; w < W; w++) out[w] &= universe ? universe[w] : hix.base_ub[w];
    stats.h2d_bytes += (universe ? W * 8 : 0) + ((size_t)n_left + n_right) * 4 + sizeof a;
    stats.d2h_bytes += W * 8;
    return B200_OK;
}

}  // namespace b200
