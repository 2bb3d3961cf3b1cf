// Facet distribution and facet stats (facet.cu) for the keyword batch (b200_query_batch::facet_*) and for
// b200_facet_distribution_batch: slot scratch, chunking, and the decoding of the kernels' outputs into the caller's arrays.
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
const SortField *field_of(const HostIndex &hix, uint16_t fid) {
    auto it = hix.sort_fields.find(fid);
    return it == hix.sort_fields.end() ? nullptr : &it->second;
}
}  // namespace

// per value a count and a first docid, then the 16-byte FacetHead
size_t Engine::facet_slot_bytes(uint16_t fid) const {
    const SortField *f = field_of(hix, fid);
    return (((size_t)(f ? f->n_values() : 0) * 8 + 15) & ~(size_t)15) + sizeof(FacetHead);
}

int Engine::reserve_facet_scratch(const std::vector<uint16_t> &fids, size_t budget, DevBuf<uint8_t> &scratch, DevBuf<FacetSlot> &slots) {
    size_t total = 0, largest = 0;
    for (uint16_t fid : fids) {
        const size_t b = facet_slot_bytes(fid);
        total += b;
        largest = std::max(largest, b);
    }
    if (scratch.reserve(std::max<size_t>(1, std::max(largest, std::min(total, budget)))) != cudaSuccess ||
        slots.reserve(std::max<size_t>(1, fids.size())) != cudaSuccess) {
        cudaGetLastError();
        return fail(B200_ERR_CAPACITY, "facet counts: a slot's scratch (8 bytes per value of its field) does not fit in device memory");
    }
    return B200_OK;
}

int Engine::reserve_facet_out(size_t n_slots, uint32_t cap, FacetOut &out) {
    const size_t n = std::max<size_t>(1, n_slots * cap);
    if (d_facet_out.reserve(n * 16 + std::max<size_t>(1, n_slots) * 16) != cudaSuccess) {
        cudaGetLastError();
        return fail(B200_ERR_CAPACITY, "facet outputs (16 bytes per entry: n_slots x facet_cap) do not fit in device memory");
    }
    out.cnt = reinterpret_cast<unsigned long long *>(d_facet_out.p);
    out.ord = reinterpret_cast<uint32_t *>(out.cnt + n);
    out.doc = out.ord + n;
    out.sum = out.doc + n;
    out.n_slots = n_slots;
    out.cap = cap;
    return B200_OK;
}

int Engine::facet_enqueue(Lane *ln, const std::vector<FacetJob> &jobs, const FacetOut &out, uint32_t max_values, DevBuf<uint8_t> &scratch,
                          DevBuf<FacetSlot> &dslots) {
    const cudaStream_t s = ln ? ln->stream : stream;
    b200_stats &st = ln ? ln->lst : stats;
    std::vector<FacetSlot> sl;
    for (size_t i = 0; i < jobs.size();) {
        // a chunk: the slots whose scratch fits (always at least one: reserve_facet_scratch made room for the largest)
        size_t used = 0;
        uint64_t bytes = 0;
        sl.clear();
        for (; i < jobs.size() && sl.size() < 65535; i++) {
            const size_t need = facet_slot_bytes(jobs[i].fid);
            if (!sl.empty() && used + need > scratch.cap) break;
            const SortField *f = field_of(hix, jobs[i].fid);
            FacetSlot x{};
            x.cand = jobs[i].cand;
            x.n_num = f ? f->n_num : 0;
            x.n_str = f ? f->n_str : 0;
            if (f) {
                x.doc_off = f->d_doc_off;
                x.doc_ord = f->d_doc_ord;
                x.disp = f->d_disp;
            }
            const uint32_t V = x.n_num + x.n_str;
            x.cnt = reinterpret_cast<uint32_t *>(scratch.p + used);
            x.first = x.cnt + V;
            x.head = reinterpret_cast<FacetHead *>(scratch.p + used + need - sizeof(FacetHead));
            x.max_values = max_values;
            x.cap = out.cap;
            const size_t k = jobs[i].slot;
            x.out_ord = out.ord + k * out.cap;
            x.out_doc = out.doc + k * out.cap;
            x.out_cnt = out.cnt + k * out.cap;
            x.out_sum = out.sum + 4 * k;
            sl.push_back(x);
            used += need;
            // algorithmic bytes: the candidate words, then (at most) every value's count and first docid twice
            bytes += (uint64_t)hix.n_words64 * 8 + (uint64_t)V * 16;
        }
        // the descriptors come from pageable memory: the copy waits for the stream, so the previous chunk is done with them
        CU(cudaMemsetAsync(scratch.p, 0, used, s), "zero facet counts");
        CU(cudaMemcpyAsync(dslots.p, sl.data(), sl.size() * sizeof(FacetSlot), cudaMemcpyHostToDevice, s), "H2D facet slots");
        st.h2d_bytes += sl.size() * sizeof(FacetSlot);
        const size_t m0 = ln ? ln->mark() : mark();
        CU(launch_facet(s, dslots.p, (uint32_t)sl.size(), hix.n_words64, hix.n_docs), "facet");
        const size_t m1 = ln ? ln->mark() : mark();
        if (ln)
            ln->time_kernel(st, B200_K_FACET, m0, m1, bytes);
        else
            time_kernel(B200_K_FACET, m0, m1, bytes);
    }
    return B200_OK;
}

int Engine::facet_results(const FacetOut &out, const uint16_t *fid, const b200_results &dst, std::vector<std::string> &err) {
    const size_t n = out.n_slots, cap = out.cap;
    err.assign(n, std::string());
    if (!n) return B200_OK;
    std::vector<uint32_t> ord(n * cap), doc(n * cap), sum(4 * n);
    std::vector<unsigned long long> cnt(n * cap);
    CU(cudaMemcpyAsync(sum.data(), out.sum, sum.size() * 4, cudaMemcpyDeviceToHost, stream), "D2H facet outputs");
    if (cap) {
        CU(cudaMemcpyAsync(ord.data(), out.ord, ord.size() * 4, cudaMemcpyDeviceToHost, stream), "D2H facet outputs");
        CU(cudaMemcpyAsync(doc.data(), out.doc, doc.size() * 4, cudaMemcpyDeviceToHost, stream), "D2H facet outputs");
        CU(cudaMemcpyAsync(cnt.data(), out.cnt, cnt.size() * 8, cudaMemcpyDeviceToHost, stream), "D2H facet outputs");
    }
    CU(cudaStreamSynchronize(stream), "sync facet outputs");
    stats.d2h_bytes += sum.size() * 4 + n * cap * 16;
    for (size_t k = 0; k < n; k++) {
        const SortField *f = field_of(hix, fid[k]);
        const uint32_t n_num = sum[4 * k], n_str = sum[4 * k + 1];
        dst.facet_n_num[k] = dst.facet_n_str[k] = 0;
        dst.facet_has_stats[k] = 0;
        dst.facet_min[k] = dst.facet_max[k] = 0;
        if ((uint64_t)n_num + n_str > cap) {
            err[k] = "facet_cap " + std::to_string(cap) + " is too small: the facet distribution of field " + std::to_string(fid[k]) + " needs " +
                     std::to_string((uint64_t)n_num + n_str) + " entries";
            continue;
        }
        if (!f) continue;
        dst.facet_n_num[k] = n_num;
        dst.facet_n_str[k] = n_str;
        for (size_t e = k * cap; e < k * cap + n_num + n_str; e++) {
            bool is_string = false;
            f->decode(true, ord[e], is_string, dst.facet_key[e]);
            dst.facet_count[e] = cnt[e];
            dst.facet_docid[e] = doc[e];
        }
        if (sum[4 * k + 3]) {  // FacetHead: ~(smallest number ordinal), largest + 1
            dst.facet_has_stats[k] = 1;
            dst.facet_min[k] = f->num_val[~sum[4 * k + 2]];
            dst.facet_max[k] = f->num_val[sum[4 * k + 3] - 1];
        }
    }
    return B200_OK;
}

int Engine::facet_distribution_batch(uint32_t n, const uint64_t *const *candidates, uint64_t n_words, const uint32_t *begin, const uint16_t *fid,
                                     const uint8_t *order, uint32_t max_values, uint32_t cap, const b200_results &dst, int32_t *status) {
    if (!n) return B200_OK;
    if (!candidates || !begin || !status) return fail(B200_ERR_INVALID, "facet_distribution_batch: null candidates / facet_begin / status");
    const uint32_t n_slots = begin[n];
    if (n_slots && (!fid || !dst.facet_n_num || !dst.facet_n_str || !dst.facet_key || !dst.facet_count || !dst.facet_docid || !dst.facet_has_stats ||
                    !dst.facet_min || !dst.facet_max))
        return fail(B200_ERR_INVALID, "facet_distribution_batch: null facet_fid or output array");
    const uint64_t W = hix.n_words64;
    if (n_words < W) return fail(B200_ERR_INVALID, "facet_distribution_batch: n_words smaller than the document range");
    for (uint32_t i = 0; i < n; i++) {
        if (!candidates[i] || begin[i + 1] < begin[i]) return fail(B200_ERR_INVALID, "facet_distribution_batch: null candidates or decreasing facet_begin");
        status[i] = B200_OK;
        for (uint32_t k = begin[i]; k < begin[i + 1] && order; k++)
            if (order[k] == 1 && !status[i]) {
                status[i] = B200_ERR_UNSUPPORTED;
                last_error = "facet order by count (sortFacetValuesBy: count) is not built";
            } else if (order[k] > 1)
                return fail(B200_ERR_INVALID, "facet_order is not 0 (alpha) or 1 (count)");
    }
    for (uint32_t k = 0; k < n_slots; k++) {
        dst.facet_n_num[k] = dst.facet_n_str[k] = 0;
        dst.facet_has_stats[k] = 0;
    }
    CU(cudaSetDevice(device), "cudaSetDevice");
    // the distinct candidate bitmaps, uploaded once each
    std::map<const uint64_t *, uint32_t> at;
    for (uint32_t i = 0; i < n; i++)
        if (!status[i] && begin[i + 1] > begin[i]) at.emplace(candidates[i], 0);
    uint32_t n_bitmaps = 0;
    for (auto &kv : at) kv.second = n_bitmaps++;
    if (d_facet_cand.reserve(std::max<size_t>(1, (size_t)n_bitmaps * W)) != cudaSuccess) {
        cudaGetLastError();
        return fail(B200_ERR_CAPACITY, "facet_distribution_batch: the candidate bitmaps do not fit in device memory");
    }
    for (auto &kv : at) {
        CU(cudaMemcpyAsync(d_facet_cand.p + (size_t)kv.second * W, kv.first, W * 8, cudaMemcpyHostToDevice, stream), "H2D facet candidates");
        stats.h2d_bytes += W * 8;
    }
    std::vector<FacetJob> jobs;
    std::vector<uint16_t> fids;
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t k = begin[i]; k < begin[i + 1] && !status[i]; k++) {
            jobs.push_back(FacetJob{d_facet_cand.p + (size_t)at[candidates[i]] * W, fid[k], k});
            fids.push_back(fid[k]);
        }
    FacetOut out;
    int rc = reserve_facet_out(n_slots, cap, out);
    if (rc == B200_OK) rc = reserve_facet_scratch(fids, (size_t)256 << 20, d_facet_scratch, d_facet_slots);
    if (rc != B200_OK) return rc;
    CU(cudaMemsetAsync(out.sum, 0, (size_t)n_slots * 16, stream), "zero facet outputs");
    if ((rc = facet_enqueue(nullptr, jobs, out, max_values, d_facet_scratch, d_facet_slots)) != B200_OK) return rc;
    std::vector<std::string> err;
    if ((rc = facet_results(out, fid, dst, err)) != B200_OK) return rc;
    resolve_timers();
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t k = begin[i]; k < begin[i + 1]; k++) {
            if (!status[i] && !err[k].empty()) {
                status[i] = B200_ERR_CAPACITY;
                last_error = err[k];
            }
            if (status[i]) dst.facet_n_num[k] = dst.facet_n_str[k] = dst.facet_has_stats[k] = 0;
        }
    return B200_OK;
}

}  // namespace b200
