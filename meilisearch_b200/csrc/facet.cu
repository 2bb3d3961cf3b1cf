// Facet distribution and facet stats (search/facet/facet_distribution.rs:110-337) over candidate bitmaps, on the device.
//
// A field's values are numbered in the Sort rule's ascending walk order: numbers ascending, then strings in byte order (host_index.h
// SortField).  That is the order of the reference's facet-level walk (facet_distribution_iter.rs:26-232), so "the first non-empty
// values in level order" are the first non-empty ordinals.  The "from documents" path (<= 3000 candidates) orders numbers by their
// f64 Display strings instead; staging keeps that order of the number ordinals (SortField::disp).
//
// facet_count_kernel: one thread per 64-document word of one slot's candidates.  It walks the set bits and each document's
// ordinals, counting into a shared-memory histogram when the field has at most FACET_SHARED_VALUES values (flushed with one global
// atomic per non-empty value and CTA) and straight into the slot's global counts otherwise; per value it keeps the smallest
// candidate (as the largest ~docid), and per slot |candidates| and the smallest / largest number ordinal (compute_stats).
// facet_select_kernel: one CTA per slot scans the counts in the reference's order with a block-wide prefix over the non-empty values
// and writes the entries facet_values returns (b200milli.h, b200_results::facet_*).
#include <cuda_runtime.h>

#include "device_types.h"

namespace b200 {

namespace {

constexpr uint32_t COUNT_THREADS = 256, SELECT_THREADS = 256;

__global__ void __launch_bounds__(COUNT_THREADS) facet_count_kernel(const FacetSlot *__restrict__ slots, uint32_t n_words, uint32_t n_docs) {
    __shared__ uint32_t s_cnt[FACET_SHARED_VALUES], s_first[FACET_SHARED_VALUES];
    const FacetSlot &sl = slots[blockIdx.y];
    const uint32_t V = sl.n_num + sl.n_str;
    const uint32_t w = blockIdx.x * COUNT_THREADS + threadIdx.x;
    unsigned long long bits = w < n_words ? __ldg(sl.cand + w) : 0ull;
    if ((uint64_t)w * 64 + 64 > n_docs) bits &= (uint64_t)w * 64 >= n_docs ? 0ull : (1ull << (n_docs - w * 64)) - 1;  // only documents
    if (!__syncthreads_or(bits != 0)) return;
    const bool in_shared = sl.doc_off && V <= FACET_SHARED_VALUES;
    if (in_shared) {
        for (uint32_t i = threadIdx.x; i < V; i += COUNT_THREADS) s_cnt[i] = s_first[i] = 0;
        __syncthreads();
    }
    uint32_t *cnt = in_shared ? s_cnt : sl.cnt, *first = in_shared ? s_first : sl.first;
    const uint32_t n_cand = (uint32_t)__popcll(bits);
    uint32_t min_inv = 0, max_p1 = 0;
    if (sl.doc_off)
        while (bits) {
            const uint32_t d = w * 64 + (uint32_t)__ffsll((long long)bits) - 1;
            bits &= bits - 1;
            const uint32_t o1 = __ldg(sl.doc_off + d + 1);
            for (uint32_t o = __ldg(sl.doc_off + d); o < o1; o++) {
                const uint32_t v = __ldg(sl.doc_ord + o);
                atomicAdd(cnt + v, 1u);
                atomicMax(first + v, ~d);
                if (v < sl.n_num) {
                    min_inv = max(min_inv, ~v);
                    max_p1 = max(max_p1, v + 1);
                }
            }
        }
    const uint32_t c = __reduce_add_sync(0xffffffffu, n_cand), mi = __reduce_max_sync(0xffffffffu, min_inv),
                   mx = __reduce_max_sync(0xffffffffu, max_p1);
    if ((threadIdx.x & 31) == 0) {
        if (c) atomicAdd(&sl.head->n_cand, (unsigned long long)c);
        if (mi) atomicMax(&sl.head->min_inv, mi);
        if (mx) atomicMax(&sl.head->max_p1, mx);
    }
    if (in_shared) {
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < V; i += COUNT_THREADS)
            if (s_cnt[i]) {
                atomicAdd(sl.cnt + i, s_cnt[i]);
                atomicMax(sl.first + i, s_first[i]);
            }
    }
}

// The first `limit` non-empty values among positions [0, n) (ordinal of position p: ord(p)), written to entries [at, ..) of the slot
// (those past `cap` are counted, not written).  Returns how many were taken: min(limit, non-empty values).
template <class Ord>
__device__ uint32_t take_first(const FacetSlot &sl, uint32_t n, Ord ord, uint32_t limit, uint32_t at, uint32_t *s_warp) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t taken = 0;
    for (uint32_t base = 0; base < n && taken < limit; base += SELECT_THREADS) {
        const uint32_t p = base + threadIdx.x;
        const uint32_t o = p < n ? ord(p) : 0u;
        const uint32_t c = p < n ? sl.cnt[o] : 0u;
        const unsigned ballot = __ballot_sync(0xffffffffu, c != 0);
        if (lane == 0) s_warp[warp] = (uint32_t)__popc(ballot);
        __syncthreads();
        uint32_t before = 0, total = 0;
        for (uint32_t k = 0; k < SELECT_THREADS / 32; k++) {
            before += k < warp ? s_warp[k] : 0u;
            total += s_warp[k];
        }
        const uint32_t k = taken + before + (uint32_t)__popc(ballot & ((1u << lane) - 1));
        if (c && k < limit && at + k < sl.cap) {
            sl.out_ord[at + k] = o;
            sl.out_cnt[at + k] = c;
            sl.out_doc[at + k] = ~sl.first[o];
        }
        __syncthreads();  // s_warp is rewritten by the next round
        taken = min(limit, taken + total);
    }
    return taken;
}

__global__ void __launch_bounds__(SELECT_THREADS) facet_select_kernel(const FacetSlot *__restrict__ slots) {
    __shared__ uint32_t s_warp[SELECT_THREADS / 32];
    const FacetSlot &sl = slots[blockIdx.x];
    const uint32_t max = sl.max_values;
    uint32_t n_num = 0, n_str = 0;
    if (sl.doc_off) {
        if (sl.head->n_cand > FACET_CANDIDATES_THRESHOLD) {
            // facet levels (facet_distribution.rs:181-253): each value is inserted, then the walk stops when the map holds `max`; the
            // strings' walk runs after the numbers' whatever happened there (:280-291), so once the numbers alone reached `max` the
            // map never holds exactly `max` again (the caller's merge stops at a first string colliding with a number)
            n_num = take_first(sl, sl.n_num, [](uint32_t p) { return p; }, max ? max : FACET_ALL, 0, s_warp);
            const uint32_t str_limit = n_num < max ? max : FACET_ALL;
            n_str = take_first(sl, sl.n_str, [&](uint32_t p) { return sl.n_num + p; }, str_limit, n_num, s_warp);
        } else {
            // from documents (:110-177): the first `max` numbers in Display-string order, then the first max - (numbers taken) strings
            n_num = take_first(sl, sl.n_num, [&](uint32_t p) { return __ldg(sl.disp + p); }, max, 0, s_warp);
            n_str = take_first(sl, sl.n_str, [&](uint32_t p) { return sl.n_num + p; }, max - n_num, n_num, s_warp);
        }
    }
    if (threadIdx.x == 0) {
        sl.out_sum[0] = n_num;
        sl.out_sum[1] = n_str;
        sl.out_sum[2] = sl.head->min_inv;
        sl.out_sum[3] = sl.head->max_p1;
    }
}

}  // namespace

cudaError_t launch_facet(cudaStream_t s, const FacetSlot *slots, uint32_t n_slots, uint32_t n_words, uint32_t n_docs) {
    if (!n_slots) return cudaSuccess;
    const dim3 grid((n_words + COUNT_THREADS - 1) / COUNT_THREADS, n_slots);
    if (grid.x) facet_count_kernel<<<grid, COUNT_THREADS, 0, s>>>(slots, n_words, n_docs);
    facet_select_kernel<<<n_slots, SELECT_THREADS, 0, s>>>(slots);
    return cudaGetLastError();
}

}  // namespace b200
