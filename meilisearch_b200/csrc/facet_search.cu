// Facet search (search/facet/search.rs:119-353) over candidate bitmaps, on the device.
//
// facet_search_match_kernel: one CTA per request sweeps its field's hyper-normalised strings in byte order, 256 at a time.  As in
// lev_match_kernel, every thread first filters its string (length, character-class signature; a plain prefix or an exact word is
// decided right there) and queues the survivors, then the queue runs the banded prefix-OSA DP densely.  A block-wide prefix over the
// matched strings' key counts appends their level-0 string keys to the request's item list, which is therefore in the reference's
// insertion order.  The None path lists the field's level-0 string keys in key order.
// facet_search_count_kernel: one warp per (request, item): a sparse posting list probes the candidate bitmap, a dense one is
// AND-popcounted against it, so the cost is the sum of the walked keys' list sizes and not |candidates|.
// facet_search_select_kernel: one CTA per request.  Lexicographic: the first `max` non-zero items.  Count: the cut count c (the
// max-th largest count) by bisection over block-wide counts, then every item with count >= c in insertion order; the host replays
// the reference's heap over them (only the items at c can be evicted, and which ones depends on the original strings).
#include <cuda_runtime.h>

#include "device_types.h"
#include "kernels.h"
#include "osa.cuh"

namespace b200 {

namespace {

constexpr uint32_t MATCH_THREADS = 256, COUNT_THREADS = 256, SELECT_THREADS = 256;

// exclusive prefix of v over the block and the block's total (blockDim.x == 256; s_warp: 8 u32)
__device__ __forceinline__ uint32_t block_scan(uint32_t v, uint32_t &total, uint32_t *s_warp) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= (uint32_t)o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    uint32_t before = 0;
    total = 0;
    for (uint32_t k = 0; k < 8; k++) {
        before += k < warp ? s_warp[k] : 0u;
        total += s_warp[k];
    }
    __syncthreads();  // s_warp is rewritten by the next call
    return before + x - v;
}

__device__ __forceinline__ uint32_t block_sum(uint32_t v, uint32_t *s_warp) {
    uint32_t total;
    block_scan(v, total, s_warp);
    return total;
}

__global__ void __launch_bounds__(MATCH_THREADS) facet_search_match_kernel(FsTables t, const FsReq *__restrict__ reqs, const uint32_t *__restrict__ q_chars) {
    __shared__ uint32_t s_q[FS_MAX_Q];
    __shared__ uint32_t s_warp[8], s_qn;
    __shared__ uint16_t s_queue[MATCH_THREADS];
    __shared__ uint8_t s_match[MATCH_THREADS];
    const FsReq &r = reqs[blockIdx.x];
    if (r.mode == FS_ALL) {
        for (uint32_t i = threadIdx.x; i < r.n_str; i += MATCH_THREADS) r.items[i] = r.k0 + i;
        if (threadIdx.x == 0) r.sum[0] = r.n_str;
        return;
    }
    const int m = (int)r.q_len, k = r.k;
    for (uint32_t i = threadIdx.x; i < (uint32_t)m; i += MATCH_THREADS) s_q[i] = q_chars[r.q_off + i];
    __syncthreads();
    const uint32_t qsig = char_signature(s_q, m);
    uint32_t n = 0;
    for (uint32_t base = r.h0; base < r.h1; base += MATCH_THREADS) {
        const uint32_t h = base + threadIdx.x;
        if (threadIdx.x == 0) s_qn = 0;
        __syncthreads();
        // phase 1: filter; a plain prefix (k = 0) or an exact word is decided here
        uint8_t match = 0;
        if (h < r.h1) {
            const uint32_t c0 = __ldg(t.char_off + h);
            const int wl = (int)(__ldg(t.char_off + h + 1) - c0);
            const uint32_t *w = t.chars + c0;
            if (r.mode == FS_EXACT || k == 0) {
                bool eq = r.mode == FS_EXACT ? wl == m : wl >= m;
                for (int i = 0; i < m && eq; i++) eq = __ldg(w + i) == s_q[i];
                match = eq;
            } else if (wl >= m - k && __popc(qsig & ~char_signature(w, min(wl, m + k))) <= k) {
                s_queue[atomicAdd(&s_qn, 1u)] = (uint16_t)threadIdx.x;
            }
        }
        s_match[threadIdx.x] = match;
        __syncthreads();
        // phase 2: the DP over the queue, densely
        for (uint32_t i = threadIdx.x; i < s_qn; i += MATCH_THREADS) {
            const uint32_t hh = base + s_queue[i];
            const uint32_t c0 = __ldg(t.char_off + hh);
            const int wl = (int)(__ldg(t.char_off + hh + 1) - c0);
            if (banded_osa(s_q, m, t.chars + c0, wl, k, true) <= k) s_match[s_queue[i]] = 1;
        }
        __syncthreads();
        // append the matched strings' keys in string order
        const uint32_t e0 = s_match[threadIdx.x] ? __ldg(t.csr_off + h) : 0u;
        const uint32_t len = s_match[threadIdx.x] ? __ldg(t.csr_off + h + 1) - e0 : 0u;
        uint32_t total;
        const uint32_t pos = n + block_scan(len, total, s_warp);
        for (uint32_t e = 0; e < len; e++) r.items[pos + e] = __ldg(t.csr_key + e0 + e);
        n += total;
    }
    if (threadIdx.x == 0) r.sum[0] = n;
}

__global__ void __launch_bounds__(COUNT_THREADS) facet_search_count_kernel(FsTables t, const FsReq *__restrict__ reqs, uint32_t n_words) {
    const FsReq &r = reqs[blockIdx.y];
    const uint32_t n = r.sum[0];
    const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (COUNT_THREADS / 32);
    for (uint32_t i = blockIdx.x * (COUNT_THREADS / 32) + (threadIdx.x >> 5); i < n; i += warps) {
        const DListRef L = t.lists[r.list_base + r.items[i]];
        uint32_t c = 0;
        if (L.dense) {
            const unsigned long long *words = reinterpret_cast<const unsigned long long *>(t.pool + L.off);
            for (uint32_t x = lane; x < n_words; x += 32) c += (uint32_t)__popcll(__ldg(words + x) & __ldg(r.cand + x));
        } else {
            const uint32_t *ids = t.pool + L.off;
            for (uint32_t x = lane; x < L.card; x += 32) {
                const uint32_t d = __ldg(ids + x);
                c += (uint32_t)(__ldg(r.cand + (d >> 6)) >> (d & 63)) & 1u;
            }
        }
        c = __reduce_add_sync(0xffffffffu, c);
        if (lane == 0) r.cnt[i] = c;
    }
}

__global__ void __launch_bounds__(SELECT_THREADS) facet_search_select_kernel(const FsReq *__restrict__ reqs, uint32_t *__restrict__ out_key,
                                                                             uint32_t *__restrict__ out_cnt, uint32_t *__restrict__ cursor) {
    __shared__ uint32_t s_warp[8], s_off;
    const FsReq &r = reqs[blockIdx.x];
    const uint32_t n = r.sum[0];
    // the number of non-zero items and the largest count
    uint32_t nz = 0, mx = 0;
    for (uint32_t i = threadIdx.x; i < n; i += SELECT_THREADS) {
        const uint32_t c = r.cnt[i];
        nz += c != 0;
        mx = max(mx, c);
    }
    const uint32_t n_hits = block_sum(nz, s_warp);
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = mx;
    __syncthreads();
    for (uint32_t k = 0; k < 8; k++) mx = max(mx, s_warp[k]);
    __syncthreads();
    const uint32_t target = min(r.max, n_hits);
    uint32_t cut = 1, take = target;
    if (r.by_count && target) {
        // the largest c with |{count >= c}| >= target: every item above it survives the heap, the ones at it are replayed on the host
        uint32_t lo = 1, hi = mx + 1, at_lo = n_hits;
        while (hi - lo > 1) {
            const uint32_t mid = lo + (hi - lo) / 2;
            uint32_t ge = 0;
            for (uint32_t i = threadIdx.x; i < n; i += SELECT_THREADS) ge += r.cnt[i] >= mid;
            ge = block_sum(ge, s_warp);
            if (ge >= target) {
                lo = mid;
                at_lo = ge;
            } else {
                hi = mid;
            }
        }
        cut = lo;
        take = at_lo;
    }
    if (threadIdx.x == 0) s_off = take ? atomicAdd(cursor, take) : 0u;
    __syncthreads();
    const uint32_t off = s_off;
    // the first `take` items with count >= cut, in insertion order
    uint32_t taken = 0;
    for (uint32_t base = 0; base < n && taken < take; base += SELECT_THREADS) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t c = i < n ? r.cnt[i] : 0u;
        const bool keep = c != 0 && c >= cut;
        uint32_t total;
        const uint32_t j = taken + block_scan(keep ? 1u : 0u, total, s_warp);
        if (keep && j < take) {
            out_key[off + j] = r.items[i];
            out_cnt[off + j] = c;
        }
        taken += total;
    }
    if (threadIdx.x == 0) {
        r.sum[1] = take;
        r.sum[2] = cut;
        r.sum[3] = off;
    }
}

}  // namespace

cudaError_t launch_facet_search_match(cudaStream_t s, const FsTables &t, const FsReq *reqs, uint32_t n, const uint32_t *q_chars) {
    if (!n) return cudaSuccess;
    facet_search_match_kernel<<<n, MATCH_THREADS, 0, s>>>(t, reqs, q_chars);
    return cudaGetLastError();
}

cudaError_t launch_facet_search_count(cudaStream_t s, const FsTables &t, const FsReq *reqs, uint32_t n, uint32_t max_items, uint32_t n_words) {
    if (!n || !max_items) return cudaSuccess;
    // enough warps for the largest request's items, at most 32 CTAs per request (the warps stride over the items)
    const dim3 grid(std::min<uint32_t>(32, (max_items + COUNT_THREADS / 32 - 1) / (COUNT_THREADS / 32)), n);
    facet_search_count_kernel<<<grid, COUNT_THREADS, 0, s>>>(t, reqs, n_words);
    return cudaGetLastError();
}

cudaError_t launch_facet_search_select(cudaStream_t s, const FsReq *reqs, uint32_t n, uint32_t *out_key, uint32_t *out_cnt, uint32_t *cursor) {
    if (!n) return cudaSuccess;
    facet_search_select_kernel<<<n, SELECT_THREADS, 0, s>>>(reqs, out_key, out_cnt, cursor);
    return cudaGetLastError();
}

}  // namespace b200
