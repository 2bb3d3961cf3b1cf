// Sort ranking rule (search/new/sort.rs) over a universe, on the device.
//
// Every document of a faceted field carries one u32 key per direction: the smallest ordinal among its values in the order a sort
// walks them, n_values when it has none (host_index.h SortField).  A stack of sort rules over a universe then orders the universe by
// the tuple (key_0, ..., key_{L-1}, docid): bucket_sort descends into the buckets of rule 0 in ascending key order, splits each one
// by rule 1, ..., and returns the buckets of the last rule in docid order (DESIGN.md §3).  One CTA produces the documents of ranks
// [lo, hi) of that order without sorting the universe:
//   1. select(r): the tuple of rank r by MSB-first radix select over the tuple's significant bits (up to 11 bits per pass, histogram
//      in shared memory); once at most SORT_COLLECT documents share the resolved prefix they are collected and sorted on chip;
//   2. the documents whose tuple lies in [tuple(lo), tuple(hi - 1)] (exactly hi - lo of them) are collected, sorted on chip and
//      written out with their keys (for the Sort scores).
// A warp reads one 64-document universe word at a time (lane l: documents 64w + l and 64w + 32 + l), so key reads coalesce.
#include <cuda_runtime.h>

#include "device_types.h"

namespace b200 {

namespace {

constexpr int SORT_THREADS = 1024;
constexpr int SORT_WARPS = SORT_THREADS / 32;
constexpr uint32_t SORT_DIGIT_BITS = 11;
constexpr uint32_t SORT_HIST = 1u << SORT_DIGIT_BITS;
constexpr uint32_t SORT_COLLECT = 4096;  // >= SORT_WINDOW
constexpr uint32_t SENTINEL = 0xffffffffu;
static_assert(SORT_COLLECT >= SORT_WINDOW, "the final window is collected in one buffer");

struct SortShared {
    uint32_t hist[SORT_HIST];
    uint32_t cand[SORT_COLLECT];
    uint32_t t_lo[SORT_MAX_LEVELS + 1], t_hi[SORT_MAX_LEVELS + 1];
    uint32_t n_cand;
    // select state
    uint32_t cw, done, r, eq;
};

__device__ __forceinline__ uint32_t tword(const SortDesc &d, uint32_t doc, uint32_t w) {
    if (w == d.n_levels) return doc;
    const uint32_t *k = d.keys[w];
    return k ? __ldg(k + doc) : 0u;
}

// lexicographic order of two documents' tuples (the docid word makes it total); SENTINEL sorts last
__device__ bool tless(const SortDesc &d, uint32_t a, uint32_t b) {
    if (a == SENTINEL) return false;
    if (b == SENTINEL) return true;
    for (uint32_t w = 0; w <= d.n_levels; w++) {
        uint32_t x = tword(d, a, w), y = tword(d, b, w);
        if (x != y) return x < y;
    }
    return false;
}

// -1 / 0 / 1: the document's tuple against T
__device__ int tcmp(const SortDesc &d, uint32_t doc, const uint32_t *T) {
    for (uint32_t w = 0; w <= d.n_levels; w++) {
        uint32_t x = tword(d, doc, w);
        if (x != T[w]) return x < T[w] ? -1 : 1;
    }
    return 0;
}

// the document's tuple starts with the resolved prefix: words [0, cw) equal, and the top `done` bits of word cw
__device__ __forceinline__ bool prefix_match(const SortDesc &d, uint32_t doc, const uint32_t *T, uint32_t cw, uint32_t done) {
    for (uint32_t w = 0; w < cw; w++)
        if (tword(d, doc, w) != T[w]) return false;
    if (done == 0 || cw > d.n_levels) return true;
    const uint32_t sh = d.bits[cw] - done;
    return (tword(d, doc, cw) >> sh) == (T[cw] >> sh);
}

// calls f(doc) for every document of the universe (warp-cooperative over 64-document words)
template <class F>
__device__ __forceinline__ void for_each_doc(const SortDesc &d, F f) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t w = warp; w < d.n_words; w += SORT_WARPS) {
        const unsigned long long bits = __ldg(d.ub + w);
        if (!bits) continue;
        if ((bits >> lane) & 1ull) f(w * 64 + lane);
        if ((bits >> (lane + 32)) & 1ull) f(w * 64 + 32 + lane);
    }
}

// bitonic sort of cand[0, n) by tuple (n <= SORT_COLLECT; padded with SENTINEL up to a power of two)
__device__ void sort_cand(const SortDesc &d, SortShared &s, uint32_t n) {
    uint32_t P = 1;
    while (P < n) P <<= 1;
    for (uint32_t i = n + threadIdx.x; i < P; i += SORT_THREADS) s.cand[i] = SENTINEL;
    __syncthreads();
    for (uint32_t k = 2; k <= P; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < P; i += SORT_THREADS) {
                const uint32_t ixj = i ^ j;
                if (ixj > i) {
                    const uint32_t a = s.cand[i], b = s.cand[ixj];
                    const bool up = (i & k) == 0;
                    if (up ? tless(d, b, a) : tless(d, a, b)) {
                        s.cand[i] = b;
                        s.cand[ixj] = a;
                    }
                }
            }
            __syncthreads();
        }
}

__device__ __forceinline__ void skip_empty_words(const SortDesc &d, SortShared &s, uint32_t *T) {
    while (s.cw <= d.n_levels && s.done == d.bits[s.cw]) {
        if (s.done == 0) T[s.cw] = 0;
        s.cw++;
        s.done = 0;
    }
}

// T = tuple of the document of rank r (0-based) of the universe; returns the number of universe passes
__device__ uint32_t select_rank(const SortDesc &d, SortShared &s, uint32_t r, uint32_t *T) {
    uint32_t passes = 0;
    if (threadIdx.x == 0) {
        s.cw = 0;
        s.done = 0;
        s.r = r;
        s.eq = SENTINEL;
        for (uint32_t w = 0; w <= d.n_levels; w++) T[w] = 0;
        skip_empty_words(d, s, T);
    }
    __syncthreads();
    for (;;) {
        const uint32_t cw = s.cw, done = s.done;
        if (s.eq <= SORT_COLLECT || cw > d.n_levels) break;
        const uint32_t nb = min(SORT_DIGIT_BITS, d.bits[cw] - done), sh = d.bits[cw] - done - nb, mask = (1u << nb) - 1u;
        for (uint32_t i = threadIdx.x; i < SORT_HIST; i += SORT_THREADS) s.hist[i] = 0;
        __syncthreads();
        for_each_doc(d, [&](uint32_t doc) {
            if (prefix_match(d, doc, T, cw, done)) atomicAdd(&s.hist[(tword(d, doc, cw) >> sh) & mask], 1u);
        });
        passes++;
        __syncthreads();
        if (threadIdx.x < 32) {
            // warp 0: lane l owns digits [64 l, 64 l + 64); find the digit whose cumulative count passes r
            const uint32_t lane = threadIdx.x, per = SORT_HIST / 32;
            uint32_t sum = 0;
            for (uint32_t i = 0; i < per; i++) sum += s.hist[lane * per + i];
            uint32_t incl = sum;
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                if ((int)lane >= o) incl += v;
            }
            const uint32_t excl = incl - sum, rr = s.r;
            const bool mine = rr >= excl && rr < incl;
            // r beyond the documents of the prefix cannot happen when hi <= |universe|; stop rather than loop
            if (lane == 31 && rr >= incl) s.eq = 0;
            if (mine) {
                uint32_t c = excl, dig = lane * per;
                while (c + s.hist[dig] <= rr) c += s.hist[dig++];
                T[cw] |= dig << sh;
                s.r = rr - c;
                s.eq = s.hist[dig];
                s.done = done + nb;
                skip_empty_words(d, s, T);
            }
        }
        __syncthreads();
    }
    // at most SORT_COLLECT documents share the resolved prefix: collect them, sort them, take the one of rank s.r among them
    const uint32_t cw = s.cw, done = s.done;
    if (threadIdx.x == 0) s.n_cand = 0;
    __syncthreads();
    for_each_doc(d, [&](uint32_t doc) {
        if (prefix_match(d, doc, T, cw, done)) {
            uint32_t at = atomicAdd(&s.n_cand, 1u);
            if (at < SORT_COLLECT) s.cand[at] = doc;
        }
    });
    passes++;
    __syncthreads();
    const uint32_t n = min(s.n_cand, SORT_COLLECT);
    sort_cand(d, s, n);
    if (threadIdx.x == 0 && n > 0) {
        const uint32_t doc = s.cand[min(s.r, n - 1)];
        for (uint32_t w = 0; w <= d.n_levels; w++) T[w] = tword(d, doc, w);
    }
    __syncthreads();
    return passes;
}

__global__ void __launch_bounds__(SORT_THREADS) sort_window_kernel(const SortDesc *__restrict__ descs, uint32_t n_descs) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SortShared &s = *reinterpret_cast<SortShared *>(smem_raw);
    const SortDesc &d = descs[blockIdx.x];
    if (d.hi <= d.lo) return;
    uint32_t passes = 0;
    if (d.lo > 0) passes += select_rank(d, s, d.lo, s.t_lo);
    passes += select_rank(d, s, d.hi - 1, s.t_hi);
    if (threadIdx.x == 0) s.n_cand = 0;
    __syncthreads();
    const bool from_first = d.lo == 0;
    for_each_doc(d, [&](uint32_t doc) {
        if ((from_first || tcmp(d, doc, s.t_lo) >= 0) && tcmp(d, doc, s.t_hi) <= 0) {
            uint32_t at = atomicAdd(&s.n_cand, 1u);
            if (at < SORT_COLLECT) s.cand[at] = doc;
        }
    });
    passes++;
    __syncthreads();
    const uint32_t n = min(s.n_cand, d.hi - d.lo);
    sort_cand(d, s, min(s.n_cand, SORT_COLLECT));
    for (uint32_t i = threadIdx.x; i < n; i += SORT_THREADS) {
        const uint32_t doc = s.cand[i];
        d.dst[i] = doc;
        for (uint32_t l = 0; l < d.n_levels; l++) d.dst_keys[(size_t)i * d.n_levels + l] = tword(d, doc, l);
    }
    if (threadIdx.x == 0) {
        d.info[0] = passes;
        d.info[1] = s.n_cand;
    }
}

}  // namespace

cudaError_t launch_sort_window(cudaStream_t s, const SortDesc *descs, uint32_t n_descs) {
    if (!n_descs) return cudaSuccess;
    static_assert(sizeof(SortShared) <= 48 * 1024, "default dynamic shared-memory limit");
    sort_window_kernel<<<n_descs, SORT_THREADS, sizeof(SortShared), s>>>(descs, n_descs);
    return cudaGetLastError();
}

}  // namespace b200
