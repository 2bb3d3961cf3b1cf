// Window of a tuple order over a document set, on the device: the documents of ranks [lo, hi) of a set ordered by a tuple of u32
// words whose last word is the docid.  Shared by the Sort rule (sort.cu) and the GeoSort rule (geo.cu); one CTA per window:
//   1. select(r): the tuple of rank r by MSB-first radix select over the tuple's significant bits (up to 11 bits per pass, histogram
//      in shared memory); once at most SEL_COLLECT documents share the resolved prefix they are collected and sorted on chip;
//   2. the documents whose tuple lies in [tuple(lo), tuple(hi - 1)] (exactly hi - lo of them) are collected, sorted on chip and
//      handed to the view's emit().
// A view V provides: THREADS (the CTA size), n_levels (the docid is word n_levels), bits[] (significant bits of each word),
// lo / hi / info, word(doc, w) (< 2^bits[w]), for_each_doc(f) over the set, and emit(row, doc).
#pragma once
#include <cuda_runtime.h>

#include "device_types.h"

namespace b200 {
namespace tsel {

constexpr uint32_t SEL_DIGIT_BITS = 11;
constexpr uint32_t SEL_HIST = 1u << SEL_DIGIT_BITS;
constexpr uint32_t SEL_COLLECT = 4096;  // >= SORT_WINDOW
constexpr uint32_t SEL_MAX_WORDS = 16;  // tuple words, docid included
constexpr uint32_t SENTINEL = 0xffffffffu;
static_assert(SEL_COLLECT >= SORT_WINDOW, "the final window is collected in one buffer");
static_assert(SEL_MAX_WORDS >= SORT_MAX_LEVELS + 1, "a Sort tuple fits");

struct SelShared {
    uint32_t hist[SEL_HIST];
    uint32_t cand[SEL_COLLECT];
    uint32_t t_lo[SEL_MAX_WORDS], t_hi[SEL_MAX_WORDS];
    uint32_t n_cand;
    // select state
    uint32_t cw, done, r, eq;
};

// lexicographic order of two documents' tuples (the docid word makes it total); SENTINEL sorts last
template <class V>
__device__ bool tless(const V &d, uint32_t a, uint32_t b) {
    if (a == SENTINEL) return false;
    if (b == SENTINEL) return true;
    for (uint32_t w = 0; w <= d.n_levels; w++) {
        uint32_t x = d.word(a, w), y = d.word(b, w);
        if (x != y) return x < y;
    }
    return false;
}

// -1 / 0 / 1: the document's tuple against T
template <class V>
__device__ int tcmp(const V &d, uint32_t doc, const uint32_t *T) {
    for (uint32_t w = 0; w <= d.n_levels; w++) {
        uint32_t x = d.word(doc, w);
        if (x != T[w]) return x < T[w] ? -1 : 1;
    }
    return 0;
}

// the document's tuple starts with the resolved prefix: words [0, cw) equal, and the top `done` bits of word cw
template <class V>
__device__ __forceinline__ bool prefix_match(const V &d, uint32_t doc, const uint32_t *T, uint32_t cw, uint32_t done) {
    for (uint32_t w = 0; w < cw; w++)
        if (d.word(doc, w) != T[w]) return false;
    if (done == 0 || cw > d.n_levels) return true;
    const uint32_t sh = d.bits[cw] - done;
    return (d.word(doc, cw) >> sh) == (T[cw] >> sh);
}

// bitonic sort of cand[0, n) by tuple (n <= SEL_COLLECT; padded with SENTINEL up to a power of two)
template <class V>
__device__ void sort_cand(const V &d, SelShared &s, uint32_t n) {
    uint32_t P = 1;
    while (P < n) P <<= 1;
    for (uint32_t i = n + threadIdx.x; i < P; i += V::THREADS) s.cand[i] = SENTINEL;
    __syncthreads();
    for (uint32_t k = 2; k <= P; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < P; i += V::THREADS) {
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

template <class V>
__device__ __forceinline__ void skip_empty_words(const V &d, SelShared &s, uint32_t *T) {
    while (s.cw <= d.n_levels && s.done == d.bits[s.cw]) {
        if (s.done == 0) T[s.cw] = 0;
        s.cw++;
        s.done = 0;
    }
}

// T = tuple of the document of rank r (0-based) of the set; returns the number of passes over the set
template <class V>
__device__ uint32_t select_rank(const V &d, SelShared &s, uint32_t r, uint32_t *T) {
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
        if (s.eq <= SEL_COLLECT || cw > d.n_levels) break;
        const uint32_t nb = min(SEL_DIGIT_BITS, d.bits[cw] - done), sh = d.bits[cw] - done - nb, mask = (1u << nb) - 1u;
        for (uint32_t i = threadIdx.x; i < SEL_HIST; i += V::THREADS) s.hist[i] = 0;
        __syncthreads();
        d.for_each_doc([&](uint32_t doc) {
            if (prefix_match(d, doc, T, cw, done)) atomicAdd(&s.hist[(d.word(doc, cw) >> sh) & mask], 1u);
        });
        passes++;
        __syncthreads();
        if (threadIdx.x < 32) {
            // warp 0: lane l owns digits [64 l, 64 l + 64); find the digit whose cumulative count passes r
            const uint32_t lane = threadIdx.x, per = SEL_HIST / 32;
            uint32_t sum = 0;
            for (uint32_t i = 0; i < per; i++) sum += s.hist[lane * per + i];
            uint32_t incl = sum;
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                if ((int)lane >= o) incl += v;
            }
            const uint32_t excl = incl - sum, rr = s.r;
            const bool mine = rr >= excl && rr < incl;
            // r beyond the documents of the prefix cannot happen when hi <= |set|; stop rather than loop
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
    // at most SEL_COLLECT documents share the resolved prefix: collect them, sort them, take the one of rank s.r among them
    const uint32_t cw = s.cw, done = s.done;
    if (threadIdx.x == 0) s.n_cand = 0;
    __syncthreads();
    d.for_each_doc([&](uint32_t doc) {
        if (prefix_match(d, doc, T, cw, done)) {
            uint32_t at = atomicAdd(&s.n_cand, 1u);
            if (at < SEL_COLLECT) s.cand[at] = doc;
        }
    });
    passes++;
    __syncthreads();
    const uint32_t n = min(s.n_cand, SEL_COLLECT);
    sort_cand(d, s, n);
    if (threadIdx.x == 0 && n > 0) {
        const uint32_t doc = s.cand[min(s.r, n - 1)];
        for (uint32_t w = 0; w <= d.n_levels; w++) T[w] = d.word(doc, w);
    }
    __syncthreads();
    return passes;
}

// the window [lo, hi) of the view's order: emit(row, doc) for row in [0, hi - lo); info[0] = passes, info[1] = documents collected
template <class V>
__device__ void window(const V &d, SelShared &s) {
    if (d.hi <= d.lo) return;
    uint32_t passes = 0;
    if (d.lo > 0) passes += select_rank(d, s, d.lo, s.t_lo);
    passes += select_rank(d, s, d.hi - 1, s.t_hi);
    if (threadIdx.x == 0) s.n_cand = 0;
    __syncthreads();
    const bool from_first = d.lo == 0;
    d.for_each_doc([&](uint32_t doc) {
        if ((from_first || tcmp(d, doc, s.t_lo) >= 0) && tcmp(d, doc, s.t_hi) <= 0) {
            uint32_t at = atomicAdd(&s.n_cand, 1u);
            if (at < SEL_COLLECT) s.cand[at] = doc;
        }
    });
    passes++;
    __syncthreads();
    const uint32_t n = min(s.n_cand, d.hi - d.lo);
    sort_cand(d, s, min(s.n_cand, SEL_COLLECT));
    for (uint32_t i = threadIdx.x; i < n; i += V::THREADS) d.emit(i, s.cand[i]);
    if (threadIdx.x == 0) {
        d.info[0] = passes;
        d.info[1] = s.n_cand;
    }
}

}  // namespace tsel
}  // namespace b200
