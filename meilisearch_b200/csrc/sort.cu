// Sort ranking rule (search/new/sort.rs) over a universe, on the device.
//
// Every document of a faceted field carries one u32 key per direction: the smallest ordinal among its values in the order a sort
// walks them, n_values when it has none (host_index.h SortField).  A stack of sort rules over a universe then orders the universe by
// the tuple (key_0, ..., key_{L-1}, docid): bucket_sort descends into the buckets of rule 0 in ascending key order, splits each one
// by rule 1, ..., and returns the buckets of the last rule in docid order (DESIGN.md §3).  One CTA produces the documents of ranks
// [lo, hi) of that order without sorting the universe (tuple_select.cuh).  The universe is a dense bitmap, optionally minus a second
// bitmap (the Null bucket of a GeoSort rule: the universe without its geo documents), or a list of docids (one GeoSort bucket).
// Over a bitmap a warp reads one 64-document word at a time (lane l: documents 64w + l and 64w + 32 + l), so key reads coalesce.
#include <cuda_runtime.h>

#include "device_types.h"
#include "tuple_select.cuh"

namespace b200 {

namespace {

struct SortView {
    static constexpr int THREADS = 1024;
    static constexpr int WARPS = THREADS / 32;
    const SortDesc &d;
    const uint32_t *bits;
    uint32_t n_levels, lo, hi;
    uint32_t *info;
    __device__ explicit SortView(const SortDesc &x) : d(x), bits(x.bits), n_levels(x.n_levels), lo(x.lo), hi(x.hi), info(x.info) {}
    __device__ __forceinline__ uint32_t word(uint32_t doc, uint32_t w) const {
        if (w == d.n_levels) return doc;
        const uint32_t *k = d.keys[w];
        return k ? __ldg(k + doc) : 0u;
    }
    template <class F>
    __device__ __forceinline__ void for_each_doc(F f) const {
        if (d.ids) {
            for (uint32_t i = threadIdx.x; i < d.n_ids; i += THREADS) f(__ldg(d.ids + i));
            return;
        }
        const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (uint32_t w = warp; w < d.n_words; w += WARPS) {
            unsigned long long bits = __ldg(d.ub + w);
            if (d.exclude) bits &= ~__ldg(d.exclude + w);
            if (!bits) continue;
            if ((bits >> lane) & 1ull) f(w * 64 + lane);
            if ((bits >> (lane + 32)) & 1ull) f(w * 64 + 32 + lane);
        }
    }
    __device__ __forceinline__ void emit(uint32_t i, uint32_t doc) const {
        d.dst[i] = doc;
        for (uint32_t l = 0; l < d.n_levels; l++) d.dst_keys[(size_t)i * d.n_levels + l] = word(doc, l);
    }
};

__global__ void __launch_bounds__(SortView::THREADS) sort_window_kernel(const SortDesc *__restrict__ descs, uint32_t n_descs) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    tsel::SelShared &s = *reinterpret_cast<tsel::SelShared *>(smem_raw);
    const SortView v(descs[blockIdx.x]);
    tsel::window(v, s);
}

}  // namespace

cudaError_t launch_sort_window(cudaStream_t s, const SortDesc *descs, uint32_t n_descs) {
    if (!n_descs) return cudaSuccess;
    static_assert(sizeof(tsel::SelShared) <= 48 * 1024, "default dynamic shared-memory limit");
    sort_window_kernel<<<n_descs, SortView::THREADS, sizeof(tsel::SelShared), s>>>(descs, n_descs);
    return cudaGetLastError();
}

}  // namespace b200
