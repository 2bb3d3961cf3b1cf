// GeoSort ranking rule (search/new/geo_sort.rs, documents/geo_sort.rs) on the device: windows of the order in which the rule's
// cache hands out the geo documents of a universe.
//
// The order (DESIGN.md §3) is a tuple order, so the windows come from the radix select of tuple_select.cuh, with the tuple words
// computed from each document's point as they are read (GeoDesc in device_types.h):
//   rtree:     squared Euclidean distance between lat_lng_to_xyz of the point and of the target (its antipode when descending), as
//              rstar's nearest_neighbor_iter ranks points (((dx*dx) + dy*dy) + dz*dz); ties by docid;
//   iterative: floor of the haversine distance (geoutils, R = 6371000 m), a stable sort by docid; reversed when descending.
// The distances are those of geo_math.cuh.  A floor the device cannot decide (geo_ambiguous) comes from the host's patch: the
// documents are listed by geo_ambiguous_kernel before the windows are selected.
#include <cuda_runtime.h>

#include "device_types.h"
#include "geo_math.cuh"
#include "tuple_select.cuh"

namespace b200 {

namespace {

// the iterative key: floor metres, or the host's where the device's distance is ambiguous
__device__ __forceinline__ uint32_t iterative_floor(const GeoDesc &d, uint32_t doc, const GeoPoint &p) {
    const GeoDist g = geo_dist(d.t_lat, d.t_lng, d.t_cos_lat, p.lat, p.lng, p.cos_lat);
    uint32_t f = floor_m(g.m);
    if (d.n_patch && geo_ambiguous(g, floor_threshold(g.m))) {
        uint32_t lo = 0, hi = d.n_patch;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) / 2;
            if ((uint32_t)(d.patch[mid] >> 32) < doc) lo = mid + 1;
            else hi = mid;
        }
        if (lo < d.n_patch && (uint32_t)(d.patch[lo] >> 32) == doc) f = (uint32_t)d.patch[lo];
    }
    return f;
}

struct GeoView {
    static constexpr int THREADS = 512;
    static constexpr int WARPS = THREADS / 32;
    static constexpr uint32_t n_levels = 4;
    const GeoDesc &d;
    const uint32_t *bits;
    uint32_t lo, hi;
    uint32_t *info;
    __device__ explicit GeoView(const GeoDesc &x) : d(x), bits(x.bits), lo(x.lo), hi(x.hi), info(x.info) {}
    // the document comes in iterative order (mode 1, or mode 2 past the split)
    __device__ __forceinline__ bool iterative(uint32_t doc, unsigned long long key) const {
        if (d.mode != 2) return d.mode == 1;
        return key > d.split_key || (key == d.split_key && doc > d.split_doc);
    }
    __device__ uint32_t word(uint32_t doc, uint32_t w) const {
        if (w == n_levels) return doc;
        const GeoPoint p = d.pts[doc];
        const unsigned long long key = d.mode == 1 ? 0ull : rtree_key(d.q, p);
        const bool it = iterative(doc, key);
        switch (w) {
            case 0: return d.mode == 2 && it ? 1u : 0u;
            case 1: return it ? 0u : (uint32_t)(key >> 32);
            case 2: {
                if (!it) return (uint32_t)key;
                const uint32_t f = iterative_floor(d, doc, p);
                return d.asc ? f : GEO_FLOOR_MAX - f;
            }
            default: return it && !d.asc ? d.doc_max - doc : 0u;
        }
    }
    template <class F>
    __device__ __forceinline__ void for_each_doc(F f) const {
        const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (uint32_t w = warp; w < d.n_words; w += WARPS) {
            const unsigned long long bits = __ldg(d.ub + w) & __ldg(d.geo + w);
            if (!bits) continue;
            if ((bits >> lane) & 1ull) f(w * 64 + lane);
            if ((bits >> (lane + 32)) & 1ull) f(w * 64 + 32 + lane);
        }
    }
    __device__ void emit(uint32_t i, uint32_t doc) const {
        const GeoPoint p = d.pts[doc];
        d.dst[i] = doc;
        d.dst_key[i] = rtree_key(d.q, p);
    }
};

__global__ void __launch_bounds__(GeoView::THREADS) geo_window_kernel(const GeoDesc *__restrict__ descs, uint32_t n_descs) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    tsel::SelShared &s = *reinterpret_cast<tsel::SelShared *>(smem_raw);
    const GeoView v(descs[blockIdx.x]);
    tsel::window(v, s);
}

// The documents of universe AND geo whose floor metres the device cannot decide, for the host to decide (one CTA per descriptor).
__global__ void __launch_bounds__(GeoView::THREADS) geo_ambiguous_kernel(const GeoDesc *__restrict__ descs, uint32_t n_descs) {
    const GeoDesc &d = descs[blockIdx.x];
    const GeoView v(d);
    v.for_each_doc([&](uint32_t doc) {
        const GeoPoint p = d.pts[doc];
        const GeoDist g = geo_dist(d.t_lat, d.t_lng, d.t_cos_lat, p.lat, p.lng, p.cos_lat);
        if (!geo_ambiguous(g, floor_threshold(g.m))) return;
        const uint32_t k = atomicAdd(d.amb_count, 1u);
        if (k < d.amb_cap) d.amb[k] = doc;
    });
}

constexpr int COUNT_THREADS = 512;

__global__ void __launch_bounds__(COUNT_THREADS) geo_count_kernel(const GeoCount *__restrict__ counts, uint32_t n) {
    __shared__ uint32_t part[COUNT_THREADS / 32];
    const GeoCount &c = counts[blockIdx.x];
    uint32_t t = 0;
    for (uint32_t w = threadIdx.x; w < c.n_words; w += COUNT_THREADS) t += __popcll(__ldg(c.ub + w) & __ldg(c.geo + w));
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t sum = 0;
        for (int i = 0; i < COUNT_THREADS / 32; i++) sum += part[i];
        *c.out = sum;
    }
}

}  // namespace

cudaError_t launch_geo_count(cudaStream_t s, const GeoCount *counts, uint32_t n) {
    if (!n) return cudaSuccess;
    geo_count_kernel<<<n, COUNT_THREADS, 0, s>>>(counts, n);
    return cudaGetLastError();
}

cudaError_t launch_geo_ambiguous(cudaStream_t s, const GeoDesc *descs, uint32_t n_descs) {
    if (!n_descs) return cudaSuccess;
    geo_ambiguous_kernel<<<n_descs, GeoView::THREADS, 0, s>>>(descs, n_descs);
    return cudaGetLastError();
}

cudaError_t launch_geo_window(cudaStream_t s, const GeoDesc *descs, uint32_t n_descs) {
    if (!n_descs) return cudaSuccess;
    static_assert(sizeof(tsel::SelShared) <= 48 * 1024, "default dynamic shared-memory limit");
    geo_window_kernel<<<n_descs, GeoView::THREADS, sizeof(tsel::SelShared), s>>>(descs, n_descs);
    return cudaGetLastError();
}

}  // namespace b200
