// GeoSort ranking rule (search/new/geo_sort.rs, documents/geo_sort.rs) on the device: windows of the order in which the rule's
// cache hands out the geo documents of a universe.
//
// The order (DESIGN.md §3) is a tuple order, so the windows come from the radix select of tuple_select.cuh, with the tuple words
// computed from each document's point as they are read (GeoDesc in device_types.h):
//   rtree:     squared Euclidean distance between lat_lng_to_xyz of the point and of the target (its antipode when descending), as
//              rstar's nearest_neighbor_iter ranks points (((dx*dx) + dy*dy) + dz*dz); ties by docid;
//   iterative: floor of the haversine distance (geoutils, R = 6371000 m), a stable sort by docid; reversed when descending.
// Points and cos(lat) are staged as computed by the host's libm; the squared distance is rounded exactly as on the host (no fused
// multiply-add), so rtree keys are bit-identical.  The haversine uses the device's sin / atan2 (within a few ULP of the host's).
#include <cuda_runtime.h>

#include "device_types.h"
#include "tuple_select.cuh"

namespace b200 {

namespace {

constexpr double EARTH_RADIUS_M = 6371000.0;

// Location::haversine_distance_to (geoutils), from the target (t) to the point (p).  sin(to_radians(d) / 2) is taken as
// sinpi(d / 360): both are within a few ULP of the true value, and sinpi needs no slow-path argument reduction (a call that
// spills registers).
__device__ __forceinline__ double haversine_m(double t_lat, double t_lng, double t_cos_lat, const GeoPoint &p) {
    const double s_lat = sinpi(__ddiv_rn(__dsub_rn(p.lat, t_lat), 360.0)), s_lng = sinpi(__ddiv_rn(__dsub_rn(p.lng, t_lng), 360.0));
    const double a = __dadd_rn(__dmul_rn(s_lat, s_lat), __dmul_rn(__dmul_rn(__dmul_rn(s_lng, s_lng), t_cos_lat), p.cos_lat));
    const double c = __dmul_rn(2.0, atan2(__dsqrt_rn(a), __dsqrt_rn(__dsub_rn(1.0, a))));
    return __dmul_rn(c, EARTH_RADIUS_M);
}

__device__ __forceinline__ unsigned long long rtree_key(const double *q, const GeoPoint &p) {
    const double dx = __dsub_rn(p.x, q[0]), dy = __dsub_rn(p.y, q[1]), dz = __dsub_rn(p.z, q[2]);
    const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
    return (unsigned long long)__double_as_longlong(d2);  // >= 0: the bits order as the values
}

__device__ __forceinline__ uint32_t floor_m(double m) { return (uint32_t)min(m, (double)GEO_FLOOR_MAX); }

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
                const uint32_t f = floor_m(haversine_m(d.t_lat, d.t_lng, d.t_cos_lat, p));
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
        d.dst_dist[i] = haversine_m(d.t_lat, d.t_lng, d.t_cos_lat, p);
        d.dst_key[i] = rtree_key(d.q, p);
    }
};

__global__ void __launch_bounds__(GeoView::THREADS) geo_window_kernel(const GeoDesc *__restrict__ descs, uint32_t n_descs) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    tsel::SelShared &s = *reinterpret_cast<tsel::SelShared *>(smem_raw);
    const GeoView v(descs[blockIdx.x]);
    tsel::window(v, s);
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

cudaError_t launch_geo_window(cudaStream_t s, const GeoDesc *descs, uint32_t n_descs) {
    if (!n_descs) return cudaSuccess;
    static_assert(sizeof(tsel::SelShared) <= 48 * 1024, "default dynamic shared-memory limit");
    geo_window_kernel<<<n_descs, GeoView::THREADS, sizeof(tsel::SelShared), s>>>(descs, n_descs);
    return cudaGetLastError();
}

}  // namespace b200
