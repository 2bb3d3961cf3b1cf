// Geo filters (search/facet/filter/index_filter.rs:465-696) on the device: `_geoRadius` and `_geoBoundingBox` clauses over the staged
// points (GeoPoint, the geo documents' bitmap).
//
// _geoRadius is `rtree.nearest_neighbor_iter(xyz(base)).take_while(haversine(base, p) <= radius + EPSILON)`: a prefix of the rtree
// order (squared chord distance d2, ties by docid), not a predicate.  Pass 1 finds, per radius clause, F = the smallest (d2, docid)
// of a point whose haversine exceeds the radius; pass 2 keeps the geo documents whose (d2, docid) < F.
// _geoBoundingBox is the AND of two inclusive range filters on the `_geo.lat` / `_geo.lng` number facets (the staged lat / lng),
// the longitude one split in two when the box wraps the antimeridian.
//
// Both passes stage GEO_FILTER_TILE_WORDS words of points per CTA in shared memory once and then loop over every clause (pass 1) or
// every slot (pass 2), so the points are read from HBM once per launch, not once per clause.
#include <cuda_runtime.h>

#include "device_types.h"
#include "geo_math.cuh"

namespace b200 {

namespace {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr uint32_t TILE_DOCS = GEO_FILTER_TILE_WORDS * 64;

// (key, doc) lexicographic minimum into *dst, by a 16-byte compare-and-swap
__device__ void first_min(GeoFirst *dst, unsigned long long key, unsigned long long doc) {
    const volatile GeoFirst *v = dst;
    GeoFirst cur{v->key, v->doc};  // a torn read only costs one more turn of the loop
    while (key < cur.key || (key == cur.key && doc < cur.doc)) {
        const GeoFirst prev = atomicCAS(dst, cur, GeoFirst{key, doc});
        if (prev.key == cur.key && prev.doc == cur.doc) return;
        cur = prev;
    }
}

// Pass 1.  One warp per clause at a time; a lane takes every 32nd document of the tile.  A point is decided by its squared chord d2
// alone unless lo <= d2 <= hi (the band, set on the host by geo_radius_band), where the haversine is computed; a haversine the
// device cannot place against the radius (geo_ambiguous) is listed for the host and passes here.  Among the points that fail, the
// lane keeps the smallest (d2, docid): documents come in ascending docid order, so a strict `<` on d2 keeps the smallest docid of a
// tie.
__global__ void __launch_bounds__(THREADS) geo_first_fail_kernel(const unsigned long long *__restrict__ geo, const GeoPoint *__restrict__ pts,
                                                                 uint32_t n_words, const GeoClause *__restrict__ clauses,
                                                                 const uint32_t *__restrict__ radius, uint32_t n_radius, GeoFirst *first,
                                                                 GeoAmb *amb, uint32_t amb_cap, uint32_t *amb_count) {
    __shared__ double sx[TILE_DOCS], sy[TILE_DOCS], sz[TILE_DOCS];
    __shared__ unsigned long long sgeo[GEO_FILTER_TILE_WORDS];
    const uint32_t w0 = blockIdx.x * GEO_FILTER_TILE_WORDS, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < GEO_FILTER_TILE_WORDS) sgeo[threadIdx.x] = w0 + threadIdx.x < n_words ? __ldg(geo + w0 + threadIdx.x) : 0ull;
    __syncthreads();
    bool any = false;
    for (uint32_t i = threadIdx.x; i < TILE_DOCS; i += THREADS)
        if (sgeo[i >> 6] >> (i & 63) & 1ull) {
            const GeoPoint &p = pts[(size_t)w0 * 64 + i];
            sx[i] = p.x;
            sy[i] = p.y;
            sz[i] = p.z;
            any = true;
        }
    if (!__syncthreads_or(any)) return;
    for (uint32_t c = warp; c < n_radius; c += WARPS) {
        const GeoClause &k = clauses[radius[c]];
        const double q[3] = {k.q[0], k.q[1], k.q[2]}, lo = k.lo, hi = k.hi, r_eps = k.r_eps;
        unsigned long long best = ~0ull, best_doc = ~0ull;
        for (uint32_t i = lane; i < TILE_DOCS; i += 32) {
            if (!(sgeo[i >> 6] >> (i & 63) & 1ull)) continue;
            const double d2 = chord2(q, sx[i], sy[i], sz[i]);
            const unsigned long long key = (unsigned long long)__double_as_longlong(d2);
            if (d2 < lo || key >= best) continue;
            const uint32_t doc = w0 * 64 + i;
            if (d2 <= hi) {
                const GeoPoint &p = pts[doc];
                const GeoDist g = geo_dist(k.t_lat, k.t_lng, k.t_cos_lat, p.lat, p.lng, p.cos_lat);
                if (geo_ambiguous(g, r_eps)) {
                    const uint32_t a = atomicAdd(amb_count, 1u);
                    if (a < amb_cap) amb[a] = GeoAmb{radius[c], doc, key};
                    continue;
                }
                if (g.m <= r_eps) continue;
            }
            best = key;
            best_doc = doc;
        }
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long ok = __shfl_xor_sync(0xffffffffu, best, o), od = __shfl_xor_sync(0xffffffffu, best_doc, o);
            if (ok < best || (ok == best && od < best_doc)) {
                best = ok;
                best_doc = od;
            }
        }
        if (lane == 0 && best != ~0ull) first_min(first + radius[c], best, best_doc);
    }
}

// Pass 2.  One warp per (slot, 64-document word): each clause's word is assembled by two ballots, complemented for NOT, and ANDed
// into the slot's universe word; a clause is skipped once the word is empty.
__global__ void __launch_bounds__(THREADS) geo_filter_kernel(const unsigned long long *__restrict__ geo, const GeoPoint *__restrict__ pts,
                                                             uint32_t n_words, const GeoClause *__restrict__ clauses,
                                                             const GeoFirst *__restrict__ first, const uint32_t *__restrict__ slot_clauses,
                                                             const GeoSlot *__restrict__ slots, uint32_t n_slots) {
    __shared__ double sx[TILE_DOCS], sy[TILE_DOCS], sz[TILE_DOCS], slat[TILE_DOCS], slng[TILE_DOCS];
    __shared__ unsigned long long sgeo[GEO_FILTER_TILE_WORDS];
    __shared__ unsigned int scount[GEO_FILTER_SLOT_CHUNK];
    const uint32_t w0 = blockIdx.x * GEO_FILTER_TILE_WORDS, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t tile_words = min(GEO_FILTER_TILE_WORDS, n_words - w0);
    if (threadIdx.x < GEO_FILTER_TILE_WORDS) sgeo[threadIdx.x] = threadIdx.x < tile_words ? __ldg(geo + w0 + threadIdx.x) : 0ull;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < TILE_DOCS; i += THREADS)
        if (sgeo[i >> 6] >> (i & 63) & 1ull) {
            const GeoPoint &p = pts[(size_t)w0 * 64 + i];
            sx[i] = p.x;
            sy[i] = p.y;
            sz[i] = p.z;
            slat[i] = p.lat;
            slng[i] = p.lng;
        }
    for (uint32_t s0 = 0; s0 < n_slots; s0 += GEO_FILTER_SLOT_CHUNK) {
        const uint32_t ns = min(GEO_FILTER_SLOT_CHUNK, n_slots - s0);
        for (uint32_t i = threadIdx.x; i < ns; i += THREADS) scount[i] = 0;
        __syncthreads();
        for (uint32_t t = warp; t < ns * tile_words; t += WARPS) {
            const GeoSlot &sl = slots[s0 + t / tile_words];
            const uint32_t wl = t % tile_words, w = w0 + wl;
            unsigned long long acc = __ldg(sl.ub + w);
            const unsigned long long g = sgeo[wl];
            for (uint32_t j = sl.c_begin; j < sl.c_end && acc; j++) {
                const uint32_t c = __ldg(slot_clauses + j);
                const GeoClause &k = clauses[c];
                bool in[2];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const uint32_t i = wl * 64 + h * 32 + lane;
                    if (!(g >> (h * 32 + lane) & 1ull)) {
                        in[h] = false;
                    } else if (k.kind == 0) {
                        const double q[3] = {k.q[0], k.q[1], k.q[2]};
                        const unsigned long long key = (unsigned long long)__double_as_longlong(chord2(q, sx[i], sy[i], sz[i]));
                        const GeoFirst f = first[c];
                        in[h] = key < f.key || (key == f.key && (unsigned long long)(w0 * 64 + i) < f.doc);
                    } else {
                        const double lat = slat[i], lng = slng[i];
                        const bool in_lng = k.right < k.left ? ((lng >= k.left && lng <= 180.0) || (lng >= -180.0 && lng <= k.right))
                                                             : (lng >= k.left && lng <= k.right);
                        in[h] = lat >= k.bottom && lat <= k.top && in_lng;
                    }
                }
                unsigned long long word = (unsigned long long)__ballot_sync(0xffffffffu, in[0]) | (unsigned long long)__ballot_sync(0xffffffffu, in[1]) << 32;
                if (k.neg) word = ~word;
                acc &= word;
            }
            if (lane == 0) {
                sl.dst[w] = acc;
                if (acc) atomicAdd(&scount[t / tile_words], (unsigned int)__popcll(acc));
            }
        }
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < ns; i += THREADS)
            if (scount[i]) atomicAdd(slots[s0 + i].count, (unsigned long long)scount[i]);
        __syncthreads();
    }
}

}  // namespace

cudaError_t launch_geo_first_fail(cudaStream_t s, const unsigned long long *geo, const GeoPoint *pts, uint32_t n_words, const GeoClause *clauses,
                                  const uint32_t *radius, uint32_t n_radius, GeoFirst *first, GeoAmb *amb, uint32_t amb_cap,
                                  uint32_t *amb_count) {
    if (!n_radius || !n_words) return cudaSuccess;
    const uint32_t tiles = (n_words + GEO_FILTER_TILE_WORDS - 1) / GEO_FILTER_TILE_WORDS;
    geo_first_fail_kernel<<<tiles, THREADS, 0, s>>>(geo, pts, n_words, clauses, radius, n_radius, first, amb, amb_cap, amb_count);
    return cudaGetLastError();
}

cudaError_t launch_geo_filter(cudaStream_t s, const unsigned long long *geo, const GeoPoint *pts, uint32_t n_words, const GeoClause *clauses,
                              const GeoFirst *first, const uint32_t *slot_clauses, const GeoSlot *slots, uint32_t n_slots) {
    if (!n_slots || !n_words) return cudaSuccess;
    const uint32_t tiles = (n_words + GEO_FILTER_TILE_WORDS - 1) / GEO_FILTER_TILE_WORDS;
    geo_filter_kernel<<<tiles, THREADS, 0, s>>>(geo, pts, n_words, clauses, first, slot_clauses, slots, n_slots);
    return cudaGetLastError();
}

}  // namespace b200
