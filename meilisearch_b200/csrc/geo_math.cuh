// The two distances of the reference's geo code, shared by GeoSort (geo.cu) and the geo filters (geo_filter.cu), and the decisions
// the reference takes on them.
// Points and cos(lat) are staged as computed by the host's libm; the squared distance is rounded exactly as on the host (no fused
// multiply-add), so rtree keys are bit-identical.  The haversine follows the reference's operations one rounding at a time, but its
// sin / atan2 are the device's, which differ from the host libm's by a few ULP; near the antipode, where 1 - a cancels, that grows
// to metres.  A haversine decision (a floor, a radius) whose device distance lies within the tolerance of geo_ambiguous of its threshold is
// ambiguous and taken on the host with libm (engine_geo.cpp, engine_search.cpp).  tests/test_gpu_geo_probe.py measures the device's
// error against the host and asserts that GEO_TAU keeps a 4x margin over it.
#pragma once
#include <cuda_runtime.h>

#include "device_types.h"

namespace b200 {

constexpr double EARTH_RADIUS_M = 6371000.0;
constexpr double GEO_DEG_TO_RAD = 3.14159265358979323846 / 180.0;  // f64::to_radians's factor, rounded once
// past this distance a is within a few ULP of 1: the host may compute a > 1 (a NaN distance) where the device does not
constexpr double GEO_ANTIPODE_M = 3.14159265358979323846 * EARTH_RADIUS_M - 1.0;
// |device haversine - host haversine| <= GEO_TAU * (max(h, 1) + R / sqrt(1 - a)): the first term covers the few ULP of relative
// error of sin / atan2, the second the cancellation in 1 - a (an absolute error of a few ULP of 1 in a moves the angle by that over
// sqrt(a (1 - a))).  The probe measured 1.66 x 2^-52 on an H100: a 154x margin (DESIGN.md, "Geo decisions at their last bits").
constexpr double GEO_TAU = 0x1p-44;

// a haversine in metres and sqrt(1 - a), the factor its error grows with near the antipode
struct GeoDist {
    double m, c1;
};

// Location::haversine_distance_to (geoutils), from the target (t) to the point (p), operation for operation:
//   sin(to_radians(p - t) / 2), a = s_lat^2 + ((s_lng^2 cos t) cos p), 2 atan2(sqrt(a), sqrt(1 - a)) R.
// a > 1 gives sqrt(negative) = NaN, and NaN propagates, as in Rust.
__device__ __forceinline__ GeoDist geo_dist(double t_lat, double t_lng, double t_cos_lat, double p_lat, double p_lng, double p_cos_lat) {
    const double s_lat = sin(__dmul_rn(__dmul_rn(__dsub_rn(p_lat, t_lat), GEO_DEG_TO_RAD), 0.5));
    const double s_lng = sin(__dmul_rn(__dmul_rn(__dsub_rn(p_lng, t_lng), GEO_DEG_TO_RAD), 0.5));
    const double a = __dadd_rn(__dmul_rn(s_lat, s_lat), __dmul_rn(__dmul_rn(__dmul_rn(s_lng, s_lng), t_cos_lat), p_cos_lat));
    const double c1 = __dsqrt_rn(__dsub_rn(1.0, a));
    const double c = __dmul_rn(2.0, atan2(__dsqrt_rn(a), c1));
    return GeoDist{__dmul_rn(c, EARTH_RADIUS_M), c1};
}
__device__ __forceinline__ double haversine_m(double t_lat, double t_lng, double t_cos_lat, double p_lat, double p_lng, double p_cos_lat) {
    return geo_dist(t_lat, t_lng, t_cos_lat, p_lat, p_lng, p_cos_lat).m;
}
__device__ __forceinline__ double haversine_m(double t_lat, double t_lng, double t_cos_lat, const GeoPoint &p) {
    return haversine_m(t_lat, t_lng, t_cos_lat, p.lat, p.lng, p.cos_lat);
}

// the device's distance cannot tell on which side of `thr` the host's falls: NaN, past GEO_ANTIPODE_M, or within the tolerance
// (each step rounded explicitly, so every kernel that includes this flags the same points)
__device__ __forceinline__ bool geo_ambiguous(const GeoDist &g, double thr) {
    const double tol = __dmul_rn(GEO_TAU, __dadd_rn(fmax(g.m, 1.0), __ddiv_rn(EARTH_RADIUS_M, g.c1)));
    return !(fabs(__dsub_rn(g.m, thr)) > tol) || !(g.m <= GEO_ANTIPODE_M);
}
// the threshold of the floor: the whole metre nearest to m (1 below it: floor cannot change between 0 and 1)
__device__ __forceinline__ double floor_threshold(double m) { return fmax(rint(m), 1.0); }

// `distance as usize`: saturating, NaN and negatives to 0; GEO_FLOOR_MAX caps it (no haversine reaches it)
__device__ __forceinline__ uint32_t floor_m(double m) { return m > 0.0 ? (uint32_t)fmin(m, (double)GEO_FLOOR_MAX) : 0u; }

// rstar's distance_2 between lat_lng_to_xyz points: ((dx*dx) + dy*dy) + dz*dz
__device__ __forceinline__ double chord2(const double *q, double x, double y, double z) {
    const double dx = __dsub_rn(x, q[0]), dy = __dsub_rn(y, q[1]), dz = __dsub_rn(z, q[2]);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// the rtree order's key: the bits of the squared distance (>= 0, so the bits order as the values)
__device__ __forceinline__ unsigned long long rtree_key(const double *q, const GeoPoint &p) {
    return (unsigned long long)__double_as_longlong(chord2(q, p.x, p.y, p.z));
}

}  // namespace b200
