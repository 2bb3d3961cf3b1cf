// The two distances of the reference's geo code, shared by GeoSort (geo.cu) and the geo filters (geo_filter.cu).
// Points and cos(lat) are staged as computed by the host's libm; the squared distance is rounded exactly as on the host (no fused
// multiply-add), so rtree keys are bit-identical.  The haversine uses the device's sin / atan2 (within a few ULP of the host's).
#pragma once
#include <cuda_runtime.h>

#include "device_types.h"

namespace b200 {

constexpr double EARTH_RADIUS_M = 6371000.0;

// Location::haversine_distance_to (geoutils), from the target (t) to the point (p).  sin(to_radians(d) / 2) is taken as
// sinpi(d / 360): both are within a few ULP of the true value, and sinpi needs no slow-path argument reduction (a call that
// spills registers).
__device__ __forceinline__ double haversine_m(double t_lat, double t_lng, double t_cos_lat, double p_lat, double p_lng, double p_cos_lat) {
    const double s_lat = sinpi(__ddiv_rn(__dsub_rn(p_lat, t_lat), 360.0)), s_lng = sinpi(__ddiv_rn(__dsub_rn(p_lng, t_lng), 360.0));
    const double a = __dadd_rn(__dmul_rn(s_lat, s_lat), __dmul_rn(__dmul_rn(__dmul_rn(s_lng, s_lng), t_cos_lat), p_cos_lat));
    const double c = __dmul_rn(2.0, atan2(__dsqrt_rn(a), __dsqrt_rn(__dsub_rn(1.0, a))));
    return __dmul_rn(c, EARTH_RADIUS_M);
}
__device__ __forceinline__ double haversine_m(double t_lat, double t_lng, double t_cos_lat, const GeoPoint &p) {
    return haversine_m(t_lat, t_lng, t_cos_lat, p.lat, p.lng, p.cos_lat);
}

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
