// The device's geo functions (meilisearch_b200/csrc/geo_math.cuh) evaluated over arrays, for tests/test_gpu_geo_probe.py: per pair
// the haversine and sqrt(1 - a), the iterative key floor_m, whether the floor and a given threshold are ambiguous, and the rtree key.
#include <cstdint>

#include "geo_math.cuh"

using namespace b200;

namespace {

__global__ void probe_kernel(int n, const double *t, const GeoPoint *p, const double *q, const double *thr, double *m, double *c1,
                             uint32_t *floor, uint8_t *amb_floor, uint8_t *amb_thr, unsigned long long *key) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const GeoPoint pt = p[i];
    const GeoDist g = geo_dist(t[3 * i], t[3 * i + 1], t[3 * i + 2], pt.lat, pt.lng, pt.cos_lat);
    m[i] = g.m;
    c1[i] = g.c1;
    floor[i] = floor_m(g.m);
    amb_floor[i] = geo_ambiguous(g, floor_threshold(g.m));
    amb_thr[i] = geo_ambiguous(g, thr[i]);
    key[i] = rtree_key(q + 3 * i, pt);
}

template <class T>
T *dev(const T *h, int n) {
    T *d = nullptr;
    cudaMalloc(&d, sizeof(T) * (size_t)n);
    if (h) cudaMemcpy(d, h, sizeof(T) * (size_t)n, cudaMemcpyHostToDevice);
    return d;
}

}  // namespace

extern "C" double geo_probe_tau() { return GEO_TAU; }
extern "C" double geo_probe_antipode_m() { return GEO_ANTIPODE_M; }

// t: n x (lat, lng, cos lat) of the targets; p: n GeoPoints (x, y, z, lat, lng, cos lat); q: n x xyz rtree targets; thr: n thresholds.
// Returns 0 or the CUDA error.
extern "C" int geo_probe(int n, const double *t, const double *p, const double *q, const double *thr, double *m, double *c1, uint32_t *floor,
                         uint8_t *amb_floor, uint8_t *amb_thr, unsigned long long *key) {
    if (n <= 0) return 0;
    double *dt = dev(t, 3 * n), *dq = dev(q, 3 * n), *dthr = dev(thr, n), *dm = dev<double>(nullptr, n), *dc1 = dev<double>(nullptr, n);
    GeoPoint *dp = dev(reinterpret_cast<const GeoPoint *>(p), n);
    uint32_t *dfloor = dev<uint32_t>(nullptr, n);
    uint8_t *daf = dev<uint8_t>(nullptr, n), *dat = dev<uint8_t>(nullptr, n);
    unsigned long long *dkey = dev<unsigned long long>(nullptr, n);
    probe_kernel<<<(n + 255) / 256, 256>>>(n, dt, dp, dq, dthr, dm, dc1, dfloor, daf, dat, dkey);
    cudaMemcpy(m, dm, 8 * (size_t)n, cudaMemcpyDeviceToHost);
    cudaMemcpy(c1, dc1, 8 * (size_t)n, cudaMemcpyDeviceToHost);
    cudaMemcpy(floor, dfloor, 4 * (size_t)n, cudaMemcpyDeviceToHost);
    cudaMemcpy(amb_floor, daf, (size_t)n, cudaMemcpyDeviceToHost);
    cudaMemcpy(amb_thr, dat, (size_t)n, cudaMemcpyDeviceToHost);
    cudaMemcpy(key, dkey, 8 * (size_t)n, cudaMemcpyDeviceToHost);
    const cudaError_t e = cudaGetLastError();
    for (void *x : {(void *)dt, (void *)dq, (void *)dthr, (void *)dm, (void *)dc1, (void *)dp, (void *)dfloor, (void *)daf, (void *)dat, (void *)dkey})
        cudaFree(x);
    return (int)e;
}
