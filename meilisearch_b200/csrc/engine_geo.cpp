// Geo filters (search/facet/filter/index_filter.rs:465-696): clause validation, the radius band, slot sharing, and the two passes of
// geo_filter.cu, for a search batch (b200_query_batch::geo_filter_*) and for b200_geo_filter_batch.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <map>

#include "engine.h"
#include "kernels.h"

namespace b200 {

#define CU(call, what)                                     \
    do {                                                   \
        cudaError_t e_ = (call);                           \
        if (e_ != cudaSuccess) return cuda_fail(e_, what); \
    } while (0)

namespace {

std::string rust_f64(double v) { return rust_f64_display(v); }

const char *const NON_FINITE = "Non finite floats are not supported";
// FilterError::AttributeNotFilterable (filter/mod.rs:82-98) goes on with the index's filterable patterns, which the library does not
// stage: the caller appends them
const char *const NOT_FILTERABLE = "Attribute `_geo/_geojson` is not filterable.";

std::string bad_lat(double lat) { return "Bad latitude `" + rust_f64(lat) + "`. Latitude must be contained between -90 and 90 degrees."; }
std::string bad_lng(double lng) {
    double n = std::fmod(lng + 180.0, 360.0);  // rem_euclid
    if (n < 0) n += 360.0;
    return "Bad longitude `" + rust_f64(lng) + "`. Longitude must be contained between -180 and 180 degrees. Hint: try using `" +
           rust_f64(n - 180.0) + "` instead.";
}

// Squared-chord bounds of a radius clause.  With theta = (radius + EPSILON) / R, a point whose true angular distance from the base is
// below theta - delta has a computed haversine within the radius, and one beyond theta + delta has one beyond it, for
//   delta = 1e-9 theta + 1e-12 rad  (at least 6 um, and a billionth of the radius).
// Why that is safe: the staged xyz are within a few ULP of the unit vectors, so the computed chord is within 1e-14 of the true one;
// near an angle theta that moves the angle by 1e-14 / cos(theta / 2), which stays far below delta while theta + delta < pi - 1e-4.
// The haversine's relative error is a few ULP there (its 1 - a term keeps at least 2.5e-9 of magnitude), so its absolute error is
// far below delta too.  Near the antipode both formulas lose resolution, so past pi - 1e-4 every point not clearly inside goes to
// the haversine (hi = infinity).  lo and hi are widened by a further 1e-12 relative against the rounding of sin here.  The band is
// some 2e-9 of the radius wide, so the haversine is computed for a handful of points per clause.
void geo_radius_band(double r_eps, double &lo, double &hi) {
    if (!(r_eps >= 0)) {  // a negative radius: every point fails, F is the first point of the order
        lo = hi = -1.0;
        return;
    }
    const double theta = r_eps / 6371000.0, delta = 1e-9 * theta + 1e-12;
    const double a = theta - delta, b = theta + delta;
    lo = a > 0 ? std::pow(2.0 * std::sin(a / 2.0), 2) * (1.0 - 1e-12) : -1.0;
    hi = b < M_PI - 1e-4 ? std::pow(2.0 * std::sin(b / 2.0), 2) * (1.0 + 1e-12) : HUGE_VAL;
}

}  // namespace

double geo_distance_host(double t_lat, double t_lng, double p_lat, double p_lng) {
    const double to_rad = M_PI / 180.0;
    const double s_lat = std::sin((p_lat - t_lat) * to_rad / 2.0), s_lng = std::sin((p_lng - t_lng) * to_rad / 2.0);
    const double a = s_lat * s_lat + s_lng * s_lng * std::cos(t_lat * to_rad) * std::cos(p_lat * to_rad);
    return 2.0 * std::atan2(std::sqrt(a), std::sqrt(1.0 - a)) * 6371000.0;
}

// One clause from the ABI's (kind, four doubles), validated in the reference's order: the coordinates finite, then their ranges, then
// the radius (finite) or top >= bottom.  Returns 0 or B200_ERR_INVALID with the reference's message.
int geo_clause(uint8_t kind, uint8_t neg, const double *a, GeoClause &c, std::string &err) {
    c = GeoClause{};
    c.kind = kind;
    c.neg = neg ? 1 : 0;
    if (kind > 1) {
        err = "geo filter clause: unknown kind (0 _geoRadius, 1 _geoBoundingBox)";
        return B200_ERR_INVALID;
    }
    const int n_coords = kind == 0 ? 2 : 4;
    for (int i = 0; i < n_coords; i++)
        if (!std::isfinite(a[i])) {
            err = NON_FINITE;
            return B200_ERR_INVALID;
        }
    for (int i = 0; i < n_coords; i += 2) {
        if (!(a[i] >= -90.0 && a[i] <= 90.0)) {
            err = bad_lat(a[i]);
            return B200_ERR_INVALID;
        }
        if (!(a[i + 1] >= -180.0 && a[i + 1] <= 180.0)) {
            err = bad_lng(a[i + 1]);
            return B200_ERR_INVALID;
        }
    }
    if (kind == 0) {
        if (!std::isfinite(a[2])) {
            err = NON_FINITE;
            return B200_ERR_INVALID;
        }
        const double to_rad = M_PI / 180.0, la = a[0] * to_rad, ln = a[1] * to_rad;
        c.q[0] = std::cos(la) * std::cos(ln);  // lat_lng_to_xyz, as the points were staged
        c.q[1] = std::cos(la) * std::sin(ln);
        c.q[2] = std::sin(la);
        c.t_lat = a[0];
        c.t_lng = a[1];
        c.t_cos_lat = std::cos(la);
        c.r_eps = a[2] + DBL_EPSILON;
        geo_radius_band(c.r_eps, c.lo, c.hi);
    } else {
        if (a[0] < a[2]) {
            err = "The top latitude `" + rust_f64(a[0]) + "` is below the bottom latitude `" + rust_f64(a[2]) + "`.";
            return B200_ERR_INVALID;
        }
        c.top = a[0];
        c.right = a[1];
        c.bottom = a[2];
        c.left = a[3];
    }
    return B200_OK;
}

namespace {

// identical clauses share one entry (and one pass-1 search): the key is the clause's defining bytes
struct ClauseSet {
    std::vector<GeoClause> clauses;
    std::map<std::string, uint32_t> index;
    uint32_t add(uint8_t kind, uint8_t neg, const double *a, const GeoClause &c) {
        double args[4] = {a[0], a[1], a[2], kind == 0 ? 0.0 : a[3]};
        std::string key(1, (char)kind);
        key.push_back((char)(neg ? 1 : 0));
        key.append(reinterpret_cast<const char *>(args), sizeof args);
        auto it = index.emplace(key, (uint32_t)clauses.size());
        if (it.second) clauses.push_back(c);
        return it.first->second;
    }
};

}  // namespace

bool Engine::geo_filterable() const { return hix.geo.lat_fid != 0xFFFF && hix.geo.lng_fid != 0xFFFF; }

int Engine::reserve_geo_bitmaps(DevBuf<unsigned long long> &buf, size_t n_bitmaps) {
    cudaError_t e = buf.reserve(std::max<size_t>(1, n_bitmaps) * hix.n_words64);
    if (e == cudaErrorMemoryAllocation) {
        cudaGetLastError();
        return fail(B200_ERR_CAPACITY, "geo filter: the batch's universe bitmaps do not fit in device memory");
    }
    CU(e, "alloc geo filter bitmaps");
    return B200_OK;
}

// The two passes for `slots` (their ub / dst set; clause lists index `slot_clauses`), counts returned in `counts`.  One synchronise.
int Engine::run_geo_filter(const std::vector<GeoClause> &clauses, const std::vector<uint32_t> &slot_clauses, std::vector<GeoSlot> &slots,
                           std::vector<uint64_t> &counts) {
    const uint32_t W = (uint32_t)hix.n_words64, n_slots = (uint32_t)slots.size();
    std::vector<uint32_t> u32;  // radius clause ids, then the slots' clause lists
    for (uint32_t c = 0; c < clauses.size(); c++)
        if (clauses[c].kind == 0) u32.push_back(c);
    const uint32_t n_radius = (uint32_t)u32.size();
    u32.insert(u32.end(), slot_clauses.begin(), slot_clauses.end());
    CU(d_gf_clause.reserve(clauses.size() + 1), "alloc geo clauses");
    CU(d_gf_first.reserve(clauses.size() + 1), "alloc geo clauses");
    CU(d_gf_amb.reserve(std::max<size_t>(d_gf_amb.cap, 1024)), "alloc geo clauses");
    CU(d_gf_u32.reserve(u32.size() + 1), "alloc geo clauses");
    CU(d_gf_slot.reserve(n_slots + 1), "alloc geo slots");
    CU(d_gf_count.reserve(n_slots + 1), "alloc geo slots");
    for (uint32_t s = 0; s < n_slots; s++) slots[s].count = d_gf_count.p + s;
    CU(cudaMemcpyAsync(d_gf_clause.p, clauses.data(), clauses.size() * sizeof(GeoClause), cudaMemcpyHostToDevice, stream), "H2D geo clauses");
    CU(cudaMemcpyAsync(d_gf_u32.p, u32.data(), u32.size() * 4, cudaMemcpyHostToDevice, stream), "H2D geo clauses");
    CU(cudaMemcpyAsync(d_gf_slot.p, slots.data(), n_slots * sizeof(GeoSlot), cudaMemcpyHostToDevice, stream), "H2D geo slots");
    CU(cudaMemsetAsync(d_gf_first.p, 0xff, clauses.size() * sizeof(GeoFirst), stream), "memset geo clauses");
    CU(cudaMemsetAsync(d_gf_count.p, 0, n_slots * 8, stream), "memset geo slots");
    stats.h2d_bytes += clauses.size() * sizeof(GeoClause) + u32.size() * 4 + n_slots * sizeof(GeoSlot);
    const uint64_t n_geo = hix.geo.n_geo;
    // algorithmic bytes: each pass reads the geo bitmap and the geo documents' points once (xyz in pass 1, xyz + lat / lng in pass
    // 2); pass 2 reads each slot's universe and writes its bitmap
    if (n_radius) {
        // pass 1; the band points it cannot decide are decided here, with libm, and the failing ones folded into F (a minimum).  The
        // list is read after the pass; when it overflowed, the pass runs again with room for all of it.
        uint32_t *amb_count = d_gf_u32.p + u32.size();
        uint32_t n_amb = 0;
        for (int attempt = 0; attempt < 2; attempt++) {
            if (attempt) CU(cudaMemsetAsync(d_gf_first.p, 0xff, clauses.size() * sizeof(GeoFirst), stream), "memset geo clauses");
            CU(cudaMemsetAsync(amb_count, 0, 4, stream), "memset geo clauses");
            const size_t m0 = mark();
            CU(launch_geo_first_fail(stream, d_geo_ub, d_geo_pts, W, d_gf_clause.p, d_gf_u32.p, n_radius, d_gf_first.p, d_gf_amb.p,
                                     (uint32_t)d_gf_amb.cap, amb_count), "geo_first_fail");
            time_kernel(B200_K_GEO_FILTER, m0, mark(), (uint64_t)W * 8 + n_geo * 24 + n_radius * (uint64_t)sizeof(GeoFirst));
            CU(cudaMemcpyAsync(&n_amb, amb_count, 4, cudaMemcpyDeviceToHost, stream), "D2H geo ambiguous");
            CU(cudaStreamSynchronize(stream), "sync");
            stats.d2h_bytes += 4;
            if (n_amb <= d_gf_amb.cap) break;
            CU(d_gf_amb.reserve(n_amb), "alloc geo ambiguous");
        }
        if (n_amb) {
            std::vector<GeoAmb> amb(n_amb);
            std::vector<GeoFirst> first(clauses.size());
            CU(cudaMemcpyAsync(amb.data(), d_gf_amb.p, n_amb * sizeof(GeoAmb), cudaMemcpyDeviceToHost, stream), "D2H geo ambiguous");
            CU(cudaMemcpyAsync(first.data(), d_gf_first.p, first.size() * sizeof(GeoFirst), cudaMemcpyDeviceToHost, stream), "D2H geo ambiguous");
            CU(cudaStreamSynchronize(stream), "sync");
            stats.d2h_bytes += n_amb * sizeof(GeoAmb) + first.size() * sizeof(GeoFirst);
            for (const GeoAmb &x : amb) {
                const GeoClause &k = clauses[x.clause];
                if (geo_distance_host(k.t_lat, k.t_lng, hix.geo.lat[x.doc], hix.geo.lng[x.doc]) <= k.r_eps) continue;
                GeoFirst &f = first[x.clause];
                if (x.key < f.key || (x.key == f.key && x.doc < f.doc)) f = GeoFirst{x.key, x.doc};
            }
            CU(cudaMemcpyAsync(d_gf_first.p, first.data(), first.size() * sizeof(GeoFirst), cudaMemcpyHostToDevice, stream), "H2D geo clauses");
            CU(cudaStreamSynchronize(stream), "sync");  // `first` is pageable and local
            stats.h2d_bytes += first.size() * sizeof(GeoFirst);
        }
    }
    const size_t m1 = mark();
    CU(launch_geo_filter(stream, d_geo_ub, d_geo_pts, W, d_gf_clause.p, d_gf_first.p, d_gf_u32.p + n_radius, d_gf_slot.p, n_slots), "geo_filter");
    time_kernel(B200_K_GEO_FILTER, m1, mark(), (uint64_t)W * 8 + n_geo * 40 + (uint64_t)n_slots * W * 16);
    counts.assign(n_slots, 0);
    CU(cudaMemcpyAsync(counts.data(), d_gf_count.p, n_slots * 8, cudaMemcpyDeviceToHost, stream), "D2H geo counts");
    stats.d2h_bytes += n_slots * 8;
    CU(cudaStreamSynchronize(stream), "sync");
    resolve_timers();
    stats.device_steps++;
    return B200_OK;
}

// The filtered universe of every query with geo clauses: documents_ids AND its universe AND its clauses.  Queries with the same
// universe pointer and the same clause list share one slot.
int Engine::geo_filter_universes(const b200_query_batch *b, GeoFiltered &gf) {
    const uint32_t NQ = b->n_queries;
    const uint64_t W = hix.n_words64;
    gf.d_univ.assign(NQ, nullptr);
    gf.count.assign(NQ, 0);
    gf.status.assign(NQ, 0);
    gf.error.assign(NQ, std::string());
    if (!b->geo_filter_kind || !b->geo_filter_args) return fail(B200_ERR_INVALID, "geo_filter_begin without geo_filter_kind / geo_filter_args");
    if (b->universes && b->n_universe_words < W) return fail(B200_ERR_INVALID, "universe bitmaps shorter than the document range");
    ClauseSet cs;
    std::map<std::pair<const uint64_t *, std::vector<uint32_t>>, uint32_t> slot_of;
    std::vector<const uint64_t *> slot_caller;
    std::vector<uint32_t> slot_clauses, q_slot(NQ, UINT32_MAX);
    std::vector<GeoSlot> slots;
    for (uint32_t q = 0; q < NQ; q++) {
        const uint32_t c0 = b->geo_filter_begin[q], c1 = b->geo_filter_begin[q + 1];
        if (c0 >= c1) continue;
        std::vector<uint32_t> ids;
        for (uint32_t k = c0; k < c1 && !gf.status[q]; k++) {
            const uint8_t kind = b->geo_filter_kind[k], neg = b->geo_filter_not ? b->geo_filter_not[k] : 0;
            GeoClause c;
            gf.status[q] = geo_clause(kind, neg, b->geo_filter_args + 4 * (size_t)k, c, gf.error[q]);
            if (!gf.status[q]) ids.push_back(cs.add(kind, neg, b->geo_filter_args + 4 * (size_t)k, c));
        }
        if (!gf.status[q] && !geo_filterable()) {
            gf.status[q] = B200_ERR_INVALID;
            gf.error[q] = NOT_FILTERABLE;
        }
        if (gf.status[q]) continue;
        const uint64_t *caller = b->universes ? b->universes[q] : nullptr;
        auto it = slot_of.emplace(std::make_pair(caller, ids), (uint32_t)slots.size());
        if (it.second) {
            slots.push_back(GeoSlot{nullptr, nullptr, nullptr, (uint32_t)slot_clauses.size(), (uint32_t)(slot_clauses.size() + ids.size())});
            slot_clauses.insert(slot_clauses.end(), ids.begin(), ids.end());
            slot_caller.push_back(caller);
        }
        q_slot[q] = it.first->second;
    }
    if (slots.empty()) return B200_OK;
    // every distinct caller universe is intersected with documents_ids and uploaded once, in one copy on the stream the kernels run
    // on, so they are ordered after it (a copy from pageable memory is staged before the call returns)
    std::map<const uint64_t *, uint32_t> caller_of;
    for (auto p : slot_caller)
        if (p) caller_of.emplace(p, (uint32_t)caller_of.size());
    int rc = reserve_geo_bitmaps(d_gf_caller, caller_of.size());
    if (rc == B200_OK) rc = reserve_geo_bitmaps(d_gf_univ, slots.size());
    if (rc != B200_OK) return rc;
    std::vector<uint64_t> host(caller_of.size() * W);
    for (auto &kv : caller_of)
        for (uint64_t w = 0; w < W; w++) host[kv.second * W + w] = kv.first[w] & hix.base_ub[w];
    if (!host.empty()) {
        CU(cudaMemcpyAsync(d_gf_caller.p, host.data(), host.size() * 8, cudaMemcpyHostToDevice, stream), "H2D universes");
        stats.h2d_bytes += host.size() * 8;
    }
    for (size_t s = 0; s < slots.size(); s++) {
        slots[s].ub = slot_caller[s] ? d_gf_caller.p + (size_t)caller_of[slot_caller[s]] * W : dix.base_ub;
        slots[s].dst = d_gf_univ.p + s * W;
    }
    std::vector<uint64_t> counts;
    rc = run_geo_filter(cs.clauses, slot_clauses, slots, counts);
    if (rc != B200_OK) return rc;
    for (uint32_t q = 0; q < NQ; q++)
        if (q_slot[q] != UINT32_MAX) {
            gf.d_univ[q] = slots[q_slot[q]].dst;
            gf.count[q] = counts[q_slot[q]];
        }
    return B200_OK;
}

// One bitmap over documents_ids per valid clause i (kind[i], args[4 i ..)) into buf; slot_of[i] = its bitmap (identical clauses share
// one), UINT32_MAX for a clause refused with status[i] / err[i].  One synchronise.
int Engine::geo_clause_bitmaps(uint32_t n, const uint8_t *kind, const double *args, DevBuf<unsigned long long> &buf, std::vector<uint32_t> &slot_of,
                               int32_t *status, std::vector<std::string> &err) {
    const uint64_t W = hix.n_words64;
    ClauseSet cs;
    slot_of.assign(n, UINT32_MAX);
    err.assign(n, std::string());
    for (uint32_t i = 0; i < n; i++) {
        GeoClause c;
        status[i] = geo_clause(kind[i], 0, args + 4 * (size_t)i, c, err[i]);
        if (!status[i] && !geo_filterable()) {
            status[i] = B200_ERR_INVALID;
            err[i] = NOT_FILTERABLE;
        }
        if (!status[i]) slot_of[i] = cs.add(kind[i], 0, args + 4 * (size_t)i, c);
    }
    if (cs.clauses.empty()) return B200_OK;
    const uint32_t n_slots = (uint32_t)cs.clauses.size();
    int rc = reserve_geo_bitmaps(buf, n_slots);
    if (rc != B200_OK) return rc;
    std::vector<uint32_t> slot_clauses(n_slots);
    std::vector<GeoSlot> slots(n_slots);
    for (uint32_t s = 0; s < n_slots; s++) {
        slot_clauses[s] = s;
        slots[s] = GeoSlot{dix.base_ub, buf.p + (size_t)s * W, nullptr, s, s + 1};
    }
    std::vector<uint64_t> counts;
    return run_geo_filter(cs.clauses, slot_clauses, slots, counts);
}

int Engine::geo_filter_batch(uint32_t n, const uint8_t *kind, const double *args, uint64_t *out, uint64_t out_words, int32_t *status) {
    const uint64_t W = hix.n_words64;
    if (n && (!kind || !args || !out || !status)) return fail(B200_ERR_INVALID, "geo_filter_batch: null kind / args / out / status");
    if (out_words < W) return fail(B200_ERR_INVALID, "geo_filter_batch: out_words smaller than the document range");
    CU(cudaSetDevice(device), "cudaSetDevice");
    for (uint32_t i = 0; i < n; i++) memset(out + (size_t)i * out_words, 0, out_words * 8);
    std::vector<uint32_t> slot_of;
    std::vector<std::string> err;
    int rc = geo_clause_bitmaps(n, kind, args, d_gf_univ, slot_of, status, err);
    if (rc != B200_OK) return rc;
    for (uint32_t i = 0; i < n; i++) {
        if (status[i]) {
            last_error = err[i];
            continue;
        }
        CU(cudaMemcpyAsync(out + (size_t)i * out_words, d_gf_univ.p + (size_t)slot_of[i] * W, W * 8, cudaMemcpyDeviceToHost, stream), "D2H geo filter");
        stats.d2h_bytes += W * 8;
    }
    CU(cudaStreamSynchronize(stream), "sync");
    return B200_OK;
}

}  // namespace b200
