// Filter programs (IndexFilter::inner_evaluate, search/facet/filter/index_filter.rs:332-696): a filter tree is compiled on the host into
// a straight-line program of filter.cu, its value leaves lowered to ordinal intervals of the field by binary search over the staged
// level-0 keys; the programs of a batch run in one launch, one slot per distinct (universe, program).
//
// Reach of a leaf's error.  Evaluating a node with the universe hint h returns val(n, h): the leaf's set, intersected with h for RANGE;
// h - val(child, h) for NOT (documents_ids without a hint); the union for OR; for AND the running bitmap r_1 = val(c_0, h),
// r_{i+1} = r_i AND val(c_i, r_i), stopping once it is empty.  Every such value is a word-local function of the leaves' words and the
// hint's, so the program computes exactly the bitmaps the reference forms, AND prefixes included; evaluation reaches child i >= 1 of an
// AND iff r_i is non-empty (the root has no hint, and a node only sees an empty hint as such a child).  The program sets one flag per
// AND prefix an error leaf sits behind, and a leaf is reached iff all the flags on its path are set.
#include <algorithm>
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

const char *const PRESENCE_DB[3] = {"facet_id_exists_docids", "facet_id_is_null_docids", "facet_id_is_empty_docids"};
const char *const PRESENCE_OP[3] = {"EXISTS", "IS NULL", "IS EMPTY"};

// OrderedF64Codec key order (facet/value_encoding.rs f64_into_bytes, then the f64 big-endian): both zeros share the ordered part
bool num_key_less(double a, double b) {
    auto ord = [](double v, uint64_t &raw) {
        memcpy(&raw, &v, 8);
        return v == 0.0 ? 1ull << 63 : (raw >> 63 ? ~raw : raw ^ (1ull << 63));
    };
    uint64_t ra, rb;
    const uint64_t oa = ord(a, ra), ob = ord(b, rb);
    return oa < ob || (oa == ob && ra < rb);
}

// a leaf's error, raised when evaluation reaches it: reached iff every flag in `flags` is set
struct ErrLeaf {
    uint32_t node;
    std::vector<uint32_t> flags;
    std::string msg;
};

struct Program {
    std::vector<FilterOp> ops;
    std::vector<uint2> iv;
    std::vector<ErrLeaf> errs;            // in pre-order
    std::vector<std::pair<uint32_t, uint32_t>> geo;  // (op, geo leaf of the batch) whose bitmap is filled in after the geo pass
    uint32_t n_flags = 0;
    int status = 0;
    int32_t error_leaf = -1;
    std::string error;
};

struct Compiler {
    const Engine &eng;
    const b200_filter_programs &p;
    uint32_t first, end;
    Program &out;
    std::vector<uint8_t> &geo_kind;  // the batch's geo leaves
    std::vector<double> &geo_args;
    std::vector<uint32_t> path;      // flags of the AND prefixes above the node being compiled

    bool fail(int code, uint32_t node, const std::string &msg) {
        if (out.status) return false;
        out.status = code;
        out.error_leaf = node == UINT32_MAX ? -1 : (int32_t)(node - first);
        out.error = msg;
        return false;
    }
    void emit(uint16_t code, uint32_t dst, uint32_t src = 0, uint32_t hint = FILTER_NO_REG) {
        FilterOp op{};
        op.code = code;
        op.dst = (uint16_t)dst;
        op.src = (uint16_t)src;
        op.hint = (uint16_t)hint;
        out.ops.push_back(op);
    }
    std::string value(uint32_t v) const { return std::string(p.value_bytes + p.value_off[v], p.value_off[v + 1] - p.value_off[v]); }
    bool values_ok(uint32_t v, uint32_t n) const {
        if ((uint64_t)v + n > p.n_values) return false;
        for (uint32_t k = v; k < v + n; k++)
            if (p.value_off[k + 1] < p.value_off[k]) return false;
        return true;
    }
    // the sorted, disjoint ordinal intervals of a value leaf into a VALUE op
    void value_op(const SortField *f, std::vector<uint2> iv, uint32_t dst, uint32_t hint, bool neg) {
        std::sort(iv.begin(), iv.end(), [](uint2 a, uint2 b) { return a.x < b.x; });
        std::vector<uint2> merged;
        for (uint2 x : iv) {
            if (x.x >= x.y) continue;
            if (!merged.empty() && x.x <= merged.back().y)
                merged.back().y = std::max(merged.back().y, x.y);
            else
                merged.push_back(x);
        }
        emit(FOP_VALUE, dst, 0, hint);
        FilterOp &op = out.ops.back();
        op.neg = neg;
        op.a = (uint32_t)out.iv.size();
        out.iv.insert(out.iv.end(), merged.begin(), merged.end());
        op.b = (uint32_t)out.iv.size();
        if (f) {
            op.doc_off = f->d_doc_off;
            op.doc_ord = f->d_doc_ord;
        }
    }
    // ordinals [a, b) of the field's numbers (then strings, offset by n_num) between two bounds
    template <class V, class Less>
    static uint2 interval(const std::vector<V> &keys, uint32_t base, uint8_t lo_kind, const V &lo, uint8_t hi_kind, const V &hi, Less less) {
        const V *b0 = keys.data(), *b1 = keys.data() + keys.size();
        const V *a = lo_kind == B200_B_UNBOUNDED ? b0
                     : lo_kind == B200_B_INCLUDED ? std::lower_bound(b0, b1, lo, less)
                                                  : std::upper_bound(b0, b1, lo, less);
        const V *b = hi_kind == B200_B_UNBOUNDED ? b1
                     : hi_kind == B200_B_INCLUDED ? std::upper_bound(b0, b1, hi, less)
                                                  : std::lower_bound(b0, b1, hi, less);
        return make_uint2(base + (uint32_t)(a - b0), base + (uint32_t)std::max(a - b0, b - b0));
    }
    // the ordinal of a string / number key of the field, or none
    static bool find_str(const SortField &f, const std::string &s, uint32_t &o) {
        auto it = std::lower_bound(f.str_val.begin(), f.str_val.end(), s);
        if (it == f.str_val.end() || *it != s) return false;
        o = f.n_num + (uint32_t)(it - f.str_val.begin());
        return true;
    }
    static bool find_num(const SortField &f, double x, uint32_t &o) {
        auto it = std::lower_bound(f.num_val.begin(), f.num_val.end(), x, num_key_less);
        if (it == f.num_val.end() || num_key_less(x, *it)) return false;
        o = (uint32_t)(it - f.num_val.begin());
        return true;
    }
    const SortField *field(uint16_t fid) const {
        auto it = eng.hix.sort_fields.find(fid);
        return it == eng.hix.sort_fields.end() ? nullptr : &it->second;
    }

    // compile the subtree at node i into register dst under hint register `hint`; returns the node after the subtree (end on failure)
    uint32_t node(uint32_t i, uint32_t hint, uint32_t dst, uint32_t depth) {
        if (out.status) return end;
        if (i >= end) return fail(B200_ERR_INVALID, UINT32_MAX, "filter: a node's children run past the program's nodes"), end;
        if (depth > B200_MAX_FILTER_DEPTH)
            return fail(B200_ERR_UNSUPPORTED, i, "filter: nesting deeper than " + std::to_string(B200_MAX_FILTER_DEPTH)), end;
        const b200_filter_node &nd = p.nodes[i];
        switch (nd.op) {
            case B200_F_AND:
            case B200_F_OR: {
                if (nd.n == 0) {
                    emit(FOP_ZERO, dst);
                    return i + 1;
                }
                uint32_t j = node(i + 1, hint, dst, depth + 1);
                for (uint32_t c = 1; c < nd.n && !out.status; c++) {
                    if (nd.op == B200_F_AND) {  // child c sees the running bitmap as its hint, and is reached iff it is non-empty
                        emit(FOP_FLAG, dst);
                        out.ops.back().a = out.n_flags;
                        path.push_back(out.n_flags++);
                        j = node(j, dst, dst + 1, depth + 1);
                        path.pop_back();
                        emit(FOP_AND, dst, dst + 1);
                    } else {
                        j = node(j, hint, dst + 1, depth + 1);
                        emit(FOP_OR, dst, dst + 1);
                    }
                }
                return j;
            }
            case B200_F_NOT: {
                const uint32_t j = node(i + 1, hint, dst, depth + 1);
                emit(FOP_NOT, dst, 0, hint);
                return j;
            }
            case B200_F_RANGE: {
                if (!values_ok(nd.value, 2) || nd.lo > B200_B_UNBOUNDED || nd.hi > B200_B_UNBOUNDED)
                    return fail(B200_ERR_INVALID, i, "filter: a RANGE leaf with bad values or bounds"), end;
                const SortField *f = field(nd.fid);
                std::vector<uint2> iv;
                if (f) {
                    const double nlo = p.value_num[nd.value], nhi = p.value_num[nd.value + 1];
                    const bool lo_ok = nd.lo == B200_B_UNBOUNDED || !std::isnan(nlo), hi_ok = nd.hi == B200_B_UNBOUNDED || !std::isnan(nhi);
                    if (nd.has_number && lo_ok && hi_ok) iv.push_back(interval(f->num_val, 0, nd.lo, nlo, nd.hi, nhi, num_key_less));
                    iv.push_back(interval(f->str_val, f->n_num, nd.lo, value(nd.value), nd.hi, value(nd.value + 1), std::less<std::string>()));
                }
                value_op(f, iv, dst, hint, false);
                return i + 1;
            }
            case B200_F_EQUAL:
            case B200_F_NOT_EQUAL:
            case B200_F_IN: {
                const uint32_t n = nd.op == B200_F_IN ? nd.n : 1;
                if (!values_ok(nd.value, n)) return fail(B200_ERR_INVALID, i, "filter: a leaf's values run past value_off"), end;
                const SortField *f = field(nd.fid);
                std::vector<uint2> iv;
                for (uint32_t v = nd.value; f && v < nd.value + n; v++) {
                    uint32_t o;
                    if (find_str(*f, value(v), o)) iv.push_back(make_uint2(o, o + 1));
                    if (!std::isnan(p.value_num[v]) && find_num(*f, p.value_num[v], o)) iv.push_back(make_uint2(o, o + 1));
                }
                value_op(f, iv, dst, FILTER_NO_REG, nd.op == B200_F_NOT_EQUAL);
                return i + 1;
            }
            case B200_F_EXISTS:
            case B200_F_IS_NULL:
            case B200_F_IS_EMPTY: {
                const int k = nd.op - B200_F_EXISTS;
                if (!eng.raw_dbs[B200_DB_FACET_ID_EXISTS_DOCIDS + k].staged)
                    return fail(B200_ERR_INVALID, i, std::string("filter: `") + PRESENCE_OP[k] + "` reads " + PRESENCE_DB[k] + ", which was not staged"), end;
                emit(FOP_BITMAP, dst);
                auto it = eng.d_presence[k].find(nd.fid);
                out.ops.back().bm = it == eng.d_presence[k].end() ? nullptr : it->second;
                return i + 1;
            }
            case B200_F_GEO_RADIUS:
            case B200_F_GEO_BBOX: {
                // a bounding box is two range conditions on _geo.lat / _geo.lng (index_filter.rs:531-696): it intersects with its hint
                const uint8_t kind = nd.op == B200_F_GEO_RADIUS ? 0 : 1;
                GeoClause c;
                std::string err;
                emit(FOP_BITMAP, dst, 0, kind == 1 ? hint : FILTER_NO_REG);  // no bitmap: a refused leaf evaluates to nothing
                // the arguments are checked first, then whether `_geo` is filterable; both errors are raised only when reached
                if (geo_clause(kind, 0, nd.args, c, err)) {
                    out.errs.push_back(ErrLeaf{i, path, err});
                } else if (!eng.geo_filterable()) {
                    out.errs.push_back(ErrLeaf{i, path, "Attribute `_geo/_geojson` is not filterable."});
                } else {
                    out.geo.emplace_back((uint32_t)out.ops.size() - 1, (uint32_t)geo_kind.size());
                    geo_kind.push_back(kind);
                    geo_args.insert(geo_args.end(), nd.args, nd.args + 4);
                }
                return i + 1;
            }
            case B200_F_EMPTY:
                emit(FOP_ZERO, dst);
                return i + 1;
            case B200_F_DENIED:
                emit(FOP_ZERO, dst);
                out.errs.push_back(ErrLeaf{i, path, "filter: the field's filterable features forbid the operator (fid " + std::to_string(nd.fid) + ")"});
                return i + 1;
            case B200_F_UNSUPPORTED:
                return fail(B200_ERR_UNSUPPORTED, i, "filter: CONTAINS, STARTS WITH, _geoPolygon, _geojson, _vectors and _shard are not implemented"), end;
            default:
                return fail(B200_ERR_INVALID, i, "filter: unknown node op " + std::to_string(nd.op)), end;
        }
    }
};

// keep only the flags some error leaf needs, renumbered; returns how many are left
uint32_t prune_flags(Program &pg) {
    std::vector<uint32_t> remap(pg.n_flags, UINT32_MAX);
    uint32_t n = 0;
    for (auto &e : pg.errs)
        for (uint32_t &f : e.flags) {
            if (remap[f] == UINT32_MAX) remap[f] = n++;
            f = remap[f];
        }
    std::vector<FilterOp> ops;
    for (FilterOp op : pg.ops) {
        if (op.code == FOP_FLAG) {
            if (remap[op.a] == UINT32_MAX) continue;
            op.a = remap[op.a];
        }
        ops.push_back(op);
    }
    pg.ops.swap(ops);
    return pg.n_flags = n;
}

}  // namespace

int Engine::run_filters(const b200_filter_programs *p, const std::vector<const unsigned long long *> &base, GeoFiltered &gf) {
    const uint32_t NQ = (uint32_t)base.size();
    const uint64_t W = hix.n_words64;
    if (!p->begin || (p->begin[NQ] > p->begin[0] && !p->nodes) || (p->n_values && (!p->value_off || !p->value_num)))
        return fail(B200_ERR_INVALID, "filter programs: null begin / nodes / value_off / value_num");
    if (p->n_values && p->value_off[p->n_values] > p->value_off[0] && !p->value_bytes) return fail(B200_ERR_INVALID, "filter programs: null value_bytes");
    gf.error_leaf.assign(NQ, -1);
    std::vector<Program> progs(NQ);
    std::vector<uint8_t> geo_kind;
    std::vector<double> geo_args;
    for (uint32_t q = 0; q < NQ; q++) {
        if (!base[q] || gf.status[q]) continue;
        const uint32_t b0 = p->begin[q], b1 = p->begin[q + 1];
        if (b1 < b0) {
            gf.status[q] = B200_ERR_INVALID;
            gf.error[q] = "filter programs: begin must not decrease";
            continue;
        }
        Compiler c{*this, *p, b0, b1, progs[q], geo_kind, geo_args, {}};
        if (c.node(b0, FILTER_NO_REG, 0, 1) != b1) c.fail(B200_ERR_INVALID, UINT32_MAX, "filter: the tree does not end at the program's last node");
        if (progs[q].status) {
            gf.status[q] = progs[q].status;
            gf.error[q] = progs[q].error;
            gf.error_leaf[q] = progs[q].error_leaf;
        }
    }
    // the geo leaves of every program, one bitmap each over documents_ids, by the geo filter kernels
    if (!geo_kind.empty()) {
        std::vector<uint32_t> slot_of;
        std::vector<int32_t> st(geo_kind.size());
        std::vector<std::string> err;
        int rc = geo_clause_bitmaps((uint32_t)geo_kind.size(), geo_kind.data(), geo_args.data(), d_ft_geo, slot_of, st.data(), err);
        if (rc != B200_OK) return rc;
        for (auto &pg : progs)
            for (auto &g : pg.geo) pg.ops[g.first].bm = d_ft_geo.p + (size_t)slot_of[g.second] * W;  // validated while compiling
    }
    // slots: queries with the same universe and the same program (ops and intervals) share one
    std::map<std::string, uint32_t> slot_of;
    std::vector<uint32_t> q_slot(NQ, UINT32_MAX);
    std::vector<FilterSlot> slots;
    std::vector<FilterOp> ops;
    std::vector<uint2> iv;
    std::vector<uint32_t> flag_base;  // per slot: its first flag
    uint32_t n_flags = 0;
    for (uint32_t q = 0; q < NQ; q++) {
        Program &pg = progs[q];
        if (!base[q] || gf.status[q]) continue;
        prune_flags(pg);
        std::string key(reinterpret_cast<const char *>(&base[q]), sizeof base[q]);
        key.append(reinterpret_cast<const char *>(pg.ops.data()), pg.ops.size() * sizeof(FilterOp));
        key.append(reinterpret_cast<const char *>(pg.iv.data()), pg.iv.size() * sizeof(uint2));
        auto it = slot_of.emplace(key, (uint32_t)slots.size());
        if (it.second) {
            FilterSlot s{};
            s.ub = base[q];
            s.op_begin = (uint32_t)ops.size();
            for (FilterOp op : pg.ops) {
                if (op.code == FOP_VALUE) {
                    op.a += (uint32_t)iv.size();
                    op.b += (uint32_t)iv.size();
                }
                ops.push_back(op);
            }
            s.op_end = (uint32_t)ops.size();
            flag_base.push_back(n_flags);
            s.all = pg.n_flags ? 1 : 0;
            iv.insert(iv.end(), pg.iv.begin(), pg.iv.end());
            n_flags += pg.n_flags;
            slots.push_back(s);
        }
        q_slot[q] = it.first->second;
    }
    if (slots.empty()) return B200_OK;
    const uint32_t n_slots = (uint32_t)slots.size();
    cudaError_t e = d_ft_univ.reserve((size_t)n_slots * W);
    if (e == cudaErrorMemoryAllocation) {
        cudaGetLastError();
        return fail(B200_ERR_CAPACITY, "filter: the batch's universe bitmaps do not fit in device memory");
    }
    CU(e, "alloc filter bitmaps");
    CU(d_ft_op.reserve(ops.size() + 1), "alloc filter ops");
    CU(d_ft_iv.reserve(iv.size() + 1), "alloc filter intervals");
    CU(d_ft_slot.reserve(n_slots), "alloc filter slots");
    CU(d_ft_flag.reserve(n_flags + 1), "alloc filter flags");
    CU(d_ft_count.reserve(n_slots), "alloc filter counts");
    for (uint32_t s = 0; s < n_slots; s++) {
        slots[s].dst = d_ft_univ.p + (size_t)s * W;
        slots[s].count = d_ft_count.p + s;
        slots[s].flags = d_ft_flag.p + flag_base[s];
    }
    CU(cudaMemcpyAsync(d_ft_op.p, ops.data(), ops.size() * sizeof(FilterOp), cudaMemcpyHostToDevice, stream), "H2D filter ops");
    if (!iv.empty()) CU(cudaMemcpyAsync(d_ft_iv.p, iv.data(), iv.size() * sizeof(uint2), cudaMemcpyHostToDevice, stream), "H2D filter intervals");
    CU(cudaMemcpyAsync(d_ft_slot.p, slots.data(), n_slots * sizeof(FilterSlot), cudaMemcpyHostToDevice, stream), "H2D filter slots");
    CU(cudaMemsetAsync(d_ft_flag.p, 0, (n_flags + 1) * 4, stream), "memset filter flags");
    CU(cudaMemsetAsync(d_ft_count.p, 0, n_slots * 8, stream), "memset filter counts");
    stats.h2d_bytes += ops.size() * sizeof(FilterOp) + iv.size() * sizeof(uint2) + n_slots * sizeof(FilterSlot);
    // algorithmic bytes: per slot its universe read and its bitmap written, and per document evaluated the ordinal runs of its value
    // leaves (its offset and the field's ordinals) and the bitmap leaves' words
    uint64_t bytes = 0;
    for (const FilterSlot &s : slots) {
        bytes += W * 16;
        for (uint32_t k = s.op_begin; k < s.op_end; k++) {
            const FilterOp &op = ops[k];
            if (op.code == FOP_VALUE && op.doc_off) {
                uint64_t n_ord = 0;
                for (auto &kv : hix.sort_fields)
                    if (kv.second.d_doc_off == op.doc_off) n_ord = kv.second.n_ord;
                bytes += (uint64_t)hix.n_docs * 4 + n_ord * 4;
            } else if (op.code == FOP_BITMAP && op.bm) {
                bytes += W * 8;
            }
        }
    }
    const size_t m0 = mark();
    CU(launch_filter(stream, d_ft_op.p, d_ft_iv.p, d_ft_slot.p, n_slots, dix.base_ub, hix.n_docs, (uint32_t)W), "filter");
    time_kernel(B200_K_FILTER, m0, mark(), bytes);
    std::vector<uint64_t> counts(n_slots);
    std::vector<uint32_t> flags(n_flags + 1);
    CU(cudaMemcpyAsync(counts.data(), d_ft_count.p, n_slots * 8, cudaMemcpyDeviceToHost, stream), "D2H filter counts");
    CU(cudaMemcpyAsync(flags.data(), d_ft_flag.p, (n_flags + 1) * 4, cudaMemcpyDeviceToHost, stream), "D2H filter flags");
    stats.d2h_bytes += n_slots * 8 + (n_flags + 1) * 4;
    CU(cudaStreamSynchronize(stream), "sync");
    resolve_timers();
    stats.device_steps++;
    for (uint32_t q = 0; q < NQ; q++) {
        if (q_slot[q] == UINT32_MAX) continue;
        const FilterSlot &s = slots[q_slot[q]];
        const uint32_t *f = flags.data() + flag_base[q_slot[q]];
        for (const ErrLeaf &el : progs[q].errs)
            if (std::all_of(el.flags.begin(), el.flags.end(), [&](uint32_t k) { return f[k] != 0; })) {
                gf.status[q] = B200_ERR_INVALID;
                gf.error[q] = el.msg;
                gf.error_leaf[q] = (int32_t)(el.node - p->begin[q]);
                break;
            }
        if (gf.status[q]) continue;
        gf.d_univ[q] = s.dst;
        gf.count[q] = counts[q_slot[q]];
    }
    return B200_OK;
}

int Engine::filter_universes(const b200_query_batch *b, GeoFiltered &gf) {
    const uint32_t NQ = b->n_queries;
    const uint64_t W = hix.n_words64;
    if (b->filter->n != NQ) return fail(B200_ERR_INVALID, "filter programs: filter->n must equal n_queries");
    if (b->universes && b->n_universe_words < W) return fail(B200_ERR_INVALID, "universe bitmaps shorter than the document range");
    if (gf.d_univ.size() != NQ) {  // no geo clauses in the batch
        gf.d_univ.assign(NQ, nullptr);
        gf.count.assign(NQ, 0);
        gf.status.assign(NQ, 0);
        gf.error.assign(NQ, std::string());
    }
    // a query's program runs over its geo-filtered universe, else over its caller's bitmap AND documents_ids (each distinct one
    // uploaded once), else over documents_ids
    std::map<const uint64_t *, uint32_t> caller_of;
    for (uint32_t q = 0; q < NQ; q++)
        if (b->filter->begin && b->filter->begin[q + 1] > b->filter->begin[q] && !gf.d_univ[q] && b->universes && b->universes[q])
            caller_of.emplace(b->universes[q], (uint32_t)caller_of.size());
    if (!caller_of.empty()) {
        cudaError_t e = d_ft_caller.reserve(caller_of.size() * W);
        if (e == cudaErrorMemoryAllocation) {
            cudaGetLastError();
            return fail(B200_ERR_CAPACITY, "filter: the batch's universe bitmaps do not fit in device memory");
        }
        CU(e, "alloc filter universes");
        std::vector<uint64_t> host(caller_of.size() * W);
        for (auto &kv : caller_of)
            for (uint64_t w = 0; w < W; w++) host[kv.second * W + w] = kv.first[w] & hix.base_ub[w];
        CU(cudaMemcpyAsync(d_ft_caller.p, host.data(), host.size() * 8, cudaMemcpyHostToDevice, stream), "H2D universes");
        stats.h2d_bytes += host.size() * 8;
        CU(cudaStreamSynchronize(stream), "sync");  // the host copy goes out of scope
    }
    std::vector<const unsigned long long *> base(NQ, nullptr);
    for (uint32_t q = 0; q < NQ; q++) {
        if (!b->filter->begin || b->filter->begin[q + 1] <= b->filter->begin[q]) continue;
        if (gf.d_univ[q])
            base[q] = gf.d_univ[q];
        else if (b->universes && b->universes[q])
            base[q] = d_ft_caller.p + (size_t)caller_of[b->universes[q]] * W;
        else
            base[q] = dix.base_ub;
    }
    return run_filters(b->filter, base, gf);
}

int Engine::filter_batch(const b200_filter_programs *p, uint64_t *out, uint64_t out_words, int32_t *status, int32_t *error_leaf) {
    const uint64_t W = hix.n_words64;
    if (!p || (p->n && (!out || !status))) return fail(B200_ERR_INVALID, "filter_batch: null programs / out / status");
    if (out_words < W) return fail(B200_ERR_INVALID, "filter_batch: out_words smaller than the document range");
    CU(cudaSetDevice(device), "cudaSetDevice");
    const uint32_t n = p->n;
    GeoFiltered gf;
    gf.d_univ.assign(n, nullptr);
    gf.count.assign(n, 0);
    gf.status.assign(n, 0);
    gf.error.assign(n, std::string());
    for (uint32_t i = 0; i < n; i++) memset(out + (size_t)i * out_words, 0, out_words * 8);
    std::vector<const unsigned long long *> base(n, nullptr);
    for (uint32_t i = 0; i < n; i++)
        if (p->begin && p->begin[i + 1] > p->begin[i]) base[i] = dix.base_ub;
    int rc = run_filters(p, base, gf);
    if (rc != B200_OK) return rc;
    for (uint32_t i = 0; i < n; i++) {
        status[i] = gf.status[i];
        if (error_leaf) error_leaf[i] = gf.error_leaf.empty() ? -1 : gf.error_leaf[i];
        if (gf.status[i]) {
            last_error = gf.error[i];
            continue;
        }
        // no program: every document (documents_ids)
        const void *src = gf.d_univ[i] ? (const void *)gf.d_univ[i] : (const void *)dix.base_ub;
        CU(cudaMemcpyAsync(out + (size_t)i * out_words, src, W * 8, cudaMemcpyDeviceToHost, stream), "D2H filter");
        stats.d2h_bytes += W * 8;
    }
    CU(cudaStreamSynchronize(stream), "sync");
    return B200_OK;
}

}  // namespace b200
