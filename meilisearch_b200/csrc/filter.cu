// Filter programs (search/facet/filter/index_filter.rs:332-696) on the device.  engine_filter.cpp compiles a filter tree into a
// straight-line program over one-bit registers (device_types.h FilterOp); a thread runs it for one document.  A warp covers 32
// documents, half of a 64-document bitmap word: the result is one ballot.  Value leaves test the document's run of ordinals in the
// field's CSR (the one facet distribution reads) against the leaf's sorted ordinal intervals; EXISTS / IS NULL / IS EMPTY and geo
// leaves read a dense bitmap (a bounding box ANDed with its hint, as the range conditions it stands for are).  A FLAG op records whether an AND prefix is non-empty anywhere (the reach of the leaves after it).
#include <cuda_runtime.h>

#include "device_types.h"

namespace b200 {

namespace {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;

__device__ __forceinline__ bool rget(const uint32_t *r, uint32_t i) { return r[i >> 5] >> (i & 31) & 1u; }
__device__ __forceinline__ void rset(uint32_t *r, uint32_t i, bool v) {
    const uint32_t m = 1u << (i & 31);
    r[i >> 5] = v ? r[i >> 5] | m : r[i >> 5] & ~m;
}

// the document has an ordinal in one of the sorted, disjoint intervals iv[a, b)
__device__ bool in_intervals(const FilterOp &op, const uint2 *__restrict__ iv, uint32_t d) {
    if (!op.doc_off || op.a == op.b) return false;
    const uint32_t j1 = __ldg(op.doc_off + d + 1);
    for (uint32_t j = __ldg(op.doc_off + d); j < j1; j++) {
        const uint32_t o = __ldg(op.doc_ord + j);
        uint32_t lo = op.a, hi = op.b;  // the first interval starting after o
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (__ldg(&iv[mid].x) <= o)
                lo = mid + 1;
            else
                hi = mid;
        }
        if (lo > op.a && o < __ldg(&iv[lo - 1].y)) return true;
    }
    return false;
}

// blockIdx.y: the slot; the block's warps stride over the slot's 32-document half words
__global__ void __launch_bounds__(THREADS) filter_kernel(const FilterOp *__restrict__ ops, const uint2 *__restrict__ iv,
                                                         const FilterSlot *__restrict__ slots, uint32_t slot0,
                                                         const unsigned long long *__restrict__ docs, uint32_t n_docs, uint32_t n_half) {
    const FilterSlot &sl = slots[slot0 + blockIdx.y];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t *ub32 = reinterpret_cast<const uint32_t *>(sl.ub), *docs32 = reinterpret_cast<const uint32_t *>(docs);
    uint32_t *dst32 = reinterpret_cast<uint32_t *>(sl.dst);
    const uint32_t op_begin = sl.op_begin, op_end = sl.op_end;
    const bool all = sl.all != 0;
    unsigned long long count = 0;
    uint32_t regs[FILTER_REG_WORDS];
    for (uint32_t h = blockIdx.x * WARPS + warp; h < n_half; h += gridDim.x * WARPS) {
        const uint32_t u = __ldg(ub32 + h);
        if (!u && !all) {
            if (lane == 0) dst32[h] = 0;
            continue;
        }
        const uint32_t d = h * 32 + lane;
        const bool valid = d < n_docs, in_docs = __ldg(docs32 + h) >> lane & 1u;
        for (uint32_t i = op_begin; i < op_end; i++) {
            const FilterOp op = ops[i];
            switch (op.code) {
                case FOP_ZERO:
                    rset(regs, op.dst, false);
                    break;
                case FOP_VALUE: {
                    bool v = valid && in_intervals(op, iv, d);
                    if (op.neg) v = in_docs && !v;
                    if (op.hint != FILTER_NO_REG) v = v && rget(regs, op.hint);
                    rset(regs, op.dst, v);
                    break;
                }
                case FOP_BITMAP: {
                    bool v = op.bm && (__ldg(op.bm + (d >> 6)) >> (d & 63) & 1ull);
                    if (op.hint != FILTER_NO_REG) v = v && rget(regs, op.hint);
                    rset(regs, op.dst, v);
                    break;
                }
                case FOP_AND:
                    rset(regs, op.dst, rget(regs, op.dst) && rget(regs, op.src));
                    break;
                case FOP_OR:
                    rset(regs, op.dst, rget(regs, op.dst) || rget(regs, op.src));
                    break;
                case FOP_NOT:
                    rset(regs, op.dst, (op.hint != FILTER_NO_REG ? rget(regs, op.hint) : in_docs) && !rget(regs, op.dst));
                    break;
                case FOP_FLAG:
                    if (__any_sync(0xffffffffu, rget(regs, op.dst)) && lane == 0 && !sl.flags[op.a]) sl.flags[op.a] = 1;
                    break;
            }
        }
        const uint32_t word = __ballot_sync(0xffffffffu, rget(regs, 0)) & u;
        if (lane == 0) {
            dst32[h] = word;
            count += __popc(word);
        }
    }
    if (lane == 0 && count) atomicAdd(sl.count, count);
}

}  // namespace

cudaError_t launch_filter(cudaStream_t s, const FilterOp *ops, const uint2 *iv, const FilterSlot *slots, uint32_t n_slots,
                          const unsigned long long *docs, uint32_t n_docs, uint32_t n_words) {
    if (!n_slots || !n_words) return cudaSuccess;
    const uint32_t n_half = 2 * n_words, max_x = (n_half + WARPS - 1) / WARPS;
    for (uint32_t s0 = 0; s0 < n_slots; s0 += 65535) {
        const uint32_t ns = n_slots - s0 < 65535 ? n_slots - s0 : 65535;
        // about 4096 CTAs in all: a slot gets fewer when there are many
        const uint32_t gx = max(1u, min(max_x, 4096u / ns));
        filter_kernel<<<dim3(gx, ns), THREADS, 0, s>>>(ops, iv, slots, s0, docs, n_docs, n_half);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace b200
