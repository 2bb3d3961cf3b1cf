// Batched vector stage on the Hopper tensor cores: distances of a tile of 64 query vectors against the staged fp16 embedding
// matrix, with the exact top-k selection fused into the epilogue (the distance matrix never exists in HBM).
//
// Replaces, for a batch of semantic / hybrid queries, B calls of VectorStore::nns_by_vector
// (crates/milli/src/vector/store.rs:638-645, reached from VectorSort::fill_buffer, ranking_rules/vector_sort.rs:58-78)
// with one exhaustive scan: distance = (1 - cos)/2 (arroy/hannoy `Cosine`), ascending, ties by docid.
//
// Per CTA (one per SM, 256 threads):
//   warp 0     TMA producer: the query tile [64 x d] once (A operand, resident: d/64 blocks of 8 KB, 128B-swizzled, K-major),
//              then matrix blocks [128 rows x 64 halfs] = two row tiles through a 4-stage ring (B operand)
//   warp 1     stages each row tile's docids (filtered rows marked) and inverse norms (NaN for rows the norm rule may send to
//              distance 0) in shared memory, one tile ahead
//   warps 2-3  epilogue: lane = query; reads the tile's 64 fp32 dots from the accumulator staging buffer, distance, compare with
//              the query's running threshold, append survivors to the query's candidate run in L2-resident scratch; a
//              warp-cooperative bitonic sort compacts a run to its k best whenever it fills up, which tightens the threshold.
//   warps 4-7  one warpgroup issues wgmma.mma_async m64n128k16 (f16 in, f32 accumulators in registers) over the k-blocks of two
//              row tiles, then writes each tile's accumulators to one of two staging buffers in shared memory for the epilogue.
//              The scan is bound by this loop, not by L2 -> SM delivery (DESIGN.md §4): the wider N halves the instructions
//              issued and the query-operand bytes read from shared memory per matrix row.
// CTA c serves query tile c % n_qtiles and the c / n_qtiles-th slice of the row tiles; vec_merge_kernel merges the slices.
// The query tile is 64 rows (one warpgroup's M) so that a 768-wide tile (96 KB), the matrix ring and the staging buffers fit in
// the 227 KB of shared memory a block may use.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>

#include "kernels.h"

namespace b200 {

namespace {

constexpr int GM = VEC_GEMM_QTILE;  // queries per tile (wgmma M of one warpgroup)
constexpr int GN = 64;              // matrix rows per tile (the epilogue's unit: row metadata, staging buffer, candidate screen)
constexpr int MN = 2 * GN;          // matrix rows per MMA (wgmma N): two tiles per instruction
constexpr int GK = 64;              // halfs per k-block = one 128-byte swizzle span
constexpr int STAGES = 4;           // B ring depth (16 KB stages: 64 KB in flight)
constexpr int NACC = 2;             // accumulator staging buffers
constexpr int ACC_LD = GM + 4;      // floats per staged column: the fragment stores and the per-query loads are bank-conflict free
constexpr int META_BUFS = 2;        // row metadata (docid, inverse norm) staged per tile by warp 1
constexpr int EPI_WARPS = GM / 32;  // epilogue warps, one query per lane
constexpr int A_BLOCK = GM * GK * 2;        // 8 KB
constexpr int B_BLOCK = MN * GK * 2;        // 16 KB
constexpr int ACC_BYTES = GN * ACC_LD * 4;  // 17 KB
constexpr int CAND_CAP = VEC_GEMM_CAND_CAP;
constexpr int KMAX = VEC_GEMM_KMAX;
static_assert(GM % 32 == 0 && 2 + EPI_WARPS <= 4, "epilogue warps must fit between warp 1 and the MMA warpgroup");

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// BACKOFF > 0: sleep that many nanoseconds after a failed poll — the single-thread roles share their scheduler with other warps,
// and a tight polling loop takes their issue slots
template <int BACKOFF = 0>
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    uint64_t spins = 0;
    while (true) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) break;
        if (BACKOFF > 0) __nanosleep(BACKOFF);
        if (++spins > (1ull << 26)) __trap();  // a lost arrival must not hang the device
    }
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int32_t c0, int32_t c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
// one lane of a converged warp (the producer loop runs warp-convergent; only the issuing instructions are predicated)
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
// wgmma shared-memory descriptor, K-major with the 128-byte swizzle: 8-row groups are 1024 B apart (stride byte offset), the
// leading byte offset is unused for swizzled K-major operands.  Fields: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46),
// layout [62,64) = 1 (128B swizzle).  A K=16 step inside the swizzle span advances the start address by 32 B.
__device__ __forceinline__ uint64_t make_sdesc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3ffff) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator accesses across the asynchronous MMA
__device__ __forceinline__ void acc_fence(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

// ---- warp-cooperative bitonic sort of 256 u64 keys, element e = i*32 + lane held in k[i]
__device__ __forceinline__ void cswap(unsigned long long &a, unsigned long long &b, bool asc) {
    unsigned long long lo = a < b ? a : b, hi = a < b ? b : a;
    a = asc ? lo : hi;
    b = asc ? hi : lo;
}
template <int SIZE, int J>
__device__ __forceinline__ void sort_step(unsigned long long (&k)[8], uint32_t lane) {
    if constexpr (J >= 32) {
        constexpr int RJ = J >> 5;
#pragma unroll
        for (int i = 0; i < 8; i++)
            if ((i & RJ) == 0) cswap(k[i], k[i | RJ], ((i * 32) & SIZE) == 0);  // lane bits do not reach SIZE >= 64
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const uint32_t e = (uint32_t)i * 32u + lane;
            const unsigned long long o = __shfl_xor_sync(0xffffffffu, k[i], J);
            const bool asc = (e & (uint32_t)SIZE) == 0;
            const bool lower = (lane & (uint32_t)J) == 0;
            const unsigned long long lo = k[i] < o ? k[i] : o, hi = k[i] < o ? o : k[i];
            k[i] = (lower == asc) ? lo : hi;
        }
    }
    if constexpr (J > 1) sort_step<SIZE, J / 2>(k, lane);
}
template <int SIZE>
__device__ __forceinline__ void sort_size(unsigned long long (&k)[8], uint32_t lane) {
    sort_step<SIZE, SIZE / 2>(k, lane);
    if constexpr (SIZE < 256) sort_size<SIZE * 2>(k, lane);
}
__device__ __forceinline__ void warp_sort256(unsigned long long (&k)[8], uint32_t lane) { sort_size<2>(k, lane); }

// Sort lane `l`'s candidate run and keep its `kk` smallest keys; returns (all lanes) the new count and threshold of that lane.
__device__ __forceinline__ void compact_run(unsigned long long *run, uint32_t c, uint32_t kk, uint32_t kp, uint32_t lane, uint32_t &new_cnt,
                                            unsigned long long &new_thr, unsigned long long &kp_key) {
    unsigned long long k[8];
    __syncwarp();  // the owning lane's appends are visible to the whole warp
#pragma unroll
    for (int i = 0; i < 8; i++) {
        uint32_t e = (uint32_t)i * 32u + lane;
        k[i] = e < c ? run[e] : ~0ull;
    }
    warp_sort256(k, lane);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 8; i++) {
        uint32_t e = (uint32_t)i * 32u + lane;
        if (e < kk) run[e] = k[i];
    }
    // key at rank kk-1
    const uint32_t ri = (kk - 1) >> 5;  // < KMAX/32 = 4
    unsigned long long mine = ri == 0 ? k[0] : (ri == 1 ? k[1] : (ri == 2 ? k[2] : k[3]));
    unsigned long long kth = __shfl_sync(0xffffffffu, mine, (kk - 1) & 31);
    const uint32_t rp = (kp - 1) >> 5;
    unsigned long long minep = rp == 0 ? k[0] : (rp == 1 ? k[1] : (rp == 2 ? k[2] : k[3]));
    unsigned long long kpth = __shfl_sync(0xffffffffu, minep, (kp - 1) & 31);
    new_cnt = c < kk ? c : kk;
    new_thr = c >= kk ? kth : ~0ull;
    kp_key = c >= kp ? kpth : ~0ull;  // this slice's kp-th best so far
    __syncwarp();
}

// Smallest value of (dot x inverse row norm) a row needs in order to possibly have key < thr, with a safety margin for the
// different rounding of the fast test: dd <= dd_thr  =>  cos >= 1 - 2 dd_thr  =>  dot*rn >= (1 - 2 dd_thr) / qn.
__device__ __forceinline__ float reject_bound(unsigned long long thr, float qn) {
    if (thr == ~0ull || !(qn > 0.f)) return __int_as_float(0xff800000);
    const float dd_thr = __uint_as_float((uint32_t)(thr >> 32));
    const float cs_min = 1.f - 2.f * dd_thr - 4e-7f;
    if (cs_min <= -1.f) return __int_as_float(0xff800000);
    const float x = cs_min / qn;
    return x - fabsf(x) * 2e-6f - 1e-30f;
}

}  // namespace

__global__ void __launch_bounds__(256, 1)
    vec_gemm_topk_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_m, uint64_t n_rows, uint32_t kblocks,
                         uint32_t n_qtiles, uint32_t n_groups, const float *__restrict__ inv_norm, const uint32_t *__restrict__ docids,
                         const float *__restrict__ q_inv_norm, const unsigned long long *__restrict__ cand, uint64_t n_cand_words, uint32_t kk,
                         unsigned long long *__restrict__ gthr /* [n_qtiles*GM][n_groups], init ~0: each slice's ceil(k/n_groups)-th best key so far */,
                         unsigned long long *__restrict__ runs /* [cta][GM][CAND_CAP] */,
                         unsigned long long *__restrict__ partial /* [n_qtiles*GM][n_groups][KMAX] */) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t *sA = smem;
    uint8_t *sB = sA + (size_t)kblocks * A_BLOCK;
    float *sAcc = reinterpret_cast<float *>(sB + STAGES * B_BLOCK);
    uint64_t *bars = reinterpret_cast<uint64_t *>(sAcc + NACC * (ACC_BYTES / 4));
    uint64_t *a_full = bars, *b_full = bars + 1, *b_empty = b_full + STAGES, *acc_full = b_empty + STAGES, *acc_empty = acc_full + NACC;
    uint64_t *meta_full = acc_empty + NACC, *meta_empty = meta_full + META_BUFS;
    // row metadata ring: static shared memory, so that the epilogue reads it with (vectorisable) LDS instead of generic loads
    __shared__ __align__(16) uint32_t s_doc[META_BUFS * GN];
    __shared__ __align__(16) float s_scale[META_BUFS * GN];
    __shared__ __align__(16) float s_norm[META_BUFS * GN];  // the rows' own inverse norms, for the NaN-scaled ones

    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t qtile = blockIdx.x % n_qtiles, group = blockIdx.x / n_qtiles;
    if (group >= n_groups) return;  // whole CTA: before any barrier
    const uint64_t n_tiles = (n_rows + GN - 1) / GN;
    const uint64_t tile_lo = n_tiles * group / n_groups, tile_hi = n_tiles * (group + 1) / n_groups;

    if (threadIdx.x == 0) {
        mbar_init(a_full, 1);
        for (int s = 0; s < STAGES; s++) {
            mbar_init(b_full + s, 1);
            mbar_init(b_empty + s, 1);
        }
        for (int b = 0; b < NACC; b++) {
            mbar_init(acc_full + b, 128);             // every thread of the MMA warpgroup, after its fragment stores
            mbar_init(acc_empty + b, EPI_WARPS * 32); // every epilogue thread, after its last read of the buffer
        }
        for (int b = 0; b < META_BUFS; b++) {
            mbar_init(meta_full + b, 1);
            mbar_init(meta_empty + b, EPI_WARPS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        const bool leader = elect_one();
        if (leader) {
            mbar_expect_tx(a_full, kblocks * A_BLOCK);
            for (uint32_t kb = 0; kb < kblocks; kb++) tma_load_2d(sA + (size_t)kb * A_BLOCK, &tmap_q, a_full, (int32_t)(kb * GK), (int32_t)(qtile * GM));
        }
        uint32_t s = 0, ph = 0;
        for (uint64_t t = tile_lo; t < tile_hi; t += 2)
            for (uint32_t kb = 0; kb < kblocks; kb++) {
                mbar_wait<128>(b_empty + s, ph ^ 1);
                if (leader) {
                    mbar_expect_tx(b_full + s, B_BLOCK);
                    tma_load_2d(sB + (size_t)s * B_BLOCK, &tmap_m, b_full + s, (int32_t)(kb * GK), (int32_t)(t * GN));
                }
                __syncwarp();
                if (++s == (uint32_t)STAGES) {
                    s = 0;
                    ph ^= 1;
                }
            }
    } else if (warp == 1) {
        // The fast reject of the epilogue compares dot x inverse row norm with a bound derived from a real cosine; it knows nothing
        // of the norm rule (distance 0 unless 0 < pn < 2^23).  Rows that rule can send to 0 for some query of the tile bypass the
        // reject: for a query with a non-zero inverse norm qn that is a zero row, or one with scale * qn >= 2^23, and the product is
        // monotonic in qn, so the tile's largest qn decides.  (Zero queries have no reject bound at all.)  Such a row is staged
        // with a NaN scale: v * NaN < bound is false for every query, and the exact test reads the row's own scale.
        float qmax = 0.f;
        for (uint32_t i = lane; i < GM; i += 32) qmax = fmaxf(qmax, q_inv_norm[qtile * GM + i]);
#pragma unroll
        for (int o = 16; o; o >>= 1) qmax = fmaxf(qmax, __shfl_xor_sync(0xffffffffu, qmax, o));
        uint32_t n = 0;
        for (uint64_t t = tile_lo; t < tile_hi; t++, n++) {
            const uint32_t mb = n % META_BUFS, mph = (n / META_BUFS) & 1;
            mbar_wait<128>(meta_empty + mb, mph ^ 1);
#pragma unroll
            for (int h = 0; h < GN / 32; h++) {
                const uint64_t r = t * GN + (uint32_t)h * 32u + lane;
                uint32_t doc = 0xffffffffu;
                float sc = 0.f, nrm = 0.f;
                if (r < n_rows) {
                    doc = __ldg(docids + r);
                    sc = nrm = __ldg(inv_norm + r);
                    if (!(sc > 0.f && sc * qmax < VEC_PN_MAX)) sc = __int_as_float(0x7fffffff);
                    if (cand && !((doc >> 6) < n_cand_words && ((__ldg(cand + (doc >> 6)) >> (doc & 63)) & 1))) doc = 0xffffffffu;
                }
                s_doc[mb * GN + h * 32 + lane] = doc;
                s_scale[mb * GN + h * 32 + lane] = sc;
                s_norm[mb * GN + h * 32 + lane] = nrm;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(meta_full + mb);
        }
    } else if (warp >= 4) {
        // MMA warpgroup: accumulators of two row tiles in registers (64 fp32 per thread), one commit group per k-block; the ring
        // stage of k-block kb is released once the group of kb + 1 is issued and that of kb has completed.  An m64n128k16 does the
        // work of two m64n64k16 in fewer issue slots and shared-memory reads of the query operand; every dot is the same sum.
        const uint32_t wq = warp - 4, g = lane >> 2, q = lane & 3;
        const uint64_t ad0 = make_sdesc(smem_u32(sA)), bd0 = make_sdesc(smem_u32(sB));
        mbar_wait(a_full, 0);
        uint32_t s = 0, ph = 0, n = 0;
        for (uint64_t t = tile_lo; t < tile_hi; t += 2) {
            float acc[64];
#pragma unroll
            for (int i = 0; i < 64; i++) acc[i] = 0.f;
            uint32_t prev = 0;
            for (uint32_t kb = 0; kb < kblocks; kb++) {
                mbar_wait(b_full + s, ph);
                wgmma_fence();
                acc_fence(acc);
                const uint64_t ad = ad0 + (uint64_t)kb * (A_BLOCK >> 4), bd = bd0 + (uint64_t)s * (B_BLOCK >> 4);
#pragma unroll
                for (uint32_t k = 0; k < GK / 16; k++) wgmma_m64n128k16(acc, ad + 2 * k, bd + 2 * k, (kb | k) != 0);  // +32 B per K=16 step
                wgmma_commit();
                acc_fence(acc);
                if (kb > 0) {
                    wgmma_wait<1>();
                    if (threadIdx.x == 128) mbar_arrive(b_empty + prev);
                }
                prev = s;
                if (++s == (uint32_t)STAGES) {
                    s = 0;
                    ph ^= 1;
                }
            }
            wgmma_wait<0>();
            acc_fence(acc);
            if (threadIdx.x == 128) mbar_arrive(b_empty + prev);
            // fragment -> staging buffer, one tile (64 rows) at a time, column-major: element (query r, row c) at c * ACC_LD + r.
            // Thread (warp wq, lane) holds queries 16 wq + g and 16 wq + g + 8, rows 8 i + 2 q and 8 i + 2 q + 1 of every n8 block i;
            // blocks 0-7 are tile t, blocks 8-15 tile t + 1.  When the slice has an odd number of tiles, the second half of its last
            // block (rows of the next slice, or zeros past the matrix) is computed and dropped.
#pragma unroll
            for (int h = 0; h < MN / GN; h++, n++) {
                if (t + h >= tile_hi) break;
                const uint32_t buf = n & 1, aph = (n >> 1) & 1;
                mbar_wait(acc_empty + buf, aph ^ 1);
                float *dst = sAcc + buf * (ACC_BYTES / 4) + wq * 16 + g;
#pragma unroll
                for (int i = 0; i < GN / 8; i++) {
                    const uint32_t c = 8 * i + 2 * q;
                    const int a = 4 * (h * (GN / 8) + i);
                    dst[c * ACC_LD] = acc[a];
                    dst[(c + 1) * ACC_LD] = acc[a + 1];
                    dst[c * ACC_LD + 8] = acc[a + 2];
                    dst[(c + 1) * ACC_LD + 8] = acc[a + 3];
                }
                mbar_arrive(acc_full + buf);
            }
        }
    } else if (warp >= 2 && warp < 2 + EPI_WARPS) {
        const uint32_t w = warp - 2;
        const uint32_t qcol = w * 32 + lane;  // this lane's query inside the tile
        const uint32_t qrow = qtile * GM + qcol;
        const float qn = q_inv_norm[qrow];
        unsigned long long *my_run = runs + ((size_t)blockIdx.x * GM + qcol) * CAND_CAP;
        unsigned long long *warp_runs = runs + ((size_t)blockIdx.x * GM + w * 32) * CAND_CAP;
        uint32_t cnt = 0;
        unsigned long long thr = ~0ull;
        float tq = __int_as_float(0xff800000);  // -inf: nothing is rejected before a threshold exists
        const uint32_t kp = (kk + n_groups - 1) / n_groups;  // per-slice share of the k best
        // When kp is small the slice's kp best keys live in registers, so its published bound is always current (it does not
        // wait for a run compaction) and the shared threshold tightens with every candidate.
        constexpr int KP_REG = 8;
        const bool reg_best = kp <= (uint32_t)KP_REG;
        unsigned long long best[KP_REG];
#pragma unroll
        for (int i = 0; i < KP_REG; i++) best[i] = ~0ull;
        unsigned long long published = ~0ull, best_kp = ~0ull;  // best_kp == best[kp - 1]
        uint32_t n = 0;
        for (uint64_t t = tile_lo; t < tile_hi; t++, n++) {
            const uint32_t buf = n % NACC, aph = (n / NACC) & 1;
            mbar_wait(acc_full + buf, aph);
            const float *col = sAcc + buf * (ACC_BYTES / 4) + qcol;
            float v[GN];
#pragma unroll
            for (int j = 0; j < GN; j++) v[j] = col[j * ACC_LD];
            const uint32_t mb = n % META_BUFS, mph = (n / META_BUFS) & 1;
            mbar_wait(meta_full + mb, mph);
            const uint32_t *tdoc = s_doc + mb * GN;
            const float *tscale = s_scale + mb * GN, *tnorm = s_norm + mb * GN;
            // pass 1, branch-free: which of the 64 rows can possibly beat this query's threshold ("dot x inverse row norm" space;
            // a NaN scale, a row the norm rule may send to 0, always passes)
            uint32_t m_lo = 0, m_hi = 0;
#pragma unroll
            for (int j = 0; j < 32; j++) {
                m_lo |= (v[j] * tscale[j] < tq) ? 0u : (1u << j);
                m_hi |= (v[j + 32] * tscale[j + 32] < tq) ? 0u : (1u << j);
            }
            uint32_t u_lo = __reduce_or_sync(0xffffffffu, m_lo), u_hi = __reduce_or_sync(0xffffffffu, m_hi);
            // pass 2: exact distance + append for the (rare) columns some lane flagged.  A compact loop over the set bits — the dot is
            // re-read from the staging buffer — instead of 64 unrolled copies: the hot loop stays small enough for the instruction cache.
            while (u_lo | u_hi) {  // warp-uniform
                const uint32_t j = u_lo ? (uint32_t)__ffs(u_lo) - 1u : 32u + (uint32_t)__ffs(u_hi) - 1u;
                if (u_lo)
                    u_lo &= u_lo - 1;
                else
                    u_hi &= u_hi - 1;
                const uint32_t mm = j < 32 ? m_lo : m_hi;
                if ((mm >> (j & 31)) & 1u) {
                    const float dot = col[j * ACC_LD];
                    const uint32_t doc = tdoc[j];
                    float pn = tscale[j] * qn;
                    // A row staged with a finite scale has 0 <= pn <= scale x (the tile's largest qn) < 2^23, so for it the norm
                    // rule is pn > 0.  A NaN scale (warp 1) takes the rule with the row's own scale.
                    if (pn != pn) {
                        pn = tnorm[j] * qn;
                        pn = pn < VEC_PN_MAX ? pn : 0.f;
                    }
                    float dd = 0.f;
                    if (pn > 0.f && isfinite(pn)) {
                        float cs = dot * pn;
                        cs = fminf(1.f, fmaxf(-1.f, cs));
                        dd = (1.f - cs) * 0.5f;
                    }
                    const unsigned long long key = ((unsigned long long)__float_as_uint(dd) << 32) | doc;
                    if (doc != 0xffffffffu && key < thr) {
                        my_run[cnt++] = key;
                        if (reg_best && key < best_kp) {  // improves this slice's kp best: sorted insertion, the largest falls off
                            unsigned long long x = key;
#pragma unroll
                            for (int i = 0; i < KP_REG; i++) {
                                const unsigned long long lo = x < best[i] ? x : best[i], hi = x < best[i] ? best[i] : x;
                                best[i] = lo;
                                x = hi;
                            }
                            best_kp = best[0];
#pragma unroll
                            for (int i = 1; i < KP_REG; i++) best_kp = (uint32_t)i < kp ? best[i] : best_kp;
                        }
                    }
                }
            }
            mbar_arrive(acc_empty + buf);
            __syncwarp();
            if (lane == 0) mbar_arrive(meta_empty + mb);
            bool changed = false;
            // compaction: when a run is nearly full — and once right after the first tile, so that every slice publishes an early
            // bound (see below) instead of appending everything for three tiles
            uint32_t need = __ballot_sync(0xffffffffu, cnt > (uint32_t)(CAND_CAP - GN) || (!reg_best && n == 0 && cnt >= kp));
            while (need) {
                uint32_t l = __ffs(need) - 1;
                need &= need - 1;
                uint32_t c = __shfl_sync(0xffffffffu, cnt, l), nc;
                unsigned long long nt, xp;
                compact_run(warp_runs + (size_t)l * CAND_CAP, c, kk, kp, lane, nc, nt, xp);
                if (lane == l) {
                    cnt = nc;
                    if (nt < thr) {
                        thr = nt;
                        changed = true;
                    }
                    // this slice holds kp = ceil(k / n_groups) keys <= xp; once every slice has published, the largest of their
                    // xp is an upper bound of the global k-th key (n_groups * kp >= k keys are <= it)
                    if (!reg_best && xp != ~0ull) gthr[(size_t)qrow * n_groups + group] = xp;
                }
            }
            if (reg_best && best_kp < published) {
                published = best_kp;
                __stcg(gthr + (size_t)qrow * n_groups + group, best_kp);
            }
            if (n < 8 || (n < 64 && (n & 3) == 1) || (n & 15) == 1) {  // every tile while the bound still moves fast, then ever more rarely
                const unsigned long long *gx = gthr + (size_t)qrow * n_groups;
                unsigned long long bound = 0;
                for (uint32_t g0 = 0; g0 < n_groups; g0 += 6) {
                    unsigned long long x[6];
#pragma unroll
                    for (int i = 0; i < 6; i++) x[i] = g0 + i < n_groups ? __ldcg(gx + g0 + i) : 0ull;  // L2 reads, issued together
#pragma unroll
                    for (int i = 0; i < 6; i++) bound = x[i] > bound ? x[i] : bound;
                }
                if (bound < thr) {
                    thr = bound;
                    changed = true;
                }
            }
            if (changed) tq = reject_bound(thr, qn);
        }
        // final: every lane's run sorted, its kk best written to this (query, group) slot
        __syncwarp();
        for (uint32_t l = 0; l < 32; l++) {
            uint32_t c = __shfl_sync(0xffffffffu, cnt, l);
            unsigned long long *run = warp_runs + (size_t)l * CAND_CAP;
            unsigned long long k[8];
#pragma unroll
            for (int i = 0; i < 8; i++) {
                uint32_t e = (uint32_t)i * 32u + lane;
                k[i] = e < c ? run[e] : ~0ull;
            }
            warp_sort256(k, lane);
            unsigned long long *out = partial + ((size_t)(qtile * GM + w * 32 + l) * n_groups + group) * KMAX;
#pragma unroll
            for (int i = 0; i < KMAX / 32; i++) {
                uint32_t e = (uint32_t)i * 32u + lane;
                out[e] = e < kk ? k[i] : ~0ull;
            }
        }
    }
    __syncthreads();
}

// fp32 queries -> fp16 padded tile rows + inverse norms (one warp per query; rows >= n_q are zero)
__global__ void vec_prep_queries_kernel(const float *__restrict__ q, uint32_t n_q, uint32_t n_pad, uint32_t d, __half *__restrict__ out,
                                        float *__restrict__ inv) {
    uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= n_pad) return;
    float s = 0.f;
    for (uint32_t i = lane; i < d; i += 32) {
        float x = w < n_q ? q[(size_t)w * d + i] : 0.f;
        out[(size_t)w * d + i] = __float2half_rn(x);
        s = fmaf(x, x, s);
    }
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
        float nrm = sqrtf(s);
        inv[w] = nrm > 0.f ? 1.0f / nrm : 0.f;
    }
}

// Merge the per-group sorted runs of one query: keep the KMAX smallest with a bitonic merge of (best ascending, run descending).
__global__ void __launch_bounds__(KMAX) vec_merge_kernel(const unsigned long long *__restrict__ partial, uint32_t n_groups, uint32_t kk,
                                                          uint32_t *__restrict__ out_ids, float *__restrict__ out_dist, uint32_t *__restrict__ out_n) {
    __shared__ unsigned long long s[2 * KMAX];
    const uint32_t q = blockIdx.x, t = threadIdx.x;
    const unsigned long long *p = partial + (size_t)q * n_groups * KMAX;
    s[t] = p[t];
    for (uint32_t g = 1; g < n_groups; g++) {
        s[2 * KMAX - 1 - t] = p[(size_t)g * KMAX + t];  // reversed: s[0..2K) is bitonic
        __syncthreads();
        {  // first step keeps the lower half only
            unsigned long long a = s[t], b = s[t + KMAX];
            s[t] = a < b ? a : b;
        }
        __syncthreads();
        for (uint32_t j = KMAX / 2; j >= 1; j >>= 1) {
            uint32_t o = t ^ j;
            unsigned long long a = s[t], b = s[o];
            __syncthreads();
            if (o > t) {
                s[t] = a < b ? a : b;
                s[o] = a < b ? b : a;
            }
            __syncthreads();
        }
    }
    __syncthreads();
    unsigned long long key = s[t];
    if (t < kk) {
        out_ids[(size_t)q * kk + t] = (uint32_t)key;
        out_dist[(size_t)q * kk + t] = __uint_as_float((uint32_t)(key >> 32));
    }
    uint32_t valid = __syncthreads_count(t < kk && key != ~0ull);
    if (t == 0) out_n[q] = valid;
}

// ------------------------------------------------------------------------------------------------ host side
namespace {
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess)
            p = nullptr;
        return reinterpret_cast<EncodeTiledFn>(p);
    }();
    return fn;
}
bool make_map(CUtensorMap *m, const void *base, uint64_t rows, uint32_t d, uint32_t box_rows) {
    EncodeTiledFn f = encode_tiled();
    if (!f) return false;
    cuuint64_t dims[2] = {d, rows};
    cuuint64_t strides[1] = {(cuuint64_t)d * 2};
    cuuint32_t box[2] = {(cuuint32_t)GK, box_rows};
    cuuint32_t estr[2] = {1, 1};
    return f(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
}  // namespace

size_t vec_gemm_smem_bytes(uint32_t d) {
    // query tile + B ring + accumulator staging + barriers + alignment slack (the 1 KB of row metadata is static)
    return (size_t)(d / GK) * A_BLOCK + (size_t)STAGES * B_BLOCK + (size_t)NACC * ACC_BYTES + 256 + 1023;
}

bool vec_gemm_supported(uint32_t d, uint32_t limit) { return d % GK == 0 && d >= GK && d <= 768 && limit >= 1 && limit <= KMAX; }

cudaError_t launch_vec_prep_queries(cudaStream_t s, const float *q, uint32_t n_q, uint32_t n_pad, uint32_t d, void *out_fp16, float *inv) {
    vec_prep_queries_kernel<<<(n_pad * 32 + 255) / 256, 256, 0, s>>>(q, n_q, n_pad, d, reinterpret_cast<__half *>(out_fp16), inv);
    return cudaGetLastError();
}

cudaError_t launch_vec_gemm_topk(cudaStream_t s, uint32_t sm_count, const void *mat_fp16, const float *inv_norm, const uint32_t *docids, uint64_t n_rows,
                                 uint32_t d, const void *q_fp16, const float *q_inv_norm, uint32_t n_qtiles, uint32_t n_groups,
                                 const unsigned long long *cand, uint64_t n_cand_words, uint32_t k, unsigned long long *gthr, unsigned long long *runs,
                                 unsigned long long *partial, uint32_t *out_ids, float *out_dist, uint32_t *out_n, uint32_t n_q) {
    if (!vec_gemm_supported(d, k) || n_qtiles * n_groups > sm_count || n_groups == 0) return cudaErrorInvalidValue;
    CUtensorMap mq, mm;
    if (!make_map(&mq, q_fp16, (uint64_t)n_qtiles * GM, d, GM) || !make_map(&mm, mat_fp16, n_rows, d, MN)) return cudaErrorNotSupported;
    cudaError_t e = cudaMemsetAsync(gthr, 0xff, (size_t)n_qtiles * GM * n_groups * 8, s);
    if (e != cudaSuccess) return e;
    const size_t smem = vec_gemm_smem_bytes(d);
    e = cudaFuncSetAttribute(vec_gemm_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    vec_gemm_topk_kernel<<<n_qtiles * n_groups, 256, smem, s>>>(mq, mm, n_rows, d / GK, n_qtiles, n_groups, inv_norm, docids, q_inv_norm, cand,
                                                                n_cand_words, k, gthr, runs, partial);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    vec_merge_kernel<<<n_q, KMAX, 0, s>>>(partial, n_groups, k, out_ids, out_dist, out_n);
    return cudaGetLastError();
}

}  // namespace b200
