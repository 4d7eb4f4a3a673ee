// knn_filter_sm90.cu — the dominant kernel: fused Q.K^T (Hopper wgmma, fp32 accumulators in registers, TMA-staged
// operand tiles) + per-query streaming top-KP selection in the epilogue.
//
// Replaces the arithmetic of faiss `Index.search` as called from lotus/vector_store/faiss_vs.py:67,75
// (knn_inner_product / knn_L2sqr: blocked sgemm + heap). The N x Q score matrix is never written to HBM.
//
// Role of this kernel in the exact pipeline (DESIGN.md §Pipeline): it is a FILTER. It computes scores with
// bf16 (or TF32) tensor-core products and fp32 accumulation and keeps, per query and per corpus split,
// the KP > k best candidates plus the value `thr` below which everything was discarded. knn_exact.cu then
// re-scores the candidates in the canonical fp64 order and certifies, with a rigorous error margin, that
// nothing discarded could belong to the true top-k; uncertified queries take the dense exact path.
//
// Kernel shape: a CTA owns 128 queries and computes 128 queries x 256 corpus rows per tile.
//   warpgroup 0: TMA producer (one lane)
//   warpgroups 1, 2: consumers; consumer g issues wgmma m64n256 for query rows 64g..64g+63 (fp32 accumulators in
//                    registers, 128 per thread) and runs the epilogue of those rows
//   K-block = one 64-byte swizzle row (32 bf16 / 16 tf32): wgmma k16 (bf16) or k8 (tf32), two per K-block.
//   smem ring of NSTAGES x (A 8 KB + B 16 KB), mbarrier full/empty pairs.
//   CTA pairs (default once there are two query tiles): a 2-CTA cluster takes two consecutive query tiles and sweeps the
//   same corpus tiles; each CTA loads HALF of every corpus tile and TMA-multicasts it into both CTAs, so the corpus bytes
//   read per SM drop by half. A stage is freed once the consumers of both CTAs are done with it.
//   Persistent: one CTA per SM, work item = (query unit, corpus split), query units fastest so that co-resident
//   workers stream the same corpus tiles and hit them in L2.
//
// Epilogue lists: the wgmma fragment spreads a query row over four lanes, so each warp passes its 16 rows x 256 scores
// through a small shared-memory transpose, 16 columns at a time; afterwards lane (r, e) = (lane & 15, lane >> 4) holds 8
// scores of row r. Candidate list ("set") e of a row collects the columns c with bit 3 of c equal to e, so a query keeps
// two lists of KP/2 per corpus split, the layout finalize merges.
#include <cuda.h>

#include "common.cuh"

namespace b2 {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 256;
constexpr int WG_M = 64;        // query rows per consumer warpgroup (wgmma M)
constexpr int KB_BYTES = 64;    // K-block: one SWIZZLE_64B row
constexpr int KSTEPS = 2;       // wgmma K steps (32 bytes each) per K-block
constexpr int STAGE_A_BYTES = BLOCK_M * KB_BYTES;
constexpr int STAGE_B_BYTES = BLOCK_N * KB_BYTES;
constexpr int STAGE_BYTES = STAGE_A_BYTES + STAGE_B_BYTES;
constexpr int NUM_THREADS = 384;   // producer warpgroup + two consumer warpgroups
constexpr int CONSUMER_WARPS = 8;
constexpr int MAX_STAGES = 8;
constexpr int SMEM_LIMIT = 232448;  // 227 KB
constexpr int SMEM_ALIGN_SLACK = 1024;  // the ring is aligned to 1024 B by hand
constexpr int BAR_BYTES = 256;
constexpr int FILTER_MAX_K = 1000;  // largest k served by the filter (finalize keeps min(k + 32, 1024) survivors per query)

// pending (not yet merged) candidates per (query row, set): a flush is triggered once any row holds PEND_FLUSH of them,
// checked after each 8-column group, so a row never holds more than PEND_FLUSH - 1 + 8 <= PEND
constexpr int PEND = 16;
constexpr int PEND_FLUSH = 8;
// per-set strides of the lists and pending buffers, padded by 16 so that the two halves of a warp (two sets, same 16 rows)
// use different banks
__host__ __device__ constexpr int list_set_stride(int kph) { return kph * BLOCK_M + 16; }
constexpr int PEND_SET_STRIDE = PEND * BLOCK_M + 16;
__host__ __device__ constexpr int list_bytes(int kp) { return 2 /*sets*/ * 2 /*score, id*/ * 4 * (list_set_stride(kp / 2) + PEND_SET_STRIDE); }
// transpose scratch: 16 rows x 16 columns per consumer warp, rows padded to 17 floats
constexpr int XP_STRIDE = 17;
constexpr int XP_WARP_FLOATS = 16 * XP_STRIDE;
__host__ __device__ constexpr int misc_bytes() { return CONSUMER_WARPS * XP_WARP_FLOATS * 4 + BAR_BYTES + SMEM_ALIGN_SLACK; }
__host__ __device__ constexpr int num_stages(int kp) {
    const int s = (SMEM_LIMIT - list_bytes(kp) - misc_bytes()) / STAGE_BYTES;
    return s > MAX_STAGES ? MAX_STAGES : s;
}
__host__ __device__ constexpr int smem_bytes(int kp) { return num_stages(kp) * STAGE_BYTES + list_bytes(kp) + misc_bytes(); }

// ---- PTX wrappers ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive on the barrier at the same offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// Bounded wait: a protocol bug must trap (sticky error the host reports) instead of hanging the GPU. No printf here: a
// function call inside the consumers' wgmma pipeline makes ptxas serialize every wgmma.
template <bool SUSPEND>
__device__ __forceinline__ void mbar_wait_impl(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    uint32_t spins = 0;
    long long t_start = 0;
    while (true) {
        if constexpr (SUSPEND) {
            asm volatile(
                "{\n\t.reg .pred p;\n\t"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
                "selp.u32 %0, 1, 0, p;\n\t}"
                : "=r"(done)
                : "r"(addr), "r"(parity), "r"(20000u)  // suspend-time hint (ns): sleep in hardware instead of spinning
                : "memory");
        } else {
            asm volatile(
                "{\n\t.reg .pred p;\n\t"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                "selp.u32 %0, 1, 0, p;\n\t}"
                : "=r"(done)
                : "r"(addr), "r"(parity)
                : "memory");
        }
        if (done) break;
        if ((++spins & 0x3ffu) == 0) {
            const long long now = clock64();
            if (t_start == 0) t_start = now;
            else if (now - t_start > 8000000000LL) __trap();  // ~4 s at 2 GHz: no legitimate wait is longer than microseconds
        }
    }
}
// the producer may sleep; the consumers must wake the moment their operands land
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { mbar_wait_impl<true>(bar, parity); }
__device__ __forceinline__ void mbar_wait_spin(uint64_t* bar, uint32_t parity) { mbar_wait_impl<false>(bar, parity); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// the box lands at the same offset in every CTA of `mask`, each completing the bytes on its own barrier at `bar`'s offset
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1,
                                                      uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
            smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// wgmma shared-memory descriptor: K-major operand tile, rows of 64 bytes, SWIZZLE_64B (the layout a TMA box
// {64 B, rows} with CU_TENSOR_MAP_SWIZZLE_64B lands in). 8-row groups are 512 B apart (SBO).
__device__ __forceinline__ uint64_t make_sw64_desc(uint32_t smem_addr) {
    uint64_t desc = 0;
    desc |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);      // start address, bits [0,14)
    desc |= (uint64_t)1 << 16;                            // leading byte offset (ignored for swizzled K-major)
    desc |= (uint64_t)((8 * KB_BYTES) >> 4) << 32;        // stride byte offset, bits [32,46)
    desc |= (uint64_t)2 << 62;                            // layout type: SWIZZLE_64B
    return desc;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads or writes across a wgmma wait
__device__ __forceinline__ void acc_fence(float (&d)[128]) {
#pragma unroll
    for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 256] (+)= A[64 x K] . B[256 x K]^T, both K-major in shared memory; scale_d == 0 overwrites D
template <bool TF32>
__device__ __forceinline__ void wgmma_64x256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    if constexpr (TF32) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
            : "l"(adesc), "l"(bdesc), "r"(scale_d));
    } else {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
            : "l"(adesc), "l"(bdesc), "r"(scale_d));
    }
}

struct FilterParams {
    const float* xnorm;  // [n], L2 only
    float* cand_score;   // [nq, n_splits, KP]
    int32_t* cand_id;    // [nq, n_splits, KP]
    float* cand_thr;     // [nq, n_splits, 2]
    int32_t nq;
    int32_t n;
    int32_t num_kb;        // K-blocks per tile = ceil(d / elements per 64 B)
    int32_t n_mtiles;      // ceil(nq / 128)
    int32_t n_munits;      // schedulable query units: n_mtiles, or ceil(n_mtiles / 2) CTA pairs
    int32_t n_splits;
    int32_t top1;             // host-side switch only: the TOP1 kernel variant is launched (k-means assignment)
    int32_t tiles_per_split;  // corpus tiles (of 256 rows) per split
    int32_t units_whole;      // two-phase schedule: the first units_whole query units (a multiple of the worker count) sweep the WHOLE
                              // corpus as one item each (split 0); only the remaining units are cut into n_splits splits
    int32_t n_ntiles;         // ceil(n / 256)
    // all-pairs (dedup) schedule: the query matrix IS the corpus; an item is one query unit sweeping only the corpus tiles
    // that can hold a column j > i (upper triangle). Query units are dealt to the `nparts` ranks in GROUPS of pair_group
    // consecutive units (group g belongs to rank g % nparts): the CTAs of one rank then walk neighbouring corpus tiles at
    // the same time and share them through L2 (dealing single tiles round-robin spreads the concurrently read corpus
    // window nparts times wider).
    int32_t pair_mode, part, nparts, pair_group, pair_items;
    int32_t pair_align;  // 1: every unit of a group starts its sweep at the group's first corpus tile (equal sweep lengths
                         // keep the CTAs of a wave on the same corpus tile for the whole launch; costs <= group/2 extra tiles)
    float pair_thr;                   // emit candidates with filter score > pair_thr
    int32_t* pair_i;                  // [pair_cap]
    int32_t* pair_j;
    unsigned long long* pair_count;   // total candidates found (may exceed pair_cap)
    unsigned long long pair_cap;
};

struct Ring {
    uint8_t* stage_base;
    uint64_t *full_bar, *empty_bar;
};

// Persistent schedule. A "worker" is a CTA (or a CTA pair); item = (query unit, corpus split), unit fastest so that
// co-resident workers stream the same corpus tiles and share them in L2.
struct Sched {
    int worker, n_workers, rank;  // rank = CTA rank inside the pair (0 in single-CTA mode)
};
template <bool TWO>
__device__ __forceinline__ Sched make_sched() {
    Sched sc;
    if constexpr (TWO) {
        sc.worker = blockIdx.x >> 1;
        sc.n_workers = gridDim.x >> 1;
        sc.rank = (int)cluster_ctarank();
    } else {
        sc.worker = blockIdx.x;
        sc.n_workers = gridDim.x;
        sc.rank = 0;
    }
    return sc;
}
__device__ __forceinline__ int num_items(const FilterParams& p) {
    if (p.pair_mode) return p.pair_items;
    return p.units_whole + (p.n_munits - p.units_whole) * p.n_splits;
}
template <bool TWO>
__device__ __forceinline__ void item_range(const FilterParams& p, const Sched& sc, int item, int& m_tile, int& split, int& t0,
                                           int& t1) {
    if (p.pair_mode) {
        // units are query tiles (single-CTA mode) or pairs of consecutive query tiles (CTA pairs: the two CTAs of a pair
        // take tiles 2u and 2u+1 and sweep the same corpus tiles)
        const int grp = item / p.pair_group;
        const int first = (grp * p.nparts + p.part) * p.pair_group;
        const int unit = first + (item - grp * p.pair_group);
        m_tile = TWO ? 2 * unit + sc.rank : unit;
        split = 0;
        const int lead_tile = (p.pair_align ? first : unit) * (TWO ? 2 : 1);
        t0 = (lead_tile * BLOCK_M) / BLOCK_N;  // first corpus tile that can contain a column > row
        t1 = p.n_ntiles;
    } else {
        int unit;
        if (item < p.units_whole) {  // phase A: one worker, one unit, every corpus tile (all workers stream the same tiles in step)
            unit = item;
            split = 0;
            t0 = 0;
            t1 = p.n_ntiles;
        } else {  // phase B: the leftover units, unit fastest, cut into n_splits splits to fill the last waves
            const int j = item - p.units_whole, rem = p.n_munits - p.units_whole;
            unit = p.units_whole + j % rem;
            split = j / rem;
            t0 = split * p.tiles_per_split;
            t1 = min(t0 + p.tiles_per_split, p.n_ntiles);
        }
        m_tile = TWO ? 2 * unit + sc.rank : unit;
    }
}

// TMA producer: one lane (per CTA) streams (query tile, corpus tile) K-blocks into the smem ring. In a CTA pair each CTA
// loads its own query rows and half of the corpus tile, multicast to both CTAs; every CTA's full barrier counts a whole stage.
template <bool TF32, int NSTAGES, bool TWO>
__device__ __forceinline__ void producer_loop(const CUtensorMap* tmap_q, const CUtensorMap* tmap_x, const FilterParams& p,
                                              const Ring& r, const Sched& sc) {
    constexpr int KB_ELEMS = KB_BYTES / (TF32 ? 4 : 2);
    const int n_items = num_items(p);
    int stage = 0;
    uint32_t phase = 0;
    for (int item = sc.worker; item < n_items; item += sc.n_workers) {
        int m_tile, split, t0, t1;
        item_range<TWO>(p, sc, item, m_tile, split, t0, t1);
        for (int t = t0; t < t1; ++t) {
            for (int kb = 0; kb < p.num_kb; ++kb) {
                mbar_wait(&r.empty_bar[stage], phase ^ 1);
                uint8_t* sa = r.stage_base + stage * STAGE_BYTES;
                uint8_t* sb = sa + STAGE_A_BYTES;
                mbar_arrive_expect_tx(&r.full_bar[stage], STAGE_BYTES);
                tma_load_2d(sa, tmap_q, &r.full_bar[stage], kb * KB_ELEMS, m_tile * BLOCK_M);
                if constexpr (TWO)
                    tma_load_2d_multicast(sb + sc.rank * (STAGE_B_BYTES / 2), tmap_x, &r.full_bar[stage], kb * KB_ELEMS,
                                          t * BLOCK_N + sc.rank * (BLOCK_N / 2), (uint16_t)3);
                else
                    tma_load_2d(sb, tmap_x, &r.full_bar[stage], kb * KB_ELEMS, t * BLOCK_N);
                if (++stage == NSTAGES) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
    }
}

// a consumer warp is done reading stage s: one arrival per warp, in both CTAs of a pair (the peer multicasts into this stage)
template <bool TWO>
__device__ __forceinline__ void release_stage(const Ring& r, int s, int rank) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
        mbar_arrive(&r.empty_bar[s]);
        if constexpr (TWO) mbar_arrive_cluster(&r.empty_bar[s], (uint32_t)(rank ^ 1));
    }
}

// Consumer warpgroup g: acc = (query rows 64g..64g+63 of the stage's A tile) . (the 256 corpus rows)^T over all K-blocks of
// one corpus tile. One wgmma group per K-block; a stage is released as soon as the group that read it has retired.
template <bool TF32, int NSTAGES, bool TWO>
__device__ __forceinline__ void mma_tile(float (&acc)[128], const Ring& r, int num_kb, int g, int rank, int& stage, uint32_t& phase) {
    const uint32_t a_off = (uint32_t)(g * WG_M * KB_BYTES);
    int prev = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait_spin(&r.full_bar[stage], phase);
        const uint32_t sa = smem_u32(r.stage_base + stage * STAGE_BYTES);
        const uint64_t adesc = make_sw64_desc(sa + a_off);
        const uint64_t bdesc = make_sw64_desc(sa + STAGE_A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < KSTEPS; ++k)  // +32 bytes per K step inside the 64-byte swizzle row (16 B units)
            wgmma_64x256<TF32>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        if (prev >= 0) {
            wgmma_wait<1>();
            release_stage<TWO>(r, prev, rank);
        }
        prev = stage;
        if (++stage == NSTAGES) {
            stage = 0;
            phase ^= 1;
        }
    }
    wgmma_wait<0>();
    acc_fence(acc);
    release_stage<TWO>(r, prev, rank);
}

// barrier init shared by both kernels; returns after the block-wide (cluster-wide) sync
template <int NSTAGES, bool TWO>
__device__ __forceinline__ Ring setup_ring(uint8_t* smem, const CUtensorMap* tmap_q, const CUtensorMap* tmap_x) {
    Ring r;
    r.stage_base = smem;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NSTAGES * STAGE_BYTES);
    r.full_bar = bars;
    r.empty_bar = bars + NSTAGES;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(tmap_q);
        tma_prefetch_desc(tmap_x);
        for (int s = 0; s < NSTAGES; ++s) {
            mbar_init(&r.full_bar[s], 1);  // the producer arms it; TMA (of both CTAs in a pair) completes the bytes
            mbar_init(&r.empty_bar[s], TWO ? 2 * CONSUMER_WARPS : CONSUMER_WARPS);  // one arrival per consumer warp (of both CTAs)
        }
        fence_barrier_init();
    }
    if constexpr (TWO) cluster_sync_all();  // the peer must see initialised barriers before any remote arrive / multicast
    else __syncthreads();
    return r;
}

template <bool TWO>
__device__ __forceinline__ void teardown_ring() {
    __syncwarp();
    if constexpr (TWO) cluster_sync_all();  // nobody leaves while the peer may still multicast into its smem or arrive on it
}

__device__ __forceinline__ uint8_t* align_smem(uint8_t* raw) {
    const uint32_t a = smem_u32(raw);
    return raw + ((1024u - (a & 1023u)) & 1023u);
}

// Replace-min insertion into the thread's candidate list (column `row` of sc/id, stride BLOCK_M): while slots are
// free just take the next one; once full, overwrite the current minimum and rescan for the new minimum (= threshold).
// Called only from flush_pending, where all 32 lanes of the warp run it in lockstep.
template <int KP>
__device__ __forceinline__ void list_insert(float* sc, int32_t* id, float s, int32_t idx, float& thr, int& minpos) {
    // fill phase (minpos < 0 encodes "-(entries so far) - 1"): slots are free, no scan needed until the list is full
    const bool filling = minpos < 0;
    const int pos = filling ? -minpos - 1 : minpos;
    sc[pos * BLOCK_M] = s;
    id[pos * BLOCK_M] = idx;
    if (filling && pos + 1 < KP) {
        minpos = -(pos + 1) - 1;
        return;  // threshold stays -inf
    }
    // new minimum: four independent (value, position) chains so the shared-memory loads and compares overlap
    static_assert(KP % 4 == 0, "list length must be a multiple of 4");
    float m[4];
    int mp[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        m[c] = sc[c * BLOCK_M];
        mp[c] = c;
    }
#pragma unroll
    for (int p = 4; p < KP; p += 4) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const float v = sc[(p + c) * BLOCK_M];
            if (v < m[c]) {
                m[c] = v;
                mp[c] = p + c;
            }
        }
    }
    // ties keep the lowest position, like the sequential scan
    if (m[1] < m[0] || (m[1] == m[0] && mp[1] < mp[0])) { m[0] = m[1]; mp[0] = mp[1]; }
    if (m[3] < m[2] || (m[3] == m[2] && mp[3] < mp[2])) { m[2] = m[3]; mp[2] = mp[3]; }
    if (m[2] < m[0] || (m[2] == m[0] && mp[2] < mp[0])) { m[0] = m[2]; mp[0] = mp[2]; }
    thr = m[0];
    minpos = mp[0];
}

// Merge every lane's pending candidates into its list. Warp-collective: the loop bound is the warp-wide
// maximum so the 32 lanes (32 different lists) execute their insertions together instead of one lane at a
// time. Returns (new threshold, position of the minimum). Inlined: a call would make ptxas serialize the wgmmas.
template <int KP>
__device__ __forceinline__ float2 flush_pending(float* my_sc, int32_t* my_id, const float* pend_sc, const int32_t* pend_id,
                                             int cnt, float thr, int minpos) {
    int mx = cnt;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    for (int i = 0; i < mx; ++i) {
        if (i < cnt) {
            const float s = pend_sc[i * BLOCK_M];
            if (s > thr) list_insert<KP>(my_sc, my_id, s, pend_id[i * BLOCK_M], thr, minpos);
        }
        __syncwarp();
    }
    return make_float2(thr, __int_as_float(minpos));
}

// L2 epilogue transform (2<q,x> - |x|^2 ranks like -|q-x|^2) and masking of the columns past the corpus end
template <bool IS_L2>
__device__ __forceinline__ void prepare8(float (&v)[8], int idx0, int valid, const float* xnorm) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (j < valid) {
            if constexpr (IS_L2) v[j] = fmaf(2.f, v[j], -__ldg(xnorm + idx0 + j));
        } else {
            v[j] = -INFINITY;
        }
    }
}

// Eight consecutive scores of the lane's (row, set). One warp vote skips the group when no lane beats its threshold (late
// in a sweep almost always); otherwise 8 branch-free predicated appends into the pending buffer and one vote on a flush.
// The pending buffers are merged into the lists by the whole warp in lockstep once any lane holds PEND_FLUSH candidates.
template <int KPH>
__device__ __forceinline__ void process8(const float (&v)[8], int idx0, float* my_sc, int32_t* my_id, float* pend_sc,
                                         int32_t* pend_id, float& thr, int& minpos, int& cnt) {
    float m = v[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) m = fmaxf(m, v[j]);
    if (!__any_sync(0xffffffffu, m > thr)) return;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (v[j] > thr) {  // cnt <= PEND_FLUSH - 1 on entry: the pending buffer cannot overflow
            pend_sc[cnt * BLOCK_M] = v[j];
            pend_id[cnt * BLOCK_M] = idx0 + j;
            ++cnt;
        }
    }
    if (__any_sync(0xffffffffu, cnt >= PEND_FLUSH)) {
        const float2 fr = flush_pending<KPH>(my_sc, my_id, pend_sc, pend_id, cnt, thr, minpos);
        thr = fr.x;
        minpos = __float_as_int(fr.y);
        cnt = 0;
    }
}

// k == 1 specialisation (k-means assignment: a few corpus tiles per item, where the list warm-up of the general epilogue
// costs more than the MMAs): each (row, set) keeps its best TWO candidates and the third-best score in registers — no smem
// lists, no pending buffer, no flush. b1 >= b2 >= b3; everything not kept scores <= b3, which is the list's discard bound.
__device__ __forceinline__ void process8_top2(const float (&v)[8], int idx0, float& b1, float& b2, float& b3, int32_t& i1,
                                              int32_t& i2) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float s = v[j];
        const int32_t id = idx0 + j;
        const bool c3 = s > b3, c2 = s > b2, c1 = s > b1;  // strict: an equal score stays behind the earlier column
        b3 = c2 ? b2 : (c3 ? s : b3);
        i2 = c1 ? i1 : (c2 ? id : i2);
        b2 = c1 ? b1 : (c2 ? s : b2);
        i1 = c1 ? id : i1;
        b1 = c1 ? s : b1;
    }
}

template <int KP, bool IS_L2, bool TF32, bool TWO, bool TOP1 = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
knn_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                  const FilterParams p) {
    constexpr int NSTAGES = num_stages(KP);
    static_assert(NSTAGES >= 2, "not enough shared memory for the operand ring");
    constexpr int KPH = KP / 2;  // candidates kept per (row, set)
    static_assert(KPH % 4 == 0, "list length must allow float4 write-out");
    constexpr int LSET = list_set_stride(KPH);

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem(smem_raw);
    float* xpose = reinterpret_cast<float*>(smem + NSTAGES * STAGE_BYTES + BAR_BYTES);  // [8 warps][16][XP_STRIDE]
    float* list_sc = xpose + CONSUMER_WARPS * XP_WARP_FLOATS;                          // [2 sets][LSET]
    int32_t* list_id = reinterpret_cast<int32_t*>(list_sc + 2 * LSET);
    float* pend_sc_base = reinterpret_cast<float*>(list_id + 2 * LSET);                // [2 sets][PEND_SET_STRIDE]
    int32_t* pend_id_base = reinterpret_cast<int32_t*>(pend_sc_base + 2 * PEND_SET_STRIDE);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const Ring ring = setup_ring<NSTAGES, TWO>(smem, &tmap_q, &tmap_x);
    const int n_items = num_items(p);
    const Sched sc = make_sched<TWO>();

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (threadIdx.x == 0) producer_loop<TF32, NSTAGES, TWO>(&tmap_q, &tmap_x, p, ring, sc);
    } else {
        setmaxnreg_inc<232>();
        // ===================== consumer warpgroup g: wgmma of 64 query rows, streaming top-KPH per (row, set) ==========
        const int g = (warp >> 2) - 1;
        const int wq = warp & 3;
        const int rr = lane & 15, e = lane >> 4;
        const int row = g * WG_M + wq * 16 + rr;  // this lane's list row inside the query tile
        float* my_sc = list_sc + e * LSET + row;
        int32_t* my_id = list_id + e * LSET + row;
        float* pend_sc = pend_sc_base + e * PEND_SET_STRIDE + row;
        int32_t* pend_id = pend_id_base + e * PEND_SET_STRIDE + row;
        float* xs = xpose + (warp - 4) * XP_WARP_FLOATS;
        // fragment coordinates of this lane: rows lane/4 and lane/4 + 8 of the warp's 16, columns 8j + 2(lane%4) + {0,1}
        const int fr = lane >> 2, fc = 2 * (lane & 3);
        int stage = 0;
        uint32_t phase = 0;
        float acc[128];
        for (int item = sc.worker; item < n_items; item += sc.n_workers) {
            int m_tile, split, t0, t1;
            item_range<TWO>(p, sc, item, m_tile, split, t0, t1);
            if constexpr (!TOP1) {
#pragma unroll 4
                for (int i = 0; i < KPH; ++i) {
                    my_sc[i * BLOCK_M] = -INFINITY;
                    my_id[i * BLOCK_M] = -1;
                }
            }
            float thr = -INFINITY;
            int minpos = -1;  // fill phase, 0 entries (see list_insert)
            int cnt = 0;      // pending candidates of this (row, set)
            float b1 = -INFINITY, b2 = -INFINITY, b3 = -INFINITY;  // TOP1: best two scores + discard bound
            int32_t i1 = -1, i2 = -1;
            for (int t = t0; t < t1; ++t) {
                mma_tile<TF32, NSTAGES, TWO>(acc, ring, p.num_kb, g, sc.rank, stage, phase);
                const int col0 = t * BLOCK_N;
                const int ncols = min(BLOCK_N, p.n - col0);
#pragma unroll
                for (int c = 0; c < BLOCK_N / 16; ++c) {  // 16-column chunks through the per-warp transpose
                    __syncwarp();
#pragma unroll
                    for (int jj = 0; jj < 2; ++jj) {
                        const int a = (2 * c + jj) * 4;
                        xs[fr * XP_STRIDE + 8 * jj + fc] = acc[a];
                        xs[fr * XP_STRIDE + 8 * jj + fc + 1] = acc[a + 1];
                        xs[(fr + 8) * XP_STRIDE + 8 * jj + fc] = acc[a + 2];
                        xs[(fr + 8) * XP_STRIDE + 8 * jj + fc + 1] = acc[a + 3];
                    }
                    __syncwarp();
                    float v[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) v[j] = xs[rr * XP_STRIDE + 8 * e + j];
                    const int off = 16 * c + 8 * e;
                    prepare8<IS_L2>(v, col0 + off, ncols - off, p.xnorm);
                    if constexpr (TOP1)
                        process8_top2(v, col0 + off, b1, b2, b3, i1, i2);
                    else
                        process8<KPH>(v, col0 + off, my_sc, my_id, pend_sc, pend_id, thr, minpos, cnt);
                }
            }
            if constexpr (TOP1) {
                // same [KPH] list layout as the general epilogue: two real entries, the rest (-inf, -1)
#pragma unroll 4
                for (int i = 2; i < KPH; ++i) {
                    my_sc[i * BLOCK_M] = -INFINITY;
                    my_id[i * BLOCK_M] = -1;
                }
                my_sc[0 * BLOCK_M] = b1;
                my_id[0 * BLOCK_M] = i1;
                my_sc[1 * BLOCK_M] = b2;
                my_id[1 * BLOCK_M] = i2;
                thr = b3;
            } else {
                const float2 fl = flush_pending<KPH>(my_sc, my_id, pend_sc, pend_id, cnt, thr, minpos);
                thr = fl.x;
                minpos = __float_as_int(fl.y);
                cnt = 0;
            }
            // write this (query, split, set) candidate list
            const int q = m_tile * BLOCK_M + row;
            if (q < p.nq) {
                const size_t lidx = ((size_t)q * p.n_splits + split) * 2 + e;
                float4* osc = reinterpret_cast<float4*>(p.cand_score + lidx * KPH);
                int4* oid = reinterpret_cast<int4*>(p.cand_id + lidx * KPH);
#pragma unroll 4
                for (int i = 0; i < KPH / 4; ++i) {
                    osc[i] = make_float4(my_sc[(4 * i + 0) * BLOCK_M], my_sc[(4 * i + 1) * BLOCK_M],
                                         my_sc[(4 * i + 2) * BLOCK_M], my_sc[(4 * i + 3) * BLOCK_M]);
                    oid[i] = make_int4(my_id[(4 * i + 0) * BLOCK_M], my_id[(4 * i + 1) * BLOCK_M],
                                       my_id[(4 * i + 2) * BLOCK_M], my_id[(4 * i + 3) * BLOCK_M]);
                }
                p.cand_thr[lidx] = thr;  // -inf unless this list overflowed
            }
        }
    }

    teardown_ring<TWO>();
}

// ---- all-pairs threshold filter (sem_dedup): same mainloop, the epilogue emits (i, j) candidates -------------------
constexpr int PAIR_STAGES = MAX_STAGES;
constexpr int PAIR_SMEM = PAIR_STAGES * STAGE_BYTES + BAR_BYTES + SMEM_ALIGN_SLACK;

template <bool TF32, bool TWO>
__global__ void __launch_bounds__(NUM_THREADS, 1)
pair_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x, const FilterParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem(smem_raw);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const Ring ring = setup_ring<PAIR_STAGES, TWO>(smem, &tmap_q, &tmap_x);
    const int n_items = num_items(p);
    const Sched sc = make_sched<TWO>();
    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (threadIdx.x == 0) producer_loop<TF32, PAIR_STAGES, TWO>(&tmap_q, &tmap_x, p, ring, sc);
    } else {
        setmaxnreg_inc<232>();
        const int g = (warp >> 2) - 1;
        const int wq = warp & 3;
        const float thr = p.pair_thr;
        int stage = 0;
        uint32_t phase = 0;
        float acc[128];
        for (int item = sc.worker; item < n_items; item += sc.n_workers) {
            int m_tile, split, t0, t1;
            item_range<TWO>(p, sc, item, m_tile, split, t0, t1);
            const int gi0 = m_tile * BLOCK_M + g * WG_M + wq * 16 + (lane >> 2);  // global rows gi0 and gi0 + 8 of this lane
            for (int t = t0; t < t1; ++t) {
                mma_tile<TF32, PAIR_STAGES, TWO>(acc, ring, p.num_kb, g, sc.rank, stage, phase);
                const int col0 = t * BLOCK_N + 2 * (lane & 3);
                float mx = acc[0];
#pragma unroll
                for (int i = 1; i < 128; ++i) mx = fmaxf(mx, acc[i]);
                if (mx > thr && gi0 < p.n) {
#pragma unroll
                    for (int i = 0; i < 128; ++i) {
                        const int gi = gi0 + 8 * ((i >> 1) & 1);
                        const int gj = col0 + 8 * (i >> 2) + (i & 1);
                        if (acc[i] > thr && gj > gi && gj < p.n && gi < p.n) {  // strict upper triangle, inside the matrix
                            const unsigned long long pos = atomicAdd(p.pair_count, 1ull);
                            if (pos < p.pair_cap) {
                                p.pair_i[pos] = gi;
                                p.pair_j[pos] = gj;
                            }
                        }
                    }
                }
            }
        }
    }
    teardown_ring<TWO>();
}

// ---- host side ---------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) {
        set_error("cuTensorMapEncodeTiled is not available from the driver (%s)", cudaGetErrorString(e));
        return nullptr;
    }
    fn = reinterpret_cast<PFN_encodeTiled>(p);
    return fn;
}

// 2-D row-major matrix [rows, cols] with `pitch` elements per row; box = {KB_BYTES of K, box_rows rows}
int make_tmap(CUtensorMap* map, const void* base, bool tf32, int64_t rows, int64_t cols, int64_t pitch, int box_rows) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) return B2_ECUDA;
    const int esz = tf32 ? 4 : 2;
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)pitch * esz};
    cuuint32_t box[2] = {(cuuint32_t)(KB_BYTES / esz), (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (gstride[0] & 15) != 0) {
        set_error("TMA operand not 16-byte aligned (base %p, pitch %lld B)", base, (long long)gstride[0]);
        return B2_EINVAL;
    }
    CUresult r = enc(map, tf32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                     const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows %lld cols %lld pitch %lld)", (int)r,
                  (long long)rows, (long long)cols, (long long)pitch);
        return B2_ECUDA;
    }
    return B2_OK;
}

template <typename Kern>
int launch_cluster(Kern kern, int grid, int smem, bool two, const CUtensorMap& tq, const CUtensorMap& tx, const FilterParams& p,
                   cudaStream_t stream) {
    // the attribute is per DEVICE (not per process): set it on every launch — a microsecond — so that a process driving
    // several GPUs (B200VS(device=i) for several i) launches correctly on each of them
    B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(NUM_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = two ? 2 : 1;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    B2_CUDA(cudaLaunchKernelEx(&cfg, kern, tq, tx, p));
    B2_LAUNCH_CHECK();
    g_stats[ST_FILTER_LAUNCHES]++;
    return B2_OK;
}

template <int KP, bool IS_L2, bool TF32, bool TWO, bool TOP1 = false>
int launch_variant(const CUtensorMap& tq, const CUtensorMap& tx, const FilterParams& p, int grid, cudaStream_t stream) {
    return launch_cluster(knn_filter_kernel<KP, IS_L2, TF32, TWO, TOP1>, grid, smem_bytes(KP), TWO, tq, tx, p, stream);
}

template <int KP, bool TWO>
int launch_kp(bool is_l2, bool tf32, const CUtensorMap& tq, const CUtensorMap& tx, const FilterParams& p, int grid,
              cudaStream_t stream) {
    if constexpr (KP == 16) {
        if (p.top1) {  // k == 1: register-resident top-2 epilogue
            if (is_l2) {
                return tf32 ? launch_variant<KP, true, true, TWO, true>(tq, tx, p, grid, stream)
                            : launch_variant<KP, true, false, TWO, true>(tq, tx, p, grid, stream);
            }
            return tf32 ? launch_variant<KP, false, true, TWO, true>(tq, tx, p, grid, stream)
                        : launch_variant<KP, false, false, TWO, true>(tq, tx, p, grid, stream);
        }
    }
    if (is_l2) {
        return tf32 ? launch_variant<KP, true, true, TWO>(tq, tx, p, grid, stream)
                    : launch_variant<KP, true, false, TWO>(tq, tx, p, grid, stream);
    }
    return tf32 ? launch_variant<KP, false, true, TWO>(tq, tx, p, grid, stream)
                : launch_variant<KP, false, false, TWO>(tq, tx, p, grid, stream);
}

template <bool TWO>
int launch_two(int kp, bool is_l2, bool tf32, const CUtensorMap& tq, const CUtensorMap& tx, const FilterParams& p, int grid,
               cudaStream_t stream) {
    switch (kp) {
        case 16: return launch_kp<16, TWO>(is_l2, tf32, tq, tx, p, grid, stream);
        case 32: return launch_kp<32, TWO>(is_l2, tf32, tq, tx, p, grid, stream);
        case 64: return launch_kp<64, TWO>(is_l2, tf32, tq, tx, p, grid, stream);
        case 72: return launch_kp<72, TWO>(is_l2, tf32, tq, tx, p, grid, stream);
        default: set_error("internal: unsupported candidate capacity %d", kp); return B2_EINVAL;
    }
}

int sm_count(int device) {
    static int cached[64] = {0};
    if (device >= 0 && device < 64 && cached[device]) return cached[device];
    int n = 132;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device);
    if (device >= 0 && device < 64) cached[device] = n;
    return n;
}

}  // namespace

int filter_kp_for_k(int k) {
    if (k <= 6) return 16;
    if (k <= 16) return 32;
    if (k <= 40) return 64;
    if (k <= FILTER_MAX_K) return 72;  // k > 40: several corpus splits share the load, see filter_min_splits_for_k
    return 0;
}

// k > 40 does not fit one candidate list (72 entries = 2 sets x 36 is what shared memory allows next to a four-stage operand
// ring), so the corpus is cut into enough splits that each (split, set) sub-list expects at most ~18 of a query's top k —
// half its capacity, 4-5 standard deviations of headroom for rows in random order. A sub-list that overflows anyway is caught
// by the certificate (its discard bound reaches the k-th exact score) and that query takes the dense path.
int filter_min_splits_for_k(int k) { return k <= 40 ? 1 : (int)ceil_div(k, 36); }

// CTA pairs need at least two query tiles; B2_FILTER_2CTA=0/1 overrides the default.
bool filter_use_pair(int64_t nq) {
    static int mode = -1;
    if (mode < 0) {
        const char* e = getenv("B2_FILTER_2CTA");
        mode = e ? (atoi(e) != 0 ? 1 : 0) : 1;  // default: CTA pairs
    }
    return mode == 1 && ceil_div(nq, BLOCK_M) >= 2;
}

// Number of corpus splits: enough work items to fill the machine, and few idle workers in the last wave.
// In pair mode a worker is a CTA pair and a query unit is two query tiles.
int filter_choose_splits(int64_t nq, int64_t n, int num_sms, bool two_cta, bool top1, int min_splits, int* units_whole) {
    if (units_whole) *units_whole = 0;
    {
        static int forced = -1;  // B2_FILTER_SPLITS: experiments only
        if (forced < 0) {
            const char* e = getenv("B2_FILTER_SPLITS");
            forced = e ? atoi(e) : 0;
        }
        if (forced > 0) {
            const int64_t nt = ceil_div(n, BLOCK_N);
            int s = (int)std::min<int64_t>(forced, nt);
            while (s > 1 && ceil_div(nt, ceil_div(nt, s)) != s) --s;
            return s;
        }
    }
    const int64_t n_mtiles = ceil_div(nq, BLOCK_M);
    const int64_t n_units = two_cta ? ceil_div(n_mtiles, 2) : n_mtiles;
    const int64_t workers = two_cta ? std::max(1, num_sms / 2) : num_sms;
    const int64_t n_ntiles = ceil_div(n, BLOCK_N);
    // cost model: an item costs its corpus tiles plus ~13 tile-times of list warm-up, the
    // kernel takes `waves` such items back to back, and every extra split adds two candidate lists per query to finalize
    const double kWarmupTiles = top1 ? 1.0 : 13.0;  // the register-resident top-2 epilogue has no list to warm up
    double best_cost = 1e300;
    int best = 0;
    for (int s = std::max(1, min_splits); s <= 256 && s <= n_ntiles; ++s) {
        const int64_t tps = ceil_div(n_ntiles, s);
        if (ceil_div(n_ntiles, tps) != s) continue;  // every split must receive tiles
        const int64_t items = n_units * s;
        const int64_t waves = ceil_div(items, workers);
        const double cost = (double)waves * ((double)tps + kWarmupTiles) * (1.0 + 0.004 * s);
        if (cost < best_cost - 1e-9) {
            best_cost = cost;
            best = s;
        }
    }
    // Two-phase schedule: as many whole waves as possible run ONE unit per worker over the whole corpus (one list warm-up per
    // wave instead of one per split, and the workers still stream the same corpus tiles in step, which is what keeps them in
    // L2); only the leftover units (< one per worker) are cut into splits, just fine enough to fill the last waves. On a
    // 125k-row shard with 100k queries: 5 x (489 + 13) + 2 x (70 + 13) = 2676 tile-times against 16 x (163 + 13) = 2816.
    static const bool two_phase_on = [] { const char* e = getenv("B2_FILTER_TWO_PHASE"); return e ? atoi(e) != 0 : true; }();
    const int64_t waves_a = n_units / workers;
    if (units_whole && two_phase_on && min_splits <= 1 && waves_a >= 1) {
        const int64_t ua = waves_a * workers, rem = n_units - ua;
        const double cost_a = (double)waves_a * ((double)n_ntiles + kWarmupTiles);
        double best2 = 1e300;
        int s2 = 1;
        if (rem == 0) {
            best2 = cost_a;
        } else {
            for (int s = 1; s <= 256 && s <= n_ntiles; ++s) {
                const int64_t tps = ceil_div(n_ntiles, s);
                if (ceil_div(n_ntiles, tps) != s) continue;
                const int64_t waves_b = ceil_div(rem * s, workers);
                const double cost = (cost_a + (double)waves_b * ((double)tps + kWarmupTiles)) * (1.0 + 0.002 * s);
                if (cost < best2 - 1e-9) {
                    best2 = cost;
                    s2 = s;
                }
            }
        }
        if (best2 < best_cost - 1e-9) {
            *units_whole = (int)ua;
            return s2;
        }
    }
    return best;
}

int launch_knn_filter(const MatView& X, const void* q_filt, int64_t q_pitch, int64_t nq, int metric, int kp,
                      int n_splits, bool two_cta, float* cand_score, int32_t* cand_id, float* cand_thr, int device,
                      cudaStream_t stream, bool top1, int units_whole) {
    if (nq <= 0 || X.n <= 0) return B2_OK;
    if (X.n > 0x7fffff00LL || nq > 0x7fffff00LL) {
        set_error("matrix too large for 32-bit row ids (n=%lld nq=%lld)", (long long)X.n, (long long)nq);
        return B2_ERANGE;
    }
    const bool tf32 = X.filt_dtype == B2_F32;
    const int kb_elems = KB_BYTES / (tf32 ? 4 : 2);
    CUtensorMap tq, tx;
    const int64_t op_cols = X.d;
    B2_TRY(make_tmap(&tq, q_filt, tf32, nq, op_cols, q_pitch, BLOCK_M));
    // pair mode: each CTA of the pair loads HALF of the 256-row corpus tile (and multicasts it to both)
    B2_TRY(make_tmap(&tx, X.filt, tf32, X.n, op_cols, X.filt_pitch, two_cta ? BLOCK_N / 2 : BLOCK_N));
    FilterParams p;
    p.xnorm = X.norm2;
    p.cand_score = cand_score;
    p.cand_id = cand_id;
    p.cand_thr = cand_thr;
    p.nq = (int32_t)nq;
    p.n = (int32_t)X.n;
    p.num_kb = (int32_t)ceil_div(X.d, kb_elems);
    p.n_mtiles = (int32_t)ceil_div(nq, BLOCK_M);
    p.n_munits = two_cta ? (p.n_mtiles + 1) / 2 : p.n_mtiles;
    p.n_ntiles = (int32_t)ceil_div(X.n, BLOCK_N);
    p.tiles_per_split = (int32_t)ceil_div(p.n_ntiles, n_splits);
    p.n_splits = n_splits;
    p.units_whole = units_whole;
    p.top1 = (top1 && kp == 16) ? 1 : 0;  // register-resident top-2 epilogue: requested by the k-means assignment path only
    p.pair_mode = 0;
    p.part = 0;
    p.nparts = 1;
    p.pair_thr = 0.f;
    p.pair_i = p.pair_j = nullptr;
    p.pair_count = nullptr;
    p.pair_cap = 0;
    if ((int64_t)p.tiles_per_split * (n_splits - 1) >= p.n_ntiles) {
        set_error("internal: empty corpus split (tiles %d, splits %d)", p.n_ntiles, n_splits);
        return B2_EINVAL;
    }
    if (units_whole < 0 || units_whole > p.n_munits) {
        set_error("internal: bad two-phase schedule (%d whole units of %d)", units_whole, p.n_munits);
        return B2_EINVAL;
    }
    const int64_t items = (int64_t)units_whole + (int64_t)(p.n_munits - units_whole) * n_splits;
    if (units_whole > 0 && n_splits > 1) {
        // whole units write split 0 only: the other lists of their queries must read as empty (id -1, bound -inf)
        B2_CUDA(cudaMemsetAsync(cand_id, 0xFF, (size_t)nq * n_splits * kp * sizeof(int32_t), stream));
        B2_TRY(launch_fill_f32(cand_thr, nq * (int64_t)n_splits * 2, -INFINITY, stream));
    }
    const bool is_l2 = metric == B2_METRIC_L2;
    if (is_l2 && !X.norm2) {
        set_error("internal: L2 filter without row norms");
        return B2_EINVAL;
    }
    int rc;
    if (two_cta) {
        const int pairs = (int)std::min<int64_t>(items, sm_count(device) / 2);
        rc = launch_two<true>(kp, is_l2, tf32, tq, tx, p, 2 * pairs, stream);
    } else {
        const int grid = (int)std::min<int64_t>(items, sm_count(device));
        rc = launch_two<false>(kp, is_l2, tf32, tq, tx, p, grid, stream);
    }
    return rc;
}

// query tiles per dealing group of the all-pairs schedule: one per SM, so that one wave of CTAs is one group
// (B2_PAIR_GROUP overrides it; the tests use a small value to exercise the dealing on small matrices)
static int pair_group_size(int device) {
    const char* e = getenv("B2_PAIR_GROUP");
    if (e && atoi(e) > 0) return atoi(e);
    return sm_count(device);
}

// All pairs i < j of X whose filter inner product exceeds thr (sem_dedup). Candidates land in pair_i/pair_j (device,
// capacity cap) in arbitrary order; *pair_count receives the total found.
int launch_pair_filter(const MatView& X, float thr, int part, int nparts, int32_t* pair_i, int32_t* pair_j,
                       unsigned long long* pair_count, unsigned long long cap, int device, cudaStream_t stream) {
    if (X.n <= 1) return B2_OK;
    if (X.n > 0x7fffff00LL) {
        set_error("matrix too large for 32-bit row ids (n=%lld)", (long long)X.n);
        return B2_ERANGE;
    }
    const bool tf32 = X.filt_dtype == B2_F32;
    const int kb_elems = KB_BYTES / (tf32 ? 4 : 2);
    CUtensorMap tq, tx;
    B2_TRY(make_tmap(&tq, X.filt, tf32, X.n, X.d, X.filt_pitch, BLOCK_M));
    B2_TRY(make_tmap(&tx, X.filt, tf32, X.n, X.d, X.filt_pitch, BLOCK_N));
    FilterParams p;
    memset(&p, 0, sizeof(p));
    p.nq = (int32_t)X.n;
    p.n = (int32_t)X.n;
    p.num_kb = (int32_t)ceil_div(X.d, kb_elems);
    static const bool two = [] { const char* e = getenv("B2_PAIR_2CTA"); return e ? atoi(e) != 0 : true; }();  // default: CTA pairs
    const bool two_cta = two && ceil_div(X.n, BLOCK_M) >= 2;
    if (two_cta) B2_TRY(make_tmap(&tx, X.filt, tf32, X.n, X.d, X.filt_pitch, BLOCK_N / 2));  // each CTA stages half a corpus tile
    p.n_mtiles = (int32_t)ceil_div(X.n, BLOCK_M);
    p.n_munits = two_cta ? (p.n_mtiles + 1) / 2 : p.n_mtiles;
    p.n_ntiles = (int32_t)ceil_div(X.n, BLOCK_N);
    p.n_splits = 1;
    p.tiles_per_split = p.n_ntiles;
    p.pair_mode = 1;
    p.part = part;
    p.nparts = nparts;
    p.pair_group = two_cta ? std::max(1, pair_group_size(device) / 2) : pair_group_size(device);  // one unit per worker
    {
        const char* e = getenv("B2_PAIR_ALIGN");
        p.pair_align = e ? (atoi(e) != 0) : 1;
    }
    p.pair_thr = thr;
    p.pair_i = pair_i;
    p.pair_j = pair_j;
    p.pair_count = pair_count;
    p.pair_cap = cap;
    // this rank's query tiles: the full groups g = part (mod nparts) plus the trailing partial group if it is ours (it is
    // then this rank's last group, so item -> tile stays a closed form)
    const int64_t full_groups = p.n_munits / p.pair_group, rem = p.n_munits % p.pair_group;
    const int64_t my_full = full_groups > part ? ceil_div(full_groups - part, (int64_t)nparts) : 0;
    const int64_t items = my_full * p.pair_group + ((rem && full_groups % nparts == part) ? rem : 0);
    p.pair_items = (int32_t)items;
    if (items <= 0) return B2_OK;
    const int grid = two_cta ? 2 * (int)std::min<int64_t>(items, sm_count(device) / 2) : (int)std::min<int64_t>(items, sm_count(device));
    if (two_cta) {
        return tf32 ? launch_cluster(pair_filter_kernel<true, true>, grid, PAIR_SMEM, true, tq, tx, p, stream)
                    : launch_cluster(pair_filter_kernel<false, true>, grid, PAIR_SMEM, true, tq, tx, p, stream);
    }
    return tf32 ? launch_cluster(pair_filter_kernel<true, false>, grid, PAIR_SMEM, false, tq, tx, p, stream)
                : launch_cluster(pair_filter_kernel<false, false>, grid, PAIR_SMEM, false, tq, tx, p, stream);
}

}  // namespace b2
