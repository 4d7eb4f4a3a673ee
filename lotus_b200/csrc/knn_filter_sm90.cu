// knn_filter_sm90.cu — the dominant kernel: fused Q.K^T (Hopper wgmma, fp32 accumulators in registers, TMA-staged
// operand tiles) + per-query streaming top-KP selection in the epilogue.
//
// Replaces the arithmetic of faiss `Index.search` as called from lotus/vector_store/faiss_vs.py:67,75
// (knn_inner_product / knn_L2sqr: blocked sgemm + heap). The N x Q score matrix is never written to HBM.
//
// Role of this kernel in the exact pipeline (DESIGN.md §Pipeline): it is a FILTER. It computes scores with
// bf16 / fp16 (or TF32) tensor-core products and fp32 accumulation and keeps, per query and per corpus split,
// the KP > k best candidates plus the value `thr` below which everything was discarded. knn_exact.cu then
// re-scores the candidates in the canonical fp64 order and certifies, with a rigorous error margin, that
// nothing discarded could belong to the true top-k; uncertified queries take the dense exact path.
//
// Kernel shape: a CTA owns 128 queries and computes 128 queries x 256 corpus rows per tile.
//   warpgroup 0: TMA producer (one lane)
//   warpgroups 1, 2: consumers; consumer g issues wgmma m64n256 for query rows 64g..64g+63 (fp32 accumulators in
//                    registers, 128 per thread) and runs the epilogue of those rows
//   K-block = one 64-byte swizzle row (32 bf16 or fp16 / 16 tf32): wgmma k16 (bf16, fp16) or k8 (tf32), two per K-block.
//   smem ring of NSTAGES x (A 8 KB + B 16 KB), mbarrier full/empty pairs.
//   Resident query K-blocks (knn filter): the query tile is the same for every corpus tile of an item, so each consumer keeps
//   its rows of the first FILTER_RES_KB K-blocks in registers (8 per K-block, loaded in the item's first tile) and issues
//   register-A wgmmas for them; in the item's later tiles those stages carry B only. Per 128 x 256 tile a CTA then pulls
//   (num_kb - FILTER_RES_KB) x 8 KB of A instead of num_kb x 8 KB (d = 768 bf16: 144 instead of 192 KB).
//   Clusters of CL CTAs (knn filter over a long corpus: FILTER_CL; k-means assignment, short corpora and dedup: CTA pairs; once
//   a chunk has CL query tiles): the
//   schedule's worker is a CTA pair that takes two consecutive query tiles (a query unit); a cluster of four runs two such
//   workers in lockstep. Every CTA of a cluster sweeps the same corpus tiles, loads 1/CL of every corpus tile and
//   TMA-multicasts it into all CL CTAs, so the corpus bytes each SM pulls from L2 drop CL-fold. A stage is freed once the
//   consumers of every CTA of the cluster are done with it.
//   Persistent: one CTA per SM, work item = (query unit, corpus split), query units fastest so that co-resident
//   workers stream the same corpus tiles and hit them in L2.
//
// Epilogue lists: the wgmma fragment spreads a query row over four lanes, so each warp passes its 16 rows x 256 scores
// through a small shared-memory transpose, 16 columns at a time; afterwards lane (r, e) = (lane & 15, lane >> 4) holds 8
// scores of row r. Before a chunk is transposed, each lane tests its fragment values against the thresholds of their
// lists, and one warp vote skips the chunk when none can enter. Candidate list ("set") e of a row collects the columns c
// with bit 3 of c equal to e, so a query keeps two lists of KP/2 per corpus split, the layout finalize merges.
#include <cuda.h>

#include <climits>
#include <type_traits>

#include "common.cuh"

namespace b2 {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 256;
constexpr int WG_M = 64;        // query rows per consumer warpgroup (wgmma M)
constexpr int KB_BYTES = 64;    // K-block: one SWIZZLE_64B row
constexpr int KSTEPS = 2;       // wgmma K steps (32 bytes each) per K-block
constexpr int KB_AREGS = 4 * KSTEPS;  // registers per consumer thread holding one K-block of its warpgroup's 64 query rows
constexpr int STAGE_A_BYTES = BLOCK_M * KB_BYTES;
constexpr int STAGE_B_BYTES = BLOCK_N * KB_BYTES;
constexpr int STAGE_BYTES = STAGE_A_BYTES + STAGE_B_BYTES;
constexpr int NUM_THREADS = 384;   // producer warpgroup + two consumer warpgroups
constexpr int CONSUMER_WARPS = 8;
constexpr int MAX_STAGES = 8;
constexpr int SMEM_LIMIT = 232448;  // 227 KB
constexpr int SMEM_ALIGN_SLACK = 1024;  // the ring is aligned to 1024 B by hand
constexpr int BAR_BYTES = 256;
// CTAs per cluster of the knn filter: each CTA pulls A (8 KB) + B / FILTER_CL from L2 per K-block, 12 KB against 16 KB for a
// pair, which lowers the energy per tile of a power-capped card. Clusters of 8 were no faster. Over a short corpus (the
// k-means centroids: a few tiles per item) clusters of 4 were slower than pairs, so the k-means assignment (TOP1) and any
// corpus of fewer than FILTER_CL_MIN_NTILES tiles keep CTA pairs (DESIGN §5).
constexpr int FILTER_CL = 4;
constexpr int FILTER_CL_MIN_NTILES = 32;
// K-blocks of its query rows that a knn filter consumer keeps in registers for a whole item (8 per K-block next to the 128
// accumulators), so that after the item's first tile those stages load only B from L2 (DESIGN §5)
constexpr int FILTER_RES_KB = 6;
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
//
// Plain arrive (default .release.cta semantics), not .release.cluster: ptxas lowers the cluster-scope release to a
// GPU-wide MEMBAR that the consumers would then pay at every stage release, in the middle of the wgmma pipeline. Nothing
// here needs that ordering. The only accesses to order are this CTA's wgmma reads of the stage against the peer's later
// TMA multicast into it: wgmma.wait_group has retired those reads before the arrive is made, and the peer's producer
// waits on this barrier before it issues the copy. No data written through memory has to become visible to anyone.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
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

// Operand kind of the filter: the element type both wgmma operands are streamed in. BF16 and F16 are 2-byte operands
// (m64n256k16, 32 elements per K-block); TF32 reads fp32 operands (m64n256k8, 16 elements per K-block); I8 reads int8
// operands (m64n256k32 into s32 accumulators, 64 elements per K-block: exact integer products and sums).
enum class Op { BF16, F16, TF32, I8 };
__host__ __device__ constexpr int op_bytes(Op op) { return op == Op::TF32 ? 4 : op == Op::I8 ? 1 : 2; }

// the 128 accumulators of an m64n256 wgmma, as operands %0..%127
#define B2_WGMMA_D                                                                                                           \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define B2_WGMMA_D_OPS                                                                                                       \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
#define B2_WGMMA_D_OPS_S32 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]), "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]), "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
#define B2_WGMMA_64X256(SHAPE_TYPES, IMM_TAIL)                                                                               \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"                                                   \
                 "wgmma.mma_async.sync.aligned." SHAPE_TYPES " " B2_WGMMA_D ", %128, %129, p, 1, 1" IMM_TAIL ";\n\t}"         \
                 : B2_WGMMA_D_OPS                                                                                          \
                 : "l"(adesc), "l"(bdesc), "r"(scale_d))
#define B2_WGMMA_64X256_RS(SHAPE_TYPES, IMM_TAIL)                                                                            \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %133, 0;\n\t"                                                   \
                 "wgmma.mma_async.sync.aligned." SHAPE_TYPES " " B2_WGMMA_D ", {%128, %129, %130, %131}, %132, p, 1, 1"   \
                 IMM_TAIL ";\n\t}"                                                                                         \
                 : B2_WGMMA_D_OPS                                                                                          \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d))

// D[64 x 256] (+)= A[64 x K] . B[256 x K]^T, both K-major in shared memory; scale_d == 0 overwrites D
template <Op OP>
__device__ __forceinline__ void wgmma_64x256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    if constexpr (OP == Op::TF32) {
        B2_WGMMA_64X256("m64n256k8.f32.tf32.tf32", "");
    } else if constexpr (OP == Op::F16) {
        B2_WGMMA_64X256("m64n256k16.f32.f16.f16", ", 0, 0");
    } else {  // Op::BF16
        B2_WGMMA_64X256("m64n256k16.f32.bf16.bf16", ", 0, 0");
    }
}
// The same product with A from registers: a[0..3] is the warp's 16-row slice of one K step in the mma fragment layout
// (load_a_frag); B stays in shared memory. Register A takes no transpose immediate, only B's.
template <Op OP>
__device__ __forceinline__ void wgmma_64x256_rs(float (&d)[128], const uint32_t* a, uint64_t bdesc, uint32_t scale_d) {
    if constexpr (OP == Op::TF32) {
        B2_WGMMA_64X256_RS("m64n256k8.f32.tf32.tf32", "");
    } else if constexpr (OP == Op::F16) {
        B2_WGMMA_64X256_RS("m64n256k16.f32.f16.f16", ", 0");
    } else {  // Op::BF16
        B2_WGMMA_64X256_RS("m64n256k16.f32.bf16.bf16", ", 0");
    }
}
// The int8 product into s32 accumulators: integer wgmma takes neither scale nor transpose immediates.
template <Op OP>
__device__ __forceinline__ void wgmma_64x256(int32_t (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    static_assert(OP == Op::I8, "s32 accumulators take int8 operands");
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 " B2_WGMMA_D ", %128, %129, p;\n\t}"
                 : B2_WGMMA_D_OPS_S32
                 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// register A: a k32 step of int8 has the byte layout of a k16 step of a 2-byte type (register j: row (lane / 4) + 8 (j & 1),
// bytes 4 (lane % 4) + 16 (j >> 1) .. + 3 of the step's 32), so load_a_frag's ldmatrix path fills it unchanged
template <Op OP>
__device__ __forceinline__ void wgmma_64x256_rs(int32_t (&d)[128], const uint32_t* a, uint64_t bdesc, uint32_t scale_d) {
    static_assert(OP == Op::I8, "s32 accumulators take int8 operands");
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %133, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 " B2_WGMMA_D ", {%128, %129, %130, %131}, %132, p;\n\t}"
                 : B2_WGMMA_D_OPS_S32
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void acc_fence(int32_t (&d)[128]) {
#pragma unroll
    for (int i = 0; i < 128; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
#undef B2_WGMMA_64X256_RS
#undef B2_WGMMA_64X256
#undef B2_WGMMA_D_OPS_S32
#undef B2_WGMMA_D_OPS
#undef B2_WGMMA_D

// Register-A fragment of one K-block: a[4k..4k+3] feed K step k of wgmma_64x256_rs. `slice` is the shared address of the
// consumer warpgroup's 64 query rows in a landed stage (K-major, 64-byte rows, SWIZZLE_64B: the 16-byte chunk c of row r
// sits at chunk c ^ ((r >> 1) & 3), r counted from a 512-byte-aligned base). Warp w of the warpgroup holds rows 16 w .. 16 w + 15.
//   2-byte operands: register j of a step holds row (lane / 4) + 8 (j & 1), elements 2 (lane % 4) + {0, 1} + 8 (j >> 1):
//                    one ldmatrix.x4, lane l addressing row l % 8 of the 8 x 8 matrix l / 8.
//   tf32:            register j holds row (lane / 4) + 8 (j & 1), element (lane % 4) + 4 (j >> 1): one 4-byte load each.
template <Op OP>
__device__ __forceinline__ void load_a_frag(uint32_t (&a)[KB_AREGS], uint32_t slice) {
    const int lane = threadIdx.x & 31;
    const int r0 = ((threadIdx.x >> 5) & 3) * 16;
    auto chunk_addr = [slice](int r, int c) { return slice + (uint32_t)(r * KB_BYTES + ((c ^ ((r >> 1) & 3)) << 4)); };
#pragma unroll
    for (int k = 0; k < KSTEPS; ++k) {
        uint32_t* f = a + 4 * k;
        if constexpr (OP == Op::TF32) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t addr = chunk_addr(r0 + (lane >> 2) + 8 * (j & 1), 2 * k + (j >> 1)) + 4 * (lane & 3);
                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(f[j]) : "r"(addr) : "memory");
            }
        } else {
            const int m = lane >> 3;
            const uint32_t addr = chunk_addr(r0 + 8 * (m & 1) + (lane & 7), 2 * k + (m >> 1));
            asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                         : "=r"(f[0]), "=r"(f[1]), "=r"(f[2]), "=r"(f[3])
                         : "r"(addr)
                         : "memory");
        }
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
    int32_t n_munits;      // schedulable query units: n_mtiles, or ceil(n_mtiles / 2) pairs of query tiles in cluster mode
                           // (clusters of four: rounded so that the units cut into splits are even, see filter_params)
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
    const int32_t* xnorm_i;  // [n] exact squared norms of int8 rows (int8 L2 filter epilogue)
};

struct Ring {
    uint8_t* stage_base;
    uint64_t *full_bar, *empty_bar;
};

// Persistent schedule. A "worker" is a CTA pair in cluster mode (a single CTA when CL == 1); item = (query unit, corpus
// split), unit fastest so that co-resident workers stream the same corpus tiles and share them in L2. A cluster of four holds
// workers 2c and 2c + 1, which must sweep the same corpus tiles item for item: they do when the number of items is even and
// the units cut into splits are even in number (the host rounds them up), since their items 2c + k W and 2c + 1 + k W are
// then the same split of neighbouring units (W, the worker count, is even).
struct Sched {
    int worker, n_workers;
    int rank;  // query tile of the unit this CTA takes (0 or 1; 0 in single-CTA mode)
    int cta;   // CTA rank inside the cluster: which 1/CL of each corpus tile it loads
};
template <int CL>
__device__ __forceinline__ Sched make_sched() {
    Sched sc;
    if constexpr (CL > 1) {
        sc.worker = blockIdx.x >> 1;
        sc.n_workers = gridDim.x >> 1;
        sc.cta = (int)cluster_ctarank();
        sc.rank = CL == 2 ? sc.cta : (sc.cta & 1);
    } else {
        sc.worker = blockIdx.x;
        sc.n_workers = gridDim.x;
        sc.rank = 0;
        sc.cta = 0;
    }
    return sc;
}
__device__ __forceinline__ int num_items(const FilterParams& p) {
    if (p.pair_mode) return p.pair_items;
    return p.units_whole + (p.n_munits - p.units_whole) * p.n_splits;
}
template <int CL>
__device__ __forceinline__ void item_range(const FilterParams& p, const Sched& sc, int item, int& m_tile, int& split, int& t0,
                                           int& t1) {
    if (p.pair_mode) {
        // units are query tiles (single-CTA mode) or pairs of consecutive query tiles (CTA pairs: the two CTAs of a pair
        // take tiles 2u and 2u+1 and sweep the same corpus tiles)
        const int grp = item / p.pair_group;
        const int first = (grp * p.nparts + p.part) * p.pair_group;
        const int unit = first + (item - grp * p.pair_group);
        m_tile = CL > 1 ? 2 * unit + sc.rank : unit;
        split = 0;
        const int lead_tile = (p.pair_align ? first : unit) * (CL > 1 ? 2 : 1);
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
        m_tile = CL > 1 ? 2 * unit + sc.rank : unit;  // past n_mtiles in a surplus unit: loads zeros, writes nothing
    }
}

// TMA producer: one lane (per CTA) streams (query tile, corpus tile) K-blocks into the smem ring. In a cluster each CTA
// loads its own query rows and 1/CL of the corpus tile, multicast to every CTA; every CTA's full barrier counts a whole stage.
// A piece of BLOCK_N / CL rows is a whole number of 512-byte SWIZZLE_64B periods, so the pieces tile the B stage exactly as
// one full-tile box would.
// The first RES_KB K-blocks of the query tile stay in the consumers' registers for the whole item (mma_tile), so after the
// item's first tile their stages carry B only. A is never multicast, so only this CTA's expected byte count changes.
template <Op OP, int NSTAGES, int CL, int RES_KB>
__device__ __forceinline__ void producer_loop(const CUtensorMap* tmap_q, const CUtensorMap* tmap_x, const FilterParams& p,
                                              const Ring& r, const Sched& sc) {
    constexpr int KB_ELEMS = KB_BYTES / op_bytes(OP);
    const int n_items = num_items(p);
    int stage = 0;
    uint32_t phase = 0;
    for (int item = sc.worker; item < n_items; item += sc.n_workers) {
        int m_tile, split, t0, t1;
        item_range<CL>(p, sc, item, m_tile, split, t0, t1);
        for (int t = t0; t < t1; ++t) {
            for (int kb = 0; kb < p.num_kb; ++kb) {
                mbar_wait(&r.empty_bar[stage], phase ^ 1);
                uint8_t* sa = r.stage_base + stage * STAGE_BYTES;
                uint8_t* sb = sa + STAGE_A_BYTES;
                const bool a_resident = t != t0 && kb < RES_KB;
                mbar_arrive_expect_tx(&r.full_bar[stage], a_resident ? STAGE_B_BYTES : STAGE_BYTES);
                if (!a_resident) tma_load_2d(sa, tmap_q, &r.full_bar[stage], kb * KB_ELEMS, m_tile * BLOCK_M);
                if constexpr (CL > 1)
                    tma_load_2d_multicast(sb + sc.cta * (STAGE_B_BYTES / CL), tmap_x, &r.full_bar[stage], kb * KB_ELEMS,
                                          t * BLOCK_N + sc.cta * (BLOCK_N / CL), (uint16_t)((1u << CL) - 1));
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

// a consumer warp is done reading stage s: one arrival per warp, in every CTA of the cluster (each of them multicasts into
// this stage). A pair keeps lane 0 arriving locally and at the peer; larger clusters spread the arrivals over lanes 0..CL-1,
// one remote arrive each, so a warp still issues one arrive instruction.
template <int CL>
__device__ __forceinline__ void release_stage(const Ring& r, int s, int cta) {
    __syncwarp();
    if constexpr (CL <= 2) {
        if ((threadIdx.x & 31) == 0) {
            mbar_arrive(&r.empty_bar[s]);
            if constexpr (CL == 2) mbar_arrive_cluster(&r.empty_bar[s], (uint32_t)(cta ^ 1));
        }
    } else {
        const uint32_t lane = threadIdx.x & 31;
        if (lane < CL) mbar_arrive_cluster(&r.empty_bar[s], lane);
    }
}

// Consumer warpgroup g: acc = (query rows 64g..64g+63 of the stage's A tile) . (the 256 corpus rows)^T over all K-blocks of
// one corpus tile. One wgmma group per K-block; a stage is released as soon as the group that read it has retired.
// K-blocks kb < RES_KB take A from `afrag`, which holds them for the whole item: the item's first tile (load_a) fills it from
// the landed stages, later tiles find no A in those stages (producer_loop). The rest read A from shared memory. The operands
// and the K order are the same either way, so are the accumulators.
template <Op OP, int NSTAGES, int CL, int RES_KB, typename AccT>
__device__ __forceinline__ void mma_tile(AccT (&acc)[128], uint32_t (&afrag)[RES_KB > 0 ? RES_KB : 1][KB_AREGS], bool load_a,
                                         const Ring& r, int num_kb, int g, int cta, int& stage, uint32_t& phase) {
    const uint32_t a_off = (uint32_t)(g * WG_M * KB_BYTES);
    int prev = -1;
    auto retire = [&]() {
        wgmma_commit();
        if (prev >= 0) {
            wgmma_wait<1>();
            release_stage<CL>(r, prev, cta);
        }
        prev = stage;
        if (++stage == NSTAGES) {
            stage = 0;
            phase ^= 1;
        }
    };
#pragma unroll
    for (int kb = 0; kb < RES_KB; ++kb) {
        if (kb < num_kb) {
            mbar_wait_spin(&r.full_bar[stage], phase);
            const uint32_t sa = smem_u32(r.stage_base + stage * STAGE_BYTES);
            if (load_a) load_a_frag<OP>(afrag[kb], sa + a_off);
            const uint64_t bdesc = make_sw64_desc(sa + STAGE_A_BYTES);
            wgmma_fence();  // orders the fragment writes (and the accumulators') before the wgmmas that read them
#pragma unroll
            for (int k = 0; k < KSTEPS; ++k)
                wgmma_64x256_rs<OP>(acc, afrag[kb] + 4 * k, bdesc + (uint64_t)(2 * k), (kb | k) != 0 ? 1u : 0u);
            retire();
        }
    }
    for (int kb = RES_KB; kb < num_kb; ++kb) {
        mbar_wait_spin(&r.full_bar[stage], phase);
        const uint32_t sa = smem_u32(r.stage_base + stage * STAGE_BYTES);
        const uint64_t adesc = make_sw64_desc(sa + a_off);
        const uint64_t bdesc = make_sw64_desc(sa + STAGE_A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < KSTEPS; ++k)  // +32 bytes per K step inside the 64-byte swizzle row (16 B units)
            wgmma_64x256<OP>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb | k) != 0 ? 1u : 0u);
        retire();
    }
    wgmma_wait<0>();
    acc_fence(acc);
    release_stage<CL>(r, prev, cta);
}

// barrier init shared by both kernels; returns after the block-wide (cluster-wide) sync
template <int NSTAGES, int CL>
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
            mbar_init(&r.full_bar[s], 1);  // the producer arms it; TMA (of every CTA in a cluster) completes the bytes
            mbar_init(&r.empty_bar[s], CL * CONSUMER_WARPS);  // one arrival per consumer warp of every CTA
        }
        fence_barrier_init();
    }
    if constexpr (CL > 1) cluster_sync_all();  // the peers must see initialised barriers before any remote arrive / multicast
    else __syncthreads();
    return r;
}

template <int CL>
__device__ __forceinline__ void teardown_ring() {
    __syncwarp();
    if constexpr (CL > 1) cluster_sync_all();  // nobody leaves while a peer may still multicast into its smem or arrive on it
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

// The same under a row mask: bit j of `live` set = column j is a selected row of the corpus; the others can enter no list
template <bool IS_L2>
__device__ __forceinline__ void prepare8_masked(float (&v)[8], int idx0, uint32_t live, const float* xnorm) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if ((live >> j) & 1u) {
            if constexpr (IS_L2) v[j] = fmaf(2.f, v[j], -__ldg(xnorm + idx0 + j));
        } else {
            v[j] = -INFINITY;
        }
    }
}

// Eight consecutive scores of the lane's (row, set), in a chunk where some lane of the warp beats its threshold (the
// consumer's gate skips the others): 8 branch-free predicated appends into the pending buffer and one vote on a flush.
// The pending buffers are merged into the lists by the whole warp in lockstep once any lane holds PEND_FLUSH candidates.
template <int KPH>
__device__ __forceinline__ void process8(const float (&v)[8], int idx0, float* my_sc, int32_t* my_id, float* pend_sc,
                                         int32_t* pend_id, float& thr, int& minpos, int& cnt) {
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

// The knn filter. Op::I8 accumulates in s32 and runs its gate on integers: the score s (IP) or 2 s - |x|^2 (L2, exact in int32
// for d < 2^15 since it equals |q|^2 - |q - x|^2) against the list thresholds rounded down. Only the chunks that pass are
// converted to fp32 (once, round to nearest), before the transpose, so the lists keep their fp32 format.
// int8 filter score of accumulator s for corpus column j: s (IP) or 2 s - |x_j|^2 (L2), exact in int32 (unsigned arithmetic:
// the intermediate 2 s may wrap, the result does not); `valid` is false past the corpus end, where the row norm is not read
template <bool IS_L2>
__device__ __forceinline__ int32_t i8_score(int32_t s, const FilterParams& p, int j, bool valid) {
    if constexpr (IS_L2) return valid ? (int32_t)(2u * (uint32_t)s - (uint32_t)__ldg(p.xnorm_i + j)) : s;
    else return s;
}

//
// MASKED: only the corpus rows whose bit is set in `mask` (bit j & 31 of word j >> 5 is row j) take part. The eight words of a
// corpus tile are the same for every query row: lane l of each consumer warp loads word l & 7 before the tile's wgmmas are
// issued and holds it across them; the epilogue fetches a chunk's word with a shuffle. A chunk whose 16 bits are clear is
// skipped outright, a tile whose 256 bits are clear skips its epilogue (its stages are consumed all the same: the producer
// does not look at the mask), and a cleared column reaches neither the gate nor the lists. So `thr` still bounds every
// SELECTED row a list discarded, which is all the certificate asks of it.
template <int KP, bool IS_L2, Op OP, int CL, bool TOP1, bool MASKED = false>
__device__ __forceinline__ void knn_filter_body(const CUtensorMap& tmap_q, const CUtensorMap& tmap_x, const FilterParams& p,
                                                const uint32_t* mask = nullptr) {
    static_assert(!(TOP1 && MASKED), "the k-means top-2 epilogue takes no row mask");
    using AccT = std::conditional_t<OP == Op::I8, int32_t, float>;
    constexpr int NSTAGES = num_stages(KP);
    static_assert(NSTAGES >= 2, "not enough shared memory for the operand ring");
    constexpr int KPH = KP / 2;  // candidates kept per (row, set)
    static_assert(KPH % 4 == 0, "list length must allow float4 write-out");
    constexpr int LSET = list_set_stride(KPH);
    // the masked epilogue's bit tests need a few registers more than the column-range compares they replace (the L2 forms
    // spilled two): a masked kernel keeps one query K-block fewer in registers
    constexpr int RES_KB = MASKED ? FILTER_RES_KB - 1 : FILTER_RES_KB;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem(smem_raw);
    float* xpose = reinterpret_cast<float*>(smem + NSTAGES * STAGE_BYTES + BAR_BYTES);  // [8 warps][16][XP_STRIDE]
    float* list_sc = xpose + CONSUMER_WARPS * XP_WARP_FLOATS;                          // [2 sets][LSET]
    int32_t* list_id = reinterpret_cast<int32_t*>(list_sc + 2 * LSET);
    float* pend_sc_base = reinterpret_cast<float*>(list_id + 2 * LSET);                // [2 sets][PEND_SET_STRIDE]
    int32_t* pend_id_base = reinterpret_cast<int32_t*>(pend_sc_base + 2 * PEND_SET_STRIDE);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const Ring ring = setup_ring<NSTAGES, CL>(smem, &tmap_q, &tmap_x);
    const int n_items = num_items(p);
    const Sched sc = make_sched<CL>();

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (threadIdx.x == 0) producer_loop<OP, NSTAGES, CL, RES_KB>(&tmap_q, &tmap_x, p, ring, sc);
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
        AccT acc[128];
        uint32_t afrag[RES_KB][KB_AREGS];  // the query tile's first RES_KB K-blocks, loaded in each item's first tile
        for (int item = sc.worker; item < n_items; item += sc.n_workers) {
            int m_tile, split, t0, t1;
            item_range<CL>(p, sc, item, m_tile, split, t0, t1);
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
            // thresholds of the lists this lane's fragment values go to: gthr[h][s] is (row fr + 8h, set s), the `thr` of
            // lane fr + 8h + 16s
            float gthr[2][2] = {{-INFINITY, -INFINITY}, {-INFINITY, -INFINITY}};
            // int8: gthr rounded down (an integer score s beats t exactly when s > floor(t); -inf maps to INT_MIN)
            int32_t gthr_i[2][2] = {{INT_MIN, INT_MIN}, {INT_MIN, INT_MIN}};
            for (int t = t0; t < t1; ++t) {
                if constexpr (MASKED) {  // the tile's 32 bytes of mask, on their way while the wgmmas run
                    if (lane == 0) asm volatile("prefetch.global.L1 [%0];" ::"l"(mask + t * (BLOCK_N / 32)));
                }
                mma_tile<OP, NSTAGES, CL, RES_KB>(acc, afrag, t == t0, ring, p.num_kb, g, sc.cta, stage, phase);
                const int col0 = t * BLOCK_N;
                const int ncols = min(BLOCK_N, p.n - col0);
                uint32_t mword = 0;  // MASKED: word (lane & 7) of the tile's mask, zero past the last word of the corpus
                if constexpr (MASKED) {
                    const int w = t * (BLOCK_N / 32) + (lane & 7);
                    if (w < (p.n + 31) >> 5) mword = __ldg(mask + w);
                    if (!__any_sync(0xffffffffu, mword != 0)) continue;  // no selected row in this tile
                }
#pragma unroll
                for (int c = 0; c < BLOCK_N / 16; ++c) {  // 16-column chunks through the per-warp transpose
                    // MASKED: bit i set = column 16 c + i is a selected row of the corpus; it stands in for the column-range
                    // tests of the unmasked epilogue, so the mask adds no compare to a chunk
                    uint32_t live = 0xffffu;
                    if constexpr (MASKED) {
                        live = (__shfl_sync(0xffffffffu, mword, c >> 1) >> (16 * (c & 1))) & 0xffffu;
                        const int rem = ncols - 16 * c;
                        if (rem < 16) live &= rem > 0 ? (1u << rem) - 1u : 0u;
                        if (live == 0) continue;  // warp-uniform: nothing selected in this chunk
                    }
                    if constexpr (!TOP1) {
                        // Gate: test the chunk's fragment values, as prepare8 transforms them, against the thresholds of
                        // their lists. When no lane holds a value above its threshold (late in a sweep almost always),
                        // process8 would append nothing, so the chunk skips the transpose and is done.
                        bool hit = false;
#pragma unroll
                        for (int jj = 0; jj < 2; ++jj) {
#pragma unroll
                            for (int h = 0; h < 4; ++h) {  // acc[a + h]: row fr + 8 (h >> 1), column 16c + 8jj + fc + (h & 1)
                                const int off = 16 * c + 8 * jj + fc + (h & 1);
                                bool in;
                                if constexpr (MASKED) in = ((live >> (8 * jj + (h & 1))) >> fc & 1u) != 0;
                                else in = off < ncols;
                                if constexpr (OP == Op::I8) {
                                    hit |= in && i8_score<IS_L2>(acc[(2 * c + jj) * 4 + h], p, col0 + off, in) > gthr_i[h >> 1][jj];
                                } else {
                                    float s = (float)acc[(2 * c + jj) * 4 + h];
                                    if constexpr (IS_L2) {
                                        if (in) s = fmaf(2.f, s, -__ldg(p.xnorm + col0 + off));
                                    }
                                    hit |= in && s > gthr[h >> 1][jj];
                                }
                            }
                        }
                        if (!__any_sync(0xffffffffu, hit)) continue;
                    }
                    __syncwarp();
#pragma unroll
                    for (int jj = 0; jj < 2; ++jj) {
                        const int a = (2 * c + jj) * 4;
                        if constexpr (OP == Op::I8) {  // the gate's integer scores, rounded to nearest: the only error
                            const int off = 16 * c + 8 * jj + fc;
                            xs[fr * XP_STRIDE + 8 * jj + fc] = (float)i8_score<IS_L2>(acc[a], p, col0 + off, off < ncols);
                            xs[fr * XP_STRIDE + 8 * jj + fc + 1] = (float)i8_score<IS_L2>(acc[a + 1], p, col0 + off + 1, off + 1 < ncols);
                            xs[(fr + 8) * XP_STRIDE + 8 * jj + fc] = (float)i8_score<IS_L2>(acc[a + 2], p, col0 + off, off < ncols);
                            xs[(fr + 8) * XP_STRIDE + 8 * jj + fc + 1] = (float)i8_score<IS_L2>(acc[a + 3], p, col0 + off + 1, off + 1 < ncols);
                        } else {
                            xs[fr * XP_STRIDE + 8 * jj + fc] = acc[a];
                            xs[fr * XP_STRIDE + 8 * jj + fc + 1] = acc[a + 1];
                            xs[(fr + 8) * XP_STRIDE + 8 * jj + fc] = acc[a + 2];
                            xs[(fr + 8) * XP_STRIDE + 8 * jj + fc + 1] = acc[a + 3];
                        }
                    }
                    __syncwarp();
                    float v[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) v[j] = xs[rr * XP_STRIDE + 8 * e + j];
                    const int off = 16 * c + 8 * e;
                    if constexpr (MASKED) prepare8_masked<IS_L2 && OP != Op::I8>(v, col0 + off, live >> (8 * e), p.xnorm);
                    else prepare8<IS_L2 && OP != Op::I8>(v, col0 + off, ncols - off, p.xnorm);  // int8: transformed already
                    if constexpr (TOP1) {
                        process8_top2(v, col0 + off, b1, b2, b3, i1, i2);
                    } else {
                        process8<KPH>(v, col0 + off, my_sc, my_id, pend_sc, pend_id, thr, minpos, cnt);
                        // a flush may have raised the thresholds the gate tests against
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
#pragma unroll
                            for (int s = 0; s < 2; ++s) gthr[h][s] = __shfl_sync(0xffffffffu, thr, fr + 8 * h + 16 * s);
                        }
                        if constexpr (OP == Op::I8) {
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
#pragma unroll
                                for (int s = 0; s < 2; ++s) gthr_i[h][s] = __float2int_rd(gthr[h][s]);
                            }
                        }
                    }
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

    teardown_ring<CL>();
}

template <int KP, bool IS_L2, Op OP, int CL, bool TOP1 = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
knn_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                  const FilterParams p) {
    knn_filter_body<KP, IS_L2, OP, CL, TOP1>(tmap_q, tmap_x, p);
}

// the int8 knn filter (IGMMA): an entry of its own, apart from the floating-point kernels (HGMMA)
template <int KP, bool IS_L2, int CL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
knn_i8_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                     const FilterParams p) {
    knn_filter_body<KP, IS_L2, Op::I8, CL, false>(tmap_q, tmap_x, p);
}

// the masked knn filter (masked search): entries of their own, so that the kernels of an unmasked search are untouched.
// mask: ceil(p.n / 32) words, see knn_filter_body
template <int KP, bool IS_L2, Op OP, int CL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
knn_masked_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                         const FilterParams p, const uint32_t* __restrict__ mask) {
    knn_filter_body<KP, IS_L2, OP, CL, false, true>(tmap_q, tmap_x, p, mask);
}

template <int KP, bool IS_L2, int CL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
knn_masked_i8_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                            const FilterParams p, const uint32_t* __restrict__ mask) {
    knn_filter_body<KP, IS_L2, Op::I8, CL, false, true>(tmap_q, tmap_x, p, mask);
}

// ---- all-pairs threshold filter (sem_dedup): same mainloop, the epilogue emits (i, j) candidates -------------------
constexpr int PAIR_STAGES = MAX_STAGES;
constexpr int PAIR_SMEM = PAIR_STAGES * STAGE_BYTES + BAR_BYTES + SMEM_ALIGN_SLACK;

// Op::I8 compares the s32 scores against the threshold rounded down (s > thr exactly when s > floor(thr))
template <Op OP, int CL>
__device__ __forceinline__ void pair_filter_body(const CUtensorMap& tmap_q, const CUtensorMap& tmap_x, const FilterParams p) {
    using AccT = std::conditional_t<OP == Op::I8, int32_t, float>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem(smem_raw);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const Ring ring = setup_ring<PAIR_STAGES, CL>(smem, &tmap_q, &tmap_x);
    const int n_items = num_items(p);
    const Sched sc = make_sched<CL>();
    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (threadIdx.x == 0) producer_loop<OP, PAIR_STAGES, CL, 0>(&tmap_q, &tmap_x, p, ring, sc);
    } else {
        setmaxnreg_inc<232>();
        const int g = (warp >> 2) - 1;
        const int wq = warp & 3;
        AccT thr;
        if constexpr (OP == Op::I8) thr = __float2int_rd(p.pair_thr);
        else thr = p.pair_thr;
        int stage = 0;
        uint32_t phase = 0;
        AccT acc[128];
        uint32_t no_afrag[1][KB_AREGS];  // every K-block reads A from shared memory
        for (int item = sc.worker; item < n_items; item += sc.n_workers) {
            int m_tile, split, t0, t1;
            item_range<CL>(p, sc, item, m_tile, split, t0, t1);
            const int gi0 = m_tile * BLOCK_M + g * WG_M + wq * 16 + (lane >> 2);  // global rows gi0 and gi0 + 8 of this lane
            for (int t = t0; t < t1; ++t) {
                mma_tile<OP, PAIR_STAGES, CL, 0>(acc, no_afrag, false, ring, p.num_kb, g, sc.cta, stage, phase);
                const int col0 = t * BLOCK_N + 2 * (lane & 3);
                AccT mx = acc[0];
#pragma unroll
                for (int i = 1; i < 128; ++i) {
                    if constexpr (OP == Op::I8) mx = max(mx, acc[i]);
                    else mx = fmaxf(mx, acc[i]);
                }
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
    teardown_ring<CL>();
}

template <Op OP, int CL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
pair_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x, const FilterParams p) {
    pair_filter_body<OP, CL>(tmap_q, tmap_x, p);
}

// the int8 all-pairs filter (IGMMA), an entry of its own like knn_i8_filter_kernel
template <int CL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
pair_i8_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x, const FilterParams p) {
    pair_filter_body<Op::I8, CL>(tmap_q, tmap_x, p);
}

// ---- range filter (range search): same mainloop and knn schedule, the epilogue emits (query, row) candidates ----------
// Every (query tile, corpus tile) pair is one tile of exactly one item (item_range, knn form). A lane's accumulators hold
// two query rows; their thresholds stay in registers for the whole item. A row is a candidate when its filter score (IP:
// <q, x>; L2: 2 <q, x> - |x|^2) is strictly above the threshold of its query; a NaN threshold (a query the exact dense path
// answers, or a row past nq) passes nothing. Op::I8 compares the exact integer scores against the thresholds rounded down.
struct RangeParams {
    const float* thr;             // [nq] candidate threshold in filter-score space
    int2* cand;                   // [cap] (query, corpus row) of each candidate, in arbitrary order
    unsigned long long* count;    // total candidates found (may exceed cap)
    unsigned long long cap;
};
constexpr int RANGE_STAGES = MAX_STAGES;
constexpr int RANGE_SMEM = RANGE_STAGES * STAGE_BYTES + BAR_BYTES + SMEM_ALIGN_SLACK;

// MASKED (masked range search): only the rows whose bit is set in `row_mask` (ceil(p.n / 32) words, laid out as for
// knn_filter_body) can become candidates, so the candidates scale with the hits among the selected rows. A tile whose 256
// bits are clear skips its epilogue (its stages are consumed all the same), a chunk whose 16 bits are clear is skipped, and
// each column's bit is ANDed with the column-range test, so bits at or past p.n (the next chunk's, on a streamed chunk)
// select nothing.
template <Op OP, bool IS_L2, int CL, bool MASKED = false>
__device__ __forceinline__ void range_filter_body(const CUtensorMap& tmap_q, const CUtensorMap& tmap_x, const FilterParams& p,
                                                  const RangeParams& rp, const uint32_t* row_mask = nullptr) {
    using AccT = std::conditional_t<OP == Op::I8, int32_t, float>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem(smem_raw);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const Ring ring = setup_ring<RANGE_STAGES, CL>(smem, &tmap_q, &tmap_x);
    const int n_items = num_items(p);
    const Sched sc = make_sched<CL>();
    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (threadIdx.x == 0) producer_loop<OP, RANGE_STAGES, CL, 0>(&tmap_q, &tmap_x, p, ring, sc);
    } else {
        setmaxnreg_inc<232>();
        const int g = (warp >> 2) - 1;
        const int wq = warp & 3;
        int stage = 0;
        uint32_t phase = 0;
        AccT acc[128];
        uint32_t no_afrag[1][KB_AREGS];  // every K-block reads A from shared memory
        for (int item = sc.worker; item < n_items; item += sc.n_workers) {
            int m_tile, split, t0, t1;
            item_range<CL>(p, sc, item, m_tile, split, t0, t1);
            const int gi0 = m_tile * BLOCK_M + g * WG_M + wq * 16 + (lane >> 2);  // query rows gi0 and gi0 + 8 of this lane
            AccT thr[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float tq = gi0 + 8 * h < p.nq ? __ldg(rp.thr + gi0 + 8 * h) : __int_as_float(0x7fc00000);
                if constexpr (OP == Op::I8) thr[h] = tq != tq ? INT_MAX : __float2int_rd(tq);  // NaN: nothing passes
                else thr[h] = tq;
            }
            for (int t = t0; t < t1; ++t) {
                if constexpr (MASKED) {  // the tile's 32 bytes of mask, on their way while the wgmmas run
                    if (lane == 0) asm volatile("prefetch.global.L1 [%0];" ::"l"(row_mask + t * (BLOCK_N / 32)));
                }
                mma_tile<OP, RANGE_STAGES, CL, 0>(acc, no_afrag, false, ring, p.num_kb, g, sc.cta, stage, phase);
                const int col0 = t * BLOCK_N + 2 * (lane & 3);
                uint32_t mword = 0;  // MASKED: word (lane & 7) of the tile's mask, zero past the last word of the corpus
                if constexpr (MASKED) {
                    const int w = t * (BLOCK_N / 32) + (lane & 7);
                    if (w < (p.n + 31) >> 5) mword = __ldg(row_mask + w);
                    if (!__any_sync(0xffffffffu, mword != 0)) continue;  // no selected row in this tile
                }
#pragma unroll
                for (int c = 0; c < BLOCK_N / 16; ++c) {  // 16-column chunks: acc[8c .. 8c + 7]
                    // MASKED: bit i set = column 16 c + i of the tile is a selected row (the same for every lane)
                    uint32_t live = 0xffffu;
                    if constexpr (MASKED) {
                        live = (__shfl_sync(0xffffffffu, mword, c >> 1) >> (16 * (c & 1))) & 0xffffu;
                        if (live == 0) continue;  // warp-uniform: nothing selected in this chunk
                    }
                    uint32_t mask = 0;
#pragma unroll
                    for (int h = 0; h < 8; ++h) {
                        const int i = 8 * c + h;
                        const int gj = col0 + 8 * (i >> 2) + (i & 1);
                        bool valid = gj < p.n;
                        if constexpr (MASKED) valid = valid && ((live >> (8 * (h >> 2) + (h & 1) + 2 * (lane & 3))) & 1u) != 0;
                        bool pass;
                        if constexpr (OP == Op::I8) {
                            pass = valid && i8_score<IS_L2>(acc[i], p, gj, valid) > thr[(i >> 1) & 1];
                        } else {
                            float s = acc[i];
                            if constexpr (IS_L2) {
                                if (valid) s = fmaf(2.f, s, -__ldg(p.xnorm + gj));
                            }
                            pass = valid && s > thr[(i >> 1) & 1];
                        }
                        mask |= pass ? 1u << h : 0u;
                    }
                    if (!__any_sync(0xffffffffu, mask != 0)) continue;
                    // warp-aggregated append: one atomic per warp and chunk, each lane writes its candidates contiguously
                    const int cnt = __popc(mask);
                    int incl = cnt;
#pragma unroll
                    for (int off = 1; off < 32; off <<= 1) {
                        const int v = __shfl_up_sync(0xffffffffu, incl, off);
                        if (lane >= off) incl += v;
                    }
                    const int total = __shfl_sync(0xffffffffu, incl, 31);
                    unsigned long long base = 0;
                    if (lane == 31) base = atomicAdd(rp.count, (unsigned long long)total);
                    base = __shfl_sync(0xffffffffu, base, 31) + (unsigned long long)(incl - cnt);
#pragma unroll
                    for (int h = 0; h < 8; ++h) {
                        if (mask & (1u << h)) {
                            const int i = 8 * c + h;
                            if (base < rp.cap) rp.cand[base] = make_int2(gi0 + 8 * ((i >> 1) & 1), col0 + 8 * (i >> 2) + (i & 1));
                            ++base;
                        }
                    }
                }
            }
        }
    }
    teardown_ring<CL>();
}

template <Op OP, bool IS_L2, int CL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
range_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x, const FilterParams p,
                    const RangeParams rp) {
    range_filter_body<OP, IS_L2, CL>(tmap_q, tmap_x, p, rp);
}

// the int8 range filter (IGMMA), an entry of its own like knn_i8_filter_kernel
template <bool IS_L2, int CL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
range_i8_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x, const FilterParams p,
                       const RangeParams rp) {
    range_filter_body<Op::I8, IS_L2, CL>(tmap_q, tmap_x, p, rp);
}

// the masked range filter (masked range search): entries of their own, so that the kernels of an unmasked range search are
// untouched. mask: ceil(p.n / 32) words, see range_filter_body
template <Op OP, bool IS_L2, int CL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
range_masked_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                           const FilterParams p, const RangeParams rp, const uint32_t* __restrict__ mask) {
    range_filter_body<OP, IS_L2, CL, true>(tmap_q, tmap_x, p, rp, mask);
}

template <bool IS_L2, int CL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
range_masked_i8_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                              const FilterParams p, const RangeParams rp, const uint32_t* __restrict__ mask) {
    range_filter_body<Op::I8, IS_L2, CL, true>(tmap_q, tmap_x, p, rp, mask);
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

// the filter operand kind of a filter copy of `filt_dtype` elements
Op filter_op(int filt_dtype) {
    switch (filt_dtype) {
        case B2_F32: return Op::TF32;
        case B2_BF16: return Op::BF16;
        case B2_I8: return Op::I8;
        default: return Op::F16;  // B2_F16
    }
}
CUtensorMapDataType tma_data_type(Op op) {
    switch (op) {
        case Op::TF32: return CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
        case Op::BF16: return CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
        case Op::I8: return CU_TENSOR_MAP_DATA_TYPE_UINT8;  // raw bytes, no conversion
        default: return CU_TENSOR_MAP_DATA_TYPE_FLOAT16;  // Op::F16
    }
}

// 2-D row-major matrix [rows, cols] with `pitch` elements per row; box = {KB_BYTES of K, box_rows rows}
int make_tmap(CUtensorMap* map, const void* base, Op op, int64_t rows, int64_t cols, int64_t pitch, int box_rows) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) return B2_ECUDA;
    const int esz = op_bytes(op);
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)pitch * esz};
    cuuint32_t box[2] = {(cuuint32_t)(KB_BYTES / esz), (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (gstride[0] & 15) != 0) {
        set_error("TMA operand not 16-byte aligned (base %p, pitch %lld B)", base, (long long)gstride[0]);
        return B2_EINVAL;
    }
    CUresult r = enc(map, tma_data_type(op), 2,
                     const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows %lld cols %lld pitch %lld)", (int)r,
                  (long long)rows, (long long)cols, (long long)pitch);
        return B2_ECUDA;
    }
    return B2_OK;
}

// The launch config of `grid` CTAs in clusters of `cl` with `smem` bytes of dynamic shared memory each; *attr backs cfg->attrs.
// Also raises kern's shared-memory limit to smem. The attribute is per DEVICE (not per process): it is set on every launch
// — a microsecond — so that a process driving several GPUs (B200VS(device=i) for several i) launches correctly on each of them.
template <typename Kern>
int cluster_config(Kern kern, int grid, int cl, int smem, cudaStream_t stream, cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr) {
    B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    *cfg = {};
    cfg->gridDim = dim3((unsigned)grid);
    cfg->blockDim = dim3(NUM_THREADS);
    cfg->dynamicSmemBytes = smem;
    cfg->stream = stream;
    attr->id = cudaLaunchAttributeClusterDimension;
    attr->val.clusterDim.x = (unsigned)cl;
    attr->val.clusterDim.y = 1;
    attr->val.clusterDim.z = 1;
    cfg->attrs = attr;
    cfg->numAttrs = 1;
    return B2_OK;
}

// Launches the filter entry `kern` (one of the *_entry selectors below) with the entry's arguments. A null entry is a
// combination no kernel is instantiated for.
template <typename Kern, typename... Args>
int launch_cluster(Kern kern, int grid, int cl, int smem, cudaStream_t stream, const Args&... args) {
    if constexpr (std::is_null_pointer_v<Kern>) {
        set_error("internal: no filter kernel for this launch (top-1 takes no int8 points, no mask and at most CTA pairs)");
        return B2_EINVAL;
    } else {
        cudaLaunchConfig_t cfg;
        cudaLaunchAttribute attr;
        B2_TRY(cluster_config(kern, grid, cl, smem, stream, &cfg, &attr));
        B2_CUDA(cudaLaunchKernelEx(&cfg, kern, args...));
        B2_LAUNCH_CHECK();
        g_stats[ST_FILTER_LAUNCHES]++;
        return B2_OK;
    }
}

// Clusters of `cl` CTAs of `kern` that the current device holds at once. A GPC only holds whole clusters, and H100 GPCs do
// not all hold a multiple of four SMs, so this can be less than sm_count / cl; a persistent grid sized past it would run a
// trailing wave.
template <typename Kern>
int co_resident_clusters(Kern kern, int smem, int cl, int* n) {
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr;
    B2_TRY(cluster_config(kern, cl, cl, smem, nullptr, &cfg, &attr));
    *n = 0;
    B2_CUDA(cudaOccupancyMaxActiveClusters(n, kern, &cfg));
    if (*n <= 0) {
        set_error("the filter kernel fits no cluster of %d CTAs (%d B of shared memory each)", cl, smem);
        return B2_ECUDA;
    }
    return B2_OK;
}

// Runtime values to template arguments: each helper calls the generic lambda f once, with the value as a
// std::integral_constant.
template <typename F>
int with_cluster(int cl, F&& f) {
    switch (cl) {
        case 1: return f(std::integral_constant<int, 1>{});
        case 2: return f(std::integral_constant<int, 2>{});
        case FILTER_CL: return f(std::integral_constant<int, FILTER_CL>{});
        default: set_error("internal: unsupported cluster size %d", cl); return B2_EINVAL;
    }
}

template <typename F>
int with_kp(int kp, F&& f) {
    switch (kp) {
        case 16: return f(std::integral_constant<int, 16>{});
        case 32: return f(std::integral_constant<int, 32>{});
        case 64: return f(std::integral_constant<int, 64>{});
        case 72: return f(std::integral_constant<int, 72>{});
        default: set_error("internal: unsupported candidate capacity %d", kp); return B2_EINVAL;
    }
}

template <typename F>
int with_op(Op op, F&& f) {
    switch (op) {
        case Op::TF32: return f(std::integral_constant<Op, Op::TF32>{});
        case Op::BF16: return f(std::integral_constant<Op, Op::BF16>{});
        case Op::I8: return f(std::integral_constant<Op, Op::I8>{});
        default: return f(std::integral_constant<Op, Op::F16>{});  // Op::F16
    }
}

template <typename F>
int with_bool(bool b, F&& f) {
    return b ? f(std::true_type{}) : f(std::false_type{});
}

// The __global__ of each filter family for one set of template arguments, nullptr where none is instantiated. These are
// the only places that know that int8 has entries of its own (IGMMA, apart from the floating-point HGMMA kernels).
// k == 1 (k-means assignment, KP = 16, CTA pairs at most): the register-resident top-2 epilogue; k-means takes no int8 points
// and no mask.
template <int KP, bool IS_L2, Op OP, int CL, bool TOP1>
auto knn_entry() {
    if constexpr (TOP1) {
        if constexpr (KP == 16 && OP != Op::I8 && CL <= 2) return knn_filter_kernel<KP, IS_L2, OP, CL, true>;
        else return nullptr;
    } else if constexpr (OP == Op::I8) {
        return knn_i8_filter_kernel<KP, IS_L2, CL>;
    } else {
        return knn_filter_kernel<KP, IS_L2, OP, CL>;
    }
}

// the masked kernels (mask != nullptr): same grid, shared memory and schedule as the unmasked ones
template <int KP, bool IS_L2, Op OP, int CL, bool TOP1>
auto knn_masked_entry() {
    if constexpr (TOP1) return nullptr;
    else if constexpr (OP == Op::I8) return knn_masked_i8_filter_kernel<KP, IS_L2, CL>;
    else return knn_masked_filter_kernel<KP, IS_L2, OP, CL>;
}

// the range filter keeps no list, so it has no KP
template <Op OP, bool IS_L2, int CL>
auto range_entry() {
    if constexpr (OP == Op::I8) return range_i8_filter_kernel<IS_L2, CL>;
    else return range_filter_kernel<OP, IS_L2, CL>;
}

template <Op OP, bool IS_L2, int CL>
auto range_masked_entry() {
    if constexpr (OP == Op::I8) return range_masked_i8_filter_kernel<IS_L2, CL>;
    else return range_masked_filter_kernel<OP, IS_L2, CL>;
}

// the all-pairs filter runs single CTAs or CTA pairs
template <Op OP, int CL>
auto pair_entry() {
    if constexpr (CL > 2) return nullptr;
    else if constexpr (OP == Op::I8) return pair_i8_filter_kernel<CL>;
    else return pair_filter_kernel<OP, CL>;
}

// The checks every filter launch opens with: nq queries against the rows of X, no work (*empty) with fewer than min_rows.
int filter_prologue(const MatView& X, int64_t nq, int64_t min_rows, bool is_l2, int cluster, int workers, bool* empty) {
    *empty = nq <= 0 || X.n < min_rows;
    if (*empty) return B2_OK;
    if (X.n > 0x7fffff00LL || nq > 0x7fffff00LL) {
        set_error("matrix too large for 32-bit row ids (n=%lld nq=%lld)", (long long)X.n, (long long)nq);
        return B2_ERANGE;
    }
    if (is_l2 && (!X.norm2 || (filter_op(X.filt_dtype) == Op::I8 && !X.norm2_i8))) {
        set_error("internal: L2 filter without row norms");
        return B2_EINVAL;
    }
    // the two CTA pairs of a cluster of four sweep the same corpus tiles only with an even worker count
    if ((cluster != 1 && cluster != 2 && cluster != FILTER_CL) || workers <= 0 || (cluster > 2 && workers % 2 != 0)) {
        set_error("internal: bad filter launch (%d workers of %d CTAs)", workers, cluster);
        return B2_EINVAL;
    }
    return B2_OK;
}

// The schedule geometry of a launch over nq queries and the rows of X in clusters of `cluster`: n_splits corpus splits, of
// which the first units_whole query units (knn's two-phase schedule) take only the first. Every other field is zero.
int filter_params(const MatView& X, Op op, int64_t nq, int cluster, int n_splits, int units_whole, FilterParams* out) {
    FilterParams p{};
    p.nq = (int32_t)nq;
    p.n = (int32_t)X.n;
    p.num_kb = (int32_t)ceil_div(X.d, KB_BYTES / op_bytes(op));
    p.n_mtiles = (int32_t)ceil_div(nq, BLOCK_M);
    p.n_munits = cluster > 1 ? (p.n_mtiles + 1) / 2 : p.n_mtiles;
    p.n_ntiles = (int32_t)ceil_div(X.n, BLOCK_N);
    p.tiles_per_split = (int32_t)ceil_div(p.n_ntiles, n_splits);
    p.n_splits = n_splits;
    p.units_whole = units_whole;
    if ((int64_t)p.tiles_per_split * (n_splits - 1) >= p.n_ntiles) {
        set_error("internal: empty corpus split (tiles %d, splits %d)", p.n_ntiles, n_splits);
        return B2_EINVAL;
    }
    if (units_whole < 0 || units_whole > p.n_munits || (cluster > 2 && units_whole % 2 != 0)) {
        set_error("internal: bad two-phase schedule (%d whole units of %d, clusters of %d)", units_whole, p.n_munits, cluster);
        return B2_EINVAL;
    }
    // clusters of four: the two CTA pairs of a cluster sweep the same corpus tiles only with an even number of whole units and
    // an even number of units cut into splits; a surplus unit past the last query tile loads zeros, writes nothing
    if (cluster > 2) p.n_munits += (p.n_munits - units_whole) & 1;
    *out = p;
    return B2_OK;
}

// CTAs of a persistent launch: no more workers than work items (as the kernel's num_items counts them). Workers are CTA pairs
// in cluster mode; in clusters of four both counts are even, so whole clusters are launched.
int filter_grid(const FilterParams& p, int cluster, int workers) {
    const int64_t items = p.pair_mode ? p.pair_items : (int64_t)p.units_whole + (int64_t)(p.n_munits - p.units_whole) * p.n_splits;
    return (cluster > 1 ? 2 : 1) * (int)std::min<int64_t>(items, workers);
}

}  // namespace

int sm_count(int device) {
    static int cached[64] = {0};
    if (device >= 0 && device < 64 && cached[device]) return cached[device];
    int n = 132;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device);
    if (device >= 0 && device < 64) cached[device] = n;
    return n;
}

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

// Clusters of FILTER_CL CTAs over a long corpus, CTA pairs for the k-means assignment and short corpora; a cluster needs at
// least that many query tiles. Smaller chunks, or B2_FILTER_2CTA=0, run single CTAs.
int filter_cluster(int64_t nq, int64_t n, bool top1) {
    static int mode = -1;
    if (mode < 0) {
        const char* e = getenv("B2_FILTER_2CTA");
        mode = e ? (atoi(e) != 0 ? 1 : 0) : 1;  // default: clusters
    }
    const int cl = top1 || ceil_div(n, BLOCK_N) < FILTER_CL_MIN_NTILES ? 2 : FILTER_CL;
    return mode == 1 && ceil_div(nq, BLOCK_M) >= cl ? cl : 1;
}

// Workers of one persistent filter launch in clusters of `cl` on the current device, which is `device`: as many as are
// co-resident (CTA pairs in cluster mode, two per cluster of four; single CTAs otherwise), cached per device. kp is the knn
// filter's candidate capacity, 0 for the range filter. Every instantiation of one family and KP has the same block, shared
// memory and register budget, so the IP / bf16 one stands for all.
int filter_workers(int device, int kp, int cl, int* workers) {
    static int cached[64][3][5] = {};
    const int ci = cl == 1 ? 0 : cl == 2 ? 1 : 2;
    const int ki = kp == 0 ? 0 : kp == 16 ? 1 : kp == 32 ? 2 : kp == 64 ? 3 : 4;
    int* slot = (device >= 0 && device < 64) ? &cached[device][ci][ki] : nullptr;
    if (slot && *slot) {
        *workers = *slot;
        return B2_OK;
    }
    B2_TRY(with_cluster(cl, [&](auto CL) {
        if (kp == 0) return co_resident_clusters(range_filter_kernel<Op::BF16, false, CL.value>, RANGE_SMEM, CL, workers);
        return with_kp(kp, [&](auto KP) {
            return co_resident_clusters(knn_filter_kernel<KP.value, false, Op::BF16, CL.value>, smem_bytes(KP), CL, workers);
        });
    }));
    if (cl > 2) *workers *= cl / 2;
    if (slot) *slot = *workers;
    return B2_OK;
}

// Number of corpus splits: enough work items to fill the `workers` workers, and few idle workers in the last wave.
// In cluster mode (cl > 1) a worker is a CTA pair and a query unit is two query tiles; in clusters of four the units cut into
// splits are rounded up to an even number (see make_sched).
int filter_choose_splits(int64_t nq, int64_t n, int workers, int cl, bool top1, int min_splits, int* units_whole) {
    if (units_whole) *units_whole = 0;
    const int64_t n_mtiles = ceil_div(nq, BLOCK_M);
    const int64_t n_units = cl > 1 ? ceil_div(n_mtiles, 2) : n_mtiles;
    auto split_units = [cl](int64_t u) { return cl > 2 ? u + (u & 1) : u; };
    const int64_t n_ntiles = ceil_div(n, BLOCK_N);
    // cost model: an item costs its corpus tiles plus ~13 tile-times of list warm-up, the
    // kernel takes `waves` such items back to back, and every extra split adds two candidate lists per query to finalize
    const double kWarmupTiles = top1 ? 1.0 : 13.0;  // the register-resident top-2 epilogue has no list to warm up
    double best_cost = 1e300;
    int best = 0;
    for (int s = std::max(1, min_splits); s <= 256 && s <= n_ntiles; ++s) {
        const int64_t tps = ceil_div(n_ntiles, s);
        if (ceil_div(n_ntiles, tps) != s) continue;  // every split must receive tiles
        const int64_t items = split_units(n_units) * s;
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
    const int64_t waves_a = n_units / workers;
    if (units_whole && min_splits <= 1 && waves_a >= 1) {
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
                const int64_t waves_b = ceil_div(split_units(rem) * s, workers);
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
                      int n_splits, int cluster, int workers, float* cand_score, int32_t* cand_id, float* cand_thr,
                      cudaStream_t stream, bool top1, int units_whole) {
    const bool is_l2 = metric == B2_METRIC_L2;
    bool empty;
    B2_TRY(filter_prologue(X, nq, 1, is_l2, cluster, workers, &empty));
    if (empty) return B2_OK;
    const Op op = filter_op(X.filt_dtype);
    CUtensorMap tq, tx;
    B2_TRY(make_tmap(&tq, q_filt, op, nq, X.d, q_pitch, BLOCK_M));
    // each CTA of a cluster loads 1/cluster of the 256-row corpus tile (and multicasts it to all of them)
    B2_TRY(make_tmap(&tx, X.filt, op, X.n, X.d, X.filt_pitch, BLOCK_N / cluster));
    FilterParams p;
    B2_TRY(filter_params(X, op, nq, cluster, n_splits, units_whole, &p));
    p.xnorm = X.norm2;
    p.xnorm_i = X.norm2_i8;
    p.cand_score = cand_score;
    p.cand_id = cand_id;
    p.cand_thr = cand_thr;
    p.top1 = (top1 && kp == 16) ? 1 : 0;  // register-resident top-2 epilogue: requested by the k-means assignment path only
    p.nparts = 1;
    if (units_whole > 0 && n_splits > 1) {
        // whole units write split 0 only: the other lists of their queries must read as empty (id -1, bound -inf)
        B2_CUDA(cudaMemsetAsync(cand_id, 0xFF, (size_t)nq * n_splits * kp * sizeof(int32_t), stream));
        B2_TRY(launch_fill_f32(cand_thr, nq * (int64_t)n_splits * 2, -INFINITY, stream));
    }
    const int grid = filter_grid(p, cluster, workers);
    return with_cluster(cluster, [&](auto CL) {
        return with_kp(kp, [&](auto KP) {
            return with_bool(is_l2, [&](auto L2) {
                return with_op(op, [&](auto OP) {
                    return with_bool(p.top1, [&](auto TOP1) {
                        if (X.mask)
                            return launch_cluster(knn_masked_entry<KP.value, L2.value, OP.value, CL.value, TOP1.value>(), grid, CL,
                                                  smem_bytes(KP), stream, tq, tx, p, X.mask);
                        return launch_cluster(knn_entry<KP.value, L2.value, OP.value, CL.value, TOP1.value>(), grid, CL, smem_bytes(KP),
                                              stream, tq, tx, p);
                    });
                });
            });
        });
    });
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
    static const bool two = [] { const char* e = getenv("B2_PAIR_2CTA"); return e ? atoi(e) != 0 : true; }();  // default: CTA pairs
    const int cluster = two && ceil_div(X.n, BLOCK_M) >= 2 ? 2 : 1;
    const int workers = sm_count(device) / cluster;
    bool empty;
    B2_TRY(filter_prologue(X, X.n, 2, false, cluster, workers, &empty));
    if (empty) return B2_OK;
    const Op op = filter_op(X.filt_dtype);
    CUtensorMap tq, tx;
    B2_TRY(make_tmap(&tq, X.filt, op, X.n, X.d, X.filt_pitch, BLOCK_M));
    B2_TRY(make_tmap(&tx, X.filt, op, X.n, X.d, X.filt_pitch, BLOCK_N / cluster));  // each CTA of a pair stages half a corpus tile
    FilterParams p;
    B2_TRY(filter_params(X, op, X.n, cluster, 1, 0, &p));
    p.pair_mode = 1;
    p.part = part;
    p.nparts = nparts;
    p.pair_group = std::max(1, pair_group_size(device) / cluster);  // one unit per worker
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
    const int grid = filter_grid(p, cluster, workers);
    return with_cluster(cluster, [&](auto CL) {
        return with_op(op, [&](auto OP) { return launch_cluster(pair_entry<OP.value, CL.value>(), grid, CL, PAIR_SMEM, stream, tq, tx, p); });
    });
}

// Corpus splits of a range filter: items carry no list, so a split costs no warm-up; the corpus is cut only as far as it
// takes to give every worker an item (and not so far that a split has no tile).
int range_filter_splits(int64_t nq, int64_t n, int workers, int cl) {
    const int64_t n_mtiles = ceil_div(nq, BLOCK_M);
    int64_t units = cl > 1 ? ceil_div(n_mtiles, 2) : n_mtiles;
    if (cl > 2) units += units & 1;
    const int64_t n_ntiles = ceil_div(n, BLOCK_N);
    int64_t s = std::max<int64_t>(1, std::min<int64_t>(n_ntiles, ceil_div(workers, units)));
    s = ceil_div(n_ntiles, ceil_div(n_ntiles, s));  // every split receives tiles
    return (int)s;
}

// Candidates (query, row) of a range search: rows of X whose filter score beats thr[query] (filter-score space, see
// RangeParams). cand (device, capacity cap) receives them in arbitrary order and *count (device, zeroed by the caller) the
// total found, which may exceed cap. cluster / workers as filter_cluster / filter_workers chose them. With X.mask set (a masked
// range search) only the selected rows become candidates.
int launch_range_filter(const MatView& X, const void* q_filt, int64_t q_pitch, int64_t nq, int metric, const float* thr, int cluster,
                        int workers, int2* cand, unsigned long long* count, unsigned long long cap, cudaStream_t stream) {
    const bool is_l2 = metric == B2_METRIC_L2;
    bool empty;
    B2_TRY(filter_prologue(X, nq, 1, is_l2, cluster, workers, &empty));
    if (empty) return B2_OK;
    const Op op = filter_op(X.filt_dtype);
    CUtensorMap tq, tx;
    B2_TRY(make_tmap(&tq, q_filt, op, nq, X.d, q_pitch, BLOCK_M));
    B2_TRY(make_tmap(&tx, X.filt, op, X.n, X.d, X.filt_pitch, BLOCK_N / cluster));
    FilterParams p;
    B2_TRY(filter_params(X, op, nq, cluster, range_filter_splits(nq, X.n, workers, cluster), 0, &p));
    p.xnorm = X.norm2;
    p.xnorm_i = X.norm2_i8;
    RangeParams rp;
    rp.thr = thr;
    rp.cand = cand;
    rp.count = count;
    rp.cap = cap;
    const int grid = filter_grid(p, cluster, workers);
    return with_cluster(cluster, [&](auto CL) {
        return with_bool(is_l2, [&](auto L2) {
            return with_op(op, [&](auto OP) {
                if (X.mask)
                    return launch_cluster(range_masked_entry<OP.value, L2.value, CL.value>(), grid, CL, RANGE_SMEM, stream, tq, tx, p, rp,
                                          X.mask);
                return launch_cluster(range_entry<OP.value, L2.value, CL.value>(), grid, CL, RANGE_SMEM, stream, tq, tx, p, rp);
            });
        });
    });
}

}  // namespace b2
