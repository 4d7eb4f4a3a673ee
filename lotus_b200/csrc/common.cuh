// common.cuh — shared declarations for libb2lotus.so (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>

#include "../../include/lotus_b200.h"

namespace b2 {

// ---- error plumbing ------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern int64_t g_stats[8];
enum { ST_LAUNCHES = 0, ST_QUERIES = 1, ST_FALLBACK = 2, ST_FILTER_LAUNCHES = 3, ST_RESCORED = 4, ST_SECOND_LEVEL = 5,
       ST_STREAM_BYTES = 6, ST_STREAM_CHUNKS = 7 };

#define B2_CUDA(expr)                                                                              \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            b2::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return B2_ECUDA;                                                                       \
        }                                                                                          \
    } while (0)

#define B2_LAUNCH_CHECK()                                                                          \
    do {                                                                                           \
        b2::g_stats[b2::ST_LAUNCHES]++;                                                            \
        cudaError_t _e = cudaGetLastError();                                                       \
        if (_e != cudaSuccess) {                                                                   \
            b2::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
            return B2_ECUDA;                                                                       \
        }                                                                                          \
    } while (0)

#define B2_TRY(expr)            \
    do {                        \
        int _rc = (expr);       \
        if (_rc != B2_OK) return _rc; \
    } while (0)

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int64_t round_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// ---- order-preserving keys --------------------------------------------------------------------------------
// ord(f) is monotone in f (for non-NaN f); -0.0 is folded onto +0.0 first.
__host__ __device__ __forceinline__ uint32_t f32_ord(float f) {
    f = f + 0.0f;
#ifdef __CUDA_ARCH__
    uint32_t u = __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, 4);
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float f32_unord(uint32_t k) {
    uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
// "best first when sorted ascending": IP wants large scores first, L2 small distances first.
__host__ __device__ __forceinline__ uint32_t best_first_key(float s, int metric) {
    uint32_t o = f32_ord(s);
    return metric == B2_METRIC_IP ? ~o : o;
}
__host__ __device__ __forceinline__ float best_first_unkey(uint32_t k, int metric) {
    return f32_unord(metric == B2_METRIC_IP ? ~k : k);
}

// ---- element types -------------------------------------------------------------------------------------------
// Every choice that depends on an element type goes through these helpers, so each of them names all four types.
// B2_I8 is read only by the kernels that take a WITH_I8 template flag (and the utility kernels, which always do): the
// finalize and filter kernels of the floating-point types keep code that never tests for it.
__host__ __device__ __forceinline__ bool dtype_valid(int dtype) {
    return dtype == B2_F32 || dtype == B2_BF16 || dtype == B2_F16 || dtype == B2_I8;
}
__host__ __device__ constexpr int esize_float(int dtype) { return dtype == B2_F32 ? 4 : (dtype == B2_BF16 || dtype == B2_F16) ? 2 : 0; }
__host__ __device__ constexpr int esize(int dtype) { return dtype == B2_I8 ? 1 : esize_float(dtype); }
// elements per 16 bytes: the row pitch of a TMA operand is a multiple of this
__host__ __device__ constexpr int tma_align_elems(int dtype) { return 16 / esize(dtype); }
// largest dimension of an int8 index: |<q, x>| <= 2^14 d must stay inside the s32 accumulators of the int8 filter; with L2
// the filter forms 2 <q, x> - |x|^2 = |q|^2 - |q - x|^2 in int32 too, and |q - x|^2 <= 255^2 d needs d < 2^15
constexpr int I8_MAX_D = (1 << 17) - 1;
constexpr int I8_L2_MAX_D = (1 << 15) - 1;

// the fp32 value of the 2-byte pattern `h` (exact for both 2-byte types)
template <int DT>
__device__ __forceinline__ float half_bits_f32(uint32_t h) {
    static_assert(DT == B2_BF16 || DT == B2_F16, "2-byte element types only");
    if constexpr (DT == B2_BF16) return __uint_as_float(h << 16);
    else return __half2float(__ushort_as_half((unsigned short)h));
}

// element i of a row-major matrix of `dtype`, as fp32 (exact)
template <bool WITH_I8 = false>
__device__ __forceinline__ float elem_f32(const void* base, int dtype, size_t i) {
    if constexpr (WITH_I8) {
        if (dtype == B2_I8) return (float)reinterpret_cast<const int8_t*>(base)[i];
    }
    switch (dtype) {
        case B2_F32: return reinterpret_cast<const float*>(base)[i];
        case B2_BF16: return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[i]);
        default: return __half2float(reinterpret_cast<const __half*>(base)[i]);  // B2_F16
    }
}

// out[i] = v rounded to nearest even in `dtype` (|v| >= 65520 becomes inf in fp16). int8 is written only from values that
// are int8 already (copies and padding of int8 rows).
__device__ __forceinline__ void store_elem(void* out, int dtype, size_t i, float v) {
    switch (dtype) {
        case B2_F32: reinterpret_cast<float*>(out)[i] = v; break;
        case B2_BF16: reinterpret_cast<__nv_bfloat16*>(out)[i] = __float2bfloat16_rn(v); break;
        case B2_I8: reinterpret_cast<int8_t*>(out)[i] = (int8_t)__float2int_rn(v); break;
        default: reinterpret_cast<__half*>(out)[i] = __float2half_rn(v); break;  // B2_F16
    }
}

// ---- a matrix the kernels can search ---------------------------------------------------------------------
// `store` holds the exact values (dtype f32, bf16 or f16, row pitch `d`). `filt` is what the wgmma filter
// streams through TMA: the stored 2-byte values (pitch multiple of 8 elements) for a bf16 or fp16 index, fp32 (pitch
// multiple of 4) read as TF32 for an fp32 index; it aliases `store` whenever the pitch already qualifies.
struct MatView {
    const void* store = nullptr;
    const void* filt = nullptr;
    const float* norm2 = nullptr;  // [n] fp32 squared norms of the exact rows (L2 filter epilogue)
    const int32_t* norm2_i8 = nullptr;  // int8 stores: [n] the same norms as exact integers (int8 L2 filter epilogue)
    int64_t n = 0;
    int32_t d = 0;
    int32_t dtype = B2_F32;       // element type of `store`
    int32_t filt_dtype = B2_F32;  // element type of `filt`: B2_BF16 -> bf16 wgmma, B2_F16 -> fp16 wgmma, B2_F32 -> tf32 wgmma
    int64_t filt_pitch = 0;  // elements
    // fp32 stores only (optional): a bf16 rounding of the rows, pitch multiple of 8. When present, searches run a FIRST level on it
    // (bf16 wgmma at twice the tf32 rate, operand error 2^-8 per fp32 operand in the certificate) and only the queries whose
    // certificate fails there go through the tf32 filter on `filt`.
    const void* filt16 = nullptr;
    int64_t filt16_pitch = 0;
    // int8 stores only: an fp16 copy of the rows (exact, pitch multiple of 8), built on the first search with fp32 / bf16 / fp16
    // queries, which cannot use the int8 filter; those searches filter on it with the fp16 wgmma
    const void* filt_f16 = nullptr;
    int64_t filt_f16_pitch = 0;
    float max_norm = 0.f;    // max_j ||x_j|| (upper bound), for the certification margin
    const float* max_norm_dev = nullptr;  // when set, the kernels read the bound from device memory instead (no host sync:
                                          // the k-means loop rebuilds its centroid view every iteration)
    // masked search (optional): ceil(n / 32) words on the device, bit j & 31 of word j >> 5 set = row j takes part. The knn
    // filter and the dense path leave the other rows out; null = every row. max_norm stays that of all rows (a looser bound).
    const uint32_t* mask = nullptr;
};

// ---- kernels / launchers (one per .cu) ------------------------------------------------------------------
// knn_filter_sm90.cu
int filter_kp_for_k(int k);  // candidate-list capacity used for a given k, 0 = k too large for the filter
int launch_knn_filter(const MatView& X, const void* q_filt, int64_t q_pitch, int64_t nq, int metric, int kp,
                      int n_splits, int cluster, int workers, float* cand_score, int32_t* cand_id, float* cand_thr,
                      cudaStream_t stream, bool top1 = false, int units_whole = 0);
int filter_cluster(int64_t nq, int64_t n, bool top1);  // CTAs per cluster of a filter launch: nq queries, n corpus rows
int filter_workers(int device, int kp, int cl, int* workers);  // co-resident workers of that launch on the current device
                                                               // (kp = 0: the range filter)
int filter_choose_splits(int64_t nq, int64_t n, int workers, int cl, bool top1 = false, int min_splits = 1,
                         int* units_whole = nullptr);  // 0: impossible; *units_whole > 0: two-phase schedule (see the definition)
int filter_min_splits_for_k(int k);
int sm_count(int device);  // multiprocessor count of a device, cached
int launch_pair_filter(const MatView& X, float thr, int part, int nparts, int32_t* pair_i, int32_t* pair_j,
                       unsigned long long* pair_count, unsigned long long cap, int device, cudaStream_t stream);
// range search: (query, row) candidates whose filter score beats thr[query] (NaN: none), see range.cu
int range_filter_splits(int64_t nq, int64_t n, int workers, int cl);
int launch_range_filter(const MatView& X, const void* q_filt, int64_t q_pitch, int64_t nq, int metric, const float* thr, int cluster,
                        int workers, int2* cand, unsigned long long* count, unsigned long long cap, cudaStream_t stream);

// knn_exact.cu
int launch_prep_queries(const void* q, int q_dtype, int64_t nq, int d, void* q_filt, int filt_dtype,
                        int64_t filt_pitch, cudaStream_t stream);
int launch_row_norms(const void* x, int dtype, int64_t n, int d, float* norm2, float* max_norm_dev,
                     cudaStream_t stream);
int launch_row_norms_i8(const void* x, int64_t n, int d, int32_t* norm2, cudaStream_t stream);  // exact, int8 rows
int launch_convert_pad(const void* x, int dtype, int64_t n, int d, void* out, int out_dtype, int64_t out_pitch,
                       cudaStream_t stream);
int launch_exact_l2_assigned(const void* pts, int dtype, int64_t m, int d, const float* cent, const int64_t* assign, float* out,
                             cudaStream_t stream);
int launch_gather_rows(const void* x, int dtype, int d, const int64_t* ids, int64_t m, int64_t n, void* out,
                       int* err_flag, cudaStream_t stream);
int launch_finalize(const MatView& X, const void* q, int q_dtype, int64_t nq, int metric, int k, int kp, int list_len,
                    int n_lists, const float* cand_score, const int32_t* cand_id, const float* cand_thr,
                    float rel_eps, float abs_eps, float q_norm_limit, const int64_t* id_map, int64_t id_offset, float* out_scores,
                    int64_t* out_idx, int32_t* flags, int32_t* sel, int32_t* sel_count, cudaStream_t stream, const float* hint = nullptr);
int finalize_capacity(int kp, int k);  // candidates finalize keeps through its merge (32 * 2^i), 0 = beyond it
// host-resident indexes: fold one corpus chunk's lists [nq, n_lists, list_len] (local ids; those below own_lo skipped) into
// running lists [nq, cap] (global ids = base + local, sorted best first) and their bound [nq]
int launch_fold_lists(const float* cand_score, const int32_t* cand_id, const float* cand_thr, int64_t nq, int n_lists, int list_len,
                      int64_t base, int64_t own_lo, int cap, float* run_score, int32_t* run_id, float* run_thr, cudaStream_t stream);
int shard_lower_bound_max_entries();
int launch_shard_lower_bound(const float* cand_score, const int32_t* cand_id, int64_t nq, int n_lists, int list_len, int j, const float* qnorm2,
                             float max_norm, float rel_eps, float abs_eps, float q_norm_limit, int metric, float* lower, cudaStream_t stream);
int launch_fill_f32(float* p, int64_t n, float v, cudaStream_t stream);
int launch_dense_topk(const MatView& X, const void* q, int q_dtype, int64_t nq, const int32_t* q_sel,
                      int64_t n_sel, int metric, int k, const int64_t* id_map, int64_t id_offset, float* dense_ws,
                      int64_t dense_ws_rows, uint64_t* sort_ws, float* out_scores, int64_t* out_idx, cudaStream_t stream);
int launch_merge_topk(const float* scores, const int64_t* idx, int g, int64_t nq, int k, int metric,
                      float* out_scores, int64_t* out_idx, cudaStream_t stream);
size_t dense_sort_ws_bytes(int64_t rows, int64_t n);  // workspace of the full-sort path for `rows` score rows
int launch_pack_topk(const float* scores, const int64_t* idx, int64_t total, uint64_t* out, cudaStream_t stream);
int launch_merge_packed(const uint64_t* packed, const int64_t* shard_offsets, int g, int64_t nq, int k, int metric, float* out_scores,
                        int64_t* out_idx, cudaStream_t stream);
int dense_max_k();         // largest k any path supports
int dense_select_max_k();  // largest k of the radix-select path (beyond it: full row sort)

}  // namespace b2
