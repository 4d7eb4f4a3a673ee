// index.cuh — the b2_index handle and the pieces of the search pipeline shared by api.cu, dedup.cu, kmeans.cu.
#pragma once
#include <algorithm>
#include <memory>
#include <vector>

#include "common.cuh"

namespace b2 {

// Device / pinned host buffers that grow on demand and free themselves. Invariant: a buffer is destroyed while its device is
// current. A handle's buffers go in b2_index_free under a DeviceGuard; function-local buffers are declared after the
// DeviceGuard of their function, so they are destroyed before the guard restores the previous device.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    int ensure(size_t bytes) {
        if (bytes <= cap) return B2_OK;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) {
            cudaGetLastError();
            set_error("cudaMalloc(%zu bytes) failed: %s", want, cudaGetErrorString(e));
            p = nullptr;
            return B2_ENOMEM;
        }
        cap = want;
        return B2_OK;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <typename T>
    T* as() { return reinterpret_cast<T*>(p); }
};

struct HostBuf {
    void* p = nullptr;
    size_t cap = 0;
    HostBuf() = default;
    HostBuf(const HostBuf&) = delete;
    HostBuf& operator=(const HostBuf&) = delete;
    ~HostBuf() { release(); }
    int ensure(size_t bytes) {
        if (bytes <= cap) return B2_OK;
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        cudaError_t e = cudaMallocHost(&p, bytes + 256);
        if (e != cudaSuccess) {
            cudaGetLastError();
            set_error("cudaMallocHost(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
            return B2_ENOMEM;
        }
        cap = bytes + 256;
        return B2_OK;
    }
    void release() {
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
    }
};

struct KmWork;  // kmeans.cu: per-handle k-means workspaces
struct KmWorkDelete {
    void operator()(KmWork* w) const;  // (defined in kmeans.cu, where KmWork is complete)
};

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// Pinned, mapped host memory (cudaHostAllocMapped): the device reads it through `dev` (UVA), the copy engines stream from it.
struct PinnedBuf {
    void* p = nullptr;
    void* dev = nullptr;
    size_t cap = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf() { release(); }
    int ensure(size_t bytes) {
        if (bytes <= cap) return B2_OK;
        release();
        cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
        if (e == cudaSuccess) e = cudaHostGetDevicePointer(&dev, p, 0);
        if (e != cudaSuccess) {
            cudaGetLastError();
            if (p) cudaFreeHost(p);
            p = dev = nullptr;
            set_error("pinning %zu bytes of host memory failed: %s", bytes, cudaGetErrorString(e));
            return B2_ENOMEM;
        }
        cap = bytes;
        return B2_OK;
    }
    void release() {
        if (p) cudaFreeHost(p);
        p = dev = nullptr;
        cap = 0;
    }
};

// Rows in pinned host memory plus what a streamed search needs of them on the device: norms, a bf16 copy for the first level of
// an fp32 store, and the stream plan (api.cu). Used for a host-resident index and for its large ids subsets.
struct HostRows {
    PinnedBuf rows;    // [n, d] in dtype, pitch d (what finalize, the dense path and gather read through UVA)
    PinnedBuf rows16;  // fp32 stores with n >= 4096: the bf16 rounding of the rows (first level), pitch d
    DevBuf norm2;      // [n] fp32 norms (+ [n] exact int32 norms of an int8 store), the max norm in `scalar`
    DevBuf scalar;
    int64_t n = 0;
    int32_t d = 0, dtype = B2_F32;
    float max_norm = 0.f;
    int64_t chunk_rows = 0;  // rows per chunk (multiple of 256 unless one chunk holds every row)
    int n_chunks = 0;
};

// The streamed-row machinery of a host-resident index: its rows, the ring of device slots and the copy stream.
struct HostStore {
    static constexpr int SLOTS = 2;
    HostRows main;
    std::unique_ptr<HostRows> sub;  // an ids subset larger than the ring, gathered on the host
    size_t ring_bytes = 0;
    DevBuf slot[SLOTS], slot16[SLOTS];  // streamed rows as the filter reads them; int8 stores: their fp16 form for float queries
    DevBuf run_score, run_id, run_thr;  // running per-query lists of the fold
    DevBuf mask_slice;  // masked search: the mask words of a chunk that does not start on a word boundary
    PinnedBuf staging_ids;
    cudaStream_t copy = nullptr;
    cudaEvent_t copied[SLOTS] = {}, freed[SLOTS] = {};
    std::vector<cudaEvent_t> ev;  // timing: per chunk copy start / end (copy stream), filter start / end (search stream)
    cudaEvent_t span0 = nullptr, span1 = nullptr, fin0 = nullptr, fin1 = nullptr;
    float copy_ms = 0.f, span_ms = 0.f, filter_ms = 0.f, finalize_ms = 0.f;  // last search
    ~HostStore();
};

// One run of the top-k filter over a view, decided in one place (plan_filter) for every caller: the plain search, the staged
// sharded search, the k-means assignment and b2_debug_filter_plan.
struct FilterChunk {  // the queries [q0, q0 + nq) of the call, filtered by one launch
    int64_t q0 = 0, nq = 0;
    int cluster = 1;      // CTAs per cluster (filter_cluster)
    int workers = 0;      // workers of the persistent launch, the co-resident ones: CTA pairs in cluster mode (filter_workers)
    int n_splits = 0;
    int units_whole = 0;  // > 0: two-phase schedule (see filter_choose_splits)
};
struct FilterPlan {
    const void* q = nullptr;  // the whole query batch (device)
    int q_dtype = B2_F32;
    int64_t nq = 0;
    int k = 0;
    bool top1 = false;       // k-means assignment: register-resident top-2 epilogue, no other path
    bool use_filter = false;  // false: the exact dense path answers every query
    bool two_level = false;   // fp32 store with a bf16 copy: a bf16 first level with a longer list, failures go to the tf32 level
    MatView X;                // the view the filter streams (filt = the bf16 copy on a two-level first level)
    int kp = 0, min_splits = 1;
    int64_t chunk = 0;  // queries per launch
    std::vector<FilterChunk> chunks;
    int64_t q_pitch = 0;
    bool q_in_place = false;  // the queries already have the filter's type and a TMA-compatible pitch
    // |filter score - exact <q, x>| <= rel_eps |q| |x| + abs_eps (|q| + |x|) (filter_rel_eps / filter_abs_eps)
    float rel_eps = 0.f;
    float abs_eps = 0.f;
    // a query whose norm reaches this is not certified from its lists: fp32 / bf16 queries rounded to fp16 for the filter
    // overflow to inf from a component of 65520 on, and such a component makes the norm at least that large
    float q_norm_limit = INFINITY;
};

// Workspace and state of one range search (range.cu): per-query thresholds, the dense query list, the filter's candidates and
// the verified hits, appended pass by pass (one pass over a device-resident view, one per streamed chunk).
struct RangeWork {
    DevBuf thr, sel, counts, cand, hit_q, hit_pos, hit_sc, keys, sc_alt, sort_tmp, lims, out_d, out_i;
    HostBuf h_count;
    const void* q = nullptr;  // the queries (device), as verification reads them
    int q_dtype = B2_F32, metric = B2_METRIC_IP, filt_dtype = B2_F32;
    int64_t nq = 0;
    float radius = 0.f;
    bool use_filter = false;
    float rel_eps = 0.f, abs_eps = 0.f, q_norm_limit = INFINITY;
    const void* q_filt = nullptr;  // the queries in the filter's type
    int64_t q_pitch = 0;
    int cluster = 1, workers = 0;
    int64_t n_dense = 0;    // queries the dense path answers (sel[1 .. n_dense])
    int64_t n_hits = 0;     // verified hits so far
    int64_t cand_peak = 0;  // most candidates one filter launch produced
    float filter_ms = 0.f;
};
// thresholds and query preparation for a search of X (for a streamed index: X.n = rows per chunk); X.filt_dtype is ignored
int range_begin(b2_index* idx, RangeWork& W, const MatView& X, int metric, const void* q_dev, int q_dtype, int64_t nq, float radius,
                cudaStream_t st);
// filter + verify the rows [own_lo, X.n) of X (X.filt / filt_dtype: the filter operand; X.store: the exact rows, row pitch
// `pitch`), reporting row j as position base + j
int range_pass(b2_index* idx, RangeWork& W, const MatView& X, int64_t pitch, int64_t base, int64_t own_lo, cudaStream_t st);
// sort the hits into W.lims [nq + 1], W.out_d / W.out_i [n_hits] (positions mapped through id_map, or + id_offset)
int range_finish(RangeWork& W, const int64_t* id_map, int64_t id_offset, cudaStream_t st);

}  // namespace b2

struct b2_index {
    using DevBuf = b2::DevBuf;
    using HostBuf = b2::HostBuf;
    using MatView = b2::MatView;
    int device = 0;
    int64_t n = 0;
    int32_t d = 0;
    int32_t dtype = B2_F32;
    int32_t metric = B2_METRIC_IP;
    DevBuf store, filt_pad, filt16, norm2, scalar;
    DevBuf filt_f16, sub_filt_f16;  // int8 stores: the fp16 copy of the rows (and of an ids subset) for floating-point queries
    MatView view;
    // per-call workspaces
    DevBuf q_in, q_filt, cand_score, cand_id, cand_thr, flags, sel, dense, out_sc, out_id, ids_dev;
    DevBuf sub_store, sub_filt, sub_filt16, sub_norm2, sort_keys;
    DevBuf defer, q_sub, sub_sc, sub_id;  // two-level search of fp32 indexes: deferred queries, their rows and results
    HostBuf h_flags;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float last_filter_ms = -1.f;
    std::unique_ptr<b2::KmWork, b2::KmWorkDelete> km;
    // row-sharded search in two stages (b2_index_search_stage1_dev / _stage2_packed_dev): what stage 1 left for stage 2
    struct Staged {
        bool active = false, filtered = false;  // filtered: the candidate lists of plan's (q, nq, k) are in the workspace
        b2::FilterPlan plan;
    } staged;
    DevBuf q_norm2;
    DevBuf q_wide;  // int8 queries on a floating-point store, widened exactly
    DevBuf mask_dev;  // masked search from host buffers: the row bitmap of the call
    b2_index* f16_twin = nullptr;  // int8 indexes: the fp16 copy k-means runs on (kmeans_view)
    // host-resident indexes (b2_index_create_host): the rows live in pinned, mapped host memory and searches stream them
    // through a ring of device slots (api.cu); `store` stays empty and `view.store` is the mapped pointer
    std::unique_ptr<b2::HostStore> host;
    std::unique_ptr<b2::RangeWork> range;  // range search workspaces, made on the first range search
    ~b2_index();  // destroys the stream and events; the buffers free themselves
};

namespace b2 {

// B2_EINVAL for the operations a host-resident index does not offer (dedup, k-means, the staged / packed sharded search)
inline int refuse_host_resident(const b2_index* idx, const char* what) {
    if (idx && idx->host) {
        set_error("%s is not available on a host-resident index", what);
        return B2_EINVAL;
    }
    return B2_OK;
}

// searchable view (filter operand, row norms, max norm) of a row-major device matrix
int build_view(const void* store, int64_t n, int d, int dtype, DevBuf& filt_pad, DevBuf& norm2, DevBuf& scalar, MatView& v,
               cudaStream_t st, DevBuf* filt16 = nullptr);
// The rows a search reads: a device view (the whole index, a gathered ids subset, either with `mask` set), or rows in pinned
// host memory that the search streams through the ring (H), X then being the view finalize and the dense path read through the
// mapped pointer.
struct SearchRows {
    MatView X;
    HostRows* H = nullptr;
    SearchRows() = default;
    SearchRows(const MatView& v) : X(v) {}  // a device view (k-means searches its centroid view)
};
// the exact top-k pipeline: wgmma filter -> finalize/certify -> dense fallback
int search_core(b2_index* idx, const SearchRows& R, int metric, const void* q_dev, int q_dtype, int64_t nq, int k,
                const int64_t* id_map, int64_t id_offset, float* out_sc, int64_t* out_id, cudaStream_t st, int level = 0);
float filter_rel_eps(int store_dtype, int filt_dtype, int q_dtype, int d);
// the index k-means runs on: idx itself, or for an int8 index its fp16 twin (exact), made on first use
int kmeans_view(b2_index* idx, b2_index** out);
float filter_abs_eps(int store_dtype, int filt_dtype, int q_dtype, int d);
// model_sms > 0: plan without a device, modelling the workers as model_sms SMs all in use (b2_debug_filter_plan)
int plan_filter(const MatView& X, const void* q, int q_dtype, int64_t nq, int k, bool top1, int device, FilterPlan& plan,
                int model_sms = 0);
// prep one chunk's queries (unless streamed in place), size the candidate workspace and run the filter between idx->ev0 and ev1
int run_filter(b2_index* idx, const FilterPlan& plan, const FilterChunk& c, int metric, cudaStream_t st);
// out[j] = x[ids[j]] for j < m, synchronised; ids outside [0, n) -> B2_ERANGE. scalar holds the device error flag.
int gather_rows_checked(const void* x, int dtype, int d, const int64_t* ids, int64_t m, int64_t n, void* out, DevBuf& scalar,
                        cudaStream_t st);

}  // namespace b2
