// api.cu — the C-ABI of libb2lotus.so (include/lotus_b200.h): handles, workspaces and the search pipeline
//   prep queries -> wgmma filter (knn_filter_sm90.cu) -> finalize/certify (knn_exact.cu) -> dense exact
//   fallback for uncertified queries.
// Reference call sites replaced: lotus/vector_store/faiss_vs.py:22-77 (see the header for the mapping).
#include <algorithm>
#include <cstring>
#include <atomic>
#include <mutex>
#include <thread>
#include <vector>

#include "index.cuh"

namespace b2 {

static thread_local std::string g_err;
int64_t g_stats[8] = {0, 0, 0, 0, 0, 0, 0, 0};

void set_error(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
}

}  // namespace b2

using namespace b2;

namespace b2 {

// Build the searchable view of a row-major matrix that already sits in device memory.
int build_view(const void* store, int64_t n, int d, int dtype, DevBuf& filt_pad, DevBuf& norm2, DevBuf& scalar,
                      MatView& v, cudaStream_t st, DevBuf* filt16) {
    v.store = store;
    v.n = n;
    v.d = d;
    v.dtype = dtype;
    v.filt_dtype = dtype;
    const int align = dtype == B2_F32 ? 4 : 8;  // TMA row pitch must be a multiple of 16 bytes
    if (d % align == 0) {
        v.filt = store;
        v.filt_pitch = d;
    } else {
        v.filt_pitch = round_up(d, align);
        B2_TRY(filt_pad.ensure((size_t)std::max<int64_t>(n, 1) * v.filt_pitch * esize(dtype)));
        B2_TRY(launch_convert_pad(store, dtype, n, d, filt_pad.p, dtype, v.filt_pitch, st));
        v.filt = filt_pad.p;
    }
    v.filt16 = nullptr;
    v.filt16_pitch = 0;
    static const bool bf16_first = [] { const char* e = getenv("B2_F32_BF16_FIRST"); return e ? atoi(e) != 0 : true; }();
    if (filt16 && dtype == B2_F32 && bf16_first && n >= 4096) {
        v.filt16_pitch = round_up(d, 8);
        B2_TRY(filt16->ensure((size_t)n * v.filt16_pitch * 2));
        B2_TRY(launch_convert_pad(store, dtype, n, d, filt16->p, B2_BF16, v.filt16_pitch, st));
        v.filt16 = filt16->p;
    }
    B2_TRY(norm2.ensure((size_t)std::max<int64_t>(n, 1) * sizeof(float)));
    B2_TRY(scalar.ensure(64));
    B2_TRY(launch_row_norms(store, dtype, n, d, norm2.as<float>(), scalar.as<float>(), st));
    float mx = 0.f;
    B2_CUDA(cudaMemcpyAsync(&mx, scalar.p, sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    v.norm2 = norm2.as<float>();
    v.max_norm = mx;
    return B2_OK;
}

// relative (to ||q||*||x||) bound on |filter score - exact score| of the inner product
float filter_rel_eps(int store_dtype, int filt_dtype, int q_dtype, int d) {
    // fp32 accumulation inside the tensor core: products are exact, every accumulation step may lose one
    // (truncated) ulp of the running magnitude; (d + 64) * 2^-23 is generous. tests/test_gpu_filter_lists.py checks every
    // list entry against this bound in its per-row form (|x| of the row, not max |x|) and pins the formula; the largest
    // measured |err| is 0.66 rel_eps |q| |x| (DESIGN.md §2).
    const double acc = (double)(d + 64) * 1.1920929e-7;
    double ex = 0.0, eq = 0.0;  // relative representation error of the corpus / query operand seen by the MMA
    if (filt_dtype == B2_F32) {  // tf32 wgmma keeps 10 explicit mantissa bits of an fp32 operand
        ex = store_dtype == B2_F32 ? 9.765625e-4 : 0.0;  // bf16 values are exact in tf32
        eq = q_dtype == B2_F32 ? 9.765625e-4 : 0.0;
    } else {  // bf16 wgmma on bf16 operands
        ex = store_dtype == B2_F32 ? 3.90625e-3 : 0.0;  // fp32 values rounded to bf16 for the filter
        eq = q_dtype == B2_F32 ? 3.90625e-3 : 0.0;
    }
    return (float)(acc + ex + eq + ex * eq + 1e-6);
}

// deferred[j] = base + sel[j] (chunk-local query numbers -> batch-wide)
__global__ void defer_append_kernel(const int32_t* sel, int64_t n, int64_t base, int64_t* deferred) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j < n) deferred[j] = base + sel[j];
}

// out[rows[j], :] = sub[j, :] for the k-wide result rows of the deferred queries
__global__ void scatter_rows_kernel(const int64_t* rows, int64_t n, int k, const float* sub_sc, const int64_t* sub_id, float* out_sc,
                                    int64_t* out_id) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n * k) return;
    const int64_t j = t / k, o = t - j * k;
    out_sc[rows[j] * k + o] = sub_sc[t];
    out_id[rows[j] * k + o] = sub_id[t];
}

__global__ void fill_pad_kernel(float* sc, int64_t* id, int64_t total, float pad) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        sc[t] = pad;
        id[t] = -1;
    }
}

// The filter run of a search: for an fp32 store with a bf16 copy (X.filt16) and a small k it is the FIRST level of a two-level
// search (bf16 filter, longer candidate list). Every caller filters exactly as planned here; b2_debug_filter_plan reports it.
int plan_filter(const MatView& X_in, const void* q, int q_dtype, int64_t nq, int k, bool top1, int num_sms, FilterPlan& p) {
    p = FilterPlan();
    p.q = q;
    p.q_dtype = q_dtype;
    p.nq = nq;
    p.k = k;
    p.top1 = top1;
    p.X = X_in;
    // candidate capacity of the bf16 first level (the 2^-8 operand error lets more rows straddle the k-th score): 0 = not used
    const int kp16 = (X_in.filt16 && X_in.n >= 4096) ? (k <= 4 ? 32 : k <= 12 ? 64 : k <= 24 ? 72 : 0) : 0;
    p.two_level = kp16 != 0;
    if (p.two_level) {
        p.X.filt = X_in.filt16;
        p.X.filt_pitch = X_in.filt16_pitch;
        p.X.filt_dtype = B2_BF16;
    }
    const MatView& X = p.X;
    p.kp = p.two_level ? kp16 : filter_kp_for_k(k);
    p.min_splits = filter_min_splits_for_k(k);
    // the filter needs a corpus worth tiling: two tiles at least, and for k > 40 enough tiles to cut into min_splits splits
    // with k well below the rows of a split. The k-means assignment has no other path.
    p.use_filter = top1 || (p.kp != 0 && X.n >= 512 && ceil_div(X.n, 256) >= p.min_splits && X.n >= 4 * (int64_t)k);
    if (!p.use_filter) return B2_OK;
    p.q_pitch = round_up(X.d, X.filt_dtype == B2_F32 ? 4 : 8);
    p.q_in_place = q_dtype == X.filt_dtype && p.q_pitch == X.d && (reinterpret_cast<uintptr_t>(q) & 15) == 0;
    p.rel_eps = filter_rel_eps(X.dtype, X.filt_dtype, q_dtype, X.d);
    // bound the candidate workspace (nqc x n_splits x kp x 8 bytes) to a few GB: fewer queries per chunk when k needs many splits
    p.chunk = top1 ? (int64_t)1 << 23
                   : std::max<int64_t>(4096, std::min<int64_t>(1 << 20, (4LL << 30) / ((int64_t)std::max(p.min_splits, 8) * p.kp * 8)));
    for (int64_t q0 = 0; q0 < nq; q0 += p.chunk) {
        FilterChunk c;
        c.q0 = q0;
        c.nq = std::min<int64_t>(p.chunk, nq - q0);
        c.two_cta = filter_use_pair(c.nq);
        // the k-means top-2 epilogue keeps the uniform split schedule
        c.n_splits = filter_choose_splits(c.nq, X.n, num_sms, c.two_cta, top1, p.min_splits, top1 ? nullptr : &c.units_whole);
        if (c.n_splits <= 0) {
            set_error("internal: no valid corpus split for k=%d over %lld rows", k, (long long)X.n);
            return B2_EINVAL;
        }
        p.chunks.push_back(c);
    }
    return B2_OK;
}

int run_filter(b2_index* idx, const FilterPlan& p, const FilterChunk& c, int metric, cudaStream_t st) {
    const MatView& X = p.X;
    const void* q_filt = reinterpret_cast<const char*>(p.q) + (size_t)c.q0 * X.d * esize(p.q_dtype);
    if (!p.q_in_place) {
        B2_TRY(idx->q_filt.ensure((size_t)c.nq * p.q_pitch * esize(X.filt_dtype)));
        B2_TRY(launch_prep_queries(q_filt, p.q_dtype, c.nq, X.d, idx->q_filt.p, X.filt_dtype, p.q_pitch, st));
        q_filt = idx->q_filt.p;
    }
    B2_TRY(idx->cand_score.ensure((size_t)c.nq * c.n_splits * p.kp * sizeof(float)));
    B2_TRY(idx->cand_id.ensure((size_t)c.nq * c.n_splits * p.kp * sizeof(int32_t)));
    B2_TRY(idx->cand_thr.ensure((size_t)c.nq * c.n_splits * 2 * sizeof(float)));  // two epilogue sets per split
    B2_CUDA(cudaEventRecord(idx->ev0, st));
    B2_TRY(launch_knn_filter(X, q_filt, p.q_pitch, c.nq, metric, p.kp, c.n_splits, c.two_cta, idx->cand_score.as<float>(),
                             idx->cand_id.as<int32_t>(), idx->cand_thr.as<float>(), idx->device, st, p.top1, c.units_whole));
    B2_CUDA(cudaEventRecord(idx->ev1, st));
    return B2_OK;
}

// rows of the dense path's score workspace (score row of 4 bytes per column, plus two sort-key buffers on the full-sort path)
// within 512 MB
static int64_t dense_rows_cap(int64_t n, bool full_sort) {
    return std::max<int64_t>(1, (int64_t)(512ull << 20) / (std::max<int64_t>(n, 1) * (full_sort ? 24 : 4)));
}

// Finalize/certify the candidate lists run_filter left for chunk c (hint: a lower bound the k-th score is known to reach, or
// null), read the one counter back and add the filter's event time to idx->last_filter_ms. The queries the certificate leaves
// open are compacted into idx->sel[1 .. 1 + *n_open]; with `fallback` the exact dense path answers them here.
static int certify(b2_index* idx, const FilterPlan& p, const FilterChunk& c, int metric, const int64_t* id_map, int64_t id_offset,
                   float* out_sc, int64_t* out_id, const float* hint, bool fallback, int64_t* n_open, cudaStream_t st) {
    const MatView& X = p.X;
    const void* qc = reinterpret_cast<const char*>(p.q) + (size_t)c.q0 * X.d * esize(p.q_dtype);
    float* osc = out_sc + (size_t)c.q0 * p.k;
    int64_t* oid = out_id + (size_t)c.q0 * p.k;
    B2_TRY(idx->flags.ensure((size_t)c.nq * sizeof(int32_t)));
    B2_TRY(idx->sel.ensure((size_t)(c.nq + 1) * sizeof(int32_t)));  // [0] = counter, [1..] = uncertified queries
    B2_TRY(idx->h_flags.ensure(64));
    int32_t* sel_count = idx->sel.as<int32_t>();
    int32_t* sel_list = sel_count + 1;
    B2_CUDA(cudaMemsetAsync(sel_count, 0, sizeof(int32_t), st));
    B2_TRY(launch_finalize(X, qc, p.q_dtype, c.nq, metric, p.k, p.kp, p.kp / 2, 2 * c.n_splits, idx->cand_score.as<float>(),
                           idx->cand_id.as<int32_t>(), idx->cand_thr.as<float>(), p.rel_eps, id_map, id_offset, osc, oid,
                           idx->flags.as<int32_t>(), sel_list, sel_count, st, hint));
    // the certificate outcome comes back as ONE counter (the failed queries are compacted on the device)
    int32_t* h_count = reinterpret_cast<int32_t*>(idx->h_flags.p);
    B2_CUDA(cudaMemcpyAsync(h_count, sel_count, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) {
        set_error("search pipeline failed on the device: %s", cudaGetErrorString(se));
        return B2_ECUDA;
    }
    float ms = -1.f;
    if (cudaEventElapsedTime(&ms, idx->ev0, idx->ev1) == cudaSuccess)
        idx->last_filter_ms = (idx->last_filter_ms < 0 ? 0.f : idx->last_filter_ms) + ms;
    const int64_t n_sel = *h_count;
    *n_open = n_sel;
    if (!fallback || n_sel == 0) return B2_OK;
    // exact fallback for the queries the certificate could not cover
    if (p.k > dense_max_k()) {
        set_error("internal: fallback with k=%d", p.k);
        return B2_ERANGE;
    }
    g_stats[ST_FALLBACK] += n_sel;
    const int64_t rows = std::min<int64_t>(dense_rows_cap(X.n, false), n_sel);
    B2_TRY(idx->dense.ensure((size_t)rows * X.n * sizeof(float)));
    return launch_dense_topk(X, qc, p.q_dtype, c.nq, sel_list, n_sel, metric, p.k, id_map, id_offset, idx->dense.as<float>(), rows,
                             nullptr, osc, oid, st);
}

// level 0: the caller's search. On a two-level plan the queries whose first-level certificate fails are deferred, gathered and
// answered by a level-1 call (tf32 filter on the same store, then the dense path for what still fails) and scattered back.
int search_core(b2_index* idx, const MatView& X_in, int metric, const void* q_dev, int q_dtype, int64_t nq, int k,
                       const int64_t* id_map, int64_t id_offset, float* out_sc, int64_t* out_id, cudaStream_t st, int level) {
    if (level == 0) idx->last_filter_ms = -1.f;
    if (nq <= 0) return B2_OK;
    if (level == 0) g_stats[ST_QUERIES] += nq;
    if (X_in.n <= 0) {
        fill_pad_kernel<<<132, 256, 0, st>>>(out_sc, out_id, nq * k, metric == B2_METRIC_L2 ? FLT_MAX : -FLT_MAX);
        B2_LAUNCH_CHECK();
        return B2_OK;
    }
    FilterPlan p;
    B2_TRY(plan_filter(X_in, q_dev, q_dtype, nq, k, false, sm_count(idx->device), p));
    const MatView& X = p.X;
    if (!p.use_filter) {
        if (k > dense_max_k()) {
            set_error("k=%d is not supported (max %d)", k, dense_max_k());
            return B2_ERANGE;
        }
        const bool full_sort = k > dense_select_max_k();  // dense path sorts whole rows: score + two key buffers per column
        const int64_t rows = std::min<int64_t>(dense_rows_cap(X.n, full_sort), nq);
        B2_TRY(idx->dense.ensure((size_t)rows * X.n * sizeof(float)));
        if (full_sort) B2_TRY(idx->sort_keys.ensure(dense_sort_ws_bytes(rows, X.n)));
        B2_TRY(launch_dense_topk(X, q_dev, q_dtype, nq, nullptr, nq, metric, k, id_map, id_offset, idx->dense.as<float>(), rows,
                                 full_sort ? idx->sort_keys.as<uint64_t>() : nullptr, out_sc, out_id, st));
        g_stats[ST_FALLBACK] += nq;
        return B2_OK;
    }
    int64_t n_deferred = 0;
    for (const FilterChunk& c : p.chunks) {
        B2_TRY(run_filter(idx, p, c, metric, st));
        int64_t n_sel = 0;
        B2_TRY(certify(idx, p, c, metric, id_map, id_offset, out_sc, out_id, nullptr, /*fallback=*/!p.two_level, &n_sel, st));
        if (p.two_level && n_sel > 0) {
            B2_TRY(idx->defer.ensure((size_t)nq * sizeof(int64_t)));
            defer_append_kernel<<<(unsigned)ceil_div(n_sel, 256), 256, 0, st>>>(idx->sel.as<int32_t>() + 1, n_sel, c.q0,
                                                                               idx->defer.as<int64_t>() + n_deferred);
            B2_LAUNCH_CHECK();
            n_deferred += n_sel;
        }
    }
    if (n_deferred > 0) {
        // second level: the deferred queries against the exact-operand (tf32) filter of the same store
        const size_t qrow = (size_t)X.d * esize(q_dtype);
        B2_TRY(idx->q_sub.ensure((size_t)n_deferred * qrow));
        B2_TRY(idx->sub_sc.ensure((size_t)n_deferred * k * sizeof(float)));
        B2_TRY(idx->sub_id.ensure((size_t)n_deferred * k * sizeof(int64_t)));
        B2_TRY(idx->scalar.ensure(64));
        int* err = reinterpret_cast<int*>(idx->scalar.as<char>() + 16);
        B2_TRY(launch_gather_rows(q_dev, q_dtype, X.d, idx->defer.as<int64_t>(), n_deferred, nq, idx->q_sub.p, err, st));
        MatView X2 = X_in;
        X2.filt16 = nullptr;
        B2_TRY(search_core(idx, X2, metric, idx->q_sub.p, q_dtype, n_deferred, k, id_map, id_offset, idx->sub_sc.as<float>(),
                           idx->sub_id.as<int64_t>(), st, /*level=*/1));
        scatter_rows_kernel<<<(unsigned)ceil_div(n_deferred * k, 256), 256, 0, st>>>(idx->defer.as<int64_t>(), n_deferred, k, idx->sub_sc.as<float>(),
                                                                                    idx->sub_id.as<int64_t>(), out_sc, out_id);
        B2_LAUNCH_CHECK();
        g_stats[ST_SECOND_LEVEL] += n_deferred;
    }
    return B2_OK;
}

int gather_rows_checked(const void* x, int dtype, int d, const int64_t* ids, int64_t m, int64_t n, void* out, DevBuf& scalar,
                        cudaStream_t st) {
    B2_TRY(scalar.ensure(64));
    int* err = reinterpret_cast<int*>(scalar.as<char>() + 16);
    B2_CUDA(cudaMemsetAsync(err, 0, sizeof(int), st));
    B2_TRY(launch_gather_rows(x, dtype, d, ids, m, n, out, err, st));
    int herr = 0;
    B2_CUDA(cudaMemcpyAsync(&herr, err, sizeof(int), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    if (herr) {
        set_error("ids contains a position outside [0, %lld)", (long long)n);
        return B2_ERANGE;
    }
    return B2_OK;
}

// searchable view for an ids subset (faiss_vs.py:57-64: temporary index over vecs[ids])
static int build_subset(b2_index* idx, const int64_t* ids_dev, int64_t m, MatView& sub, cudaStream_t st) {
    B2_TRY(idx->sub_store.ensure((size_t)std::max<int64_t>(m, 1) * idx->d * esize(idx->dtype)));
    B2_TRY(gather_rows_checked(idx->store.p, idx->dtype, idx->d, ids_dev, m, idx->n, idx->sub_store.p, idx->scalar, st));
    return build_view(idx->sub_store.p, m, idx->d, idx->dtype, idx->sub_filt, idx->sub_norm2, idx->scalar, sub, st, &idx->sub_filt16);
}

// Runs body(lo, hi) over [0, count) in chunks of 2^20 elements on up to 16 host threads.
template <typename Body>
static void for_each_chunk(int64_t count, const Body& body) {
    const int64_t kChunk = 1 << 20;
    const int64_t nchunks = ceil_div(count, kChunk);
    unsigned hw = std::thread::hardware_concurrency();
    const int nthreads = (int)std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(hw ? hw : 1, 16), nchunks));
    std::atomic<int64_t> next{0};
    auto work = [&]() {
        for (int64_t c = next.fetch_add(1); c < nchunks; c = next.fetch_add(1)) body(c * kChunk, std::min(count, c * kChunk + kChunk));
    };
    if (nthreads <= 1) {
        work();
        return;
    }
    std::vector<std::thread> pool;
    for (int t = 0; t < nthreads; ++t) pool.emplace_back(work);
    for (auto& t : pool) t.join();
}

}  // namespace b2

b2_index::~b2_index() {
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (stream) cudaStreamDestroy(stream);
}

// =====================================================================================================================
extern "C" {

int b2_abi_version(void) { return B2_ABI_VERSION; }
const char* b2_last_error(void) { return g_err.c_str(); }

int b2_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    int ok = 0;
    for (int i = 0; i < n; ++i) {
        int major = 0, minor = 0;
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, i);
        cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, i);
        if (major == 9 && minor == 0) ok++;
    }
    return ok;
}

int b2_max_k(void) { return dense_max_k(); }

int b2_index_create(const void* x, int64_t n, int32_t d, int32_t dtype, int32_t metric, int32_t device, int32_t x_on_device,
                    b2_index** out) {
    if (!out) { set_error("out is NULL"); return B2_EINVAL; }
    *out = nullptr;
    if (n < 0 || d <= 0 || (n > 0 && !x)) { set_error("bad matrix shape n=%lld d=%d", (long long)n, d); return B2_EINVAL; }
    if (dtype != B2_F32 && dtype != B2_BF16) { set_error("dtype must be B2_F32 or B2_BF16"); return B2_EINVAL; }
    if (metric != B2_METRIC_IP && metric != B2_METRIC_L2) { set_error("metric must be B2_METRIC_IP or B2_METRIC_L2"); return B2_EINVAL; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        set_error("no CUDA device: libb2lotus has no CPU fallback");
        return B2_ENODEV;
    }
    if (device < 0 || device >= ndev) { set_error("device %d out of range (%d visible)", device, ndev); return B2_EINVAL; }
    int major = 0, minor = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device);
    cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device);
    if (major != 9 || minor != 0) { set_error("device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, major, minor); return B2_ENODEV; }
    DeviceGuard guard(device);
    b2_index* idx = new b2_index();
    idx->device = device;
    idx->n = n;
    idx->d = d;
    idx->dtype = dtype;
    idx->metric = metric;
    auto fail = [&](int rc) { b2_index_free(idx); return rc; };
    if (cudaStreamCreateWithFlags(&idx->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&idx->ev0) != cudaSuccess || cudaEventCreate(&idx->ev1) != cudaSuccess) {
        set_error("stream/event creation failed: %s", cudaGetErrorString(cudaGetLastError()));
        return fail(B2_ECUDA);
    }
    const size_t bytes = (size_t)std::max<int64_t>(n, 1) * d * esize(dtype);
    int rc = idx->store.ensure(bytes);
    if (rc != B2_OK) return fail(rc);
    if (n > 0) {
        // a device-resident source was produced on some other stream (e.g. torch's): our private stream is
        // non-blocking, so order the copy after everything already submitted to the device
        if (x_on_device && cudaDeviceSynchronize() != cudaSuccess) {
            set_error("device synchronisation before the copy failed: %s", cudaGetErrorString(cudaGetLastError()));
            return fail(B2_ECUDA);
        }
        cudaError_t e = cudaMemcpyAsync(idx->store.p, x, (size_t)n * d * esize(dtype),
                                        x_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, idx->stream);
        if (e != cudaSuccess) { set_error("copy of the matrix failed: %s", cudaGetErrorString(e)); return fail(B2_ECUDA); }
    }
    rc = build_view(idx->store.p, n, d, dtype, idx->filt_pad, idx->norm2, idx->scalar, idx->view, idx->stream, &idx->filt16);
    if (rc != B2_OK) return fail(rc);
    *out = idx;
    return B2_OK;
}

void b2_index_free(b2_index* idx) {
    if (!idx) return;
    DeviceGuard guard(idx->device);
    delete idx;
}

int64_t b2_index_ntotal(const b2_index* idx) { return idx ? idx->n : -1; }
int32_t b2_index_dim(const b2_index* idx) { return idx ? idx->d : -1; }
int32_t b2_index_dtype(const b2_index* idx) { return idx ? idx->dtype : -1; }
int32_t b2_index_metric(const b2_index* idx) { return idx ? idx->metric : -1; }
int32_t b2_index_device(const b2_index* idx) { return idx ? idx->device : -1; }
const void* b2_index_data_dev(const b2_index* idx) { return idx ? idx->store.p : nullptr; }
float b2_last_filter_ms(const b2_index* idx) { return idx ? idx->last_filter_ms : -1.f; }

static int check_search_args(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k) {
    if (!idx) { set_error("Index not loaded"); return B2_EINVAL; }
    if (nq < 0 || (nq > 0 && !q)) { set_error("bad query batch"); return B2_EINVAL; }
    if (q_dtype != B2_F32 && q_dtype != B2_BF16) { set_error("q_dtype must be B2_F32 or B2_BF16"); return B2_EINVAL; }
    if (k <= 0) { set_error("k must be positive (got %d)", k); return B2_EINVAL; }
    if (k > dense_max_k()) { set_error("k=%d is not supported (max %d)", k, dense_max_k()); return B2_ERANGE; }
    return B2_OK;
}

int b2_index_search_dev(b2_index* idx, const void* q_dev, int64_t nq, int32_t q_dtype, int32_t k, const int64_t* ids_dev,
                        int64_t n_ids, int64_t id_offset, float* out_scores_dev, int64_t* out_idx_dev, void* stream) {
    B2_TRY(check_search_args(idx, q_dev, nq, q_dtype, k));
    if (nq == 0) return B2_OK;
    if (!out_scores_dev || !out_idx_dev) { set_error("output buffers are NULL"); return B2_EINVAL; }
    DeviceGuard guard(idx->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (ids_dev) {
        if (n_ids < 0) { set_error("n_ids < 0"); return B2_EINVAL; }
        MatView sub;
        B2_TRY(build_subset(idx, ids_dev, n_ids, sub, st));
        B2_TRY(search_core(idx, sub, idx->metric, q_dev, q_dtype, nq, k, ids_dev, 0, out_scores_dev, out_idx_dev, st));
    } else {
        B2_TRY(search_core(idx, idx->view, idx->metric, q_dev, q_dtype, nq, k, nullptr, id_offset, out_scores_dev, out_idx_dev, st));
    }
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
}

int b2_index_search(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, const int64_t* ids, int64_t n_ids,
                    float* out_scores, int64_t* out_idx) {
    B2_TRY(check_search_args(idx, q, nq, q_dtype, k));
    if (nq == 0) return B2_OK;
    if (!out_scores || !out_idx) { set_error("output buffers are NULL"); return B2_EINVAL; }
    DeviceGuard guard(idx->device);
    cudaStream_t st = idx->stream;
    const size_t qbytes = (size_t)nq * idx->d * esize(q_dtype);
    B2_TRY(idx->q_in.ensure(qbytes));
    B2_TRY(idx->out_sc.ensure((size_t)nq * k * sizeof(float)));
    B2_TRY(idx->out_id.ensure((size_t)nq * k * sizeof(int64_t)));
    B2_CUDA(cudaMemcpyAsync(idx->q_in.p, q, qbytes, cudaMemcpyHostToDevice, st));
    const int64_t* ids_dev = nullptr;
    if (ids) {
        if (n_ids < 0) { set_error("n_ids < 0"); return B2_EINVAL; }
        bool identity = n_ids == idx->n;
        for (int64_t i = 0; identity && i < n_ids; ++i) identity = ids[i] == i;
        if (!identity) {
            B2_TRY(idx->ids_dev.ensure((size_t)std::max<int64_t>(n_ids, 1) * sizeof(int64_t)));
            B2_CUDA(cudaMemcpyAsync(idx->ids_dev.p, ids, (size_t)n_ids * sizeof(int64_t), cudaMemcpyHostToDevice, st));
            ids_dev = idx->ids_dev.as<int64_t>();
        }
    }
    if (ids_dev) {
        MatView sub;
        B2_TRY(build_subset(idx, ids_dev, n_ids, sub, st));
        B2_TRY(search_core(idx, sub, idx->metric, idx->q_in.p, q_dtype, nq, k, ids_dev, 0, idx->out_sc.as<float>(), idx->out_id.as<int64_t>(), st));
    } else {
        B2_TRY(search_core(idx, idx->view, idx->metric, idx->q_in.p, q_dtype, nq, k, nullptr, 0, idx->out_sc.as<float>(),
                           idx->out_id.as<int64_t>(), st));
    }
    B2_CUDA(cudaMemcpyAsync(out_scores, idx->out_sc.p, (size_t)nq * k * sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(out_idx, idx->out_id.p, (size_t)nq * k * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("search failed on the device: %s", cudaGetErrorString(e)); return B2_ECUDA; }
    return B2_OK;
}

int b2_merge_topk_dev(const float* scores_dev, const int64_t* idx_dev, int32_t g, int64_t nq, int32_t k, int32_t metric,
                      int32_t device, float* out_scores_dev, int64_t* out_idx_dev, void* stream) {
    if (g <= 0 || k <= 0 || nq < 0) { set_error("bad merge shape g=%d nq=%lld k=%d", g, (long long)nq, k); return B2_EINVAL; }
    if (nq == 0) return B2_OK;
    if (!scores_dev || !idx_dev || !out_scores_dev || !out_idx_dev) { set_error("NULL buffer"); return B2_EINVAL; }
    DeviceGuard guard(device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(launch_merge_topk(scores_dev, idx_dev, g, nq, k, metric, out_scores_dev, out_idx_dev, st));
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
}

int b2_index_search_packed_dev(b2_index* idx, const void* q_dev, int64_t nq, int32_t q_dtype, int32_t k, uint64_t* out_packed_dev,
                               void* stream) {
    B2_TRY(check_search_args(idx, q_dev, nq, q_dtype, k));
    if (nq == 0) return B2_OK;
    if (!out_packed_dev) { set_error("output buffer is NULL"); return B2_EINVAL; }
    if (idx->n > 0xfffffffeLL) { set_error("packed lists hold 32-bit local ids"); return B2_ERANGE; }
    DeviceGuard guard(idx->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(idx->out_sc.ensure((size_t)nq * k * sizeof(float)));
    B2_TRY(idx->out_id.ensure((size_t)nq * k * sizeof(int64_t)));
    B2_TRY(search_core(idx, idx->view, idx->metric, q_dev, q_dtype, nq, k, nullptr, 0, idx->out_sc.as<float>(), idx->out_id.as<int64_t>(), st));
    B2_TRY(launch_pack_topk(idx->out_sc.as<float>(), idx->out_id.as<int64_t>(), nq * (int64_t)k, out_packed_dev, st));
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
}

// ---- row-sharded search in two stages ---------------------------------------------------------------------------------------
// stage 1: filter this shard, report per query a lower bound on the exact score of its j best local candidates (asynchronous:
// nothing is copied to the host). The caller all-reduces (MIN) the bounds over the ranks with j = ceil(k / ranks): k rows of the
// whole index are then known to reach that score. stage 2: finalize with that bound as a hint — rows that cannot reach it are
// not re-scored and the certificate only has to beat the hint — and pack. Shapes the staged path does not cover (dense path,
// fp32 two-level search, more than one query chunk, too many candidate entries) report -inf bounds and stage 2 runs the plain
// search, so the pair of calls is always valid.
int b2_index_search_stage1_dev(b2_index* idx, const void* q_dev, int64_t nq, int32_t q_dtype, int32_t k, int32_t j, float* lower_dev,
                               void* stream) {
    B2_TRY(check_search_args(idx, q_dev, nq, q_dtype, k));
    if (nq == 0) return B2_OK;
    if (!lower_dev || j <= 0) { set_error("bad stage-1 arguments"); return B2_EINVAL; }
    DeviceGuard guard(idx->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    b2_index::Staged& sg = idx->staged;
    sg = b2_index::Staged();
    sg.active = true;
    const MatView& X = idx->view;
    FilterPlan& p = sg.plan;
    B2_TRY(plan_filter(X, q_dev, q_dtype, nq, k, false, sm_count(idx->device), p));
    if (!p.use_filter || p.two_level || p.chunks.size() != 1 || 2 * p.chunks[0].n_splits * (p.kp / 2) > shard_lower_bound_max_entries() ||
        j > k) {
        return launch_fill_f32(lower_dev, nq, -INFINITY, st);  // stage 2 will run the plain search
    }
    idx->last_filter_ms = -1.f;
    const FilterChunk& c = p.chunks[0];
    B2_TRY(run_filter(idx, p, c, idx->metric, st));
    sg.filtered = true;
    B2_TRY(idx->q_norm2.ensure((size_t)nq * sizeof(float)));
    B2_TRY(idx->scalar.ensure(64));
    B2_TRY(launch_row_norms(q_dev, q_dtype, nq, X.d, idx->q_norm2.as<float>(), idx->scalar.as<float>() + 8, st));
    B2_TRY(launch_shard_lower_bound(idx->cand_score.as<float>(), idx->cand_id.as<int32_t>(), nq, 2 * c.n_splits, p.kp / 2, j,
                                    idx->q_norm2.as<float>(), X.max_norm, p.rel_eps, idx->metric, lower_dev, st));
    g_stats[ST_QUERIES] += nq;
    return B2_OK;
}

int b2_index_search_stage2_packed_dev(b2_index* idx, const float* hint_dev, uint64_t* out_packed_dev, void* stream) {
    if (!idx) { set_error("Index not loaded"); return B2_EINVAL; }
    b2_index::Staged sg = idx->staged;
    idx->staged.active = false;
    if (!sg.active) { set_error("stage 2 without a stage 1"); return B2_EINVAL; }
    if (!out_packed_dev) { set_error("output buffer is NULL"); return B2_EINVAL; }
    const FilterPlan& p = sg.plan;
    if (!sg.filtered) return b2_index_search_packed_dev(idx, p.q, p.nq, p.q_dtype, p.k, out_packed_dev, stream);
    if (idx->n > 0xfffffffeLL) { set_error("packed lists hold 32-bit local ids"); return B2_ERANGE; }
    DeviceGuard guard(idx->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(idx->out_sc.ensure((size_t)p.nq * p.k * sizeof(float)));
    B2_TRY(idx->out_id.ensure((size_t)p.nq * p.k * sizeof(int64_t)));
    // uncertified queries: the exact local top-k (a superset of what the merge needs)
    int64_t n_sel = 0;
    B2_TRY(certify(idx, p, p.chunks[0], idx->metric, nullptr, 0, idx->out_sc.as<float>(), idx->out_id.as<int64_t>(), hint_dev,
                   /*fallback=*/true, &n_sel, st));
    B2_TRY(launch_pack_topk(idx->out_sc.as<float>(), idx->out_id.as<int64_t>(), p.nq * (int64_t)p.k, out_packed_dev, st));
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
}

int b2_merge_topk_packed_dev(const uint64_t* packed_dev, const int64_t* shard_offsets, int32_t g, int64_t nq, int32_t k, int32_t metric,
                             int32_t device, float* out_scores_dev, int64_t* out_idx_dev, void* stream) {
    if (g <= 0 || k <= 0 || nq < 0 || !shard_offsets) { set_error("bad merge shape g=%d nq=%lld k=%d", g, (long long)nq, k); return B2_EINVAL; }
    if (nq == 0) return B2_OK;
    if (!packed_dev || !out_scores_dev || !out_idx_dev) { set_error("NULL buffer"); return B2_EINVAL; }
    DeviceGuard guard(device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(launch_merge_packed(packed_dev, shard_offsets, g, nq, k, metric, out_scores_dev, out_idx_dev, st));
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
}

int b2_index_gather(b2_index* idx, const int64_t* ids, int64_t m, void* out, int32_t out_on_device) {
    if (!idx) { set_error("Index not loaded"); return B2_EINVAL; }
    if (m < 0 || (m > 0 && (!ids || !out))) { set_error("bad gather arguments"); return B2_EINVAL; }
    if (m == 0) return B2_OK;
    DeviceGuard guard(idx->device);
    cudaStream_t st = idx->stream;
    const size_t row_bytes = (size_t)idx->d * esize(idx->dtype);
    const int64_t* ids_dev = ids;
    void* out_dev = out;
    if (!out_on_device) {
        B2_TRY(idx->ids_dev.ensure((size_t)m * sizeof(int64_t)));
        B2_CUDA(cudaMemcpyAsync(idx->ids_dev.p, ids, (size_t)m * sizeof(int64_t), cudaMemcpyHostToDevice, st));
        ids_dev = idx->ids_dev.as<int64_t>();
        B2_TRY(idx->sub_store.ensure((size_t)m * row_bytes));
        out_dev = idx->sub_store.p;
    }
    B2_TRY(gather_rows_checked(idx->store.p, idx->dtype, idx->d, ids_dev, m, idx->n, out_dev, idx->scalar, st));
    if (!out_on_device) {
        B2_CUDA(cudaMemcpyAsync(out, out_dev, (size_t)m * row_bytes, cudaMemcpyDeviceToHost, st));
        B2_CUDA(cudaStreamSynchronize(st));
    }
    return B2_OK;
}

// Host-side marshalling helper (no device work): round-to-nearest-even fp32 -> bf16 bit patterns, NaN kept quiet, and
// report whether every value was already bf16-representable (then the 2-byte form is EXACT and the plugin ships it).
int b2_host_f32_to_bf16(const float* x, int64_t count, uint16_t* out, int32_t* all_exact) {
    if (count < 0 || (count > 0 && (!x || !out))) { set_error("bad conversion arguments"); return B2_EINVAL; }
    std::atomic<int> inexact{0};
    for_each_chunk(count, [&](int64_t lo, int64_t hi) {
        const uint32_t* u = reinterpret_cast<const uint32_t*>(x);
        int chunk_inexact = 0;
        for (int64_t i = lo; i < hi; ++i) {
            const uint32_t v = u[i];
            chunk_inexact |= (v & 0xffffu) != 0;
            const bool is_nan = (v & 0x7fffffffu) > 0x7f800000u;
            out[i] = is_nan ? (uint16_t)((v >> 16) | 0x0040u) : (uint16_t)((v + 0x7fffu + ((v >> 16) & 1u)) >> 16);
        }
        if (chunk_inexact) inexact.store(1);
    });
    if (all_exact) *all_exact = inexact.load() ? 0 : 1;
    return B2_OK;
}

// Host-side marshalling helper: bf16 bit patterns -> float32 (exact), threaded.
int b2_host_bf16_to_f32(const uint16_t* x, int64_t count, float* out) {
    if (count < 0 || (count > 0 && (!x || !out))) { set_error("bad conversion arguments"); return B2_EINVAL; }
    uint32_t* o = reinterpret_cast<uint32_t*>(out);
    for_each_chunk(count, [&](int64_t lo, int64_t hi) {
        for (int64_t i = lo; i < hi; ++i) o[i] = (uint32_t)x[i] << 16;
    });
    return B2_OK;
}

// The filter's work schedule for a (queries, rows, k) shape on `num_sms` SMs, as plan_filter decides it for a bf16 index (the
// first query chunk when the batch takes several) — no device work: lets the CPU test-suite check that every (query unit,
// corpus tile) pair is covered exactly once for the shapes the GPU tests do not reach.
int b2_debug_filter_plan(int64_t nq, int64_t n, int32_t k, int32_t num_sms, int32_t* kp, int32_t* n_splits, int32_t* units_whole,
                         int32_t* two_cta) {
    if (nq <= 0 || n <= 0 || k <= 0 || num_sms <= 0 || !kp || !n_splits || !units_whole || !two_cta) { set_error("bad arguments"); return B2_EINVAL; }
    MatView X;  // a bf16 view of n rows: one-level search
    X.n = n;
    X.d = 8;
    X.dtype = X.filt_dtype = B2_BF16;
    FilterPlan p;
    B2_TRY(plan_filter(X, nullptr, B2_BF16, nq, k, false, num_sms, p));
    const FilterChunk c = p.use_filter ? p.chunks[0] : FilterChunk();
    *kp = p.use_filter ? p.kp : 0;
    *n_splits = c.n_splits;
    *units_whole = c.units_whole;
    *two_cta = c.two_cta ? 1 : 0;
    return B2_OK;
}

// The raw candidate lists of one filter run on host queries, planned and launched exactly as search_core (level 0 / 1) or the
// k-means assignment (top1) does it, so the tests can check the kernel's contract list by list instead of through finalize.
int b2_debug_filter_lists(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, int32_t top1, int32_t level,
                          int32_t* plan, float* rel_eps, float* cand_score, int32_t* cand_id, float* cand_thr) {
    B2_TRY(check_search_args(idx, q, nq, q_dtype, k));
    if (nq == 0 || !plan || !rel_eps || (level != 0 && level != 1)) { set_error("bad arguments"); return B2_EINVAL; }
    const bool lists = cand_score && cand_id && cand_thr;
    DeviceGuard guard(idx->device);
    cudaStream_t st = idx->stream;
    MatView X = idx->view;
    if (level == 1 || top1) X.filt16 = nullptr;  // the second level drops the bf16 copy; the k-means centroid view has none
    const size_t qbytes = (size_t)nq * idx->d * esize(q_dtype);
    if (lists) {
        B2_TRY(idx->q_in.ensure(qbytes));
        B2_CUDA(cudaMemcpyAsync(idx->q_in.p, q, qbytes, cudaMemcpyHostToDevice, st));
    }
    FilterPlan p;
    B2_TRY(plan_filter(X, lists ? idx->q_in.p : nullptr, q_dtype, nq, k, top1 != 0, sm_count(idx->device), p));
    const FilterChunk c = p.use_filter ? p.chunks[0] : FilterChunk();
    plan[0] = p.use_filter ? 1 : 0;
    plan[1] = p.use_filter ? p.kp : 0;
    plan[2] = c.n_splits;
    plan[3] = c.units_whole;
    plan[4] = c.two_cta ? 1 : 0;
    plan[5] = p.two_level ? 1 : 0;
    plan[6] = p.X.filt_dtype;
    plan[7] = (int32_t)p.chunks.size();
    *rel_eps = p.rel_eps;
    if (p.chunks.size() > 1) { set_error("%lld queries take %zu query chunks; one is supported", (long long)nq, p.chunks.size()); return B2_ERANGE; }
    if (!lists || !p.use_filter) return B2_OK;
    B2_TRY(run_filter(idx, p, c, idx->metric, st));
    const size_t entries = (size_t)nq * c.n_splits * p.kp;
    B2_CUDA(cudaMemcpyAsync(cand_score, idx->cand_score.p, entries * sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(cand_id, idx->cand_id.p, entries * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(cand_thr, idx->cand_thr.p, (size_t)nq * c.n_splits * 2 * sizeof(float), cudaMemcpyDeviceToHost, st));
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("filter failed on the device: %s", cudaGetErrorString(e)); return B2_ECUDA; }
    return B2_OK;
}

int b2_stats(int64_t* out, int32_t cap) {
    int n = cap < 8 ? cap : 8;
    for (int i = 0; i < n; ++i) out[i] = g_stats[i];
    return n;
}
void b2_stats_reset(void) { memset(g_stats, 0, sizeof(g_stats)); }

}  // extern "C"
