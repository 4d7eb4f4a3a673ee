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

// fp32 stores of at least 4096 rows keep a bf16 copy for the first level of a two-level search (B2_F32_BF16_FIRST=0: no copy)
static bool f32_bf16_first() {
    static const bool on = [] { const char* e = getenv("B2_F32_BF16_FIRST"); return e ? atoi(e) != 0 : true; }();
    return on;
}

// Build the searchable view of a row-major matrix that already sits in device memory.
int build_view(const void* store, int64_t n, int d, int dtype, DevBuf& filt_pad, DevBuf& norm2, DevBuf& scalar,
                      MatView& v, cudaStream_t st, DevBuf* filt16) {
    v.store = store;
    v.n = n;
    v.d = d;
    v.dtype = dtype;
    v.filt_dtype = dtype;
    const int align = tma_align_elems(dtype);  // TMA row pitch must be a multiple of 16 bytes
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
    v.filt_f16 = nullptr;
    v.filt_f16_pitch = 0;
    if (filt16 && dtype == B2_F32 && f32_bf16_first() && n >= 4096) {
        v.filt16_pitch = round_up(d, 8);
        B2_TRY(filt16->ensure((size_t)n * v.filt16_pitch * 2));
        B2_TRY(launch_convert_pad(store, dtype, n, d, filt16->p, B2_BF16, v.filt16_pitch, st));
        v.filt16 = filt16->p;
    }
    // int8 stores keep the exact integer norms after the fp32 ones (int8 L2 filter epilogue)
    B2_TRY(norm2.ensure((size_t)std::max<int64_t>(n, 1) * (dtype == B2_I8 ? 2 : 1) * sizeof(float)));
    B2_TRY(scalar.ensure(64));
    B2_TRY(launch_row_norms(store, dtype, n, d, norm2.as<float>(), scalar.as<float>(), st));
    v.norm2_i8 = nullptr;
    if (dtype == B2_I8) {
        v.norm2_i8 = reinterpret_cast<const int32_t*>(norm2.as<float>() + std::max<int64_t>(n, 1));
        B2_TRY(launch_row_norms_i8(store, n, d, const_cast<int32_t*>(v.norm2_i8), st));
    }
    float mx = 0.f;
    B2_CUDA(cudaMemcpyAsync(&mx, scalar.p, sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    v.norm2 = norm2.as<float>();
    v.max_norm = mx;
    return B2_OK;
}

// Relative representation error of one operand of `dtype` seen by a wgmma of `filt_dtype`: 0 when the value is exact.
//   tf32 keeps 10 explicit mantissa bits of an fp32 value (2^-10); bf16 and fp16 values are exact in tf32.
//   bf16 wgmma: fp32 values are rounded to bf16 (2^-8); fp16 values (11-bit significand) are rounded too, also 2^-8.
//   fp16 wgmma: fp32 and bf16 values are rounded to fp16 (2^-11 relative, plus the absolute term of filter_abs_eps for the
//   subnormal range). bf16 values that are fp16-normal would be exact, but a bf16 value can lie outside fp16's range.
//   int8 values (|v| <= 128) are exact in every filter type; the int8 wgmma only ever sees int8 operands.
static double operand_rel_err(int dtype, int filt_dtype) {
    if (dtype == B2_I8 || filt_dtype == B2_I8) return 0.0;
    switch (filt_dtype) {
        case B2_F32: return dtype == B2_F32 ? 9.765625e-4 : 0.0;
        case B2_BF16: return dtype == B2_BF16 ? 0.0 : 3.90625e-3;
        default: return dtype == B2_F16 ? 0.0 : 4.8828125e-4;  // B2_F16
    }
}

// relative (to ||q||*||x||) bound on |filter score - exact score| of the inner product
float filter_rel_eps(int store_dtype, int filt_dtype, int q_dtype, int d) {
    // fp32 accumulation inside the tensor core: products are exact, every accumulation step may lose one
    // (truncated) ulp of the running magnitude; (d + 64) * 2^-23 is generous. tests/test_gpu_filter_lists.py checks every
    // list entry against this bound in its per-row form (|x| of the row, not max |x|) and pins the formula; the largest
    // measured |err| is 0.66 rel_eps |q| |x| (DESIGN.md §2).
    // The int8 wgmma accumulates exactly in s32; its one error is the conversion of the sum s to fp32, at most 2^-24 |s| <=
    // 2^-24 |q| |x| (and none while |s| < 2^24).
    const double acc = filt_dtype == B2_I8 ? 5.9604644775390625e-8 : (double)(d + 64) * 1.1920929e-7;
    // relative representation error of the corpus / query operand seen by the MMA
    const double ex = operand_rel_err(store_dtype, filt_dtype), eq = operand_rel_err(q_dtype, filt_dtype);
    return (float)(acc + ex + eq + ex * eq + 1e-6);
}

// Absolute part of the bound, in |filter - exact| <= rel_eps |q| |x| + abs_eps (|q| + |x|). Rounding v to fp16 (round to
// nearest even) errs by at most 2^-11 |v| + 2^-25 (half the subnormal spacing 2^-24), so a rounded side adds at most
// 2^-25 * sum_i |other_i| <= 2^-25 sqrt(d) |other| to the inner product. Zero unless a side is rounded to fp16. (No search
// rounds both sides: an fp16 filter streams an fp16 store or, in k-means, fp32 centroids against fp16 points; the cross term
// of two rounded sides would need more than this.)
float filter_abs_eps(int store_dtype, int filt_dtype, int q_dtype, int d) {
    if (filt_dtype != B2_F16) return 0.f;
    auto exact = [](int dt) { return dt == B2_F16 || dt == B2_I8; };  // int8 values are exact in fp16
    const int rounded = (exact(store_dtype) ? 0 : 1) + (exact(q_dtype) ? 0 : 1);
    return (float)(rounded * 2.9802322387695312e-8 * sqrt((double)d) * (1.0 + 1e-6));
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

// out[w] = the 32 mask bits from bit0 + 32 w on, for w < words (bits at or past nbits read as zero): the mask of a streamed
// corpus chunk that does not start on a word boundary
__global__ void mask_slice_kernel(const uint32_t* mask, int64_t bit0, int64_t nbits, int64_t words, uint32_t* out) {
    const int64_t src_words = (nbits + 31) >> 5;
    for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < words; w += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = bit0 + 32 * w, i = b >> 5;
        const uint32_t lo = i < src_words ? mask[i] : 0u, hi = i + 1 < src_words ? mask[i + 1] : 0u;
        out[w] = __funnelshift_r(lo, hi, (uint32_t)(b & 31));
    }
}

// The filter run of a search: for an fp32 store with a bf16 copy (X.filt16) and a small k it is the FIRST level of a two-level
// search (bf16 filter, longer candidate list). Every caller filters exactly as planned here; b2_debug_filter_plan reports it.
int plan_filter(const MatView& X_in, const void* q, int q_dtype, int64_t nq, int k, bool top1, int device, FilterPlan& p,
                int model_sms) {
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
    if (X_in.dtype == B2_I8 && q_dtype != B2_I8) {  // floating-point queries on an int8 store: its fp16 copy (exact)
        if (!X_in.filt_f16 && model_sms <= 0) {
            set_error("internal: int8 store without its fp16 copy");
            return B2_EINVAL;
        }
        p.X.filt = X_in.filt_f16;
        p.X.filt_pitch = X_in.filt_f16_pitch;
        p.X.filt_dtype = B2_F16;
    }
    const MatView& X = p.X;
    p.kp = p.two_level ? kp16 : filter_kp_for_k(k);
    p.min_splits = filter_min_splits_for_k(k);
    // the filter needs a corpus worth tiling: two tiles at least, and for k > 40 enough tiles to cut into min_splits splits
    // with k well below the rows of a split. The k-means assignment has no other path.
    p.use_filter = top1 || (p.kp != 0 && X.n >= 512 && ceil_div(X.n, 256) >= p.min_splits && X.n >= 4 * (int64_t)k);
    if (!p.use_filter) return B2_OK;
    p.q_pitch = round_up(X.d, tma_align_elems(X.filt_dtype));
    p.q_in_place = q_dtype == X.filt_dtype && p.q_pitch == X.d && (reinterpret_cast<uintptr_t>(q) & 15) == 0;
    p.rel_eps = filter_rel_eps(X.dtype, X.filt_dtype, q_dtype, X.d);
    p.abs_eps = filter_abs_eps(X.dtype, X.filt_dtype, q_dtype, X.d);
    if (X.filt_dtype == B2_F16 && q_dtype != B2_F16) p.q_norm_limit = 65504.f;  // rounded queries: see FilterPlan
    // bound the candidate workspace (nqc x n_splits x kp x 8 bytes) to a few GB: fewer queries per chunk when k needs many splits
    p.chunk = top1 ? (int64_t)1 << 23
                   : std::max<int64_t>(4096, std::min<int64_t>(1 << 20, (4LL << 30) / ((int64_t)std::max(p.min_splits, 8) * p.kp * 8)));
    for (int64_t q0 = 0; q0 < nq; q0 += p.chunk) {
        FilterChunk c;
        c.q0 = q0;
        c.nq = std::min<int64_t>(p.chunk, nq - q0);
        c.cluster = filter_cluster(c.nq, X.n, top1);
        if (model_sms > 0) c.workers = std::max(1, model_sms / c.cluster) * (c.cluster > 2 ? c.cluster / 2 : 1);
        else B2_TRY(filter_workers(device, p.kp, c.cluster, &c.workers));
        // the k-means top-2 epilogue keeps the uniform split schedule
        c.n_splits = filter_choose_splits(c.nq, X.n, c.workers, c.cluster, top1, p.min_splits, top1 ? nullptr : &c.units_whole);
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
    B2_TRY(launch_knn_filter(X, q_filt, p.q_pitch, c.nq, metric, p.kp, c.n_splits, c.cluster, c.workers,
                             idx->cand_score.as<float>(), idx->cand_id.as<int32_t>(), idx->cand_thr.as<float>(), st, p.top1,
                             c.units_whole));
    B2_CUDA(cudaEventRecord(idx->ev1, st));
    return B2_OK;
}

// The candidate lists finalize reads for one query chunk: per query n_lists lists of list_len entries, each with its bound in
// thr. The filter leaves 2 * n_splits lists of kp / 2 (two epilogue sets per split); a streamed search folds the lists of every
// corpus chunk into one list of finalize_capacity(kp, k) entries.
struct CandLists {
    const float* score;
    const int32_t* id;
    const float* thr;
    int list_len, n_lists;
};

// the lists run_filter left for chunk c
static CandLists filter_lists(b2_index* idx, const FilterPlan& p, const FilterChunk& c) {
    return {idx->cand_score.as<float>(), idx->cand_id.as<int32_t>(), idx->cand_thr.as<float>(), p.kp / 2, 2 * c.n_splits};
}

// rows of the dense path's score workspace (score row of 4 bytes per column, plus two sort-key buffers on the full-sort path)
// within 512 MB
static int64_t dense_rows_cap(int64_t n, bool full_sort) {
    return std::max<int64_t>(1, (int64_t)(512ull << 20) / (std::max<int64_t>(n, 1) * (full_sort ? 24 : 4)));
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

// The fp16 copy of an int8 view that fp32 / bf16 / fp16 queries are filtered against, made once and kept in `buf`.
static int ensure_f16_copy(MatView& v, DevBuf& buf, cudaStream_t st) {
    if (v.dtype != B2_I8 || v.filt_f16) return B2_OK;
    v.filt_f16_pitch = round_up(v.d, tma_align_elems(B2_F16));
    B2_TRY(buf.ensure((size_t)std::max<int64_t>(v.n, 1) * v.filt_f16_pitch * 2));
    B2_TRY(launch_convert_pad(v.store, B2_I8, v.n, v.d, buf.p, B2_F16, v.filt_f16_pitch, st));
    v.filt_f16 = buf.p;
    return B2_OK;
}

// Queries as the store's pipeline takes them. int8 queries on a floating-point store are widened exactly, to fp16 on an fp16
// store and to bf16 otherwise, so that the store's own finalize kernel serves them and every filter level sees an operand of
// no representation error (bf16 is exact in tf32 and on an fp32 store's bf16 first level alike); other queries on an int8
// store need its fp16 copy.
static int adapt_queries(b2_index* idx, const void*& q, int32_t& q_dtype, int64_t nq, cudaStream_t st) {
    if (q_dtype == B2_I8 && idx->dtype != B2_I8 && nq > 0) {
        const int wide = idx->dtype == B2_F16 ? B2_F16 : B2_BF16;
        B2_TRY(idx->q_wide.ensure((size_t)nq * idx->d * 2));
        B2_TRY(launch_convert_pad(q, B2_I8, nq, idx->d, idx->q_wide.p, wide, idx->d, st));
        q = idx->q_wide.p;
        q_dtype = wide;
    }
    // (a host-resident index converts each streamed chunk instead)
    if (q_dtype != B2_I8 && !idx->host) B2_TRY(ensure_f16_copy(idx->view, idx->filt_f16, st));
    return B2_OK;
}

// searchable view for an ids subset (faiss_vs.py:57-64: temporary index over vecs[ids])
static int build_subset(b2_index* idx, const int64_t* ids_dev, int64_t m, int q_dtype, MatView& sub, cudaStream_t st) {
    B2_TRY(idx->sub_store.ensure((size_t)std::max<int64_t>(m, 1) * idx->d * esize(idx->dtype)));
    B2_TRY(gather_rows_checked(idx->view.store, idx->dtype, idx->d, ids_dev, m, idx->n, idx->sub_store.p, idx->scalar, st));
    B2_TRY(build_view(idx->sub_store.p, m, idx->d, idx->dtype, idx->sub_filt, idx->sub_norm2, idx->scalar, sub, st, &idx->sub_filt16));
    return q_dtype != B2_I8 ? ensure_f16_copy(sub, idx->sub_filt_f16, st) : B2_OK;
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

// ---- host-resident indexes ------------------------------------------------------------------------------------------------
// The rows stay in pinned, mapped host memory. A search streams them in chunks through a ring of device slots on a copy stream
// owned by the handle, filters every chunk with the unchanged filter kernel, folds the chunk's lists into running per-query
// lists (fold_lists_kernel) and certifies once at the end; finalize and the dense path read the rows through the mapped
// pointer. Norms stay on the device.

constexpr size_t kDefaultRingBytes = 1ull << 30;

// device bytes one streamed row takes in the ring: the filter-ready row (TMA pitch), plus its fp16 form for an int8 store
static size_t ring_row_bytes(int d, int dtype) {
    size_t b = (size_t)round_up(d, tma_align_elems(dtype)) * esize(dtype);
    if (dtype == B2_I8) b += (size_t)round_up(d, tma_align_elems(B2_F16)) * 2;
    return b;
}

// Chunks of a corpus of n rows for a ring of ring_bytes (0 = the default) of HostStore::SLOTS slots: chunk c owns the rows
// [c * rows, min(n, (c + 1) * rows)) and streams the `rows` rows from min(c * rows, n - rows) on, so every chunk has the same
// shape (and the same filter plan); the last one re-streams the tail of its predecessor and the fold skips those rows.
static int stream_plan(int64_t n, int d, int dtype, size_t ring_bytes, int64_t* chunk_rows, int* n_chunks) {
    const size_t rb = ring_bytes ? ring_bytes : kDefaultRingBytes;
    const size_t row = ring_row_bytes(d, dtype);
    const int64_t cap = (int64_t)(rb / ((size_t)HostStore::SLOTS * row)) / 256 * 256;
    if (cap < 256) {
        set_error("ring_bytes=%zu holds fewer than 256 rows per slot (%d slots, %zu bytes per row)", rb, HostStore::SLOTS, row);
        return B2_EINVAL;
    }
    if (n <= cap) {
        *chunk_rows = n;
        *n_chunks = n > 0 ? 1 : 0;
        return B2_OK;
    }
    const int64_t nc = ceil_div(n, cap);
    const int64_t rows = std::min<int64_t>(cap, round_up(ceil_div(n, nc), 256));  // balanced: the overlap stays below 256 nc
    *chunk_rows = rows;
    *n_chunks = (int)ceil_div(n, rows);
    return B2_OK;
}

// norms (canonical, per row: bit for bit those of a device build), max norm, bf16 copy and plan of rows already in H.rows
static int host_rows_init(HostRows& H, int64_t n, int d, int dtype, size_t ring_bytes, cudaStream_t st) {
    H.n = n;
    H.d = d;
    H.dtype = dtype;
    B2_TRY(stream_plan(n, d, dtype, ring_bytes, &H.chunk_rows, &H.n_chunks));
    if (dtype == B2_F32 && f32_bf16_first() && n >= 4096) {
        B2_TRY(H.rows16.ensure((size_t)n * d * 2));
        B2_TRY(b2_host_f32_to_bf16(reinterpret_cast<const float*>(H.rows.p), n * d, reinterpret_cast<uint16_t*>(H.rows16.p), nullptr));
    }
    B2_TRY(H.norm2.ensure((size_t)std::max<int64_t>(n, 1) * (dtype == B2_I8 ? 2 : 1) * sizeof(float)));
    B2_TRY(H.scalar.ensure(64));
    B2_TRY(launch_row_norms(H.rows.dev, dtype, n, d, H.norm2.as<float>(), H.scalar.as<float>(), st));
    if (dtype == B2_I8)
        B2_TRY(launch_row_norms_i8(H.rows.dev, n, d, reinterpret_cast<int32_t*>(H.norm2.as<float>() + std::max<int64_t>(n, 1)), st));
    B2_CUDA(cudaMemcpyAsync(&H.max_norm, H.scalar.p, sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
}

// the view finalize, the dense path and gathers read: the rows through the mapped pointer, the device norms
static MatView host_view(HostRows& H) {
    MatView v;
    v.store = H.rows.dev;
    v.n = H.n;
    v.d = H.d;
    v.dtype = v.filt_dtype = H.dtype;
    v.filt_pitch = round_up(H.d, tma_align_elems(H.dtype));
    v.norm2 = H.norm2.as<float>();
    v.norm2_i8 = H.dtype == B2_I8 ? reinterpret_cast<const int32_t*>(H.norm2.as<float>() + std::max<int64_t>(H.n, 1)) : nullptr;
    v.max_norm = H.max_norm;
    return v;
}

// the rows x[ids] of a host-resident index gathered on the host, by threads, into hs.sub (pinned), with their norms and plan
static int gather_host_subset(b2_index* idx, const int64_t* ids_host, const int64_t* ids_dev, int64_t n_ids, cudaStream_t st) {
    HostStore& hs = *idx->host;
    if (!ids_host) {
        B2_TRY(hs.staging_ids.ensure((size_t)n_ids * sizeof(int64_t)));
        B2_CUDA(cudaMemcpyAsync(hs.staging_ids.p, ids_dev, (size_t)n_ids * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        B2_CUDA(cudaStreamSynchronize(st));
        ids_host = reinterpret_cast<const int64_t*>(hs.staging_ids.p);
    }
    for (int64_t i = 0; i < n_ids; ++i) {
        if (ids_host[i] < 0 || ids_host[i] >= idx->n) {
            set_error("ids contains a position outside [0, %lld)", (long long)idx->n);
            return B2_ERANGE;
        }
    }
    if (!hs.sub) hs.sub.reset(new HostRows());
    HostRows& S = *hs.sub;
    const size_t row = (size_t)idx->d * esize(idx->dtype);
    B2_TRY(S.rows.ensure((size_t)n_ids * row));
    const char* src = reinterpret_cast<const char*>(hs.main.rows.p);
    char* dst = reinterpret_cast<char*>(S.rows.p);
    for_each_chunk(n_ids, [&](int64_t lo, int64_t hi) {
        for (int64_t i = lo; i < hi; ++i) memcpy(dst + (size_t)i * row, src + (size_t)ids_host[i] * row, row);
    });
    return host_rows_init(S, n_ids, idx->d, idx->dtype, hs.ring_bytes, st);
}

// The rows a search of idx reads: the whole index, or the ids subset (ids_dev on the device, what the results map through;
// ids_host the same ids on the host, or null). A subset of a device-resident index, or of a host-resident one whose rows fit
// in the ring, is gathered into a device view and searched as a device-resident index is; a larger subset of a host-resident
// index is gathered on the host, by threads, into pinned staging and streamed.
static int select_rows(b2_index* idx, const int64_t* ids_host, const int64_t* ids_dev, int64_t n_ids, int q_dtype, cudaStream_t st,
                       SearchRows* rows) {
    *rows = SearchRows();
    HostStore* hs = idx->host.get();
    if (ids_dev && (!hs || (size_t)n_ids * ring_row_bytes(idx->d, idx->dtype) <= hs->ring_bytes))
        return build_subset(idx, ids_dev, n_ids, q_dtype, rows->X, st);
    if (!hs) {
        rows->X = idx->view;
        return B2_OK;
    }
    if (ids_dev) B2_TRY(gather_host_subset(idx, ids_host, ids_dev, n_ids, st));
    rows->H = ids_dev ? hs->sub.get() : &hs->main;
    rows->X = host_view(*rows->H);
    return B2_OK;
}

// The filter plan of a search of R. For streamed rows it is the plan of one chunk (every chunk streams chunk_rows rows, so one
// plan serves them all): level 1 (the second level of an fp32 store) streams the fp32 rows; level 0 of an fp32 store streams the
// bf16 copy when the plan takes two levels.
static int plan_rows(b2_index* idx, const SearchRows& R, const void* q_dev, int q_dtype, int64_t nq, int k, bool top1, int level,
                     FilterPlan& p) {
    if (!R.H) return plan_filter(R.X, q_dev, q_dtype, nq, k, top1, idx->device, p);
    const HostRows& H = *R.H;
    MatView Xc = R.X;
    Xc.n = H.chunk_rows;
    if (level == 0 && H.rows16.p) {
        Xc.filt16 = H.rows16.dev;  // (the plan only tests it; each chunk's slot replaces it)
        Xc.filt16_pitch = round_up(H.d, tma_align_elems(B2_BF16));
    }
    if (H.dtype == B2_I8 && q_dtype != B2_I8) {
        Xc.filt_f16 = H.rows.dev;  // (likewise: each chunk's fp16 form replaces it)
        Xc.filt_f16_pitch = round_up(H.d, tma_align_elems(B2_F16));
    }
    return plan_filter(Xc, q_dev, q_dtype, nq, k, top1, idx->device, p);
}

static int ensure_events(std::vector<cudaEvent_t>& ev, size_t count) {
    while (ev.size() < count) {
        cudaEvent_t e = nullptr;
        B2_CUDA(cudaEventCreate(&e));
        ev.push_back(e);
    }
    return B2_OK;
}

// Streams the rows of H through the ring of device slots; the copy of chunk ch + 1 (on the copy stream) is issued before chunk
// ch is processed. Xc describes every chunk (Xc.n = H.chunk_rows; norms and mask those of all of H), and Xc.filt_dtype names the
// filter operand: the rows, their bf16 copy (the first level of an fp32 store) or, for float queries on an int8 store, their
// fp16 form, converted in the slot when `convert`. Chunk ch reaches on_slot(X, pitch, base, own_lo) as the view X of its slot:
// the rows [base, base + X.n) of H, exact in X.store at `pitch` elements per row, of which the first own_lo belong to the previous
// chunk (only the last chunk re-streams its predecessor's tail). The slot is released once on_slot's work is queued; then
// then(base, own_lo) runs.
template <typename OnSlot, typename Then>
static int stream_chunks(b2_index* idx, HostRows& H, const MatView& Xc, bool convert, cudaStream_t st, const OnSlot& on_slot,
                         const Then& then) {
    HostStore& hs = *idx->host;
    const int d = H.d;
    const bool via_f16 = Xc.filt_dtype == B2_F16 && H.dtype == B2_I8;
    const int src_dtype = via_f16 ? H.dtype : Xc.filt_dtype;
    const char* src = reinterpret_cast<const char*>(src_dtype == H.dtype ? H.rows.p : H.rows16.p);
    const size_t src_row = (size_t)d * esize(src_dtype);
    const int64_t pitch = via_f16 ? d : round_up(d, tma_align_elems(src_dtype));  // elements per slot row
    const size_t slot_pitch = (size_t)pitch * esize(src_dtype);
    const int64_t f16_pitch = round_up(d, tma_align_elems(B2_F16));
    const int64_t R = H.chunk_rows;
    for (int s = 0; s < HostStore::SLOTS; ++s) {
        B2_TRY(hs.slot[s].ensure((size_t)R * slot_pitch));
        if (via_f16) B2_TRY(hs.slot16[s].ensure((size_t)R * f16_pitch * 2));
    }
    const int nc = H.n_chunks;
    B2_TRY(ensure_events(hs.ev, (size_t)4 * nc));
    auto issue_copy = [&](int ch) -> int {
        const int s = ch % HostStore::SLOTS;
        const int64_t base = std::min<int64_t>((int64_t)ch * R, H.n - R);
        B2_CUDA(cudaStreamWaitEvent(hs.copy, hs.freed[s], 0));  // the slot's previous chunk has been processed
        B2_CUDA(cudaEventRecord(hs.ev[4 * ch], hs.copy));
        B2_CUDA(cudaMemcpy2DAsync(hs.slot[s].p, slot_pitch, src + (size_t)base * src_row, src_row, src_row, (size_t)R,
                                  cudaMemcpyHostToDevice, hs.copy));
        B2_CUDA(cudaEventRecord(hs.ev[4 * ch + 1], hs.copy));
        B2_CUDA(cudaEventRecord(hs.copied[s], hs.copy));
        g_stats[ST_STREAM_BYTES] += R * (int64_t)src_row;
        return B2_OK;
    };
    B2_CUDA(cudaEventRecord(hs.span0, st));
    B2_TRY(issue_copy(0));
    for (int ch = 0; ch < nc; ++ch) {
        if (ch + 1 < nc) B2_TRY(issue_copy(ch + 1));
        const int s = ch % HostStore::SLOTS;
        const int64_t base = std::min<int64_t>((int64_t)ch * R, H.n - R);
        B2_CUDA(cudaStreamWaitEvent(st, hs.copied[s], 0));
        MatView X = Xc;
        X.store = X.filt = hs.slot[s].p;
        X.filt_pitch = pitch;
        if (via_f16) {
            if (convert) B2_TRY(launch_convert_pad(hs.slot[s].p, B2_I8, R, d, hs.slot16[s].p, B2_F16, f16_pitch, st));
            X.filt = hs.slot16[s].p;
            X.filt_pitch = f16_pitch;
        }
        X.norm2 = Xc.norm2 + base;
        X.norm2_i8 = Xc.norm2_i8 ? Xc.norm2_i8 + base : nullptr;
        if (Xc.mask) {
            // the chunk's rows start at a word of the mask, except those of a last chunk that re-streams its predecessor's tail
            if (base % 32 == 0) {
                X.mask = Xc.mask + base / 32;
            } else {
                const int64_t words = ceil_div(R, 32);
                B2_TRY(hs.mask_slice.ensure((size_t)words * sizeof(uint32_t)));
                mask_slice_kernel<<<(unsigned)std::min<int64_t>(ceil_div(words, 256), 1024), 256, 0, st>>>(Xc.mask, base, H.n, words,
                                                                                                      hs.mask_slice.as<uint32_t>());
                B2_LAUNCH_CHECK();
                X.mask = hs.mask_slice.as<uint32_t>();
            }
        }
        B2_CUDA(cudaEventRecord(hs.ev[4 * ch + 2], st));
        B2_TRY(on_slot(X, pitch, base, (int64_t)ch * R - base));
        B2_CUDA(cudaEventRecord(hs.ev[4 * ch + 3], st));
        B2_CUDA(cudaEventRecord(hs.freed[s], st));  // the slot may take its next chunk
        B2_TRY(then(base, (int64_t)ch * R - base));
        g_stats[ST_STREAM_CHUNKS]++;
    }
    B2_CUDA(cudaEventRecord(hs.span1, st));
    return B2_OK;
}

// Filter the query chunk qc of plan p over every corpus chunk of H and fold the lists into hs.run_* ([qc.nq, cap] and [qc.nq]).
static int stream_filter_fold(b2_index* idx, HostRows& H, const FilterPlan& p, const FilterChunk& qc, int metric, int cap,
                              cudaStream_t st) {
    HostStore& hs = *idx->host;
    // the queries in the filter's form, once for every corpus chunk
    FilterPlan pc = p;
    FilterChunk c = qc;
    c.q0 = 0;
    const void* qsrc = reinterpret_cast<const char*>(p.q) + (size_t)qc.q0 * H.d * esize(p.q_dtype);
    pc.q = qsrc;
    if (!p.q_in_place) {
        B2_TRY(idx->q_filt.ensure((size_t)qc.nq * p.q_pitch * esize(p.X.filt_dtype)));
        B2_TRY(launch_prep_queries(qsrc, p.q_dtype, qc.nq, H.d, idx->q_filt.p, p.X.filt_dtype, p.q_pitch, st));
        pc.q = idx->q_filt.p;
        pc.q_in_place = true;
    }
    B2_TRY(hs.run_score.ensure((size_t)qc.nq * cap * sizeof(float)));
    B2_TRY(hs.run_id.ensure((size_t)qc.nq * cap * sizeof(int32_t)));
    B2_TRY(hs.run_thr.ensure((size_t)qc.nq * sizeof(float)));
    B2_CUDA(cudaMemsetAsync(hs.run_id.p, 0xFF, (size_t)qc.nq * cap * sizeof(int32_t), st));
    B2_TRY(launch_fill_f32(hs.run_thr.as<float>(), qc.nq, -INFINITY, st));
    return stream_chunks(
        idx, H, p.X, /*convert=*/true, st,
        [&](const MatView& X, int64_t, int64_t, int64_t) {
            pc.X = X;
            return run_filter(idx, pc, c, metric, st);
        },
        [&](int64_t base, int64_t own_lo) {
            const CandLists L = filter_lists(idx, pc, c);
            return launch_fold_lists(L.score, L.id, L.thr, c.nq, L.n_lists, L.list_len, base, own_lo, cap, hs.run_score.as<float>(),
                                     hs.run_id.as<int32_t>(), hs.run_thr.as<float>(), st);
        });
}

// event times of the last stream_filter_fold and the finalize after it (after the search stream was synchronised)
static void stream_times_add(b2_index* idx, int nc) {
    HostStore& hs = *idx->host;
    float ms = 0.f, filt = 0.f;
    for (int ch = 0; ch < nc; ++ch) {
        if (cudaEventElapsedTime(&ms, hs.ev[4 * ch], hs.ev[4 * ch + 1]) == cudaSuccess) hs.copy_ms += ms;
        if (cudaEventElapsedTime(&ms, hs.ev[4 * ch + 2], hs.ev[4 * ch + 3]) == cudaSuccess) filt += ms;
    }
    if (cudaEventElapsedTime(&ms, hs.span0, hs.span1) == cudaSuccess) hs.span_ms += ms;
    if (cudaEventElapsedTime(&ms, hs.fin0, hs.fin1) == cudaSuccess) hs.finalize_ms += ms;
    hs.filter_ms += filt;
    idx->last_filter_ms = (idx->last_filter_ms < 0 ? 0.f : idx->last_filter_ms) + filt;
}

// The candidate lists of query chunk c of a search of R: the filter run over a device view, or over every streamed chunk of
// R.H with the lists folded into one of `cap` entries.
static int chunk_lists(b2_index* idx, const SearchRows& R, const FilterPlan& p, const FilterChunk& c, int metric, int cap,
                       CandLists* L, cudaStream_t st) {
    if (!R.H) {
        B2_TRY(run_filter(idx, p, c, metric, st));
        *L = filter_lists(idx, p, c);
        return B2_OK;
    }
    B2_TRY(stream_filter_fold(idx, *R.H, p, c, metric, cap, st));
    HostStore& hs = *idx->host;
    *L = {hs.run_score.as<float>(), hs.run_id.as<int32_t>(), hs.run_thr.as<float>(), cap, 1};
    return B2_OK;
}

// Finalize/certify the lists L of chunk c over the rows R (hint: a lower bound the k-th score is known to reach, or null), read
// the one counter back and add the filter's event time to idx->last_filter_ms (for streamed rows: every chunk's, with the
// copy, span and finalize times in the stream times). The queries the certificate leaves open are compacted into
// idx->sel[1 .. 1 + *n_open]; with `fallback` the exact dense path answers them here.
static int certify(b2_index* idx, const FilterPlan& p, const FilterChunk& c, const SearchRows& R, const CandLists& L, int metric,
                   const int64_t* id_map, int64_t id_offset, float* out_sc, int64_t* out_id, const float* hint, bool fallback,
                   int64_t* n_open, cudaStream_t st) {
    const MatView& X = R.X;
    const void* qc = reinterpret_cast<const char*>(p.q) + (size_t)c.q0 * X.d * esize(p.q_dtype);
    float* osc = out_sc + (size_t)c.q0 * p.k;
    int64_t* oid = out_id + (size_t)c.q0 * p.k;
    B2_TRY(idx->flags.ensure((size_t)c.nq * sizeof(int32_t)));
    B2_TRY(idx->sel.ensure((size_t)(c.nq + 1) * sizeof(int32_t)));  // [0] = counter, [1..] = uncertified queries
    B2_TRY(idx->h_flags.ensure(64));
    int32_t* sel_count = idx->sel.as<int32_t>();
    int32_t* sel_list = sel_count + 1;
    B2_CUDA(cudaMemsetAsync(sel_count, 0, sizeof(int32_t), st));
    if (R.H) B2_CUDA(cudaEventRecord(idx->host->fin0, st));
    B2_TRY(launch_finalize(X, qc, p.q_dtype, c.nq, metric, p.k, p.kp, L.list_len, L.n_lists, L.score, L.id, L.thr, p.rel_eps,
                           p.abs_eps, p.q_norm_limit, id_map, id_offset, osc, oid, idx->flags.as<int32_t>(), sel_list, sel_count, st,
                           hint));
    if (R.H) B2_CUDA(cudaEventRecord(idx->host->fin1, st));
    // the certificate outcome comes back as ONE counter (the failed queries are compacted on the device)
    int32_t* h_count = reinterpret_cast<int32_t*>(idx->h_flags.p);
    B2_CUDA(cudaMemcpyAsync(h_count, sel_count, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) {
        set_error("search pipeline failed on the device: %s", cudaGetErrorString(se));
        return B2_ECUDA;
    }
    float ms = -1.f;
    if (R.H)
        stream_times_add(idx, R.H->n_chunks);
    else if (cudaEventElapsedTime(&ms, idx->ev0, idx->ev1) == cudaSuccess)
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
// Streamed rows give the results of the same rows in device memory, bit for bit.
int search_core(b2_index* idx, const SearchRows& R, int metric, const void* q_dev, int q_dtype, int64_t nq, int k,
                const int64_t* id_map, int64_t id_offset, float* out_sc, int64_t* out_id, cudaStream_t st, int level) {
    const MatView& X = R.X;
    if (level == 0) {
        idx->last_filter_ms = -1.f;
        if (R.H) {
            HostStore& hs = *idx->host;
            hs.copy_ms = hs.span_ms = hs.filter_ms = hs.finalize_ms = 0.f;
        }
    }
    if (nq <= 0) return B2_OK;
    if (level == 0) g_stats[ST_QUERIES] += nq;
    if (X.n <= 0) {
        fill_pad_kernel<<<132, 256, 0, st>>>(out_sc, out_id, nq * k, metric == B2_METRIC_L2 ? FLT_MAX : -FLT_MAX);
        B2_LAUNCH_CHECK();
        return B2_OK;
    }
    FilterPlan p;
    B2_TRY(plan_rows(idx, R, q_dev, q_dtype, nq, k, false, level, p));
    // streamed rows fold their lists into one of `cap` entries, which finalize has to be able to hold
    const int cap = R.H && p.use_filter ? finalize_capacity(p.kp, k) : 0;
    if (!p.use_filter || (R.H && cap == 0)) {
        // the dense path over every row (streamed rows: read through the mapped pointer)
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
        CandLists L;
        B2_TRY(chunk_lists(idx, R, p, c, metric, cap, &L, st));
        int64_t n_sel = 0;
        B2_TRY(certify(idx, p, c, R, L, metric, id_map, id_offset, out_sc, out_id, nullptr, /*fallback=*/!p.two_level, &n_sel, st));
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
        SearchRows R2 = R;
        R2.X.filt16 = nullptr;
        B2_TRY(search_core(idx, R2, metric, idx->q_sub.p, q_dtype, n_deferred, k, id_map, id_offset, idx->sub_sc.as<float>(),
                           idx->sub_id.as<int64_t>(), st, /*level=*/1));
        scatter_rows_kernel<<<(unsigned)ceil_div(n_deferred * k, 256), 256, 0, st>>>(idx->defer.as<int64_t>(), n_deferred, k, idx->sub_sc.as<float>(),
                                                                                    idx->sub_id.as<int64_t>(), out_sc, out_id);
        B2_LAUNCH_CHECK();
        g_stats[ST_SECOND_LEVEL] += n_deferred;
    }
    return B2_OK;
}

// ---- range search (range.cu) ----------------------------------------------------------------------------------------------
// The filter operand of a device-resident view: float queries on an int8 store use its fp16 copy (exact). An fp32 store filters
// with tf32 on its own rows (its bf16 first-level copy is a knn optimisation; a range search would only admit more candidates).
static MatView range_filter_view(const MatView& X, int q_dtype) {
    MatView v = X;
    if (X.dtype == B2_I8 && q_dtype != B2_I8) {
        v.filt = X.filt_f16;
        v.filt_pitch = X.filt_f16_pitch;
        v.filt_dtype = B2_F16;
    }
    return v;
}

// The range search of R: one pass over a device view, or one pass per streamed chunk, filtered and verified while its slot holds
// it (the copy of the next chunk runs meanwhile), so verification reads device memory only; the last chunk skips the rows its
// predecessor covered. An int8 store with float queries filters the fp16 form of each chunk and verifies against the int8 rows.
static int range_rows(b2_index* idx, RangeWork& W, const SearchRows& R, const void* q_dev, int q_dtype, int64_t nq, float radius,
                      cudaStream_t st) {
    if (!R.H) {
        B2_TRY(range_begin(idx, W, R.X, idx->metric, q_dev, q_dtype, nq, radius, st));
        return range_pass(idx, W, range_filter_view(R.X, q_dtype), R.X.d, 0, 0, st);
    }
    MatView Xc = R.X;
    Xc.n = R.H->chunk_rows;
    B2_TRY(range_begin(idx, W, Xc, idx->metric, q_dev, q_dtype, nq, radius, st));
    if (nq <= 0 || R.H->n <= 0) return B2_OK;
    return stream_chunks(
        idx, *R.H, range_filter_view(Xc, q_dtype), /*convert=*/W.use_filter, st,
        [&](const MatView& X, int64_t pitch, int64_t base, int64_t own_lo) {
            return range_pass(idx, W, X, pitch, base, own_lo, st);  // synchronises: the slot is free afterwards
        },
        [](int64_t, int64_t) { return B2_OK; });
}

}  // namespace b2

namespace b2 {
HostStore::~HostStore() {
    if (copy) {
        cudaStreamSynchronize(copy);
        cudaStreamDestroy(copy);
    }
    for (int s = 0; s < SLOTS; ++s) {
        if (copied[s]) cudaEventDestroy(copied[s]);
        if (freed[s]) cudaEventDestroy(freed[s]);
    }
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
    for (cudaEvent_t e : {span0, span1, fin0, fin1})
        if (e) cudaEventDestroy(e);
}
}  // namespace b2

namespace b2 {
// k-means over an int8 index runs on an fp16 twin of it (same rows, exact in fp16), made on the first k-means call and kept
// with the handle: the existing fp16 k-means path (fp16 TOP1 filter, fp16 accumulate) then serves int8 points unchanged
int kmeans_view(b2_index* idx, b2_index** out) {
    *out = idx;
    if (idx->dtype != B2_I8) return B2_OK;
    if (!idx->f16_twin) {
        DevBuf tmp;
        B2_TRY(tmp.ensure((size_t)std::max<int64_t>(idx->n, 1) * idx->d * 2));
        B2_TRY(launch_convert_pad(idx->store.p, B2_I8, idx->n, idx->d, tmp.p, B2_F16, idx->d, idx->stream));
        B2_CUDA(cudaStreamSynchronize(idx->stream));
        b2_index* t = nullptr;
        B2_TRY(b2_index_create(tmp.p, idx->n, idx->d, B2_F16, idx->metric, idx->device, 1, &t));
        B2_CUDA(cudaStreamSynchronize(t->stream));
        idx->f16_twin = t;
    }
    *out = idx->f16_twin;
    return B2_OK;
}
}  // namespace b2

b2_index::~b2_index() {
    if (f16_twin) b2_index_free(f16_twin);
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

// the checks both create entry points make before any device work
static int check_create_args(const void* x, int64_t n, int32_t d, int32_t dtype, int32_t metric, b2_index** out) {
    if (!out) { set_error("out is NULL"); return B2_EINVAL; }
    *out = nullptr;
    if (n < 0 || d <= 0 || (n > 0 && !x)) { set_error("bad matrix shape n=%lld d=%d", (long long)n, d); return B2_EINVAL; }
    if (!dtype_valid(dtype)) { set_error("dtype must be B2_F32, B2_BF16, B2_F16 or B2_I8"); return B2_EINVAL; }
    if (dtype == B2_I8 && d > I8_MAX_D) { set_error("an int8 index needs d < 2^17 (got %d): its s32 accumulators would overflow", d); return B2_EINVAL; }
    if (dtype == B2_I8 && metric == B2_METRIC_L2 && d > I8_L2_MAX_D) {
        set_error("an int8 L2 index needs d < 2^15 (got %d): 2 <q, x> - |x|^2 would overflow int32", d);
        return B2_EINVAL;
    }
    if (metric != B2_METRIC_IP && metric != B2_METRIC_L2) { set_error("metric must be B2_METRIC_IP or B2_METRIC_L2"); return B2_EINVAL; }
    return B2_OK;
}

static int check_create_device(int32_t device) {
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
    return B2_OK;
}

int b2_index_create(const void* x, int64_t n, int32_t d, int32_t dtype, int32_t metric, int32_t device, int32_t x_on_device,
                    b2_index** out) {
    B2_TRY(check_create_args(x, n, d, dtype, metric, out));
    B2_TRY(check_create_device(device));
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

int b2_index_create_host(const void* x, int64_t n, int32_t d, int32_t dtype, int32_t metric, int32_t device, int64_t ring_bytes,
                         b2_index** out) {
    B2_TRY(check_create_args(x, n, d, dtype, metric, out));
    if (n >= (1LL << 31)) { set_error("a host-resident index holds fewer than 2^31 rows (got %lld): its row ids are int32", (long long)n); return B2_EINVAL; }
    if (ring_bytes < 0) { set_error("ring_bytes < 0"); return B2_EINVAL; }
    {
        int64_t rows = 0;
        int nc = 0;
        B2_TRY(stream_plan(n, d, dtype, (size_t)ring_bytes, &rows, &nc));
    }
    B2_TRY(check_create_device(device));
    DeviceGuard guard(device);
    b2_index* idx = new b2_index();
    idx->device = device;
    idx->n = n;
    idx->d = d;
    idx->dtype = dtype;
    idx->metric = metric;
    idx->host.reset(new HostStore());
    HostStore& hs = *idx->host;
    hs.ring_bytes = ring_bytes ? (size_t)ring_bytes : kDefaultRingBytes;
    auto fail = [&](int rc) { b2_index_free(idx); return rc; };
    bool ok = cudaStreamCreateWithFlags(&idx->stream, cudaStreamNonBlocking) == cudaSuccess &&
              cudaStreamCreateWithFlags(&hs.copy, cudaStreamNonBlocking) == cudaSuccess && cudaEventCreate(&idx->ev0) == cudaSuccess &&
              cudaEventCreate(&idx->ev1) == cudaSuccess;
    for (int s = 0; ok && s < HostStore::SLOTS; ++s)
        ok = cudaEventCreateWithFlags(&hs.copied[s], cudaEventDisableTiming) == cudaSuccess &&
             cudaEventCreateWithFlags(&hs.freed[s], cudaEventDisableTiming) == cudaSuccess;
    for (cudaEvent_t* e : {&hs.span0, &hs.span1, &hs.fin0, &hs.fin1}) ok = ok && cudaEventCreate(e) == cudaSuccess;
    if (!ok) {
        set_error("stream/event creation failed: %s", cudaGetErrorString(cudaGetLastError()));
        return fail(B2_ECUDA);
    }
    const size_t bytes = (size_t)n * d * esize(dtype);
    int rc = hs.main.rows.ensure(std::max<size_t>(bytes, 1));
    if (rc != B2_OK) return fail(rc);
    const char* src = reinterpret_cast<const char*>(x);
    char* dst = reinterpret_cast<char*>(hs.main.rows.p);
    for_each_chunk((int64_t)ceil_div((int64_t)bytes, 1 << 12), [&](int64_t lo, int64_t hi) {  // threaded copy, 4 KB pages
        const size_t b0 = (size_t)lo << 12, b1 = std::min(bytes, (size_t)hi << 12);
        memcpy(dst + b0, src + b0, b1 - b0);
    });
    rc = host_rows_init(hs.main, n, d, dtype, hs.ring_bytes, idx->stream);
    if (rc != B2_OK) return fail(rc);
    idx->view = host_view(hs.main);
    *out = idx;
    return B2_OK;
}

int32_t b2_index_resident(const b2_index* idx) { return idx ? (idx->host ? 1 : 0) : -1; }

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
const void* b2_index_data_dev(const b2_index* idx) { return idx && !idx->host ? idx->store.p : nullptr; }
float b2_last_filter_ms(const b2_index* idx) { return idx ? idx->last_filter_ms : -1.f; }

static int check_search_args(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k) {
    if (!idx) { set_error("Index not loaded"); return B2_EINVAL; }
    if (nq < 0 || (nq > 0 && !q)) { set_error("bad query batch"); return B2_EINVAL; }
    if (!dtype_valid(q_dtype)) { set_error("q_dtype must be B2_F32, B2_BF16, B2_F16 or B2_I8"); return B2_EINVAL; }
    if (k <= 0) { set_error("k must be positive (got %d)", k); return B2_EINVAL; }
    if (k > dense_max_k()) { set_error("k=%d is not supported (max %d)", k, dense_max_k()); return B2_ERANGE; }
    return B2_OK;
}

// The inputs of a call on host buffers, staged on the device: the queries in idx->q_in (then adapted, see adapt_queries) and,
// unless they list every row in order, the ids in idx->ids_dev (*ids_dev = null: the whole index).
static int stage_host_call(b2_index* idx, const void* q, int64_t nq, int32_t& q_dtype, const int64_t* ids, int64_t n_ids,
                           cudaStream_t st, const void** q_dev, const int64_t** ids_dev) {
    const size_t qbytes = (size_t)nq * idx->d * esize(q_dtype);
    B2_TRY(idx->q_in.ensure(qbytes));
    B2_CUDA(cudaMemcpyAsync(idx->q_in.p, q, qbytes, cudaMemcpyHostToDevice, st));
    *q_dev = idx->q_in.p;
    B2_TRY(adapt_queries(idx, *q_dev, q_dtype, nq, st));
    *ids_dev = nullptr;
    if (!ids) return B2_OK;
    if (n_ids < 0) { set_error("n_ids < 0"); return B2_EINVAL; }
    bool identity = n_ids == idx->n;
    for (int64_t i = 0; identity && i < n_ids; ++i) identity = ids[i] == i;
    if (identity) return B2_OK;
    B2_TRY(idx->ids_dev.ensure((size_t)std::max<int64_t>(n_ids, 1) * sizeof(int64_t)));
    B2_CUDA(cudaMemcpyAsync(idx->ids_dev.p, ids, (size_t)n_ids * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    *ids_dev = idx->ids_dev.as<int64_t>();
    return B2_OK;
}

// the top-k results of a call on host buffers (idx->out_sc / out_id, sized for nq x k) copied back, waited for
static int download_topk(b2_index* idx, int64_t nq, int k, float* out_scores, int64_t* out_idx, cudaStream_t st) {
    B2_CUDA(cudaMemcpyAsync(out_scores, idx->out_sc.p, (size_t)nq * k * sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(out_idx, idx->out_id.p, (size_t)nq * k * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("search failed on the device: %s", cudaGetErrorString(e)); return B2_ECUDA; }
    return B2_OK;
}

int b2_index_search_dev(b2_index* idx, const void* q_dev, int64_t nq, int32_t q_dtype, int32_t k, const int64_t* ids_dev,
                        int64_t n_ids, int64_t id_offset, float* out_scores_dev, int64_t* out_idx_dev, void* stream) {
    B2_TRY(check_search_args(idx, q_dev, nq, q_dtype, k));
    if (nq == 0) return B2_OK;
    if (!out_scores_dev || !out_idx_dev) { set_error("output buffers are NULL"); return B2_EINVAL; }
    DeviceGuard guard(idx->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(adapt_queries(idx, q_dev, q_dtype, nq, st));
    if (ids_dev && n_ids < 0) { set_error("n_ids < 0"); return B2_EINVAL; }
    SearchRows R;
    B2_TRY(select_rows(idx, nullptr, ids_dev, n_ids, q_dtype, st, &R));
    B2_TRY(search_core(idx, R, idx->metric, q_dev, q_dtype, nq, k, ids_dev, ids_dev ? 0 : id_offset, out_scores_dev, out_idx_dev, st));
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
    B2_TRY(idx->out_sc.ensure((size_t)nq * k * sizeof(float)));
    B2_TRY(idx->out_id.ensure((size_t)nq * k * sizeof(int64_t)));
    const void* q_dev = nullptr;
    const int64_t* ids_dev = nullptr;
    B2_TRY(stage_host_call(idx, q, nq, q_dtype, ids, n_ids, st, &q_dev, &ids_dev));
    SearchRows R;
    B2_TRY(select_rows(idx, ids, ids_dev, n_ids, q_dtype, st, &R));
    B2_TRY(search_core(idx, R, idx->metric, q_dev, q_dtype, nq, k, ids_dev, 0, idx->out_sc.as<float>(), idx->out_id.as<int64_t>(), st));
    return download_topk(idx, nq, k, out_scores, out_idx, st);
}

// ---- masked search: the rows a bitmap selects, searched in place (no gathered copy of the subset) ----------------------------
static int check_masked_args(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, const uint32_t* mask) {
    if (!idx && b2_device_count() == 0) { set_error("no CUDA device: libb2lotus has no CPU fallback"); return B2_ENODEV; }
    B2_TRY(check_search_args(idx, q, nq, q_dtype, k));
    if (!mask && idx->n > 0) { set_error("mask is NULL"); return B2_EINVAL; }
    return B2_OK;
}

// mask_dev: ceil(n / 32) words on the index's device
static int masked_search(b2_index* idx, const void* q_dev, int q_dtype, int64_t nq, int k, const uint32_t* mask_dev, int64_t id_offset,
                         float* out_sc, int64_t* out_id, cudaStream_t st) {
    SearchRows R;
    B2_TRY(select_rows(idx, nullptr, nullptr, 0, q_dtype, st, &R));
    R.X.mask = mask_dev;
    return search_core(idx, R, idx->metric, q_dev, q_dtype, nq, k, nullptr, id_offset, out_sc, out_id, st);
}

static int upload_mask(b2_index* idx, const uint32_t* mask, cudaStream_t st) {
    const size_t bytes = (size_t)ceil_div(idx->n, 32) * sizeof(uint32_t);
    B2_TRY(idx->mask_dev.ensure(std::max<size_t>(bytes, 4)));
    if (bytes) B2_CUDA(cudaMemcpyAsync(idx->mask_dev.p, mask, bytes, cudaMemcpyHostToDevice, st));
    return B2_OK;
}

int b2_index_search_masked_dev(b2_index* idx, const void* q_dev, int64_t nq, int32_t q_dtype, int32_t k, const uint32_t* mask_dev,
                               int64_t id_offset, float* out_scores_dev, int64_t* out_idx_dev, void* stream) {
    B2_TRY(check_masked_args(idx, q_dev, nq, q_dtype, k, mask_dev));
    if (nq == 0) return B2_OK;
    if (!out_scores_dev || !out_idx_dev) { set_error("output buffers are NULL"); return B2_EINVAL; }
    DeviceGuard guard(idx->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(adapt_queries(idx, q_dev, q_dtype, nq, st));
    B2_TRY(masked_search(idx, q_dev, q_dtype, nq, k, mask_dev, id_offset, out_scores_dev, out_idx_dev, st));
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
}

int b2_index_search_masked(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, const uint32_t* mask,
                           float* out_scores, int64_t* out_idx) {
    B2_TRY(check_masked_args(idx, q, nq, q_dtype, k, mask));
    if (nq == 0) return B2_OK;
    if (!out_scores || !out_idx) { set_error("output buffers are NULL"); return B2_EINVAL; }
    DeviceGuard guard(idx->device);
    cudaStream_t st = idx->stream;
    B2_TRY(idx->out_sc.ensure((size_t)nq * k * sizeof(float)));
    B2_TRY(idx->out_id.ensure((size_t)nq * k * sizeof(int64_t)));
    const void* q_dev = nullptr;
    const int64_t* no_ids = nullptr;
    B2_TRY(stage_host_call(idx, q, nq, q_dtype, nullptr, 0, st, &q_dev, &no_ids));
    B2_TRY(upload_mask(idx, mask, st));
    B2_TRY(masked_search(idx, q_dev, q_dtype, nq, k, idx->mask_dev.as<uint32_t>(), 0, idx->out_sc.as<float>(),
                         idx->out_id.as<int64_t>(), st));
    return download_topk(idx, nq, k, out_scores, out_idx, st);
}

// The range search of the ids subset (ids, n_ids), or of the rows a bitmap selects (mask: ceil(n / 32) host words), or of the
// whole index. A masked search reads the rows in place; its candidates and dense rows are selected rows only, reported by
// their positions in the index.
static int range_search(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, float radius, const int64_t* ids, int64_t n_ids,
                        const uint32_t* mask, int64_t* lims, float* out_d, int64_t* out_i, int64_t cap, int64_t* n_results) {
    if (!idx) { set_error("Index not loaded"); return B2_EINVAL; }
    if (nq < 0 || (nq > 0 && !q)) { set_error("bad query batch"); return B2_EINVAL; }
    if (!dtype_valid(q_dtype)) { set_error("q_dtype must be B2_F32, B2_BF16, B2_F16 or B2_I8"); return B2_EINVAL; }
    if (!lims || !n_results) { set_error("lims / n_results are NULL"); return B2_EINVAL; }
    if (cap < 0 || (cap > 0 && (!out_d || !out_i))) { set_error("bad output buffers (cap=%lld)", (long long)cap); return B2_EINVAL; }
    if (ids && n_ids < 0) { set_error("n_ids < 0"); return B2_EINVAL; }
    if (nq > 0x7fffff00LL) { set_error("too many queries for one range search (nq=%lld)", (long long)nq); return B2_ERANGE; }
    *n_results = 0;
    if (nq == 0 || radius != radius) {  // a NaN radius: every comparison is false
        for (int64_t i = 0; i <= nq; ++i) lims[i] = 0;
        return B2_OK;
    }
    DeviceGuard guard(idx->device);
    cudaStream_t st = idx->stream;
    if (!idx->range) idx->range.reset(new RangeWork());
    RangeWork& W = *idx->range;
    idx->last_filter_ms = -1.f;
    const void* q_dev = nullptr;
    const int64_t* ids_dev = nullptr;
    B2_TRY(stage_host_call(idx, q, nq, q_dtype, ids, n_ids, st, &q_dev, &ids_dev));
    SearchRows R;
    B2_TRY(select_rows(idx, ids, ids_dev, n_ids, q_dtype, st, &R));
    if (mask) {
        B2_TRY(upload_mask(idx, mask, st));
        R.X.mask = idx->mask_dev.as<uint32_t>();
    }
    B2_TRY(range_rows(idx, W, R, q_dev, q_dtype, nq, radius, st));
    B2_TRY(range_finish(W, ids_dev, 0, st));
    B2_CUDA(cudaMemcpyAsync(lims, W.lims.p, (size_t)(nq + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("range search failed on the device: %s", cudaGetErrorString(e)); return B2_ECUDA; }
    if (W.use_filter && W.n_dense < nq) idx->last_filter_ms = W.filter_ms;
    const int64_t total = lims[nq];
    *n_results = total;
    if (total > cap) {
        set_error("range search found %lld results, more than cap=%lld", (long long)total, (long long)cap);
        return B2_ERANGE;
    }
    if (total > 0) {
        B2_CUDA(cudaMemcpyAsync(out_d, W.out_d.p, (size_t)total * sizeof(float), cudaMemcpyDeviceToHost, st));
        B2_CUDA(cudaMemcpyAsync(out_i, W.out_i.p, (size_t)total * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("range search failed on the device: %s", cudaGetErrorString(e)); return B2_ECUDA; }
    }
    return B2_OK;
}

int b2_index_range_search(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, float radius, const int64_t* ids, int64_t n_ids,
                          int64_t* lims, float* out_d, int64_t* out_i, int64_t cap, int64_t* n_results) {
    return range_search(idx, q, nq, q_dtype, radius, ids, n_ids, nullptr, lims, out_d, out_i, cap, n_results);
}

int b2_index_range_search_masked(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, float radius, const uint32_t* mask,
                                 int64_t* lims, float* out_d, int64_t* out_i, int64_t cap, int64_t* n_results) {
    if (!idx && b2_device_count() == 0) { set_error("no CUDA device: libb2lotus has no CPU fallback"); return B2_ENODEV; }
    if (idx && !mask && idx->n > 0) { set_error("mask is NULL"); return B2_EINVAL; }
    return range_search(idx, q, nq, q_dtype, radius, nullptr, 0, mask, lims, out_d, out_i, cap, n_results);
}

int b2_debug_range_stats(const b2_index* idx, int64_t* out4) {
    if (!idx || !out4) { set_error("NULL argument"); return B2_EINVAL; }
    const RangeWork* W = idx->range.get();
    out4[0] = W ? W->cand_peak : 0;
    out4[1] = W ? W->n_hits : 0;
    out4[2] = W ? W->n_dense : 0;
    out4[3] = W ? (int64_t)W->use_filter : 0;
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
    B2_TRY(refuse_host_resident(idx, "b2_index_search_packed_dev"));
    if (idx->n > 0xfffffffeLL) { set_error("packed lists hold 32-bit local ids"); return B2_ERANGE; }
    DeviceGuard guard(idx->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(idx->out_sc.ensure((size_t)nq * k * sizeof(float)));
    B2_TRY(idx->out_id.ensure((size_t)nq * k * sizeof(int64_t)));
    B2_TRY(adapt_queries(idx, q_dev, q_dtype, nq, st));
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
    B2_TRY(refuse_host_resident(idx, "b2_index_search_stage1_dev"));
    DeviceGuard guard(idx->device);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    B2_TRY(adapt_queries(idx, q_dev, q_dtype, nq, st));
    b2_index::Staged& sg = idx->staged;
    sg = b2_index::Staged();
    sg.active = true;
    const MatView& X = idx->view;
    FilterPlan& p = sg.plan;
    B2_TRY(plan_filter(X, q_dev, q_dtype, nq, k, false, idx->device, p));
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
                                    idx->q_norm2.as<float>(), X.max_norm, p.rel_eps, p.abs_eps, p.q_norm_limit, idx->metric, lower_dev, st));
    g_stats[ST_QUERIES] += nq;
    return B2_OK;
}

int b2_index_search_stage2_packed_dev(b2_index* idx, const float* hint_dev, uint64_t* out_packed_dev, void* stream) {
    if (!idx) { set_error("Index not loaded"); return B2_EINVAL; }
    B2_TRY(refuse_host_resident(idx, "b2_index_search_stage2_packed_dev"));
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
    const FilterChunk& c = p.chunks[0];
    B2_TRY(certify(idx, p, c, p.X, filter_lists(idx, p, c), idx->metric, nullptr, 0, idx->out_sc.as<float>(), idx->out_id.as<int64_t>(),
                   hint_dev, /*fallback=*/true, &n_sel, st));
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
    if (idx->host && !out_on_device) {  // host rows to host memory: threaded copies, no device work
        for (int64_t i = 0; i < m; ++i) {
            if (ids[i] < 0 || ids[i] >= idx->n) { set_error("ids contains a position outside [0, %lld)", (long long)idx->n); return B2_ERANGE; }
        }
        const char* src = reinterpret_cast<const char*>(idx->host->main.rows.p);
        for_each_chunk(m, [&](int64_t lo, int64_t hi) {
            for (int64_t i = lo; i < hi; ++i) memcpy(reinterpret_cast<char*>(out) + (size_t)i * row_bytes, src + (size_t)ids[i] * row_bytes, row_bytes);
        });
        return B2_OK;
    }
    const int64_t* ids_dev = ids;
    void* out_dev = out;
    if (!out_on_device) {
        B2_TRY(idx->ids_dev.ensure((size_t)m * sizeof(int64_t)));
        B2_CUDA(cudaMemcpyAsync(idx->ids_dev.p, ids, (size_t)m * sizeof(int64_t), cudaMemcpyHostToDevice, st));
        ids_dev = idx->ids_dev.as<int64_t>();
        B2_TRY(idx->sub_store.ensure((size_t)m * row_bytes));
        out_dev = idx->sub_store.p;
    }
    B2_TRY(gather_rows_checked(idx->view.store, idx->dtype, idx->d, ids_dev, m, idx->n, out_dev, idx->scalar, st));
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
// first query chunk when the batch takes several) — no device work: the worker count is modelled as every SM in use, and
// *two_cta receives the cluster size. Lets the CPU test-suite check that every (query unit, corpus tile) pair is covered
// exactly once for the shapes the GPU tests do not reach.
int b2_debug_filter_plan(int64_t nq, int64_t n, int32_t k, int32_t num_sms, int32_t* kp, int32_t* n_splits, int32_t* units_whole,
                         int32_t* two_cta) {
    if (nq <= 0 || n <= 0 || k <= 0 || num_sms <= 0 || !kp || !n_splits || !units_whole || !two_cta) { set_error("bad arguments"); return B2_EINVAL; }
    MatView X;  // a bf16 view of n rows: one-level search
    X.n = n;
    X.d = 8;
    X.dtype = X.filt_dtype = B2_BF16;
    FilterPlan p;
    B2_TRY(plan_filter(X, nullptr, B2_BF16, nq, k, false, -1, p, num_sms));
    const FilterChunk c = p.use_filter ? p.chunks[0] : FilterChunk();
    *kp = p.use_filter ? p.kp : 0;
    *n_splits = c.n_splits;
    *units_whole = c.units_whole;
    *two_cta = c.cluster;
    return B2_OK;
}

// The raw candidate lists of one filter run on host queries, planned and launched exactly as search_core (level 0 / 1) or the
// k-means assignment (top1) does it, so the tests can check the kernel's contract list by list instead of through finalize.
// mask (host, nullable): the row bitmap of a masked search.
static int debug_filter_lists(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, int32_t top1, int32_t level,
                              const uint32_t* mask, int32_t* plan, float* rel_eps, float* cand_score, int32_t* cand_id,
                              float* cand_thr) {
    B2_TRY(check_search_args(idx, q, nq, q_dtype, k));
    if (nq == 0 || !plan || !rel_eps || (level != 0 && level != 1)) { set_error("bad arguments"); return B2_EINVAL; }
    const bool lists = cand_score && cand_id && cand_thr;
    DeviceGuard guard(idx->device);
    cudaStream_t st = idx->stream;
    const uint32_t* mask_dev = nullptr;
    if (mask) {
        B2_TRY(upload_mask(idx, mask, st));
        mask_dev = idx->mask_dev.as<uint32_t>();
    }
    if (idx->host && top1) { set_error("the k-means assignment is not available on a host-resident index"); return B2_EINVAL; }
    const void* q_dev = nullptr;
    if (lists) {
        const int64_t* no_ids = nullptr;
        B2_TRY(stage_host_call(idx, q, nq, q_dtype, nullptr, 0, st, &q_dev, &no_ids));
    } else if (q_dtype != B2_I8 && !idx->host) {
        B2_TRY(ensure_f16_copy(idx->view, idx->filt_f16, st));
    }
    SearchRows R;
    B2_TRY(select_rows(idx, nullptr, nullptr, 0, q_dtype, st, &R));
    R.X.mask = mask_dev;
    if (level == 1 || top1) R.X.filt16 = nullptr;  // the second level drops the bf16 copy; the k-means centroid view has none
    FilterPlan p;
    B2_TRY(plan_rows(idx, R, q_dev, q_dtype, nq, k, top1 != 0, level, p));
    const int cap = R.H && p.use_filter ? finalize_capacity(p.kp, k) : 0;
    const FilterChunk c = p.use_filter ? p.chunks[0] : FilterChunk();
    // streamed rows: the folded lists after the last corpus chunk, the one list of `cap` entries finalize reads, reported as one
    // split of two halves of cap / 2 (kp = cap) with its bound in both thr entries
    const int kp = R.H ? cap : p.use_filter ? p.kp : 0;  // 0: no lists, the dense path answers
    plan[0] = kp ? 1 : 0;
    plan[1] = kp;
    plan[2] = R.H ? 1 : c.n_splits;
    plan[3] = R.H ? 0 : c.units_whole;
    plan[4] = c.cluster;
    plan[5] = p.two_level ? 1 : 0;
    plan[6] = p.X.filt_dtype;
    plan[7] = (int32_t)p.chunks.size();
    *rel_eps = p.rel_eps;
    if (p.chunks.size() > 1) { set_error("%lld queries take %zu query chunks; one is supported", (long long)nq, p.chunks.size()); return B2_ERANGE; }
    if (!lists || !kp) return B2_OK;
    CandLists L;
    B2_TRY(chunk_lists(idx, R, p, c, idx->metric, cap, &L, st));
    const size_t entries = (size_t)nq * L.n_lists * L.list_len;
    B2_CUDA(cudaMemcpyAsync(cand_score, L.score, entries * sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(cand_id, L.id, entries * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (L.n_lists == 1) {
        for (int h = 0; h < 2; ++h)
            B2_CUDA(cudaMemcpy2DAsync(cand_thr + h, 2 * sizeof(float), L.thr, sizeof(float), sizeof(float), (size_t)nq, cudaMemcpyDeviceToHost, st));
    } else {
        B2_CUDA(cudaMemcpyAsync(cand_thr, L.thr, (size_t)nq * L.n_lists * sizeof(float), cudaMemcpyDeviceToHost, st));
    }
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("filter failed on the device: %s", cudaGetErrorString(e)); return B2_ECUDA; }
    return B2_OK;
}

int b2_debug_filter_lists(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, int32_t top1, int32_t level,
                          int32_t* plan, float* rel_eps, float* cand_score, int32_t* cand_id, float* cand_thr) {
    return debug_filter_lists(idx, q, nq, q_dtype, k, top1, level, nullptr, plan, rel_eps, cand_score, cand_id, cand_thr);
}

int b2_debug_filter_lists_masked(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, int32_t level,
                                 const uint32_t* mask, int32_t* plan, float* rel_eps, float* cand_score, int32_t* cand_id,
                                 float* cand_thr) {
    if (idx && !mask && idx->n > 0) { set_error("mask is NULL"); return B2_EINVAL; }
    return debug_filter_lists(idx, q, nq, q_dtype, k, 0, level, mask, plan, rel_eps, cand_score, cand_id, cand_thr);
}

// The chunking of a host-resident index (no device work): rows per chunk, chunks, ring slots.
int b2_debug_stream_plan(int64_t n, int32_t d, int32_t dtype, int64_t ring_bytes, int64_t* chunk_rows, int64_t* n_chunks, int32_t* slots) {
    if (n < 0 || d <= 0 || !dtype_valid(dtype) || ring_bytes < 0 || !chunk_rows || !n_chunks || !slots) { set_error("bad arguments"); return B2_EINVAL; }
    int nc = 0;
    B2_TRY(stream_plan(n, d, dtype, (size_t)ring_bytes, chunk_rows, &nc));
    *n_chunks = nc;
    *slots = HostStore::SLOTS;
    return B2_OK;
}

// Event times of the last search of a host-resident index: [0] copies (copy stream), [1] the span from the first copy to the
// last fold on the search stream, [2] the filter launches, [3] finalize. Sums over query chunks and levels.
int b2_debug_stream_times(const b2_index* idx, float* out4) {
    if (!idx || !out4) { set_error("bad arguments"); return B2_EINVAL; }
    if (!idx->host) { set_error("not a host-resident index"); return B2_EINVAL; }
    const HostStore& hs = *idx->host;
    out4[0] = hs.copy_ms;
    out4[1] = hs.span_ms;
    out4[2] = hs.filter_ms;
    out4[3] = hs.finalize_ms;
    return B2_OK;
}

int b2_debug_filter_eps(int32_t store_dtype, int32_t filt_dtype, int32_t q_dtype, int32_t d, float* rel_eps, float* abs_eps) {
    if (!dtype_valid(store_dtype) || !dtype_valid(filt_dtype) || !dtype_valid(q_dtype) || d <= 0 || !rel_eps || !abs_eps) {
        set_error("bad arguments");
        return B2_EINVAL;
    }
    *rel_eps = filter_rel_eps(store_dtype, filt_dtype, q_dtype, d);
    *abs_eps = filter_abs_eps(store_dtype, filt_dtype, q_dtype, d);
    return B2_OK;
}

int b2_stats(int64_t* out, int32_t cap) {
    int n = cap < 8 ? cap : 8;
    for (int i = 0; i < n; ++i) out[i] = g_stats[i];
    return n;
}
void b2_stats_reset(void) { memset(g_stats, 0, sizeof(g_stats)); }

}  // extern "C"
