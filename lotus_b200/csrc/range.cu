// range.cu — range search (b2_index_range_search): every row whose canonical score is above the radius (IP) or whose
// canonical squared distance is below it (L2), for each query.
//
//   range_thr_kernel    : per query (one warp), the candidate threshold in filter-score space (DESIGN.md §2): radius minus the
//                         filter's error margin, so that no row whose canonical result passes can score at or below it. A
//                         query whose margin is not finite gets NaN (no filter candidates) and is listed for the dense path.
//   range filter        : knn_filter_sm90.cu (range_filter_kernel): (query, row) pairs whose filter score beats the threshold.
//                         A masked range search (b2_index_range_search_masked) runs range_masked_filter_kernel, which emits
//                         selected rows only.
//   range_verify_kernel : one warp per (query, row) pair: the canonical score (canonical.cuh, the arithmetic finalize uses)
//                         and the strict comparison; a passing pair becomes a hit (query, position, score). The dense path is
//                         the same kernel over every row of a query (every selected row, in a masked search).
//   assembly            : one radix sort of the hits by (query << 32 | position), lims by binary search, unpack to D / I.
#include <cub/cub.cuh>

#include "canonical.cuh"
#include "index.cuh"

namespace b2 {

namespace {

constexpr int SMEM_LIMIT_BYTES = 232448;  // 227 KB of shared memory per block

// thr[q] and the dense list (sel[0] = count, sel[1..] = queries) of a range search
__global__ void range_thr_kernel(const void* q, int q_dtype, int64_t nq, int d, int metric, float radius, float rel_eps, float abs_eps,
                                 float max_norm, float q_norm_limit, int use_filter, float* thr, int32_t* sel) {
    const int lane = threadIdx.x & 31;
    const int64_t qi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (qi >= nq) return;
    // canonical squared norm of the query, as finalize forms it
    double acc = 0.0;
    const int d4 = ((d + 3) >> 2) << 2;
    for (int g = lane; g < (d4 >> 2); g += 32) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int i = 4 * g + e;
            const double v = i < d ? (double)elem_f32<true>(q, q_dtype, (size_t)qi * d + i) : 0.0;
            acc = fma(v, v, acc);
        }
    }
    const double qn2 = butterfly_sum(acc);
    if (lane != 0) return;
    const double qn = sqrt(qn2), mx = (double)max_norm, r = (double)radius;
    double t;
    if (metric == B2_METRIC_L2) {
        // dist < r  <=>  s = 2 <q, x> - |x|^2 > |q|^2 - r; eps_s is finalize's margin of a filter score in s-space
        const double eps_s = 2.0 * (double)rel_eps * qn * mx + 2.4e-7 * (mx * mx + 2.0 * qn * mx) + 1e-30 + 2.0 * (double)abs_eps * (qn + mx);
        t = qn2 - r - eps_s - 4.8e-7 * (fabs(r) + qn2);
    } else {
        const double eps = (double)rel_eps * qn * mx + 1e-30 + (double)abs_eps * (qn + mx);
        t = r - eps - 2.4e-7 * fabs(r);
    }
    const bool limited = q_norm_limit < INFINITY && !(qn2 < (double)q_norm_limit * (double)q_norm_limit);
    const float tf = __double2float_rd(t);
    if (!use_filter || limited || !isfinite(tf)) {
        thr[qi] = __int_as_float(0x7fc00000);  // NaN: the filter passes nothing for this query
        sel[1 + atomicAdd(sel, 1)] = (int32_t)qi;
    } else {
        thr[qi] = tf;
    }
}

struct VerifyParams {
    const void* store;  // rows [0, n) of this pass, row pitch `pitch` elements of dtype
    int dtype, d;
    int64_t n, pitch;
    const void* q;
    int q_dtype, metric;
    float radius;
    const int2* cand;          // candidate mode: (query, row) pairs
    int64_t n_cand;
    const int32_t* dense_sel;  // dense mode (cand == nullptr): every row of [own_lo, n) for each of the n_dense queries
    int64_t n_dense;
    int64_t own_lo;  // rows below own_lo belong to an earlier pass (the re-streamed tail of a host-resident chunk)
    const uint32_t* mask;  // masked range search: bit j is row j of this pass; the dense mode skips the cleared rows (null: none)
    int64_t base;    // position reported for row 0
    int32_t* hit_q;
    int32_t* hit_pos;
    float* hit_sc;
    unsigned long long* hit_count;
    unsigned long long hit_cap;
};

// One warp per pair; each warp takes a contiguous run of pairs (the filter appends a warp's candidates together, the dense
// mode walks the rows of one query), so the query staged in shared memory is reloaded only when it changes.
__global__ void range_verify_kernel(const VerifyParams p) {
    extern __shared__ __align__(16) float vq[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int d4 = ((p.d + 3) >> 2) << 2;
    float* q_s = vq + (size_t)warp * d4;
    const int64_t rows = p.n - p.own_lo;
    const int64_t total = p.cand ? p.n_cand : p.n_dense * rows;
    const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int64_t w = blockIdx.x * (int64_t)(blockDim.x >> 5) + warp;
    const int64_t per = (total + n_warps - 1) / n_warps;
    const int64_t t0 = w * per, t1 = min(total, t0 + per);
    const bool vec = (p.d % 4) == 0 && (p.pitch % 4) == 0;
    const size_t esz = esize(p.dtype);
    const bool is_l2 = p.metric == B2_METRIC_L2;
    int64_t cur = -1;
    for (int64_t t = t0; t < t1; ++t) {
        int64_t qi, j;
        if (p.cand) {
            const int2 c = p.cand[t];
            qi = c.x;
            j = c.y;
        } else {
            qi = p.dense_sel[t / rows];
            j = p.own_lo + t % rows;
            if (p.mask && !((p.mask[j >> 5] >> (j & 31)) & 1u)) continue;  // (warp-uniform)
        }
        if (j < p.own_lo) continue;  // (warp-uniform)
        if (qi != cur) {
            __syncwarp();
            for (int i = lane; i < d4; i += 32) q_s[i] = i < p.d ? elem_f32<true>(p.q, p.q_dtype, (size_t)qi * p.d + i) : 0.f;
            __syncwarp();
            cur = qi;
        }
        const char* row = reinterpret_cast<const char*>(p.store) + (size_t)j * p.pitch * esz;
        const double part = is_l2 ? canonical_partial<true, true>(q_s, row, p.dtype, p.d, vec, lane)
                                   : canonical_partial<false, true>(q_s, row, p.dtype, p.d, vec, lane);
        const float s = (float)butterfly_sum(part);
        if (lane == 0 && (is_l2 ? s < p.radius : s > p.radius)) {
            const unsigned long long h = atomicAdd(p.hit_count, 1ull);
            if (h < p.hit_cap) {
                p.hit_q[h] = (int32_t)qi;
                p.hit_pos[h] = (int32_t)(p.base + j);
                p.hit_sc[h] = s;
            }
        }
    }
}

__global__ void range_keys_kernel(const int32_t* hit_q, const int32_t* hit_pos, int64_t n, uint64_t* keys) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x)
        keys[t] = ((uint64_t)(uint32_t)hit_q[t] << 32) | (uint32_t)hit_pos[t];
}

// lims[q] = first hit of query q in the sorted keys (q = nq: the total)
__global__ void range_lims_kernel(const uint64_t* keys, int64_t n, int64_t nq, int64_t* lims) {
    const int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (q > nq) return;
    const uint64_t want = (uint64_t)q << 32;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < want) lo = mid + 1;
        else hi = mid;
    }
    lims[q] = lo;
}

__global__ void range_unpack_kernel(const uint64_t* keys, const float* sc, int64_t n, const int64_t* id_map, int64_t id_offset,
                                    float* out_d, int64_t* out_i) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pos = (int64_t)(uint32_t)(keys[t] & 0xffffffffu);
        out_i[t] = id_map ? id_map[pos] : pos + id_offset;
        out_d[t] = sc[t];
    }
}

// b grows to hold `want` bytes, keeping its first `keep` bytes
int grow_keep(DevBuf& b, size_t keep, size_t want, cudaStream_t st) {
    if (want <= b.cap) return B2_OK;
    DevBuf nb;
    B2_TRY(nb.ensure(std::max(want, 2 * b.cap)));
    if (keep) B2_CUDA(cudaMemcpyAsync(nb.p, b.p, keep, cudaMemcpyDeviceToDevice, st));
    std::swap(b.p, nb.p);
    std::swap(b.cap, nb.cap);
    return B2_OK;
}

int read_count(const unsigned long long* dev, RangeWork& W, cudaStream_t st, unsigned long long* out) {
    B2_CUDA(cudaMemcpyAsync(W.h_count.p, dev, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
        set_error("range search failed on the device: %s", cudaGetErrorString(e));
        return B2_ECUDA;
    }
    *out = *reinterpret_cast<unsigned long long*>(W.h_count.p);
    return B2_OK;
}

// canonical verification of `n_pairs` pairs (candidates, or the dense rows of the dense queries) appended to the hits; a hit
// buffer that overflows grows to the exact size and the same pairs are verified again
int verify_pairs(RangeWork& W, VerifyParams vp, int64_t n_pairs, cudaStream_t st) {
    if (n_pairs <= 0) return B2_OK;
    const int d4 = (int)round_up(vp.d, 4);
    const int warps = (int)std::max<int64_t>(1, std::min<int64_t>(8, (96 << 10) / ((int64_t)d4 * 4)));
    const size_t smem = (size_t)warps * d4 * 4;
    if (smem > (size_t)SMEM_LIMIT_BYTES) {
        set_error("range search supports d <= %d (got %d)", SMEM_LIMIT_BYTES / 4 - 4, vp.d);
        return B2_EINVAL;
    }
    B2_CUDA(cudaFuncSetAttribute(range_verify_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>(ceil_div(n_pairs, warps), 132 * 32));
    const int64_t before = W.n_hits;
    for (int attempt = 0; attempt < 2; ++attempt) {
        vp.hit_q = W.hit_q.as<int32_t>();
        vp.hit_pos = W.hit_pos.as<int32_t>();
        vp.hit_sc = W.hit_sc.as<float>();
        vp.hit_count = W.counts.as<unsigned long long>() + 1;
        vp.hit_cap = std::min(W.hit_q.cap / sizeof(int32_t), std::min(W.hit_pos.cap / sizeof(int32_t), W.hit_sc.cap / sizeof(float)));
        range_verify_kernel<<<(unsigned)blocks, warps * 32, smem, st>>>(vp);
        B2_LAUNCH_CHECK();
        unsigned long long total = 0;
        B2_TRY(read_count(vp.hit_count, W, st, &total));
        if (total <= vp.hit_cap) {
            W.n_hits = (int64_t)total;
            g_stats[ST_RESCORED] += n_pairs;
            return B2_OK;
        }
        const size_t want = (size_t)total + (size_t)(total >> 3);
        B2_TRY(grow_keep(W.hit_q, (size_t)before * 4, want * 4, st));
        B2_TRY(grow_keep(W.hit_pos, (size_t)before * 4, want * 4, st));
        B2_TRY(grow_keep(W.hit_sc, (size_t)before * 4, want * 4, st));
        const unsigned long long reset = (unsigned long long)before;
        B2_CUDA(cudaMemcpyAsync(vp.hit_count, &reset, sizeof(reset), cudaMemcpyHostToDevice, st));
    }
    set_error("internal: range search hit buffer overflowed twice");
    return B2_ERANGE;
}

}  // namespace

int range_begin(b2_index* idx, RangeWork& W, const MatView& X, int metric, const void* q_dev, int q_dtype, int64_t nq, float radius,
                cudaStream_t st) {
    W.q = q_dev;
    W.q_dtype = q_dtype;
    W.nq = nq;
    W.metric = metric;
    W.radius = radius;
    W.n_hits = 0;
    W.n_dense = 0;
    W.cand_peak = 0;
    W.filter_ms = 0.f;
    W.filt_dtype = X.dtype == B2_I8 && q_dtype != B2_I8 ? B2_F16 : X.dtype;  // float queries on an int8 store: its fp16 copy
    W.use_filter = X.n >= 512 && nq > 0;
    W.rel_eps = filter_rel_eps(X.dtype, W.filt_dtype, q_dtype, X.d);
    W.abs_eps = filter_abs_eps(X.dtype, W.filt_dtype, q_dtype, X.d);
    W.q_norm_limit = W.filt_dtype == B2_F16 && q_dtype != B2_F16 ? 65504.f : INFINITY;  // as plan_filter
    B2_TRY(W.thr.ensure((size_t)std::max<int64_t>(nq, 1) * sizeof(float)));
    B2_TRY(W.sel.ensure((size_t)(nq + 1) * sizeof(int32_t)));
    B2_TRY(W.counts.ensure(2 * sizeof(unsigned long long)));
    B2_TRY(W.h_count.ensure(64));
    B2_TRY(W.hit_q.ensure(1 << 20));
    B2_TRY(W.hit_pos.ensure(1 << 20));
    B2_TRY(W.hit_sc.ensure(1 << 20));
    B2_CUDA(cudaMemsetAsync(W.sel.p, 0, sizeof(int32_t), st));
    B2_CUDA(cudaMemsetAsync(W.counts.p, 0, 2 * sizeof(unsigned long long), st));
    if (nq <= 0) return B2_OK;
    range_thr_kernel<<<(unsigned)ceil_div(nq, 8), 256, 0, st>>>(q_dev, q_dtype, nq, X.d, metric, radius, W.rel_eps, W.abs_eps, X.max_norm,
                                                             W.q_norm_limit, W.use_filter ? 1 : 0, W.thr.as<float>(), W.sel.as<int32_t>());
    B2_LAUNCH_CHECK();
    int32_t n_dense = 0;
    B2_CUDA(cudaMemcpyAsync(&n_dense, W.sel.p, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    W.n_dense = n_dense;
    g_stats[ST_QUERIES] += nq;
    g_stats[ST_FALLBACK] += n_dense;
    if (W.use_filter && n_dense < nq) {
        W.q_pitch = round_up(X.d, tma_align_elems(W.filt_dtype));
        B2_TRY(idx->q_filt.ensure((size_t)nq * W.q_pitch * esize(W.filt_dtype)));
        B2_TRY(launch_prep_queries(q_dev, q_dtype, nq, X.d, idx->q_filt.p, W.filt_dtype, W.q_pitch, st));
        W.q_filt = idx->q_filt.p;
        W.cluster = filter_cluster(nq, X.n, false);
        B2_TRY(filter_workers(idx->device, 0, W.cluster, &W.workers));
    }
    return B2_OK;
}

int range_pass(b2_index* idx, RangeWork& W, const MatView& X, int64_t pitch, int64_t base, int64_t own_lo, cudaStream_t st) {
    if (W.nq <= 0 || X.n <= own_lo) return B2_OK;
    VerifyParams vp = {};
    vp.store = X.store;
    vp.dtype = X.dtype;
    vp.d = X.d;
    vp.n = X.n;
    vp.pitch = pitch;
    vp.q = W.q;
    vp.q_dtype = W.q_dtype;
    vp.metric = W.metric;
    vp.radius = W.radius;
    vp.own_lo = own_lo;
    vp.base = base;
    vp.mask = X.mask;  // the filter of a masked search reads it too, so its candidates are selected rows only
    if (W.use_filter && W.n_dense < W.nq) {
        unsigned long long* count = W.counts.as<unsigned long long>();
        if (W.cand.cap < sizeof(int2)) B2_TRY(W.cand.ensure((size_t)std::max<int64_t>(1 << 20, 64 * W.nq) * sizeof(int2)));
        unsigned long long found = 0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            const unsigned long long cap = W.cand.cap / sizeof(int2);
            B2_CUDA(cudaMemsetAsync(count, 0, sizeof(unsigned long long), st));
            B2_CUDA(cudaEventRecord(idx->ev0, st));
            B2_TRY(launch_range_filter(X, W.q_filt, W.q_pitch, W.nq, W.metric, W.thr.as<float>(), W.cluster, W.workers, W.cand.as<int2>(),
                                       count, cap, st));
            B2_CUDA(cudaEventRecord(idx->ev1, st));
            B2_TRY(read_count(count, W, st, &found));
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, idx->ev0, idx->ev1) == cudaSuccess) W.filter_ms += ms;
            if (found <= cap) break;
            // the candidate buffer overflowed: run the filter again with room for every candidate
            W.cand.release();
            B2_TRY(W.cand.ensure((size_t)found * sizeof(int2)));
            if (attempt == 1) {
                set_error("internal: range candidate buffer overflowed twice");
                return B2_ERANGE;
            }
        }
        W.cand_peak = std::max<int64_t>(W.cand_peak, (int64_t)found);
        vp.cand = W.cand.as<int2>();
        vp.n_cand = (int64_t)found;
        B2_TRY(verify_pairs(W, vp, (int64_t)found, st));
    }
    if (W.n_dense > 0) {
        vp.cand = nullptr;
        vp.n_cand = 0;
        vp.dense_sel = W.sel.as<int32_t>() + 1;
        vp.n_dense = W.n_dense;
        B2_TRY(verify_pairs(W, vp, W.n_dense * (X.n - own_lo), st));
    }
    return B2_OK;
}

int range_finish(RangeWork& W, const int64_t* id_map, int64_t id_offset, cudaStream_t st) {
    const int64_t n = W.n_hits;
    B2_TRY(W.lims.ensure((size_t)(W.nq + 1) * sizeof(int64_t)));
    B2_TRY(W.out_d.ensure((size_t)std::max<int64_t>(n, 1) * sizeof(float)));
    B2_TRY(W.out_i.ensure((size_t)std::max<int64_t>(n, 1) * sizeof(int64_t)));
    B2_TRY(W.keys.ensure((size_t)std::max<int64_t>(n, 1) * 2 * sizeof(uint64_t)));
    B2_TRY(W.sc_alt.ensure((size_t)std::max<int64_t>(n, 1) * sizeof(float)));
    uint64_t* keys = W.keys.as<uint64_t>();
    uint64_t* keys_alt = keys + std::max<int64_t>(n, 1);
    if (n > 0) {
        range_keys_kernel<<<(unsigned)std::min<int64_t>(ceil_div(n, 256), 132 * 16), 256, 0, st>>>(W.hit_q.as<int32_t>(), W.hit_pos.as<int32_t>(),
                                                                                                 n, keys);
        B2_LAUNCH_CHECK();
        int qbits = 1;
        while (qbits < 32 && ((int64_t)1 << qbits) < W.nq) ++qbits;
        cub::DoubleBuffer<uint64_t> kb(keys, keys_alt);
        cub::DoubleBuffer<float> vb(W.hit_sc.as<float>(), W.sc_alt.as<float>());
        size_t tmp = 0;
        B2_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, kb, vb, n, 0, 32 + qbits, st));
        B2_TRY(W.sort_tmp.ensure(tmp));
        B2_CUDA(cub::DeviceRadixSort::SortPairs(W.sort_tmp.p, tmp, kb, vb, n, 0, 32 + qbits, st));
        keys = kb.Current();
        range_unpack_kernel<<<(unsigned)std::min<int64_t>(ceil_div(n, 256), 132 * 16), 256, 0, st>>>(keys, vb.Current(), n, id_map, id_offset,
                                                                                                   W.out_d.as<float>(), W.out_i.as<int64_t>());
        B2_LAUNCH_CHECK();
    }
    range_lims_kernel<<<(unsigned)ceil_div(W.nq + 1, 256), 256, 0, st>>>(keys, n, W.nq, W.lims.as<int64_t>());
    B2_LAUNCH_CHECK();
    return B2_OK;
}

}  // namespace b2
