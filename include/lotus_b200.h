/*
 * lotus_b200.h — C-ABI of libb2lotus.so, the H100 (sm_90a) vector-store backend for LOTUS.
 *
 * This is the drop-in boundary for ONE hot path of lotus-data/lotus: the faiss-backed
 * `lotus.vector_store.FaissVS` and the faiss.Kmeans call in `lotus.utils.cluster`.
 * Every entry point below replaces one faiss call site of the reference (citations are
 * relative to the reference tree, lotus-data/lotus @ 136ae4f4):
 *
 *   b2_index_create        <- faiss.index_factory + Index.add      lotus/vector_store/faiss_vs.py:23-24, :63-64
 *   b2_index_search        <- Index.search (whole index)           lotus/vector_store/faiss_vs.py:75
 *                             tmp_index.search + id remap (ids=)   lotus/vector_store/faiss_vs.py:57-72
 *   b2_index_gather        <- pickle.load(vecs)[ids]               lotus/vector_store/faiss_vs.py:38-41
 *   b2_threshold_pairs     <- sem_sim_join(K=N) + `_scores > thr`  lotus/sem_ops/sem_dedup.py:45-46
 *   b2_connected_components<- DFS over the pair set                lotus/sem_ops/sem_dedup.py:58-84
 *   b2_kmeans              <- faiss.Kmeans(d,k,niter).train +
 *                             kmeans.index.search(x, 1)            lotus/utils.py:61-65
 *   b2_merge_topk_dev      <- (no reference call site: the reference is single process; this is the
 *                             k-way merge after the NCCL all-gather of per-shard candidates)
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / CUDA types in any signature (a stream is passed as void*).
 *   - every function returns 0 on success, a negative B2_E* code on failure; the message for the calling
 *     thread's last failure is b2_last_error().
 *   - "host" entry points take HOST buffers and do their own H2D/D2H copies (these are what a plugin calls);
 *     "_dev" entry points take DEVICE buffers that live on the index's device, enqueue on `stream`
 *     (a cudaStream_t cast to void*, NULL = the legacy default stream) and return after the results are
 *     complete in the output buffers (they synchronise `stream` before returning).
 *   - the caller owns every in/out buffer; the library owns the b2_index handle and its device memory.
 *   - one in-flight call per handle (the reference's FaissVS is not re-entrant either).
 *   - there is NO CPU fallback: without a CUDA device every compute entry point returns B2_ENODEV.
 *
 * Result semantics (identical to faiss IndexFlatIP / IndexFlatL2 as restated in oracle/faiss_flat.c):
 *   - metric IP: larger is better, rows sorted best first; metric L2: squared distance, ascending.
 *   - fewer than k results: index -1 and score -FLT_MAX (IP) / +FLT_MAX (L2).
 *   - scores are the canonical fp32 score: the dot product (or sum of squared differences) accumulated
 *     in fp64 in a fixed order and rounded once to fp32 (see oracle/faiss_flat.c `orc_dot_canonical`).
 *   - exact ties follow faiss's heap (utils/Heap.h): L2 -> (dist asc, id asc); IP -> (score desc, id desc),
 *     with the retention window at rank k described in DESIGN.md §Ties.
 */
#ifndef LOTUS_B200_H
#define LOTUS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_ABI_VERSION 1

#if defined(__GNUC__)
#define B2_API __attribute__((visibility("default")))
#else
#define B2_API
#endif

/* element types of embedding matrices. B2_F16 is IEEE binary16: its values and their pairwise products are exact in fp32,
 * so an fp16 index is searched on the 2-byte tensor-core path with no operand error, and the results are those of the
 * fp32 upcast of the stored values. fp32 / bf16 queries on an fp16 index are rounded to fp16 for the filter only (a query
 * component of magnitude >= 65520 sends that query to the exact dense path); the reported scores always use the
 * query as given. */
enum { B2_F32 = 0, B2_BF16 = 1, B2_F16 = 2 };
/* B2_I8: signed 8-bit integers (two's complement), e.g. quantized embeddings. An int8 index with int8 queries is filtered on
 * the int8 tensor cores (s8 x s8 -> s32, exact integer accumulation), so its results are those of the fp32 upcast of the
 * stored values. fp32 / bf16 / fp16 queries on an int8 index are filtered against an fp16 copy of the rows (exact), built
 * on the first such search and kept with the handle (2 more bytes per element). int8 queries on the other indexes are
 * widened exactly. An int8 index needs d < 2^17 (the s32 accumulator range), and d < 2^15 with B2_METRIC_L2 (the filter
 * forms 2 <q, x> - |x|^2 in int32). b2_threshold_pairs runs the int8 pair filter; its threshold is in units of int8 inner
 * products. k-means runs on an fp16 copy of the rows (exact), made on the first k-means call and kept with the handle.
 * The code is kept apart from the floating-point types. */
enum { B2_I8 = 8 };
/* metrics; numeric values match faiss.METRIC_INNER_PRODUCT / faiss.METRIC_L2 */
enum { B2_METRIC_IP = 0, B2_METRIC_L2 = 1 };

/* error codes */
enum {
    B2_OK = 0,
    B2_EINVAL = -1,   /* bad argument */
    B2_ENODEV = -2,   /* no CUDA device / wrong architecture */
    B2_ECUDA = -3,    /* CUDA runtime or driver error */
    B2_ENOMEM = -4,   /* allocation failed */
    B2_ERANGE = -5    /* k or an id out of the supported range */
};

typedef struct b2_index b2_index;

/* ---- library ---------------------------------------------------------------------------------------- */
B2_API int b2_abi_version(void);
B2_API const char* b2_last_error(void);
/* number of visible CUDA devices that are sm_90 (H100); 0 when there is none */
B2_API int b2_device_count(void);
/* largest k supported by b2_index_search */
B2_API int b2_max_k(void);

/* ---- index lifetime (faiss_vs.py:22-36) -------------------------------------------------------------- */
/* Build a flat index over x[n,d] (row-major, `dtype` elements). x is a HOST pointer unless x_on_device != 0.
 * The matrix is copied; the caller may free x afterwards. */
B2_API int b2_index_create(const void* x, int64_t n, int32_t d, int32_t dtype, int32_t metric, int32_t device,
                    int32_t x_on_device, b2_index** out);
/* Build a HOST-RESIDENT flat index over the host matrix x[n,d]: for corpora larger than free device memory. The rows are
 * copied into a library-owned pinned, mapped host allocation (B2_ENOMEM, with the size in the message, when it cannot be
 * pinned); only their norms (4 bytes per row, 8 for B2_I8), a ring of two chunk slots of ring_bytes in all (0 = 1 GiB) and
 * per-search workspaces live on the device. fp32 indexes of at least 4096 rows also keep a bf16 rounding of the rows in
 * pinned memory (2 more bytes per element): the first level of a search streams it. A search streams the rows through the
 * ring in chunks (rows per chunk from ring_bytes, a multiple of 256), copying the next chunk while the filter runs over the
 * current one, and returns results bit-identical to b2_index_create's index over the same rows. n < 2^31; every dtype with
 * the limits of b2_index_create. b2_index_search / _search_dev (with or without ids), b2_index_gather, b2_last_filter_ms (the
 * sum over chunks) and b2_debug_filter_lists (the folded lists) serve it; b2_index_data_dev returns NULL, and
 * b2_threshold_pairs, the k-means entry points and b2_index_search_packed_dev / _stage1_dev / _stage2_packed_dev return
 * B2_EINVAL ("not available on a host-resident index"). An ids subset whose rows fit in the ring is gathered into device
 * memory and searched there; a larger one is gathered on the host and streamed. */
B2_API int b2_index_create_host(const void* x, int64_t n, int32_t d, int32_t dtype, int32_t metric, int32_t device,
                                int64_t ring_bytes, b2_index** out);
/* where the rows of an index live: 0 = device memory (b2_index_create), 1 = host memory (b2_index_create_host) */
B2_API int32_t b2_index_resident(const b2_index* idx);
B2_API void b2_index_free(b2_index* idx);
B2_API int64_t b2_index_ntotal(const b2_index* idx);
B2_API int32_t b2_index_dim(const b2_index* idx);
B2_API int32_t b2_index_dtype(const b2_index* idx);
B2_API int32_t b2_index_metric(const b2_index* idx);
B2_API int32_t b2_index_device(const b2_index* idx);
/* device pointer of the stored matrix [n,d] in `dtype` (for zero-copy hand-off to torch) */
B2_API const void* b2_index_data_dev(const b2_index* idx);

/* ---- search (faiss_vs.py:43-77) ---------------------------------------------------------------------- */
/* q[nq,d] in q_dtype. ids == NULL: search the whole index. ids != NULL (n_ids entries, positions into the
 * index, any order): search only those rows and report the ORIGINAL ids (the reference builds a temporary
 * index over vecs[ids] and remaps; ties follow the order of `ids`).
 * out_scores[nq,k] float32, out_idx[nq,k] int64. HOST buffers. */
B2_API int b2_index_search(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, const int64_t* ids,
                    int64_t n_ids, float* out_scores, int64_t* out_idx);

/* DEVICE buffers; ids_dev may be NULL. id_offset is added to every reported id when ids_dev == NULL
 * (row-sharded multi-GPU: global id = local id + shard offset). */
B2_API int b2_index_search_dev(b2_index* idx, const void* q_dev, int64_t nq, int32_t q_dtype, int32_t k,
                        const int64_t* ids_dev, int64_t n_ids, int64_t id_offset, float* out_scores_dev,
                        int64_t* out_idx_dev, void* stream);

/* Masked search: only the rows a bitmap selects take part, searched in place. mask holds ceil(n / 32) little-endian 32-bit
 * words, bit (j & 31) of word (j >> 5) set = row j takes part; bits at or past n are ignored. The result is that of
 * b2_index_search with ids = the ascending list of the set rows, bit for bit (indices and score bits, and the -1 / -+FLT_MAX
 * padding when fewer than k rows are selected, an all-zero mask included), but no copy of the subset is made: the filter
 * kernel sweeps the whole index and leaves the cleared rows out, so a subset of a device-resident index costs no device
 * memory beyond the bitmap and one of a host-resident index no gather on the host. It sweeps all n rows whatever the mask
 * selects. Every dtype, both metrics, both residencies, k up to b2_max_k(). HOST buffers. */
B2_API int b2_index_search_masked(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, const uint32_t* mask,
                                  float* out_scores, int64_t* out_idx);
/* DEVICE buffers (mask_dev included); id_offset is added to every reported id, as in b2_index_search_dev. */
B2_API int b2_index_search_masked_dev(b2_index* idx, const void* q_dev, int64_t nq, int32_t q_dtype, int32_t k,
                                      const uint32_t* mask_dev, int64_t id_offset, float* out_scores_dev, int64_t* out_idx_dev,
                                      void* stream);

/* k-way merge of g per-shard result lists: scores[g,nq,k], idx[g,nq,k] (each list sorted best first, shard
 * s holding ids below those of shard s+1) -> out[nq,k]. DEVICE buffers on `device`. */
B2_API int b2_merge_topk_dev(const float* scores_dev, const int64_t* idx_dev, int32_t g, int64_t nq, int32_t k,
                      int32_t metric, int32_t device, float* out_scores_dev, int64_t* out_idx_dev, void* stream);

/* The same two steps with ONE 8-byte word per entry — (float32 score bits << 32) | local row id, 0xffffffff = no result — so
 * the row-sharded exchange is a single all-gather of nq*k*8 bytes per rank (25.6 MB at 100k x 32) instead of scores + int64 ids
 * (38 MB in two collectives). b2_index_search_packed_dev searches the whole index and reports LOCAL ids;
 * b2_merge_topk_packed_dev takes packed[g,nq,k] plus shard_offsets[g] (HOST array: global id of row 0 of shard s) and writes
 * float32 scores and int64 GLOBAL ids. */
B2_API int b2_index_search_packed_dev(b2_index* idx, const void* q_dev, int64_t nq, int32_t q_dtype, int32_t k,
                               uint64_t* out_packed_dev, void* stream);
B2_API int b2_merge_topk_packed_dev(const uint64_t* packed_dev, const int64_t* shard_offsets, int32_t g, int64_t nq, int32_t k,
                             int32_t metric, int32_t device, float* out_scores_dev, int64_t* out_idx_dev, void* stream);

/* Row-sharded search in two stages, so that the ranks can tell each other how good the merged top k will be BEFORE the exact
 * re-scoring. Stage 1 filters this shard (wgmma kernel) and writes lower_dev[nq]: for every query a lower bound on the exact
 * score of its j best local candidates (-inf when unknown); it only enqueues work on `stream`. The caller all-reduces (MIN)
 * lower_dev over the ranks with j = ceil(k / ranks) — k rows of the whole index are then known to reach that score — and hands
 * the result to stage 2, which re-scores only the local candidates that can still reach it (about k / ranks instead of k + 2),
 * certifies against it, and writes the packed [nq,k] list like b2_index_search_packed_dev. q_dev must stay valid until
 * stage 2 returns. One staged search in flight per handle. */
B2_API int b2_index_search_stage1_dev(b2_index* idx, const void* q_dev, int64_t nq, int32_t q_dtype, int32_t k, int32_t j,
                               float* lower_dev, void* stream);
B2_API int b2_index_search_stage2_packed_dev(b2_index* idx, const float* hint_dev, uint64_t* out_packed_dev, void* stream);

/* ---- range search (faiss IndexFlat.range_search) ------------------------------------------------------ */
/* Every row whose canonical score is strictly greater than `radius` (B2_METRIC_IP), or whose canonical squared distance is
 * strictly less than it (B2_METRIC_L2), for each query q[nq,d] in q_dtype. HOST buffers, in the layout of faiss's Python
 * range_search: lims[nq+1] int64; out_d / out_i [lims[nq]] hold query i's hits at [lims[i], lims[i+1]), in ascending row id,
 * with the same canonical float32 values b2_index_search reports. ids != NULL: only those rows (positions into the index, any
 * order, repeats allowed), as a temporary index over x[ids]: a query's hits follow the order of `ids` and report the original
 * ids. A NaN radius matches nothing. lims and *n_results are filled on success and also when the call returns B2_ERANGE
 * because cap < *n_results; the caller then retries with cap = *n_results. Every index residency and dtype. */
B2_API int b2_index_range_search(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, float radius, const int64_t* ids,
                                 int64_t n_ids, int64_t* lims, float* out_d, int64_t* out_i, int64_t cap, int64_t* n_results);
/* Masked range search: b2_index_range_search over the rows a bitmap selects, searched in place. mask is laid out as for
 * b2_index_search_masked (ceil(n / 32) little-endian words, bits at or past n ignored). The result equals b2_index_range_search
 * with ids = the ascending list of the set rows, bit for bit (lims, ids and score bits; an all-zero mask gives lims of zeros),
 * and the argument checks, the NaN radius and B2_ERANGE behave as there. No copy of the subset is made: the range filter
 * sweeps all n rows and only selected rows become candidates, so the candidate buffer scales with the hits among them.
 * Every dtype, both metrics, both residencies. HOST buffers. */
B2_API int b2_index_range_search_masked(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, float radius,
                                        const uint32_t* mask, int64_t* lims, float* out_d, int64_t* out_i, int64_t cap,
                                        int64_t* n_results);

/* ---- row gather (faiss_vs.py:38-41) ------------------------------------------------------------------ */
/* out[m,d] in the index's dtype = x[ids]; HOST out unless out_on_device != 0 (then ids is a device pointer too) */
B2_API int b2_index_gather(b2_index* idx, const int64_t* ids, int64_t m, void* out, int32_t out_on_device);

/* ---- dedup (sem_dedup.py:45-84) ---------------------------------------------------------------------- */
/* All unordered pairs i<j with canonical score(i,j) > threshold (IP; strict, as sem_dedup.py:46).
 * out_i/out_j: HOST arrays of capacity cap; *n_pairs receives the number found (may exceed cap: then only the
 * first cap pairs in (i,j) order are stored and the call returns B2_ERANGE).
 * part/nparts: process only the row-tile slice `part` of `nparts` (multi-GPU sharding of the pair space);
 * pass 0,1 for everything. Pairs are returned sorted by (i,j). */
B2_API int b2_threshold_pairs(b2_index* idx, float threshold, int32_t part, int32_t nparts, int64_t* out_i,
                       int64_t* out_j, int64_t cap, int64_t* n_pairs);
/* labels[n] = smallest row id of the connected component of each row under the pair list (HOST buffers). */
B2_API int b2_connected_components(int64_t n, const int64_t* pi, const int64_t* pj, int64_t n_pairs, int32_t device,
                            int64_t* labels);

/* ---- k-means (lotus/utils.py:61-65) ------------------------------------------------------------------ */
/* faiss.Kmeans(d, k, niter=niter, seed=1234, max_points_per_centroid=256).train(x[ids]) followed by
 * index.search(x[ids], 1). ids may be NULL (all rows). out_assign[m] int64, out_centroids[k,d] float32
 * (nullable), out_obj[niter] float32 (nullable, the objective of every iteration). HOST buffers.
 * full_lloyd != 0 trains on every point instead of faiss's 256*k subsample. */
B2_API int b2_kmeans(b2_index* idx, const int64_t* ids, int64_t m, int32_t k, int32_t niter, int64_t seed,
              int32_t full_lloyd, int64_t* out_assign, float* out_centroids, float* out_obj);
/* one assignment pass against given centroids[k,d] (float32, HOST): out_assign[m] int64, out_dist[m] float32
 * (nullable). This is `kmeans.index.search(x, 1)` with explicit centroids. */
B2_API int b2_kmeans_assign(b2_index* idx, const int64_t* ids, int64_t m, const float* centroids, int32_t k,
                     int64_t* out_assign, float* out_dist);

/* DEVICE-buffer forms for the row-sharded multi-GPU Lloyd loop (lotus_b200/distributed.py sharded_kmeans): nothing visits
 * the host between the assignment, the per-shard sums and the NCCL all-reduce of [k,d] sums + [k] counts.
 * b2_kmeans_assign_dev: assign_dev[m] int64 (and dist_dev[m] float32 when non-NULL: the canonical distance to the winner)
 * for the rows ids_dev[0..m) (NULL = all rows) against centroids_dev[k,d] float32.
 * b2_kmeans_accumulate_dev: sums_dev[k,d] float32 = per-centroid sums of the member rows in point order (NOT divided),
 * counts_dev[k] float32; when obj_dev is non-NULL, *obj_dev += sum of squared distances of the rows to
 * centroids_dev[assign] (float64; centroids_dev = the centroids the assignment was made against).
 * All pointers live on the index's device; both calls enqueue on `stream` and synchronise it before returning. */
B2_API int b2_kmeans_assign_dev(b2_index* idx, const int64_t* ids_dev, int64_t m, const float* centroids_dev, int32_t k,
                         int64_t* assign_dev, float* dist_dev, void* stream);
B2_API int b2_kmeans_accumulate_dev(b2_index* idx, const int64_t* ids_dev, int64_t m, const int64_t* assign_dev, int32_t k,
                             const float* centroids_dev, float* sums_dev, float* counts_dev, double* obj_dev, void* stream);

/* per-shard centroid update for multi-GPU Lloyd: for the rows ids[0..m) (or all) and their assignment assign[m],
 * out_sums[k,d] float32 = sum of the member rows of each centroid (point order, fp32, NOT divided), out_counts[k] float32.
 * The caller all-reduces sums and counts over the ranks and divides. HOST buffers. (faiss/Clustering.cpp compute_centroids
 * before its normalisation loop; lotus/utils.py:61-62 calls it through faiss.Kmeans.train.) */
B2_API int b2_kmeans_accumulate(b2_index* idx, const int64_t* ids, int64_t m, const int64_t* assign, int32_t k, float* out_sums,
                         float* out_counts);

/* ---- host-side marshalling (no device work) ------------------------------------------------------------ */
/* out[i] = bfloat16 bit pattern of x[i] (round to nearest even, NaN stays a quiet NaN); *all_exact (nullable) = 1 when
 * every x[i] was already bfloat16-representable, i.e. the 2-byte form loses nothing. The plugin uses it to ship query
 * vectors that came out of a bf16 index (faiss_vs.py:38-41 -> sem_sim_join.py:130-134) in their exact 2-byte form. */
B2_API int b2_host_f32_to_bf16(const float* x, int64_t count, uint16_t* out, int32_t* all_exact);
/* the exact inverse: out[i] = float32 value of the bfloat16 bit pattern x[i] (row gathers of a bf16 index, faiss_vs.py:38-41) */
B2_API int b2_host_bf16_to_f32(const uint16_t* x, int64_t count, float* out);

/* The filter kernel's work schedule for a shape (no device work; used by the CPU tests): kp = candidate-list capacity (0 = the
 * shape goes to the dense path), n_splits = corpus splits, units_whole = leading query units that sweep the whole corpus as one
 * item each (two-phase schedule), two_cta = CTAs per cluster (1 = single CTAs; otherwise a query unit is two query tiles and
 * there are num_sms / 2 workers, CTA pairs). */
B2_API int b2_debug_filter_plan(int64_t nq, int64_t n, int32_t k, int32_t num_sms, int32_t* kp, int32_t* n_splits,
                         int32_t* units_whole, int32_t* two_cta);
/* The filter kernel's raw candidate lists for host queries q[nq,d] (q_dtype), planned and launched exactly as a search does
 * (level 0; level 1 = the tf32 second level of an fp32 index, which drops its bf16 copy) or, with top1 != 0, as the k-means
 * assignment does (register top-2 epilogue). plan[8] receives: use_filter, kp, n_splits, units_whole, cluster, two_level,
 * filter operand dtype, query chunks; *rel_eps the filter's error bound relative to |q|*|x|. With every list buffer non-NULL
 * and use_filter set, the filter runs and fills (HOST buffers) cand_score / cand_id [nq, n_splits, 2 sets, kp/2] and
 * cand_thr [nq, n_splits, 2]; with any of them NULL only the plan is reported. B2_ERANGE when nq needs more than one query
 * chunk. For testing; not part of the search path. */
B2_API int b2_debug_filter_lists(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, int32_t top1, int32_t level,
                          int32_t* plan, float* rel_eps, float* cand_score, int32_t* cand_id, float* cand_thr);
/* b2_debug_filter_lists for a masked search (mask: HOST, as b2_index_search_masked takes it): no cleared row is on any list,
 * and a list's bound holds for the selected rows it discarded. */
B2_API int b2_debug_filter_lists_masked(b2_index* idx, const void* q, int64_t nq, int32_t q_dtype, int32_t k, int32_t level,
                                        const uint32_t* mask, int32_t* plan, float* rel_eps, float* cand_score, int32_t* cand_id,
                                        float* cand_thr);
/* The chunking of a host-resident index of n rows (no device work): *chunk_rows rows per chunk (a multiple of 256 unless
 * one chunk holds every row), *n_chunks chunks, *slots device slots of the ring. Chunk c owns the rows
 * [c * chunk_rows, min(n, (c + 1) * chunk_rows)); it streams chunk_rows rows from min(c * chunk_rows, n - chunk_rows) on,
 * so the last chunk re-streams the tail of its predecessor and the search skips those rows there. B2_EINVAL when a slot
 * of ring_bytes / slots holds fewer than 256 rows. */
B2_API int b2_debug_stream_plan(int64_t n, int32_t d, int32_t dtype, int64_t ring_bytes, int64_t* chunk_rows, int64_t* n_chunks,
                                int32_t* slots);
/* CUDA-event times (ms) of the last search of a host-resident index: out4[0] the host-to-device copies (copy stream),
 * [1] the span of the streamed filter on the search stream (first chunk wait to last fold), [2] the filter launches, [3]
 * finalize. [1] - [2] is the part of the pipeline not spent in the filter: copies the filter did not hide, plus the folds. */
B2_API int b2_debug_stream_times(const b2_index* idx, float* out4);
/* The filter's error model for one operand combination (no device work): |filter score - exact inner product| <=
 * rel_eps * |q| * |x| + abs_eps * (|q| + |x|) for a store of `store_dtype` filtered as `filt_dtype` (B2_F32 = tf32 wgmma,
 * B2_BF16 / B2_F16 = 2-byte wgmma) with queries of `q_dtype`, dimension d. abs_eps is non-zero only where an operand is
 * rounded to fp16 (its subnormal spacing). For testing; the search paths use the same function. */
B2_API int b2_debug_filter_eps(int32_t store_dtype, int32_t filt_dtype, int32_t q_dtype, int32_t d, float* rel_eps, float* abs_eps);
/* The last b2_index_range_search or b2_index_range_search_masked of this handle: out4[0] the most candidates one range-filter
 * launch produced (the peak size of the candidate buffer), [1] the hits, [2] the queries the exact dense path answered, [3] 1
 * if the filter ran. */
B2_API int b2_debug_range_stats(const b2_index* idx, int64_t* out4);

/* ---- instrumentation ---------------------------------------------------------------------------------- */
/* counters since the last b2_stats_reset(): [0] kernels launched by this library, [1] queries answered,
 * [2] queries that took the exact dense fallback, [3] wgmma filter launches, [4] rows rescored exactly,
 * [5] queries of fp32 indexes that the bf16 first-level filter could not certify and the tf32 level answered,
 * [6] bytes copied host-to-device by searches of host-resident indexes, [7] corpus chunks those searches filtered.
 * Returns how many counters were written (<= cap). */
B2_API int b2_stats(int64_t* out, int32_t cap);
B2_API void b2_stats_reset(void);
/* device time (ms) of the dominant kernel (the wgmma filter) in the last search on this handle, measured
 * with CUDA events on the stream it was launched on; <0 when unavailable. */
B2_API float b2_last_filter_ms(const b2_index* idx);

#ifdef __cplusplus
}
#endif
#endif /* LOTUS_B200_H */
