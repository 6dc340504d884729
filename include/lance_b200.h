/*
 * lance_b200.h -- C ABI of the H100-native IVF-PQ / IVF-FLAT hot path.
 *
 * This is the drop-in boundary for lancedb/lance: every entry point replaces one function (or one
 * trait method) of the reference's `lance-index::vector::{kmeans,ivf,pq,flat}` / `lance-linalg`
 * crates; the reference file:line it replaces is cited above each declaration (paths relative to
 * /root/reference/rust).  INTEGRATION.md shows the Rust `extern "C"` block + shim a maintainer adds.
 *
 * Conventions
 *   - Plain pointers and sizes only.  Every data pointer may be a HOST pointer (pageable or pinned)
 *     or a DEVICE pointer of the current device; the library detects which (cudaPointerGetAttributes)
 *     and stages host buffers through the device itself.  Outputs are written where they point.
 *   - Caller allocates inputs AND outputs; the library never frees or keeps a caller pointer after
 *     the call returns, except inside an `lb2_index` handle, which owns private device copies.
 *   - Vectors are Arrow FixedSizeList values buffers: contiguous row-major n x d.
 *   - Every function returns lb2_status and never unwinds/aborts across the boundary; the message
 *     of the last failure on the calling thread is available from lb2_last_error().
 *   - There is NO CPU fallback: without a usable CUDA device every compute entry point returns
 *     LB2_NO_DEVICE.
 *   - Calls are blocking (results are complete on return).  All entry points are thread-safe;
 *     each calling thread uses the CUDA device selected by lb2_set_device() on that thread and its
 *     own CUDA stream, so concurrent callers (the reference searches up to ncpu-2 partitions at a
 *     time, rust/lance/src/io/exec/knn.rs:881) overlap on the device.  Calls that only read a handle
 *     (searches, transform, export, optimize / split / join into a new handle) may share it across
 *     threads; a call that changes or frees a handle (lb2_index_set_partition_index, the _load* calls,
 *     lb2_index_destroy, lb2_partition_index_destroy) needs exclusive access to it.
 *   - Stream variants: lb2_set_stream() orders every later call of the thread on a caller-owned
 *     cudaStream_t; lb2_index_search_async() enqueues a whole search and returns without waiting.
 */
#ifndef LANCE_B200_H_
#define LANCE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  LB2_OK = 0,
  LB2_INVALID_ARG = 1,
  LB2_UNSUPPORTED = 2, /* valid request that this build does not implement (never silently emulated) */
  LB2_CUDA_ERROR = 3,
  LB2_NCCL_ERROR = 4,
  LB2_OOM = 5,
  LB2_NO_DEVICE = 6
} lb2_status;

/* element type of a vector buffer (arrow DataType of the FixedSizeList child) */
typedef enum { LB2_F32 = 0, LB2_F16 = 1, LB2_BF16 = 2, LB2_U8 = 3 } lb2_dtype;

/* lance_linalg::distance::DistanceType (lance-linalg/src/distance.rs) */
typedef enum { LB2_L2 = 0, LB2_COSINE = 1, LB2_DOT = 2 } lb2_metric;

typedef struct lb2_index lb2_index; /* device-resident IVF_PQ / IVF_FLAT index */

/* ---- runtime -------------------------------------------------------------------------------- */
const char* lb2_version(void);
size_t lb2_last_error(char* buf, size_t len); /* copies the calling thread's last message */
int lb2_device_count(void);                   /* 0 when no CUDA device is usable */
lb2_status lb2_set_device(int device);
lb2_status lb2_synchronize(void);
/* Give cached device memory back: the calling thread's bulk-copy staging buffer (host-sourced builds keep one
 * of up to LB2_STAGING_CACHE_MB, default 1024 MB, between calls so that the copy of the next build starts at
 * once) and every free block of the stream-ordered pool.  The reference has no counterpart (its buffers are
 * Arrow arrays dropped with the batch); call it when a burst of index builds is over. */
lb2_status lb2_trim_memory(void);
/* Bind the calling thread's library context to a caller-owned CUDA stream (cudaStream_t passed as
 * void*): all work of later calls from this thread -- kernels, copies, stream-ordered allocations --
 * is enqueued on it, after whatever the caller enqueued before.  Blocking entry points still wait for
 * their own results (that is a cudaStreamSynchronize of this stream).  NULL returns to the thread's
 * private stream.  The stream must belong to the thread's device and outlive the binding. */
lb2_status lb2_set_stream(void* cuda_stream);
/* device / pinned-host buffers for callers that keep data resident (bench, the Rust shim's ring) */
lb2_status lb2_malloc(void** ptr, size_t bytes);
lb2_status lb2_free(void* ptr);
lb2_status lb2_malloc_host(void** ptr, size_t bytes); /* pinned */
lb2_status lb2_free_host(void* ptr);
lb2_status lb2_memcpy(void* dst, const void* src, size_t bytes); /* direction auto-detected */
/* instrumentation: number of kernels this library launched on the calling thread's device since
 * the last reset, and per-kernel CUDA-event timing (name = kernel family, e.g. "pq_scan"). */
lb2_status lb2_launch_count(uint64_t* count, int reset);
lb2_status lb2_profile_enable(int on);
lb2_status lb2_profile_get(const char* name, uint64_t* launches, double* total_ms);
lb2_status lb2_profile_reset(void);
/* all entries as "name\tlaunches\ttotal_ms\n" lines; returns the full length (like snprintf) */
size_t lb2_profile_dump(char* buf, size_t len);
lb2_status lb2_timer_start(void);          /* CUDA event on the library's stream */
lb2_status lb2_timer_stop(float* ms_out);  /* records, synchronises, returns elapsed ms */

/* ---- lance-linalg distance API -------------------------------------------------------------- */
/* l2_distance_batch / dot_distance_batch / cosine_distance_batch
 * (lance-linalg/src/distance/l2.rs:194-203, dot.rs:164-172, cosine.rs:266-290):
 * out[i] = dist(from, to[i]) for i < n.  f32 L2/Dot are bit-exact to the reference's 16-lane order. */
lb2_status lb2_distance_batch(const void* from, const void* to, uint64_t n, uint32_t d,
                              lb2_dtype dtype, lb2_metric metric, float* out);
/* normalize_fsl (lance-linalg/src/kernels.rs:141-146,201-211): out[i] = x[i] / ||x[i]|| */
lb2_status lb2_normalize(const void* vectors, uint64_t n, uint32_t d, lb2_dtype dtype, void* out);

/* ---- k-means (lance-index/src/vector/kmeans.rs) --------------------------------------------- */
typedef struct {
  uint32_t max_iters;      /* KMeansParams::max_iters, default 50 (kmeans.rs:92-103) */
  double tolerance;        /* 1e-4 */
  uint32_t redos;          /* 1.  Every redo restarts from the same rng state (kmeans.rs:645-653), so without a
                              balance bias redos > 1 equals one run; with a bias redos > 1 -> LB2_UNSUPPORTED */
  float balance_factor;    /* BEFORE the division by n that train_kmeans applies (kmeans.rs:1344);
                              IVF training passes 1.0 (rust/lance/src/index/vector/ivf.rs:1858) */
  uint32_t hierarchical_k; /* 16: for k > 256 (and no init_centroids) the reference's hierarchical
                              scheme is used (kmeans.rs:746-1003, 1027); 0/1 = flat Lloyd for every k */
  uint64_t sample_rate;    /* 256: only the first sample_rate*k rows are used (kmeans.rs:1328-1340) */
  uint64_t seed;           /* the reference is unseeded (kmeans.rs:645); we are reproducible */
  const void* init_centroids; /* KMeanInit::Incremental (k x d, same dtype) or NULL = random rows */
  lb2_metric metric;       /* L2 or DOT (cosine callers normalise first, as the reference does) */
  uint32_t partition_index;       /* lb2_partition_index_mode of a build's full pass (below): EXACT (the default),
                                     AUTO or HNSW.  A build whose mode resolves to the graph assigns every row
                                     through lb2_partition_index_* over its trained centroids, and the index keeps
                                     the rule (lb2_index_set_partition_index).  lb2_kmeans_train refuses any other
                                     value than EXACT with LB2_INVALID_ARG: training never uses the graph. */
  uint32_t partition_index_batch; /* the graph's insert_batch: 0 or 1 serial (the default), B >= 2 in rounds */
} lb2_kmeans_params;
void lb2_kmeans_params_default(lb2_kmeans_params* p);

/* train_kmeans<T>(array, params, dimension, k, sample_rate) -> KMeans  (kmeans.rs:1309-1347) */
lb2_status lb2_kmeans_train(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, uint32_t k,
                            const lb2_kmeans_params* params, void* centroids_out, double* loss_out,
                            uint32_t* iters_out);

/* compute_partitions_arrow_array / compute_partitions_with_dists (kmeans.rs:1187-1294):
 * part_out[i] = argmin_k dist(vectors[i], centroids[k]) (first minimum), dist_out[i] that distance,
 * valid_out[i] = 0 where the reference returns None (all NaN/Inf).  dist_out/valid_out nullable. */
lb2_status lb2_compute_partitions(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                                  lb2_metric metric, const void* vectors, uint64_t n,
                                  uint32_t* part_out, float* dist_out, uint8_t* valid_out);

/* kmeans_find_partitions_arrow_array (kmeans.rs:1076-1158), batched over nq queries:
 * ids/dists are [nq][nprobes], ascending by (distance, id). */
lb2_status lb2_find_partitions(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                               lb2_metric metric, const void* queries, uint64_t nq,
                               uint32_t nprobes, uint32_t* ids_out, float* dists_out);

/* compute_residual (lance-index/src/vector/residual.rs:111-154): out[i] = v[i] - centroids[part[i]] */
lb2_status lb2_compute_residual(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                                const void* vectors, uint64_t n, const uint32_t* part_ids,
                                void* out);

/* ---- partition index: an HNSW graph over the centroids (lance-index/src/vector/utils.rs:26-108) --------------------
 * PartitionTransformer::new (ivf/transform.rs:48-68) asks SimpleIndex::may_train_index for a graph over the centroids,
 * and transform (:112-124) then assigns each row by one graph search instead of the exact scan.  The modes are the
 * values of LANCE_USE_HNSW_SPEEDUP_INDEXING (utils.rs:26-44): EXACT = "disabled", AUTO = unset (or any other value),
 * HNSW = "enabled".  EXACT is this library's default everywhere. */
typedef enum {
  LB2_PARTITION_INDEX_EXACT = 0, /* never the graph */
  LB2_PARTITION_INDEX_AUTO = 1,  /* the graph when k * d >= 1 000 000 (centroids.len() of the flat values array) */
  LB2_PARTITION_INDEX_HNSW = 2   /* always the graph */
} lb2_partition_index_mode;
typedef struct lb2_partition_index lb2_partition_index;
/* may_train_index's decision (utils.rs:67-91), on the host only: *uses_graph_out = 1 when `mode` resolves to the
 * graph for a k x d model whose columns have element type `dtype`.  Only an f32 model has a graph (utils.rs:83-90);
 * u8 columns have f32 models and follow f32, f16 / bf16 models are always exact. */
lb2_status lb2_partition_index_uses_graph(uint64_t k, uint32_t d, lb2_dtype dtype, lb2_partition_index_mode mode,
                                          int* uses_graph_out);
/* SimpleIndex::try_new (utils.rs:53-59): HNSW::index_vectors (hnsw/builder.rs:742-775) over FlatFloatStorage of the
 * k centroids (f32, [k][d]; node i is centroid i) under L2 or dot, with HnswBuildParams::default() (max_level 7),
 * ef_construction 15 and m 12.  *out = NULL whenever the mode resolves to the exact scan, as may_train_index returns
 * None.  The graph is IVF_HNSW_FLAT's graph of one partition holding the centroids, bit for bit: its distances are
 * the f32 16-lane rule (below), the level of node i >= 1 comes from the counter-based draw of (seed, partition 0,
 * node i) (the reference's rayon build and unseeded levels are not reproducible), and insert_batch B >= 2 builds in
 * IVF_HNSW_SQ's deterministic rounds (0 or 1: the serial build).  Cosine -> LB2_INVALID_ARG (the IVF transformer
 * normalises first and assigns under L2, ivf.rs:149-166: normalise and pass L2); d % 4 != 0 or a communicator of more
 * than one rank with a mode that resolves to the graph -> LB2_UNSUPPORTED. */
lb2_status lb2_partition_index_build(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                                     lb2_partition_index_mode mode, uint64_t seed, uint32_t insert_batch,
                                     lb2_partition_index** out);
/* PartitionTransformer::transform's partition step (ivf/transform.rs:112-124).  pi == NULL is the exact scan:
 * lb2_compute_partitions with the same arguments.  Otherwise SimpleIndex::search (utils.rs:93-108) of every row:
 * search_basic (hnsw/builder.rs:164-235) with k = 1, ef = 15, no bounds and no prefilter (entry node 0, greedy_search
 * at every level from max_level - 1 down to 0, beam_search at level 0), part_out[i] / dist_out[i] the first result.
 * The distance is the f32 16-lane rule of lb2_compute_partitions (l2.rs / dot.rs with LANES = 16), so dist_out is the
 * reference's CENTROID_DIST for the row and partition.  k, d and the metric must be pi's; the graph reads its own copy
 * of the centroids, so `centroids` is only read when pi == NULL.  Rows are f32 or u8 (held as f32), on the host
 * (streamed in chunks, LB2_CHUNK_ROWS / LB2_MAX_RESIDENT_MB) or the device.  valid_out[i] = 0, part_out[i] = 0 and
 * dist_out[i] = NaN for
 *  - a row with a NaN or infinite element: KeepFiniteVectors drops it before the partition step (ivf.rs:149-166);
 *  - a finite row whose search keeps no result: beam_search admits f32::MIN <= dist < f32::MAX only (graph.rs:
 *    290-291), so a row whose every distance it meets overflows has none, and the reference's `res[0]` panics
 *    (utils.rs:106).  The exact scan drops such a row too (kmeans.rs:1187-1246 returns None).
 * Every other row is valid, with the graph's answer. */
lb2_status lb2_partition_index_assign(const lb2_partition_index* pi, const void* centroids, uint32_t k, uint32_t d,
                                      lb2_dtype dtype, lb2_metric metric, const void* vectors, uint64_t n,
                                      uint32_t* part_out, float* dist_out, uint8_t* valid_out);
/* the graph's shape (each output nullable), and the graph in the layout of lb2_index_export_hnsw_flat for one
 * partition of k rows: levels[k], counts0[k], neighbors0 / dists0 [k][2m], counts_up / neighbors_up / dists_up over
 * the num_upper_rows upper-level rows ([.][m]); unused list slots are zero */
lb2_status lb2_partition_index_info(const lb2_partition_index* pi, uint32_t* k, uint32_t* d, uint32_t* max_level,
                                    uint32_t* m, uint32_t* ef_construction, uint64_t* num_upper_rows);
lb2_status lb2_partition_index_export(const lb2_partition_index* pi, uint8_t* levels_out, uint32_t* counts0_out,
                                      uint32_t* neighbors0_out, float* dists0_out, uint32_t* counts_up_out,
                                      uint32_t* neighbors_up_out, float* dists_up_out);
lb2_status lb2_partition_index_destroy(lb2_partition_index* pi); /* NULL is a no-op */
/* Builds: lb2_kmeans_params.partition_index selects the rule of the full pass of every build that takes the params
 * (IVF_PQ, IVF_FLAT, IVF_SQ, IVF_RQ and the three IVF_HNSW kinds); the graph is built over the trained centroids
 * (under L2 for a cosine index, whose rows are normalised first; dot for dot) with level seed
 * seed ^ 0x7061727469646978 ("partidix"; `seed` the build's seed) and insert_batch partition_index_batch.  Each
 * row's partition, CENTROID_DIST (IVF_RQ's dist_v_c and factors) and residual (IVF_PQ's codes) follow the graph's
 * answer; rows without one are dropped, as the exact scan drops its None rows.  EXACT builds are unchanged. */
/* The partition rule of an index handle: the mode, the graph's level seed and insert_batch, and the graph over the
 * index's centroids when the mode resolves to one for the index's column type (the rule and refusals of
 * lb2_partition_index_build; cosine indexes use L2 on normalised rows).  It serves lb2_index_transform, the
 * nearest-new-centroid transform of IVF_RQ rows in lb2_index_split (ivf.rs:301-304), and every index that
 * lb2_index_optimize / _split / _join / _update return, which inherit the rule and build the graph over their own
 * centroids.  Builds set it from their parameters; an index opened with lb2_index_create* / _load* /
 * _load_storage starts EXACT (LANCE_USE_HNSW_SPEEDUP_INDEXING's mapping is the caller's: see INTEGRATION.md).
 * EXACT drops the graph.  lb2_index_load_storage keeps the rule. */
lb2_status lb2_index_set_partition_index(lb2_index* index, lb2_partition_index_mode mode, uint64_t seed,
                                         uint32_t insert_batch);

/* ---- product quantisation (lance-index/src/vector/pq*.rs) ------------------------------------ */
typedef struct {
  uint32_t num_sub_vectors; /* PQBuildParams (pq/builder.rs:27-59): 16; any divisor of d (every sub-vector width
                               d / num_sub_vectors has an exact device route) */
  uint32_t num_bits;        /* 8 or 4 */
  uint32_t max_iters;       /* 50 */
  uint32_t kmeans_redos;    /* 1 (PQ k-means has no balance bias: any value equals one run, see redos above) */
  uint64_t sample_rate;     /* 256 */
  const void* codebook;     /* user codebook to continue from, or NULL */
  uint64_t seed;
} lb2_pq_params;
void lb2_pq_params_default(lb2_pq_params* p);

/* PQBuildParams::build(data, distance_type) -> ProductQuantizer (pq/builder.rs:162-194):
 * codebook_out is the flat [M][2^nbits][d/M] layout of pq/utils.rs:59-76; iters_out[M] nullable.  Every M that
 * divides d trains on the device, at every sub-vector width d / M. */
lb2_status lb2_pq_train(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype,
                        lb2_metric metric, const lb2_pq_params* params, void* codebook_out,
                        uint32_t* iters_out);

/* ProductQuantizer::quantize / transform_impl (pq.rs:116-191,430).  When `centroids`
 * ([num_centroids][d]) and `part_ids` are given the residual (residual.rs:161-205) is fused: codes of
 * v - centroids[part]; a part id >= num_centroids is LB2_INVALID_ARG.
 * codes_out is row-major [n][M] (8-bit) or [n][M/2] (4-bit: byte i = code[2i+1] << 4 | code[2i],
 * pq.rs:168-173; 16 codewords per sub-space, M even).  Every sub-vector width d / M is encoded exactly (the
 * reference's 16-lane order from width 16 on). */
lb2_status lb2_pq_encode(const void* codebook, uint32_t num_sub_vectors, uint32_t num_bits,
                         uint32_t d, lb2_dtype dtype, lb2_metric metric, const void* centroids,
                         uint32_t num_centroids, const uint32_t* part_ids, const void* vectors, uint64_t n,
                         uint8_t* codes_out);

/* build_distance_table_l2 / _dot (pq/distance.rs:24-92): lut_out[M * 2^nbits] f32 */
lb2_status lb2_pq_build_lut(const void* codebook, uint32_t num_sub_vectors, uint32_t num_bits,
                            uint32_t d, lb2_metric metric, const float* query, float* lut_out);

/* compute_pq_distance (pq/distance.rs:109-144) on TRANSPOSED codes [M][n], as the reference's
 * storage holds them; PQDistCalculator::distance_all's Dot correction (pq/storage.rs:957-958)
 * is applied when metric == LB2_DOT. */
lb2_status lb2_pq_scan(const float* lut, uint32_t num_sub_vectors, uint32_t num_bits,
                       lb2_metric metric, const uint8_t* codes_transposed, uint64_t n,
                       float* dists_out);

/* 4-bit PQ: compute_pq_distance_4bit (pq/distance.rs:147-242) with PQDistCalculator::distance_all's
 * Dot correction.  lut = M x 16 f32 (lb2_pq_build_lut with num_bits = 4), codes_transposed = packed
 * [M/2][n].  The first min(max(200, k_hint), n) rows and the last n % 16 rows are exact f32 sums; the
 * rest is the reference's u8-quantised table with saturating u8 accumulation, dequantised.  k_hint =
 * the k of the search (DistCalculator::distance_all(k_hint), flat/index.rs:99). */
lb2_status lb2_pq_scan_4bit(const float* lut, uint32_t num_sub_vectors, lb2_metric metric,
                            const uint8_t* codes_transposed, uint64_t n, uint64_t k_hint,
                            float* dists_out);

/* FlatIndex::search fast path over a distance array (flat/index.rs:97-127): the k smallest
 * (distance, position) pairs; out sorted ascending by (distance, row id).  *count_out <= k. */
lb2_status lb2_flat_topk(const float* dists, const uint64_t* row_ids, uint64_t n, uint32_t k,
                         uint64_t* ids_out, float* dists_out, uint32_t* count_out);
/* The same with FlatIndex::search's range branch (flat/index.rs:100-115): only rows with
 * lower <= dist < upper (f32::total_cmp order; an absent bound is f32::MIN / f32::MAX, as the reference
 * unwraps it) are offered to the heap.  Both calls return exactly the SET the reference's BinaryHeap ends
 * with -- also when more rows tie at the k-th distance than fit (the heap's sift order is restated). */
lb2_status lb2_flat_topk_range(const float* dists, const uint64_t* row_ids, uint64_t n, uint32_t k,
                               int has_lower, float lower, int has_upper, float upper,
                               uint64_t* ids_out, float* dists_out, uint32_t* count_out);

/* flat_knn over one vector column (rust/lance/src/dataset/scanner.rs:3336-3411), batched over nq queries: the plan
 * of a nearest() query without an index (scanner.rs:2912-2941) and its unindexed half (knn_combined, :2946-3027).
 *   - every row's distance to the query is compute_distance's (lance-index/src/vector/flat.rs:94-150), with the
 *     function of the element type, the same arithmetic as the refine step: f32 L2 / dot, f16 L2 and bf16 in 16 f32
 *     lanes; f16 dot in 32 lanes (dot_scalar); u8 L2 / dot as exact integer sums; cosine within the f64 bound;
 *   - a row whose allow bit is clear (a null vector, or one the prefilter removes) is never returned;
 *   - the optional range keeps lower <= distance < upper (LanceFilterExec, scanner.rs:3342-3377; NaN fails it);
 *   - SortExec(_distance, _rowid).fetch(k) (scanner.rs:3450-3466): the k smallest (distance, row id) pairs in the
 *     f32 total order (a NaN the device produces is positive and sorts after +inf), ties at the k-th distance going
 *     to the smallest row ids.  (On x86 the reference turns inf - inf into a NEGATIVE NaN, which sorts first; such
 *     rows sort last here.)
 * vectors [n][d] and queries [nq][d] are of element type `dtype`; host or device memory (device rows are read in
 * place, host rows are staged in chunks).  Outputs [nq][k] ascending by (distance, row id); unused slots row id
 * UINT64_MAX, distance +inf; counts_out [nq] nullable.  LB2_INVALID_ARG: k == 0; LB2_UNSUPPORTED: k > 1024, or a d
 * whose tile of queries and rows does not fit the device's shared memory. */
typedef struct {
  uint32_t k;                    /* 1..1024 */
  const uint64_t* allow_bitmap;  /* nullable; (n+63)/64 words, bit i = row i (input order) may be returned.  The
                                    caller clears null vectors here too (Arrow validity AND prefilter). */
  uint32_t has_lower_bound, has_upper_bound;
  float lower_bound, upper_bound;
} lb2_flat_search_params;
lb2_status lb2_flat_search(const void* vectors, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                           const uint64_t* row_ids /* NULL = 0..n; must be distinct */, const void* queries,
                           uint64_t nq, const lb2_flat_search_params* p, uint64_t* row_ids_out, float* dists_out,
                           uint32_t* counts_out);
/* flat_knn for a batch of queries that differ in k, range and prefilter, as separate nearest() plans without an index
 * (use_index(false), tables without an index, ground truth with per-query filters: scanner.rs:2912-2941) reach the
 * column.  Row q of the outputs is bit for bit lb2_flat_search of query q alone with its own k, range and bitmap
 * (filter_bitmaps[params[q].filter], or no bitmap for UINT32_MAX): ids, distance bits and counts.  Rows are
 * [nq][k_stride]; slots k_q .. k_stride - 1 hold UINT64_MAX / +inf; counts_out is nullable.  Each bitmap ((n+63)/64
 * words, host or device, a NULL entry admits every row) is staged once however many queries name it.  Every query's
 * k and filter reach the scan kernel from a per-query table on the device, so the number of kernel launches depends
 * on n, nq and the chunking of host rows, not on how many distinct (k, range, filter) sets the batch holds.
 * Refused before anything is written: what lb2_flat_search refuses for any query (the message names the query), and
 * with LB2_INVALID_ARG k_stride below the largest k, and a filter index that is neither below num_filters nor
 * UINT32_MAX. */
typedef struct {
  uint32_t k;                          /* 1..1024 */
  uint32_t filter;                     /* index into filter_bitmaps[], UINT32_MAX = no filter */
  uint32_t has_lower_bound, has_upper_bound;
  float lower_bound, upper_bound;
} lb2_flat_query_params;
lb2_status lb2_flat_search_batch(const void* vectors, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                                 const uint64_t* row_ids /* NULL = 0..n; must be distinct */, const void* queries,
                                 uint64_t nq, const lb2_flat_query_params* params /* [nq] */,
                                 const uint64_t* const* filter_bitmaps /* [num_filters] */, uint32_t num_filters,
                                 uint32_t k_stride, uint64_t* row_ids_out /* [nq][k_stride] */, float* dists_out,
                                 uint32_t* counts_out);

/* IvfTransformer::transform for IVF_PQ (lance-index/src/vector/ivf.rs:188-236,357): for a batch,
 * [normalise if cosine] -> partition id -> residual -> PQ code, in one pass over the vectors.
 * `metric` is the index metric: it selects the partition assignment and whether residuals are taken
 * (not for dot, PQBuildParams::use_residual); the PQ codes are L2 codes in every case, because the
 * index builder trains its quantizer with DistanceType::L2 (rust/lance/src/index/vector/builder.rs:460).
 * valid_out[i] = 0 marks rows KeepFiniteVectors would drop (transform.rs:112-159).  Any num_sub_vectors that divides
 * d, as lb2_pq_encode; so lb2_index_transform and lb2_index_optimize maintain IVF_PQ and IVF_HNSW_PQ indexes of every
 * sub-vector width, reference-built ones included. */
lb2_status lb2_ivfpq_transform(const void* centroids, uint32_t k, const void* codebook,
                               uint32_t num_sub_vectors, uint32_t num_bits, uint32_t d,
                               lb2_dtype dtype, lb2_metric metric, const void* vectors, uint64_t n,
                               uint32_t* part_out, uint8_t* codes_out, uint8_t* valid_out);

/* ---- device-resident index: IVFIndex<FlatIndex, ProductQuantizer> ----------------------------
 * (rust/lance/src/index/vector/ivf/v2.rs:104; storage lance-index/src/vector/pq/storage.rs:151) */
lb2_status lb2_index_create(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                            lb2_metric metric, const void* codebook, uint32_t num_sub_vectors,
                            uint32_t num_bits, lb2_index** out);
/* num_bits = 8 or 4 (4: 16 codewords per sub-space, codes are [n][M/2] packed bytes, M even; searches
 * use compute_pq_distance_4bit's flat-rows + u8-quantised-table rule with k_hint = k, and exact
 * row-by-row distances when a prefilter is given, as the reference does).
 * load the (row_id, __ivf_part_id, __pq_code) shuffle output (builder.rs:685-937): rows are grouped
 * by partition on the device (stable, i.e. input order inside a partition). Replaces prior content. */
lb2_status lb2_index_load(lb2_index* index, const uint32_t* part_ids, const uint8_t* codes,
                          const uint64_t* row_ids /* NULL = 0..n */, uint64_t n);
/* IVFIndex::find_partitions + search_in_partition for a BATCH of queries, then the global merge
 * SortExec(_distance, _rowid).fetch(k) (v2.rs:455-500, rust/lance/src/dataset/scanner.rs:3450-3466).
 * Outputs [nq][k]; unused slots: row id = UINT64_MAX, distance = +inf; counts_out[nq] nullable. */
lb2_status lb2_index_search(lb2_index* index, const void* queries, uint64_t nq, uint32_t k,
                            uint32_t nprobes, uint64_t* row_ids_out, float* dists_out,
                            uint32_t* counts_out);
/* The same, followed by the refine step of the reference's plan (Take vectors + flat KNN re-rank,
 * rust/lance/src/dataset/scanner.rs:2884-2905; lance-index/src/vector/flat.rs:95-148): the index
 * returns k * refine_factor candidates, their EXACT distances to the query are recomputed from the
 * raw column `vectors` ([>= max row id + 1][d], element type = the index's dtype, row id = row
 * number; device-resident for speed) with the index's true metric, and the k best by
 * (distance, row id) are returned.  k * refine_factor <= 1024. */
lb2_status lb2_index_search_refine(lb2_index* index, const void* vectors, uint64_t num_vectors,
                                   const void* queries, uint64_t nq, uint32_t k, uint32_t nprobes,
                                   uint32_t refine_factor, uint64_t* row_ids_out, float* dists_out,
                                   uint32_t* counts_out);
/* Extended search: prefilter and refine in one call.
 * Prefilter = the reference's PreFilter / RowIdMask (lance-index/src/prefilter.rs:27-51): when the
 * mask is not empty FlatIndex::search visits the partition row by row and skips rows for which
 * RowIdMask::selected(row_id) is false BEFORE they can enter the heap (flat/index.rs:129-165).
 * Here the mask is a bitmap over STORAGE positions (the order of lb2_index_export's row_ids, i.e.
 * partition-local offset + part_offsets[p]); bit i (word i/64, bit i%64) set = row may be returned.
 * lb2_index_row_mask builds it on the device from the RowIdMask's allow / block lists.
 * allow_bitmap NULL = the fast unfiltered path. Host or device pointer, (num_rows+63)/64 words. */
typedef struct {
  uint32_t k;
  uint32_t nprobes;
  uint32_t refine_factor;       /* 0 = no refine step */
  const void* refine_vectors;   /* raw column, see lb2_index_search_refine; required when refine_factor > 0 */
  uint64_t num_vectors;
  const uint64_t* allow_bitmap; /* nullable */
  /* range query (Query::lower_bound / upper_bound, lance-index/src/vector.rs:83-86): inside a partition
   * only rows with lower <= _distance < upper enter the top-k (flat/index.rs:100-115, index distances);
   * with refine the plan filters the exact distances the same way afterwards (scanner.rs:3342-3377) */
  uint32_t has_lower_bound, has_upper_bound;
  float lower_bound, upper_bound;
} lb2_search_params;
lb2_status lb2_index_search_ex(lb2_index* index, const void* queries, uint64_t nq,
                               const lb2_search_params* params, uint64_t* row_ids_out, float* dists_out,
                               uint32_t* counts_out);
/* Search with a minimum and a maximum number of probes, as ANNIvfSubIndexExec runs a query
 * (rust/lance/src/io/exec/knn.rs:714-1130).  lb2_index_search_ex is the case minimum == maximum
 * (Scanner::nprobes, scanner.rs:1103-1111); a plain nearest() query is minimum 1, maximum None
 * (scanner.rs:1064-1077).  Per query, with kc = k * max(1, refine_factor) and K partitions:
 *   - P = the L = min(maximum or K, K) nearest partitions, ascending by (distance, id);
 *   - early pruning (knn.rs:1117-1130): the count of P's distances <= d0 * f (Rust's partition_point),
 *     f = 0.6 / 7 / 81 for k = 1 / 2..=10 / > 10; min_np = min(max(minimum, pruned), L) (adjust_probes,
 *     knn.rs:1108-1115);
 *   - c_p = min(kc, rows of p the allow bitmap and the range admit) (flat/index.rs:97-165);
 *     found0 = min(k, sum of c over P[0, min_np)) (initial_search, knn.rs:837-882);
 *   - the search stops there if L <= min_np or found0 >= k;
 *   - shortcut (knn.rs:746-783): with max_len and mask_ids given and found0 < max_len <= k, the mask ids
 *     the initial search did not return are added at +inf, and nothing more is searched;
 *   - late search (knn.rs:714-835): late partition t = P[min_np + t] is searched while
 *     found0 + sum of c over the late partitions u <= t - late_width is below min(k, max_len if given).
 *     In the reference how many late partitions run depends on when futures complete; this rule is
 *     take_while ahead of buffered(late_width) with in-order completion (DESIGN.md section 2).
 * The result is the top kc by (distance, row id) of the partitions searched and the shortcut rows, then
 * refine and the range filter as in lb2_index_search_ex (shortcut rows get exact distances there).
 * nprobes_out[q] (nullable) = partitions searched (the reference's partitions_searched).
 * The ranking sorts all K centroid distances per query whatever the number of probes.  With a range
 * bound c_p depends on the distances, so P[0, L) is scanned and cut afterwards: such a search costs
 * as much as one with nprobes = L.
 * LB2_INVALID_ARG: sp->nprobes != 0, minimum_nprobes == 0, maximum_nprobes < minimum_nprobes,
 * late_width == 0, or max_len / mask_ids without sp->allow_bitmap.  LB2_UNSUPPORTED on a thread with a
 * communicator of more than one rank (each rank's c_p would count only its own shard). */
typedef struct {
  uint32_t minimum_nprobes;   /* Query::minimum_nprobes, >= 1 */
  uint32_t maximum_nprobes;   /* Query::maximum_nprobes; 0 = None (every partition); else >= minimum */
  uint32_t late_width;        /* partitions the late search keeps in flight, >= 1 (get_num_compute_intensive_cpus()) */
  uint32_t has_max_len;       /* RowIdMask::max_len() is Some (there is an allow list) */
  uint64_t max_len;
  const uint64_t* mask_ids;   /* RowIdMask::iter_ids(), ascending; NULL = not iterable (no shortcut) */
  uint64_t num_mask_ids;
} lb2_probe_params;
lb2_status lb2_index_search_probed(lb2_index* index, const void* queries, uint64_t nq,
                                   const lb2_search_params* sp /* nprobes must be 0 */,
                                   const lb2_probe_params* pp, uint64_t* row_ids_out, float* dists_out,
                                   uint32_t* counts_out, uint32_t* nprobes_out /* nullable, [nq] */);
/* A batch of queries with their own parameters, as separate nearest() plans reach the index (each its own Query,
 * lance-index/src/vector.rs:72-116, and its own PreFilter mask, prefilter.rs:27-51), searched in one device pass.
 * Row q of the output is bit for bit what the single-parameter call returns for query q alone with q's parameters
 * and filter: lb2_index_search_ex for a fixed nprobes (nprobes_out[q] = min(nprobes, K)),
 * lb2_index_search_probed for nprobes = 0 (its minimum / maximum nprobes, the filter's max_len and mask_ids, and
 * late_width), and lb2_index_search_hnsw when ef is set on an IVF_HNSW_* index.  Rows are [nq][k_stride]; slots
 * k_q .. k_stride - 1 hold UINT64_MAX / +inf.  counts_out [nq] and nprobes_out [nq] are nullable.  Filters are
 * staged once each and shared by every query that names them; refine_vectors / num_vectors are the raw column of
 * every query with refine_factor > 0 (as lb2_search_params); late_width is the probe rule's (>= 1).
 * Every query's own k, probes, refine factor, range, filter and ef reach the scan kernels from a per-query table on
 * the device, so the number of kernel launches depends on the routes the batch needs, not on how many parameter
 * sets or filters it holds.
 * Refused before anything is launched or written: a query its own call would refuse (that call's status; the
 * message names the query), and with LB2_INVALID_ARG: k_stride below the largest k, a filter index that is neither
 * below num_filters nor UINT32_MAX, ef on a non-HNSW index, refine_factor > 0 without refine_vectors, late_width 0.
 * LB2_UNSUPPORTED: a thread whose communicator has more than one rank. */
typedef struct {
  const uint64_t* allow_bitmap; /* storage positions, as lb2_index_row_mask builds it; host or device */
  uint32_t has_max_len;         /* RowIdMask::max_len(): used by minimum / maximum nprobes queries only */
  uint64_t max_len;
  const uint64_t* mask_ids;     /* ditto; NULL = not iterable */
  uint64_t num_mask_ids;
} lb2_query_filter;
typedef struct {
  uint32_t k;                                /* >= 1 */
  uint32_t nprobes;                          /* > 0: fixed probes (search_ex); 0: minimum / maximum below */
  uint32_t minimum_nprobes, maximum_nprobes; /* as lb2_probe_params */
  uint32_t refine_factor;                    /* 0 = no refine */
  uint32_t filter;                           /* index into filters[], UINT32_MAX = no prefilter */
  uint32_t ef;                               /* IVF_HNSW_* only; 0 = k' + k' / 2 */
  uint32_t has_lower_bound, has_upper_bound;
  float lower_bound, upper_bound;
} lb2_query_params;
lb2_status lb2_index_search_batch(lb2_index* index, const void* queries, uint64_t nq,
                                  const lb2_query_params* params /* [nq] */, const lb2_query_filter* filters,
                                  uint32_t num_filters, const void* refine_vectors, uint64_t num_vectors,
                                  uint32_t late_width, uint32_t k_stride, uint64_t* row_ids_out /* [nq][k_stride] */,
                                  float* dists_out, uint32_t* counts_out, uint32_t* nprobes_out);
/* A refined batch over rows the caller takes, as the reference plans a refined query: the ANN node returns _rowid
 * candidates, the scanner takes their vectors (self.take(ann_node, vector_projection)) and runs flat_knn over only
 * those rows (rust/lance/src/dataset/scanner.rs:2884-2905).  Row ids are Lance _rowid values (fragment << 32 |
 * offset, or stable row ids), so the raw column is never indexed by them; lb2_index_search_batch's refine_vectors
 * is a dense column indexed by row id and cannot serve such a table.
 *
 * lb2_index_search_candidates: the index half.  Row q of cand_ids_out / cand_dists_out [nq][kc_stride] is exactly the
 * list lb2_index_search_batch re-ranks for query q: k'_q = k_q * max(1, refine_factor_q) entries (k_q without
 * refine), index distances in the merge's order, probe-rule shortcut rows at +inf included; slots from
 * cand_counts_out[q] on hold UINT64_MAX / +inf.  nprobes_out (nullable) is lb2_index_search_batch's.  k and
 * refine_factor stay separate, since the probe rule uses k as well as k' (early pruning, found0, the stop test):
 * a query with k' and refine factor 0 is not the same list.  With distinct_ids_out (capacity nq * kc_stride),
 * *num_distinct_out = m receives the number of distinct row ids over every valid slot of the batch, distinct_ids_out
 * those ids ascending (entries m.. hold UINT64_MAX), and positions_out [nq][kc_stride] the index of each slot's id in
 * that list (UINT64_MAX for an unused slot), so each row is taken once, in row-address order.  The three go
 * together, each host or device.  Refused as lb2_index_search_batch refuses, except that refine_factor > 0 needs no
 * vectors, and with LB2_INVALID_ARG kc_stride below the largest k'. */
lb2_status lb2_index_search_candidates(lb2_index* index, const void* queries, uint64_t nq,
                                       const lb2_query_params* params /* [nq] */, const lb2_query_filter* filters,
                                       uint32_t num_filters, uint32_t late_width, uint32_t kc_stride,
                                       uint64_t* cand_ids_out /* [nq][kc_stride] */, float* cand_dists_out,
                                       uint32_t* cand_counts_out, uint32_t* nprobes_out /* nullable */,
                                       uint64_t* distinct_ids_out /* nullable, capacity nq * kc_stride */,
                                       uint64_t* num_distinct_out,
                                       uint64_t* positions_out /* [nq][kc_stride]; required iff distinct_ids_out */);
/* lb2_index_refine_taken: the exact re-rank, flat_knn over the taken rows (scanner.rs:2884-2905, flat.rs:95-148) with
 * the arithmetic of lb2_index_search_batch's refine: the index's true metric on the original (not normalised) query
 * in the index's element type, the k best by (distance, row id) under the f32 total order, then the query's range
 * (scanner.rs:3342-3377).  Of params[q] only k, refine_factor and the bounds are read.  Candidate c of query q is
 * the row taken[positions[q][c]] ([m][d], the index's element type; host pageable, pinned or device) with row id
 * cand_ids[q][c]; a position >= m scores NaN (sorted last), as a row id past num_vectors does there.  A query with
 * refine factor 0 returns the first k of its list as they are.  So candidates, a take of distinct_ids, and this
 * call equal lb2_index_search_batch with the column as refine_vectors bit for bit.  Rows are [nq][k_stride], slots
 * k_q.. UINT64_MAX / +inf; counts_out is nullable.  Only the m taken rows cross to the device; host rows past
 * 512 MB are staged in query slabs, each slab's own rows at a time.
 * LB2_INVALID_ARG: k == 0, k' above kc_stride, k_stride below the largest k, positions NULL with a refine query,
 * taken NULL with m > 0.  LB2_UNSUPPORTED: k' > 1024. */
lb2_status lb2_index_refine_taken(lb2_index* index, const void* queries /* [nq][d], the index's element type */,
                                  uint64_t nq, const lb2_query_params* params, uint32_t kc_stride,
                                  const uint64_t* cand_ids, const float* cand_dists, const uint32_t* cand_counts,
                                  const void* taken /* [m][d], the index's element type */, uint64_t m,
                                  const uint64_t* positions /* [nq][kc_stride] */, uint32_t k_stride,
                                  uint64_t* row_ids_out /* [nq][k_stride] */, float* dists_out, uint32_t* counts_out);
/* knn_combined (rust/lance/src/dataset/scanner.rs:2946-3027): a nearest() query on an index that does not yet cover
 * every row of its table.  The reference takes the raw vectors of the ANN rows and re-scores them exactly, runs a
 * flat KNN with the index metric over the unindexed rows (with the query's prefilter), and sorts the union by
 * (_distance, _rowid), range-filtered, fetched to k.  Since the refine step's distances already are exact, this is:
 *   1. the index search (lb2_index_search_ex, or lb2_index_search_probed when pp != NULL) with refine factor
 *      max(1, sp->refine_factor);
 *   2. lb2_flat_search over *u with the index's metric, sp->k and sp's range, on the original (not normalised)
 *      query;
 *   3. the two k-lists of every query merged by (distance, row id).
 * Plan selection stays with the caller: with fast_search, or without unindexed fragments, the plain index search
 * answers; unindexed fragments whose rows are all filtered or deleted still take this call (u->n rows with clear
 * allow bits, or u->n == 0), because the ANN rows are re-scored either way.
 * Queries are of the index's element type.  LB2_INVALID_ARG: k == 0, sp->refine_vectors NULL, u or u->row_ids NULL,
 * nprobes_out without pp, and what lb2_index_search_ex / _probed refuse.  LB2_UNSUPPORTED: k * max(1, refine_factor)
 * > 1024, what lb2_flat_search refuses, and a thread whose communicator has more than one rank (as
 * lb2_index_search_probed). */
typedef struct {
  const void* vectors;           /* [n][d], the index's element type */
  uint64_t n;
  const uint64_t* row_ids;       /* required: the unindexed rows' _rowid values */
  const uint64_t* allow_bitmap;  /* nullable, over these rows: the query filter + null vectors */
} lb2_unindexed_rows;
lb2_status lb2_index_search_combined(lb2_index* index, const void* queries, uint64_t nq,
                                     const lb2_search_params* sp /* refine_vectors required; nprobes 0 with pp */,
                                     const lb2_probe_params* pp /* nullable */, const lb2_unindexed_rows* u,
                                     uint64_t* row_ids_out, float* dists_out, uint32_t* counts_out,
                                     uint32_t* nprobes_out /* nullable; requires pp */);
/* knn_combined for a mixed batch (scanner.rs:2946-3027): lb2_index_search_batch's per-query parameters over an index
 * that does not cover every row, in one call.  Row q is what lb2_index_search_combined defines for query q alone:
 *   1. the index half: lb2_index_search_batch's search of q (its probes, range, filter and ef) with refine factor
 *      max(1, refine_factor_q) against refine_vectors;
 *   2. the flat half: lb2_flat_search_batch over u's rows with the index metric, k_q and q's range on the original
 *      (not normalised) query, admitting the rows of u->filter_bitmaps[filter_q] (u->rows.allow_bitmap for a query
 *      without a filter);
 *   3. the two lists merged by (distance, row id), first k_q.
 * For a query without ef, row q and nprobes_out[q] equal lb2_index_search_combined of q alone bit for bit (with a
 * fixed nprobes, or with the probe rule and the filter's max_len and mask_ids for nprobes 0).  A query with ef
 * (IVF_HNSW_*) equals the merge of lb2_index_search_batch (ef, refine factor max(1, rf)) and lb2_flat_search.  The
 * unindexed rows are read once for the whole batch.  Rows are [nq][k_stride], slots k_q.. UINT64_MAX / +inf;
 * counts_out and nprobes_out are nullable.
 * Refused before anything is written: what lb2_index_search_batch and lb2_flat_search_batch refuse, and with
 * LB2_INVALID_ARG refine_vectors NULL, u or u->rows.row_ids NULL, u->rows.vectors NULL with n > 0, and
 * u->filter_bitmaps NULL with num_filters > 0.  LB2_UNSUPPORTED: a thread whose communicator has more than one
 * rank. */
typedef struct {
  lb2_unindexed_rows rows;                /* the unindexed rows; rows.allow_bitmap serves queries without a filter */
  const uint64_t* const* filter_bitmaps;  /* [num_filters]: validity AND filter f over these rows; NULL entry = all */
} lb2_unindexed_batch;
lb2_status lb2_index_search_combined_batch(lb2_index* index, const void* queries, uint64_t nq,
                                           const lb2_query_params* params /* [nq] */, const lb2_query_filter* filters,
                                           uint32_t num_filters, const void* refine_vectors, uint64_t num_vectors,
                                           uint32_t late_width, const lb2_unindexed_batch* u, uint32_t k_stride,
                                           uint64_t* row_ids_out /* [nq][k_stride] */, float* dists_out,
                                           uint32_t* counts_out, uint32_t* nprobes_out);
/* Incremental update of an IVF_PQ index (SURVEY 8f-4).
 * The reference expresses an optimize step as per-partition AssignOp::Add / AssignOp::Remove lists against a new
 * centroid set (rust/lance/src/index/vector/builder.rs:1219-1333 split_partition_impl, :1476-1530
 * join_partition_impl, :1534-1650 build_assign_batch) and merges them with the stored partitions.  This call is that
 * merge for lists the caller built (lb2_index_split / lb2_index_join below make the lists of a split or join
 * themselves) and returns a NEW index:
 *   - new_centroids [new_k][d] in the model's element type (NULL = unchanged, then new_k must equal the old k);
 *   - part_map[old_k] (nullable = identity): new partition id of every old partition, UINT32_MAX = the partition's
 *     rows are dropped (split: the split partition's rows come back through the add list; join: ids after the
 *     deleted partition shift down by one);
 *   - remove_row_ids (sorted ascending): old rows to drop (AssignOp::Remove; also deletions);
 *   - add_*: n_add rows already transformed (partition id, PQ code, row id); inside a partition the surviving old
 *     rows keep their order and the added rows follow in list order.
 * Appending new data to an index (optimize without retraining) is the add list alone. */
lb2_status lb2_index_update(const lb2_index* old_index, const void* new_centroids, uint32_t new_k,
                            const uint32_t* part_map, const uint32_t* add_part_ids, const uint8_t* add_codes,
                            const uint64_t* add_row_ids, uint64_t n_add, const uint64_t* remove_row_ids,
                            uint64_t n_remove, lb2_index** out);
/* ---- optimize / remap of every index kind ----------------------------------------------------------------------
 * lb2_index_transform: IvfTransformer::transform with the index's own model (lance-index/src/vector/ivf.rs:149-328),
 * the "new rows" half of shuffle_data during an optimize (rust/lance/src/index/vector/builder.rs:685-829).  vectors
 * [n][d] in the index's element type; per row the partition id, the payload the kind stores ([n][row_bytes]) and
 * valid (0 = a row the kind's build drops: KeepFiniteVectors, transform.rs:112-159).  The payload is exactly what the
 * kind's build stores for the same row:
 *   IVF_PQ   the codes of lb2_ivfpq_transform (row_bytes M, or M / 2 for 4-bit codes);
 *   IVF_FLAT the row, normalised under cosine, in the stored element type (u8 columns held as f32; row_bytes d * 4
 *            or d * 2);
 *   IVF_SQ   scale_to_u8 of the (normalised) row with the index's bounds (sq.rs:263-277; row_bytes d);
 *   IVF_RQ   the codes and factors of lb2_ivfrq_transform (row_bytes d * num_bits / 8).
 * The graph kinds transform as their base kind does.  Every output may be NULL; add_out / scale_out must be NULL
 * unless the index is IVF_RQ. */
lb2_status lb2_index_transform(const lb2_index* index, const void* vectors, uint64_t n, uint32_t* part_out,
                               uint8_t* payload_out, float* add_out, float* scale_out, uint8_t* valid_out);
/* lb2_index_optimize: the merge of IvfIndexBuilder::build_partitions / take_partition_batches (builder.rs:685-935)
 * composed with IvfIndexBuilder::remap (builder.rs:256-359), for every kind; returns a NEW index of the old one's
 * kind.  In this order:
 *   1. the old rows in storage order, minus the ids in remove_row_ids and the partitions part_map sends to
 *      UINT32_MAX; the rest move to part_map[p] (nullable = identity);
 *   2. the add list appended (payload as lb2_index_transform writes it; IVF_RQ: with its factors, required);
 *   3. a stable grouping by partition: inside a partition the surviving old rows first, then the added rows in list
 *      order (lb2_index_update's order);
 *   4. the row-id mapping applied to every row, old and added, without changing the order (storage.remap,
 *      pq/storage.rs:499-540, bq/storage.rs:661): an id mapped to UINT64_MAX (None) is dropped, an id mapped to a
 *      value is rewritten, an id that is not in remap_old_ids is kept as it is.
 * The model stays: codebook, SQ bounds and RQ rotation; new_centroids (in the model's element type) replaces the
 * centroids, and new_k must equal the old k without them.  As with lb2_index_update the caller is responsible for the
 * centroids: an old partition whose centroid changes must come back through the add list (removed from the old rows
 * by part_map or remove_row_ids), because its PQ residual codes or RQ factors were computed against the old centroid.
 * Graphs (IVF_HNSW_*): the new index has one per partition iff the old one has, with the old max_level, m and
 * ef_construction.  A new partition whose rows are all the rows of one old partition q, in the same order, with none of
 * q's rows removed or remapped to None and nothing added, keeps q's graph verbatim (every node id and distance depends
 * only on the partition's payload sequence; the reference's rebuild, hnsw/builder.rs:777-785, gives the same graph
 * up to its unseeded level draws).  Every other partition with at least 2 rows gets the graph of the kind's build over
 * its new storage, its level draws keyed by (seed, new partition id, node), inserted in rounds of insert_batch (0: the
 * B the old index was built with, 1 for a loaded graph); the new index records the B it used.  insert_batch above
 * 65 536 is LB2_INVALID_ARG for a graph kind; the other kinds ignore it.
 * LB2_INVALID_ARG before the new index is made: remap_old_ids not strictly ascending, a graph kind's insert_batch
 * above 65 536, a part id or part_map entry at or above new_k, missing or extra RQ factors, a changed new_k without new_centroids, more than 2^32 - 1 rows.  Under a
 * communicator the non-graph kinds merge each shard's rows (as lb2_index_update); the graph kinds return
 * LB2_UNSUPPORTED with more than one rank. */
typedef struct {
  const void* new_centroids; /* [new_k][d], nullable */
  uint32_t new_k;
  const uint32_t* part_map;  /* [old k], nullable = identity; UINT32_MAX = drop the old partition's rows */
  const uint32_t* add_part_ids;
  const uint8_t* add_payload; /* [n_add][row_bytes], as lb2_index_transform writes it */
  const float* add_rq_add;    /* IVF_RQ: required with n_add > 0; other kinds: must be NULL */
  const float* add_rq_scale;
  const uint64_t* add_row_ids;
  uint64_t n_add;
  const uint64_t* remove_row_ids; /* sorted ascending */
  uint64_t n_remove;
  const uint64_t* remap_old_ids; /* strictly ascending */
  const uint64_t* remap_new_ids; /* UINT64_MAX = None: the row is dropped */
  uint64_t n_remap;
  uint64_t seed;                 /* the level draws of the graphs that are rebuilt */
  uint32_t insert_batch;         /* B of the graphs that are rebuilt (IVF_HNSW_SQ's rounds); 0: the old index's B */
} lb2_optimize_params;
lb2_status lb2_index_optimize(const lb2_index* old_index, const lb2_optimize_params* p, lb2_index** out);
/* ---- partition split and join (optimize_indices / remap, rust/lance/src/index/vector/builder.rs:1152-1814) -------
 * The host owns the dataset: it fetches a partition's raw rows by row id (load_partition_raw_vectors, :1118-1147);
 * every other step is one of these calls.
 * lb2_index_partition_to_split (should_split, :1152-1176): a partition's size is its stored rows plus the rows of
 *   new_part_ids (the add list's partitions); the largest partition strictly above MAX_PARTITION_SIZE_FACTOR (4) x
 *   target, the first of equal sizes.  lb2_index_partition_to_join (should_join, :1343-1394): a partition's size is
 *   its rows the remap (strictly ascending old ids; UINT64_MAX = None) does not map to None; the smallest strictly
 *   below MIN_PARTITION_SIZE_PERCENT (25) x target / 100, never with one partition.  target is
 *   IndexType::target_partition_size (lance-index/src/lib.rs:284-295): 4096 for IVF_FLAT, 8192 for IVF_PQ, IVF_SQ and
 *   IVF_RQ, 1 Mi for the graph kinds.  *part = UINT32_MAX when none qualifies.
 * lb2_index_reassign_candidates (select_reassign_candidates_impl, :1788-1814): every centroid ranked by
 *   lb2_distance_batch(c_part, centroids) under the index metric, the first min(65, K) by (distance, id), `part`
 *   dropped, min(65, K) - 1 kept: ids[64], *count.  The host fetches these partitions' raw rows for a split.
 * lb2_index_split (split_partition_impl, :1219-1333): returns a NEW index of K + 1 partitions.
 *   - c1, c2: lb2_kmeans_train(k = 2) on the first 512 of the partition's raw rows (normalised under cosine, trained
 *     with L2), max_iters 50, redos 1, tolerance 1e-4, no balance factor, seeded by opt.seed; c1 replaces centroid
 *     `part`, c2 is centroid K.
 *   - d0 / d1 / d2 = lb2_distance_batch(c, row) on the raw rows; candidate distances lb2_distance_batch(row, c) (the
 *     orientation matters for cosine).  A row of the split partition (assign_vectors with deleted_original_partition,
 *     :1690-1749) whose d0 <= d1 && d0 <= d2 goes to the first minimum over the candidates by total_cmp when that is
 *     <= d1 and <= d2 (reassign_vectors, :1754-1785); every other row goes to c1 when d1 <= d2, else to c2.  A row of
 *     a candidate partition stays when its d0 (to its own centroid) is <= d1 and <= d2, else it moves to c1 or c2 by
 *     the same rule.  With K = 1 there are no candidates and such a row takes the c1 / c2 rule (the reference
 *     unwraps an empty minimum there).
 *   - the result is lb2_index_optimize of: the old rows without the split partition's and the moved rows; opt's add
 *     list without its rows of `part` and the moved rows; then the moved rows in add-op order (the split rows in
 *     ascending row id, then the candidate partitions in candidate order), with the payload of
 *     lb2_index_transform under the new centroids -- IVF_PQ residuals to the decided partition, IVF_RQ codes and
 *     factors from its nearest new centroid (ivf.rs:301-304) stored in the decided partition.
 *   - one stated difference (DESIGN.md section 2): every row is placed once, at its decision; the reference's
 *     build_partitions also keeps the split partition's old copies in partition `part`.
 *   A split partition without raw rows changes nothing but opt (:1184-1189).  LB2_INVALID_ARG: a bad part, one raw
 *   row, row ids not ascending within a group or candidate groups out of candidate order, a raw row that is not a row
 *   (stored or in opt's add list) of the partition it is passed for, a raw row the transform would drop (a non-finite
 *   element, a zero row under cosine; a moved row also when the new model's transform finds no finite distance to
 *   any centroid, ivf.rs:166), an add list without its partition ids, payload or row ids, opt.new_centroids / part_map / remap set.  LB2_UNSUPPORTED: u8 columns (the reference's
 *   arrow_batch_func cannot take u8 rows against its f32 centroids: l2.rs:205-266), more than one rank.
 * lb2_index_join (join_partition_impl, :1476-1530): a NEW index of K - 1 partitions: centroid `part` deleted, every
 *   raw row of `part` to the first minimum over its candidates (ids above `part` shift down by one), composed with the
 *   removals and the remap as lb2_index_optimize applies them (to old and moved rows alike). */
typedef struct {
  uint32_t part;
  const void* vectors;             /* [n][d] the partition's raw rows, the index's element type */
  const uint64_t* row_ids;         /* [n] ascending */
  uint64_t n;
  const void* cand_vectors;        /* [n_cand][d] the candidate partitions' raw rows */
  const uint64_t* cand_row_ids;    /* [n_cand] */
  const uint32_t* cand_part_ids;   /* [n_cand] grouped in candidate order, ascending row ids within a group */
  uint64_t n_cand;
  lb2_optimize_params opt;         /* add list, removals, seed, insert_batch; new_centroids, part_map and the remap
                                      NULL (the split's own), new_k ignored */
  void* new_centroids_out;         /* nullable: [new k][d] in the model type */
  uint32_t* dest_out;              /* nullable: [n + n_cand] new partition of each raw row, UINT32_MAX = stays */
} lb2_split_params;
typedef struct {
  uint32_t part;
  const void* vectors;             /* [n][d] the partition's raw rows */
  const uint64_t* row_ids;         /* [n] ascending */
  uint64_t n;
  const uint64_t* remove_row_ids;  /* sorted ascending */
  uint64_t n_remove;
  const uint64_t* remap_old_ids;   /* strictly ascending */
  const uint64_t* remap_new_ids;   /* UINT64_MAX = None */
  uint64_t n_remap;
  uint64_t seed;
  uint32_t insert_batch;
  uint32_t* dest_out;              /* nullable: [n] new partition of each raw row */
} lb2_join_params;
lb2_status lb2_index_partition_to_split(const lb2_index* index, const uint32_t* new_part_ids, uint64_t n_new,
                                        uint32_t* part);
lb2_status lb2_index_partition_to_join(const lb2_index* index, const uint64_t* remap_old_ids,
                                       const uint64_t* remap_new_ids, uint64_t n_remap, uint32_t* part);
lb2_status lb2_index_reassign_candidates(const lb2_index* index, uint32_t part, uint32_t* ids_out /*[64]*/,
                                         uint32_t* count);
lb2_status lb2_index_split(const lb2_index* old_index, const lb2_split_params* p, lb2_index** out);
lb2_status lb2_index_join(const lb2_index* old_index, const lb2_join_params* p, lb2_index** out);
/* Asynchronous search (SURVEY 8b "Threading": `_async` variants taking a stream/event).  Same
 * arguments and results as lb2_index_search_ex, but the call only ENQUEUES the work on `cuda_stream`
 * (cudaStream_t; NULL = the calling thread's current library stream) and returns: probe selection, LUT
 * build, scan, tie replay, merge and the optional refine run in stream order, with no host round trip.
 * Buffers must be device memory or pinned host memory and stay valid until the stream reaches the end of
 * the search; if `done_event` (cudaEvent_t) is not NULL it is recorded there.  Errors detected while
 * enqueueing are returned; the results are defined once the stream (or the event) has completed. */
lb2_status lb2_index_search_async(lb2_index* index, const void* queries, uint64_t nq,
                                  const lb2_search_params* params, uint64_t* row_ids_out, float* dists_out,
                                  uint32_t* counts_out, void* cuda_stream, void* done_event);
/* bitmap_out[(num_rows+63)/64]: bit i = RowIdMask::selected(row id stored at position i)
 * (lance-core/src/utils/mask.rs:84-93: in the allow list if there is one, and not in the block
 * list if there is one). Lists are sorted ascending (RoaringTreemap order); has_* = list present. */
lb2_status lb2_index_row_mask(const lb2_index* index, const uint64_t* allow_ids, uint64_t n_allow,
                              int has_allow, const uint64_t* block_ids, uint64_t n_block, int has_block,
                              uint64_t* bitmap_out);
lb2_status lb2_index_info(const lb2_index* index, uint32_t* k, uint32_t* d, uint32_t* num_sub_vectors,
                          uint32_t* num_bits, uint64_t* num_rows);
/* export for the host to write index files: any pointer may be NULL.
 * part_offsets[k+1]; codes [num_rows][M] and row_ids [num_rows] in partition order. */
lb2_status lb2_index_export(const lb2_index* index, void* centroids_out, void* codebook_out,
                            uint64_t* part_offsets_out, uint8_t* codes_out, uint64_t* row_ids_out);
/* One partition in the layout the reference's storage holds and merge_partitions writes (`__pq_code` with
 * "transposed": true -- lance-index/src/vector/pq/storage.rs:52-67,430-450; rust/lance/src/index/vector/builder.rs:
 * 938-1079): codes column-major [code bytes per row][n_p], row ids [n_p].  Call with NULL outputs first to get
 * *num_rows_out.  tests/: the bytes equal the reference's own fixture test_data/v0.27.1/pq_in_schema. */
lb2_status lb2_index_export_partition(const lb2_index* index, uint32_t partition, uint8_t* codes_transposed_out,
                                      uint64_t* row_ids_out, uint64_t* num_rows_out);
/* ---- a whole index in the reference's storage layout (every kind) ----------------------------------------------
 * The columns merge_partitions writes (rust/lance/src/index/vector/builder.rs:938-1079): each partition's storage
 * batch is written on its own, so `auxiliary.idx` (and for the graph kinds `index.idx`) holds the partitions back to
 * back, partition 0 first, with part_lengths[p] rows (an empty partition adds none).  Here every column is that
 * concatenation.  Row-wise columns, per partition in storage order:
 *   _rowid            u64 [num_rows] (ROW_ID_FIELD).
 *   payload [num_bytes], num_bytes = num_rows x the kind's bytes per row:
 *     IVF_PQ, IVF_HNSW_PQ     `__pq_code` with "transposed": true (pq/storage.rs:52-67,430-450): each partition's
 *                             codes column-major [code bytes per row][n_p], the bytes lb2_index_export_partition gives.
 *     IVF_SQ, IVF_HNSW_SQ     `__sq_code` [n_p][d] (sq/storage.rs:38-45,280-300).
 *     IVF_FLAT, IVF_HNSW_FLAT `flat` rows [n_p][d] in the stored element type, f32 / f16 / bf16 (flat/storage.rs:27,
 *                             109-120).  u8 columns: LB2_INVALID_ARG both ways.  The reference's u8 flat storage is
 *                             its binary Hamming storage (FlatBinStorage, flat/storage.rs:190-300), while this library
 *                             holds u8 rows as f32 under L2 / cosine / dot, so no stored column matches them.
 *     IVF_RQ                  `__rabit_code` packed (RabitQuantizationMetadata::packed, bq/storage.rs:48-55): the
 *                             packing restarts at every partition, because try_from_batch packs each partition's
 *                             batch on its own (bq/storage.rs:607-640) and merge_partitions writes each partition's
 *                             storage separately.  In a partition of n_p rows of cl = code_dim / 8 bytes, with
 *                             nb = n_p / 32 full blocks (pack_codes, bq/storage.rs:477-543): byte b*32*cl + i*32 + j,
 *                             j < 16, is (c[32b + PERM0[j]][i] & 15) | (c[32b + PERM0[j] + 16][i] & 15) << 4, and
 *                             byte b*32*cl + i*32 + 16 + j the same of the high nibbles (>> 4); PERM0 = 0, 8, 1, 9,
 *                             .. 7, 15 (lance-linalg/src/simd/dist_table.rs:10).  The last n_p % 32 rows follow
 *                             transposed, [cl][n_p % 32].  unpack_codes (:546-600) is the inverse.
 *   add_factors, scale_factors  f32 [num_rows]: IVF_RQ's `__add_factors` / `__scale_factors`; NULL for other kinds.
 * Graph kinds, also (HNSW::to_batch / HNSW::load, hnsw/builder.rs:579-640,788-833; the `lance:hnsw` metadata list
 * of hnsw/index.rs:57-110 gives each partition's HnswMetadata {entry_point, params, level_offsets}, :283-303):
 *   max_level, m, ef_construction   HnswBuildParams of every partition (params).
 *   entry_point       u32 [K]: 0 -- node 0 of every non-empty partition is the entry point (:354-376) and the
 *                     device search starts there; anything else is LB2_INVALID_ARG.
 *   level_offsets     u64 [K][max_level + 1]: partition-local, 0 first; level l's rows are level_offsets[p][l] ..
 *                     level_offsets[p][l + 1] - 1 of the partition's batch.
 *   vector_id         u32 [num_graph_rows] `__vector_id`: for each partition, for each level 0 .. max_level - 1, the
 *                     nodes that have the level, ascending (partition-local ids).  num_graph_rows = num_rows + the
 *                     upper-level rows of the device layout (lb2_index_hnsw_*_info).
 *   list_offsets      u64 [num_graph_rows + 1]: the Arrow list offsets of `__neighbors` and `_distance`, over the
 *                     concatenation (a partition's own offsets are its slice minus its first entry); 0 first,
 *                     num_edges last.
 *   neighbors         u32 [num_edges] `__neighbors`, distances f32 [num_edges] `_distance`: each row's list in the
 *                     order of level_neighbors_ranked, which the device layout keeps (graph/builder.rs:33-48).
 *   An empty partition has no rows and level_offsets all 0.  HNSW::load gives every node all levels; a loaded graph
 *   gives a node the levels whose batches hold it, which searches the same (no list names a node above its levels).
 * lb2_index_export_storage: out->num_partitions, num_rows, num_bytes, max_level, m, ef_construction,
 *   num_graph_rows and num_edges are set (max_level = 0 without a graph); each non-NULL buffer is written.  Call
 *   with NULL buffers first to size them.  Buffers are host or device memory.
 * lb2_index_load_storage: loads into a handle made by the kind's lb2_index_create* call (or one that already holds
 *   rows; the content is replaced, graph included).  max_level = 0 loads no graph; max_level >= 1 attaches one, as
 *   lb2_index_load_hnsw_* does, to an IVF_SQ, IVF_PQ or IVF_FLAT handle.  Every input is checked before the handle
 *   changes; LB2_INVALID_ARG, the handle as it was, for: num_partitions other than the index's; a part length above
 *   num_rows, or part_lengths not summing to num_rows; num_bytes other than num_rows x bytes per row; IVF_RQ without
 *   factors or other kinds with them; list offsets that descend or do not run from 0 to num_edges; a vector_id at or
 *   above n_p, or not ascending within its level; level_offsets that do not start at 0 and ascend by at most n_p per
 *   level, whose level 0 is not every row of the partition, or that do not add up to num_graph_rows; a node present
 *   at level l but absent at l - 1; more than 2m neighbours at level 0 or more than m above; a neighbour that is not
 *   a node of its partition at that level, or is named twice in a list; a non-empty partition whose node 0 lacks a
 *   level (lb2_index_load_hnsw_sq's check); an entry_point other than 0. */
typedef struct {
  uint32_t num_partitions;  /* K */
  uint64_t num_rows, num_bytes;
  uint64_t* part_lengths;   /* [K] */
  uint64_t* row_ids;        /* _rowid */
  uint8_t* payload;         /* __pq_code / __sq_code / flat / __rabit_code values */
  float* add_factors;
  float* scale_factors;
  uint32_t max_level, m, ef_construction;
  uint64_t num_graph_rows, num_edges;
  uint32_t* entry_point;
  uint64_t* level_offsets;
  uint32_t* vector_id;
  uint64_t* list_offsets;
  uint32_t* neighbors;
  float* distances;
} lb2_index_storage;
lb2_status lb2_index_export_storage(const lb2_index* index, lb2_index_storage* out);
lb2_status lb2_index_load_storage(lb2_index* index, const lb2_index_storage* storage);
lb2_status lb2_index_destroy(lb2_index* index);

/* IvfIndexBuilder::build (rust/lance/src/index/vector/builder.rs:236): sample -> train IVF ->
 * residuals -> train PQ -> assign + encode every row -> group by partition, all on the device. */
typedef struct {
  uint32_t num_partitions;
  lb2_kmeans_params ivf;  /* balance_factor 1.0, sample_rate 256 (ivf/builder.rs:62-78) */
  lb2_pq_params pq;
  uint64_t seed;          /* training-sample selection */
} lb2_ivfpq_build_params;
void lb2_ivfpq_build_params_default(lb2_ivfpq_build_params* p);
typedef struct {
  float ms_ivf_train, ms_pq_train, ms_transform, ms_group, ms_total; /* CUDA-event times */
  uint32_t ivf_iters, pq_iters_max;
  double ivf_loss;
} lb2_build_stats;
lb2_status lb2_ivfpq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype,
                           lb2_metric metric, const lb2_ivfpq_build_params* params,
                           const uint64_t* row_ids /* NULL = 0..n */, lb2_index** out,
                           lb2_build_stats* stats /* nullable */);

/* ---- IVF_FLAT: IVFIndex<FlatIndex, FlatQuantizer> (lance-index/src/vector/flat/{index,storage}.rs) --
 * The partitions hold the raw f32 vectors (normalised first when the metric is cosine, as
 * IvfTransformer::new_flat does, lance-index/src/vector/ivf.rs:149-185); search scores every row of
 * the probed partitions exactly (FlatDistanceCal::distance_all, flat/storage.rs:397-403) and keeps
 * the k smallest (FlatIndex::search, flat/index.rs:82-177).  lb2_index_search / _info / _destroy
 * work on both index kinds. */
typedef struct {
  uint32_t num_partitions;
  lb2_kmeans_params ivf;
  uint64_t seed;
} lb2_ivfflat_build_params;
void lb2_ivfflat_build_params_default(lb2_ivfflat_build_params* p);
lb2_status lb2_ivfflat_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype,
                             lb2_metric metric, const lb2_ivfflat_build_params* params,
                             const uint64_t* row_ids, lb2_index** out, lb2_build_stats* stats);
lb2_status lb2_index_create_flat(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                                 lb2_metric metric, lb2_index** out);
/* vectors [n][d] (already normalised for cosine), grouped by partition on the device (stable) */
lb2_status lb2_index_load_flat(lb2_index* index, const uint32_t* part_ids, const void* vectors,
                               const uint64_t* row_ids, uint64_t n);
lb2_status lb2_index_export_flat(const lb2_index* index, void* centroids_out,
                                 uint64_t* part_offsets_out, void* vectors_out,
                                 uint64_t* row_ids_out);

/* ---- IVF_SQ: IVFIndex<FlatIndex, ScalarQuantizer> (lance-index/src/vector/sq*.rs) ---------------
 * create_index(.., "IVF_SQ") builds an IvfIndexBuilder<FlatIndex, ScalarQuantizer> (rust/lance/src/index/vector.rs:
 * 429-450).  One byte per dimension: code = scale_to_u8 of the vector (normalised first under cosine) with the
 * index's bounds; no residuals (Quantization::use_residual is false, quantizer.rs:52).  A search encodes the
 * (normalised) query with the same bounds and ranks rows by an exact integer distance, so its results are
 * bit-identical to the reference, ties at the k-th distance included.  d % 4 == 0 and d * 255^2 < 2^32.
 * lb2_index_search / _search_refine / _search_ex / _search_async / _search_sharded / _row_mask / _info
 * (num_sub_vectors 0, num_bits 8) / _repartition / _destroy take an IVF_SQ handle; lb2_index_update, _load,
 * _export and _export_partition do not. */
/* ScalarQuantizer::build (lance-index/src/vector/sq.rs:67-89,152-182): the bounds are the fold of every one of the
 * n * d elements as f64 from (f64::MAX, f64::MIN) with f64::min / f64::max (NaN elements are ignored). */
lb2_status lb2_sq_train(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, double* lower_out,
                        double* upper_out);
/* ScalarQuantizer::quantize = scale_to_u8 (sq.rs:263-277): codes_out[n][d], code = ((v - lower) * 255 / (upper -
 * lower)) in f64, then `as u8` (truncation toward zero, saturating, NaN -> 0); all codes are 0 when lower == upper. */
lb2_status lb2_sq_encode(const void* vectors, uint64_t n, uint32_t d, lb2_dtype dtype, double lower, double upper,
                         uint8_t* codes_out);
/* IvfIndexBuilder<FlatIndex, ScalarQuantizer>::build (rust/lance/src/index/vector/builder.rs:398-468): the IVF stage
 * of lb2_ivfflat_build (same sample, seed and assignment), then the bounds over sample_rate * 2^num_bits rows drawn
 * with seed + 1 (normalised under cosine, rows that are not finite dropped, values as the index stores them), then
 * every kept row encoded and grouped by partition.  The quantizer stage is timed in stats->ms_pq_train.
 * num_bits other than 8 -> LB2_UNSUPPORTED (the reference has no SQ4, sq.rs:115); so is a build with a
 * communicator of more than one rank. */
typedef struct {
  uint32_t num_partitions;
  lb2_kmeans_params ivf;
  uint32_t num_bits;    /* SQBuildParams (sq/builder.rs:7-28): 8 */
  uint64_t sample_rate; /* 256 */
  uint64_t seed;        /* training-sample selection */
} lb2_ivfsq_build_params;
void lb2_ivfsq_build_params_default(lb2_ivfsq_build_params* p);
lb2_status lb2_ivfsq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                           const lb2_ivfsq_build_params* params, const uint64_t* row_ids, lb2_index** out,
                           lb2_build_stats* stats);
/* An index from a reference-built model: centroids in the model type of `dtype`, the `lance:sq` metadata's bounds
 * {dim, num_bits, bounds} (lance-index/src/vector/sq/storage.rs:38-45); finite, lower <= upper (else
 * LB2_INVALID_ARG). */
lb2_status lb2_index_create_sq(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                               double lower, double upper, lb2_index** out);
/* codes [n][d] (the __sq_code column), grouped by partition on the device (stable) */
lb2_status lb2_index_load_sq(lb2_index* index, const uint32_t* part_ids, const uint8_t* codes,
                             const uint64_t* row_ids, uint64_t n);
/* any pointer may be NULL: bounds_out[2] = {lower, upper}; part_offsets[k+1]; codes [num_rows][d] and row_ids
 * [num_rows] in partition order */
lb2_status lb2_index_export_sq(const lb2_index* index, void* centroids_out, double* bounds_out,
                               uint64_t* part_offsets_out, uint8_t* codes_out, uint64_t* row_ids_out);

/* ---- IVF_HNSW_SQ: IVFIndex<HNSW, ScalarQuantizer> (lance-index/src/vector/hnsw/builder.rs) ------------------
 * An IVF_SQ index (same IVF stage, bounds and codes for the same arguments) with an HNSW graph per partition over
 * the partition's SQ codes; every distance, row to row and query to row, is the SQ distance of lb2_index_search on
 * IVF_SQ (sq/storage.rs:387-444, storage.rs:102-105).  Node i of partition p is its storage position
 * part_offsets[p] + i.  The graph of a partition is HNSW::index_vectors (builder.rs:742-775) with the nodes
 * inserted 1 .. n_p - 1 in ascending order (the reference inserts in parallel); node 0 has max_level levels and is
 * the entry point (:354-376), node i >= 1 gets 1 + random_level() levels (:386-393) from a u32 draw keyed by (seed,
 * p, i) compared against floor(2^32 / m^l).  Ties in select_neighbors_heuristic (hnsw.rs:60-88) keep their order.
 *
 * Batched insertion (insert_batch = B >= 2; 0 and 1 insert one node at a time, as above): a deterministic stand-in
 * for the reference's concurrent inserts.  The graph is a function of (data, seed, m, ef_construction, max_level, B)
 * alone, whatever the number of warps in flight.  A partition with n_p >= 2 rows is built in rounds: the first round
 * starts at s = 1, a round starting at s inserts nodes s .. e - 1 with e = min(n_p, s + min(B, s)), and the next
 * round starts at e (rounds of 1, 2, 4, .. nodes until B, then B).  Each round has two phases:
 *   1. every node i of the round runs insert's descent and beam searches (builder.rs:396-463) over the graph as it
 *      stood at the start of the round, and its own lists are the pruned results, as in the serial build (no list
 *      names a node of the round yet, so no node of the round reaches another);
 *   2. the back-links, as if applied for i ascending, level 0 .. i's top level, entries in list order, each with the
 *      serial rule (enter the target's list when closer than its LAST entry or the list is short, then prune).  Every
 *      target is a node < s and a list takes at most one entry per node, so this is each target list taking its
 *      entries in ascending i, distinct lists independently.
 * Levels, level draws, the entry point and every distance and tie rule are the serial build's; with B = 1 every
 * round holds one node and the graph is the serial graph byte for byte.
 * Searches go through lb2_index_search / _refine / _ex / _probed / _combined / _async / _sharded with the default ef
 * k' + k' / 2, k' = k * refine_factor (:563-573), or through lb2_index_search_hnsw with an explicit ef: each probed
 * partition is HNSW::search (builder.rs:678-739); ef < k' is LB2_INVALID_ARG (:687-692).  A prefilter that leaves fewer than
 * n_p * 10 / 100 rows of a partition takes the flat branch (:238-280, range lower < d <= upper), otherwise the
 * graph (:164-201, range lower <= d < upper).  lb2_index_repartition, _update and _load_sq refuse the index; so
 * does a build with a communicator of more than one rank.
 *
 * The graph crosses the ABI in the device layout: levels[n] (levels per row), level 0 dense (counts0[n],
 * neighbors0 / dists0 [n][2m]) and the upper levels node by node in storage order: a row with L levels owns L - 1
 * consecutive upper rows, levels 1 .. L-1 (counts_up[r], neighbors_up / dists_up [r][m]).  Lists are in the order of
 * level_neighbors_ranked (graph/builder.rs:33-48); neighbour ids are partition-local.  A built graph's slots past
 * a list's count hold zeros. */
typedef struct {
  lb2_ivfsq_build_params sq;
  uint32_t max_level;       /* HnswBuildParams (hnsw/builder.rs:63-72): 7 */
  uint32_t m;               /* 20; level 0 keeps up to 2m neighbours, the others m */
  uint32_t ef_construction; /* 150 */
  uint32_t insert_batch;    /* B of the batched insertion above: 0 or 1 serial (the default 1), at most 65 536 */
} lb2_ivfhnswsq_build_params;
void lb2_ivfhnswsq_build_params_default(lb2_ivfhnswsq_build_params* p);
/* IvfIndexBuilder<HNSW, ScalarQuantizer>::build: lb2_ivfsq_build, then every partition's graph on the device (serial:
 * one warp per partition, the largest partitions first; batched: one warp per inserting node, then one per
 * back-linked list, all partitions advancing round by round); the level draws use params->sq.seed. */
lb2_status lb2_ivfhnswsq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                               const lb2_ivfhnswsq_build_params* params, const uint64_t* row_ids, lb2_index** out,
                               lb2_build_stats* stats);
/* attach a graph (host or device arrays in the layout above) to an IVF_SQ index made by lb2_index_create_sq +
 * lb2_index_load_sq; every neighbour must be a node of its partition that has the level (else LB2_INVALID_ARG) */
lb2_status lb2_index_load_hnsw_sq(lb2_index* index, uint32_t max_level, uint32_t m, uint32_t ef_construction,
                                  const uint8_t* levels, const uint32_t* counts0, const uint32_t* neighbors0,
                                  const float* dists0, const uint32_t* counts_up, const uint32_t* neighbors_up,
                                  const float* dists_up);
/* the graph's parameters and its number of upper-level rows (any pointer may be NULL) */
lb2_status lb2_index_hnsw_sq_info(const lb2_index* index, uint32_t* max_level, uint32_t* m, uint32_t* ef_construction,
                                  uint64_t* num_upper_rows);
/* the graph in the layout above; any pointer may be NULL */
lb2_status lb2_index_export_hnsw_sq(const lb2_index* index, uint8_t* levels_out, uint32_t* counts0_out,
                                    uint32_t* neighbors0_out, float* dists0_out, uint32_t* counts_up_out,
                                    uint32_t* neighbors_up_out, float* dists_up_out);
/* lb2_index_search_ex (pp NULL) or lb2_index_search_probed (pp set; nprobes_out nullable) of an IVF_HNSW_SQ index with
 * the graph search's ef for this call (Query::ef, HnswQueryParams::ef, builder.rs:563-573); ef = 0: k' + k' / 2 */
lb2_status lb2_index_search_hnsw(lb2_index* index, const void* queries, uint64_t nq, const lb2_search_params* sp,
                                 const lb2_probe_params* pp, uint32_t ef, uint64_t* row_ids_out, float* dists_out,
                                 uint32_t* counts_out, uint32_t* nprobes_out);

/* ---- IVF_HNSW_PQ: IVFIndex<HNSW, ProductQuantizer> (rust/lance/src/index/vector.rs:494-520) ---------------------
 * An IVF_PQ index (same IVF stage, codebook and codes for the same arguments) with an HNSW graph per partition over
 * the partition's PQ storage (lance-index/src/vector/pq/storage.rs:600-1037).  Levels, insertion order (batched
 * rounds included), tie handling, the graph layout, ef, the prefilter switch and the refusals are IVF_HNSW_SQ's
 * (above); the distances are the PQ storage's, and cosine is L2 on the normalised rows throughout (the storage carries L2, pq/storage.rs:465-468):
 *  - query to node (search): PQDistCalculator::distance (storage.rs:891-919) on the IVF_PQ scan's table of the
 *    query (its residual to the probed centroid under L2 / cosine, the raw query under dot): 8-bit codes the
 *    m-ascending f32 sum of table[m][code[m]], the distance of lb2_index_search on IVF_PQ; 4-bit codes the sum, in
 *    byte order, of table[2i][lo] + table[2i+1][hi] (f32 entries, not the 4-bit scan's quantised table); dot
 *    subtracts M - 1;
 *  - node to node while node i is inserted: the same sum on the table of node i's decoded codes
 *    (dist_calculator_from_id, storage.rs:675-749), entry point included; these are the distances in the lists;
 *  - the heuristic (hnsw.rs:82): dist_between (storage.rs:751-841), the distance of the two decoded rows with the
 *    column type's rule (16 f32 lanes; 32 lanes for f16 / bf16 dot).
 * The graph crosses the ABI in IVF_HNSW_SQ's layout. */
typedef struct {
  lb2_ivfpq_build_params pq;
  uint32_t max_level;       /* HnswBuildParams (hnsw/builder.rs:63-72): 7 */
  uint32_t m;               /* 20; level 0 keeps up to 2m neighbours, the others m */
  uint32_t ef_construction; /* 150 */
  uint32_t insert_batch;    /* as lb2_ivfhnswsq_build_params.insert_batch */
} lb2_ivfhnswpq_build_params;
void lb2_ivfhnswpq_build_params_default(lb2_ivfhnswpq_build_params* p);
/* IvfIndexBuilder<HNSW, ProductQuantizer>::build (vector.rs:507-520): lb2_ivfpq_build, then every partition's graph on
 * the device (as lb2_ivfhnswsq_build's, serial or batched); the level draws use params->pq.seed.  The graph
 * stage is counted in stats->ms_total only.  A communicator of more than one rank is LB2_UNSUPPORTED. */
lb2_status lb2_ivfhnswpq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                               const lb2_ivfhnswpq_build_params* params, const uint64_t* row_ids, lb2_index** out,
                               lb2_build_stats* stats);
/* attach a graph (host or device arrays in the IVF_HNSW_SQ layout) to an IVF_PQ index made by lb2_index_create +
 * lb2_index_load; the checks of lb2_index_load_hnsw_sq.  `dtype` of lb2_index_create picks the heuristic's rule. */
lb2_status lb2_index_load_hnsw_pq(lb2_index* index, uint32_t max_level, uint32_t m, uint32_t ef_construction,
                                  const uint8_t* levels, const uint32_t* counts0, const uint32_t* neighbors0,
                                  const float* dists0, const uint32_t* counts_up, const uint32_t* neighbors_up,
                                  const float* dists_up);
/* as lb2_index_hnsw_sq_info / lb2_index_export_hnsw_sq for an IVF_HNSW_PQ index */
lb2_status lb2_index_hnsw_pq_info(const lb2_index* index, uint32_t* max_level, uint32_t* m, uint32_t* ef_construction,
                                  uint64_t* num_upper_rows);
lb2_status lb2_index_export_hnsw_pq(const lb2_index* index, uint8_t* levels_out, uint32_t* counts0_out,
                                    uint32_t* neighbors0_out, float* dists0_out, uint32_t* counts_up_out,
                                    uint32_t* neighbors_up_out, float* dists_up_out);

/* ---- IVF_HNSW_FLAT: IVFIndex<HNSW, FlatQuantizer> (rust/lance/src/index/vector.rs:473-493) -----------------------
 * An IVF_FLAT index (same IVF stage, vectors and row ids for the same arguments) with an HNSW graph per partition over
 * the partition's FlatFloatStorage (lance-index/src/vector/flat/storage.rs:31-185,345-410): the stored rows as they
 * are, normalised under cosine by the IVF transformer, no residuals.  Levels, insertion order, tie handling, the graph
 * layout, ef, the prefilter switch and the refusals are IVF_HNSW_SQ's (above).  The storage keeps the index's distance
 * type, cosine included (builder.rs:841, flat/storage.rs:108-158,353-366), and every distance is the one
 * lb2_index_search on IVF_FLAT computes for the pair: the column's stored element type (f32 / f16 / bf16; u8 held as
 * f32) with 16 f32 lanes under L2 and dot, and under cosine 16 f32 FMA lanes for <q, y> and <y, y>, the xor tree and
 * 1 - xy / |q| / sqrt(yy), |q| the query role's norm from the same 16 FMA lanes:
 *  - query to node (search): the (normalised) query in the query role;
 *  - node to node while node i is inserted (dist_calculator_from_id): node i in the query role; these are the
 *    distances in the lists;
 *  - the heuristic (hnsw.rs:82): dist_between(u, v) with the candidate u in the query role and the accepted neighbour
 *    v as the row.  Cosine is not symmetric in its rounding, so the orientation is part of the definition.
 * The graph crosses the ABI in IVF_HNSW_SQ's layout. */
typedef struct {
  lb2_ivfflat_build_params flat;
  uint32_t max_level;       /* HnswBuildParams (hnsw/builder.rs:63-72): 7 */
  uint32_t m;               /* 20; level 0 keeps up to 2m neighbours, the others m */
  uint32_t ef_construction; /* 150 */
  uint32_t insert_batch;    /* as lb2_ivfhnswsq_build_params.insert_batch */
} lb2_ivfhnswflat_build_params;
void lb2_ivfhnswflat_build_params_default(lb2_ivfhnswflat_build_params* p);
/* IvfIndexBuilder<HNSW, FlatQuantizer>::build: lb2_ivfflat_build, then every partition's graph on the device (as
 * lb2_ivfhnswsq_build's, serial or batched); the level draws use params->flat.seed.  The graph stage is counted in
 * stats->ms_total only.  A communicator of more than one rank is LB2_UNSUPPORTED. */
lb2_status lb2_ivfhnswflat_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                                 const lb2_ivfhnswflat_build_params* params, const uint64_t* row_ids, lb2_index** out,
                                 lb2_build_stats* stats);
/* attach a graph (host or device arrays in the IVF_HNSW_SQ layout) to an IVF_FLAT index made by lb2_index_create_flat +
 * lb2_index_load_flat; the checks of lb2_index_load_hnsw_sq.  lb2_index_load_flat, lb2_index_update and
 * lb2_index_repartition refuse an index that has a graph. */
lb2_status lb2_index_load_hnsw_flat(lb2_index* index, uint32_t max_level, uint32_t m, uint32_t ef_construction,
                                    const uint8_t* levels, const uint32_t* counts0, const uint32_t* neighbors0,
                                    const float* dists0, const uint32_t* counts_up, const uint32_t* neighbors_up,
                                    const float* dists_up);
/* as lb2_index_hnsw_sq_info / lb2_index_export_hnsw_sq for an IVF_HNSW_FLAT index; lb2_index_export_flat exports its
 * IVF_FLAT part */
lb2_status lb2_index_hnsw_flat_info(const lb2_index* index, uint32_t* max_level, uint32_t* m,
                                    uint32_t* ef_construction, uint64_t* num_upper_rows);
lb2_status lb2_index_export_hnsw_flat(const lb2_index* index, uint8_t* levels_out, uint32_t* counts0_out,
                                      uint32_t* neighbors0_out, float* dists0_out, uint32_t* counts_up_out,
                                      uint32_t* neighbors_up_out, float* dists_up_out);
/* lb2_index_search_hnsw takes an IVF_HNSW_SQ, IVF_HNSW_PQ or IVF_HNSW_FLAT index. */

/* ---- IVF_RQ: IVFIndex<FlatIndex, RabitQuantizer> (lance-index/src/vector/bq/) ------------------------------------
 * create_index(.., "IVF_RQ") builds an IvfIndexBuilder<FlatIndex, RabitQuantizer> (rust/lance/src/index/vector.rs:
 * 452-470).  code_dim = d * num_bits; the rotation R is code_dim x code_dim, of which the first d columns are used.
 * Per row (IvfTransformer::with_rq, ivf.rs:281-328; RQTransformer, bq/transform.rs:70-220): normalised under cosine
 * (L2 from there on), partition and dist_v_c, residual = v - c, rot[j] = dot(R[j, :d], residual); code bit j =
 * rot[j] >= +0.0 by sign bit, LSB-first, code_dim / 8 bytes; add / scale factors.  A search rotates the (normalised)
 * query's residual to each probed centroid the same way and scores rows from the reference's 4-bit tables
 * (bq/storage.rs:160-445).  The rotation of a data row is defined as that same 16-lane f32 dot (the reference's GEMM
 * has no specified order), so codes, factors and results are bit-identical to the restatement, ties included.
 * f32 columns only: bf16 / u8 -> LB2_INVALID_ARG (the reference rejects them, bq/builder.rs:194-210), f16 ->
 * LB2_UNSUPPORTED; code_dim % 8 != 0 -> LB2_INVALID_ARG; a code_dim whose tables do not fit shared memory, or a
 * build with more than one rank -> LB2_UNSUPPORTED.
 * lb2_index_search / _search_refine / _search_ex / _search_async / _search_sharded / _row_mask / _info
 * (num_sub_vectors 0, num_bits) / _destroy take an IVF_RQ handle; lb2_index_update, _load, _export and
 * _export_partition reject it with LB2_INVALID_ARG, lb2_index_repartition with LB2_UNSUPPORTED. */
/* random_orthogonal (bq/builder.rs:309-367): the Q factor of a Householder QR of a standard-normal f64 matrix,
 * cast to f32; ours is drawn with Philox from `seed` (the reference's rng is unseeded).  rotation_out[code_dim]
 * [code_dim], row-major. */
lb2_status lb2_rq_rotation(uint32_t code_dim, uint64_t seed, float* rotation_out);
/* the batch transform of rows to append (replaces the transformer chain of ivf.rs:281-328): part_out[n],
 * codes_out[n][code_dim / 8], add_out[n], scale_out[n], valid_out[n] (0: the row is not finite, or zero under
 * cosine; its outputs are 0).  Any output may be NULL. */
lb2_status lb2_ivfrq_transform(const void* centroids, uint32_t k, const void* rotation, uint32_t d, uint32_t num_bits,
                               lb2_dtype dtype, lb2_metric metric, const void* vectors, uint64_t n, uint32_t* part_out,
                               uint8_t* codes_out, float* add_out, float* scale_out, uint8_t* valid_out);
/* IvfIndexBuilder<FlatIndex, RabitQuantizer>::build: the IVF stage of lb2_ivfflat_build (same sample, seed and
 * centroids), the rotation from seed + 1 (timed in stats->ms_pq_train), every kept row transformed
 * (stats->ms_transform) and grouped by partition. */
typedef struct {
  uint32_t num_partitions;
  lb2_kmeans_params ivf;
  uint32_t num_bits; /* RQBuildParams (bq/builder.rs:30-45): 1 */
  uint64_t seed;     /* training sample; the rotation uses seed + 1 */
} lb2_ivfrq_build_params;
void lb2_ivfrq_build_params_default(lb2_ivfrq_build_params* p);
lb2_status lb2_ivfrq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                           const lb2_ivfrq_build_params* params, const uint64_t* row_ids, lb2_index** out,
                           lb2_build_stats* stats);
/* An index from a reference-built model: centroids and the `lance:rabit` rotation (code_dim x code_dim) in the model
 * type of `dtype` (bq/storage.rs:40-60). */
lb2_status lb2_index_create_rq(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                               const void* rotation, uint32_t num_bits, lb2_index** out);
/* codes [n][code_dim / 8] row-major (unpacked: unpack_codes, bq/storage.rs:546-600), the __add_factors and
 * __scale_factors columns, grouped by partition on the device (stable) */
lb2_status lb2_index_load_rq(lb2_index* index, const uint32_t* part_ids, const uint8_t* codes, const float* add_factors,
                             const float* scale_factors, const uint64_t* row_ids, uint64_t n);
/* any pointer may be NULL: rotation [code_dim][code_dim]; part_offsets[k+1]; codes [num_rows][code_dim / 8],
 * add / scale [num_rows] and row_ids [num_rows] in partition order */
lb2_status lb2_index_export_rq(const lb2_index* index, void* centroids_out, void* rotation_out,
                               uint64_t* part_offsets_out, uint8_t* codes_out, float* add_out, float* scale_out,
                               uint64_t* row_ids_out);

/* ---- multi-GPU (one process per GPU) -----------------------------------------------------------
 * With a communicator every training / build call takes THIS RANK'S ROW SHARD: the k-means loops
 * (flat and hierarchical) exchange their packed per-cluster partial results once per Lloyd iteration
 * (one collective, reduced in rank order on every rank -> bit-identical models on all ranks), the
 * transform and the index are local to the shard. */
/* unique_id is the 128-byte ncclUniqueId produced by rank 0 (lb2_comm_unique_id) and broadcast by
 * the host runtime (torch.distributed / MPI / the Rust side). */
lb2_status lb2_comm_unique_id(void* unique_id_128);
lb2_status lb2_comm_init(const void* unique_id_128, int rank, int nranks);
lb2_status lb2_comm_destroy(void);
lb2_status lb2_comm_info(int* rank, int* nranks); /* (0, 1) without a communicator */
/* Search of a ROW-SHARDED index (every rank built / loaded its own rows, row ids global): the local
 * lb2_index_search_ex result of every rank is exchanged in one collective and merged by (_distance,
 * _rowid) -- the reference's final SortExec.fetch(k) (rust/lance/src/dataset/scanner.rs:3450-3466) --
 * so every rank returns the global top-k.  All ranks must call it with the same queries and params. */
lb2_status lb2_index_search_sharded(lb2_index* index, const void* queries, uint64_t nq,
                                    const lb2_search_params* params, uint64_t* row_ids_out, float* dists_out,
                                    uint32_t* counts_out);
/* Partition ownership by device all-to-all (SURVEY 8e "partition build" / 8f-4).  The reference groups the
 * transformed rows by partition with a host/disk shuffler (rust/lance-index/src/vector/v3/shuffler.rs:105).
 * For a build sharded by rows over G ranks this call is that shuffle on the device: every rank passes its
 * row-shard index (same model on all ranks, global row ids); afterwards rank g holds ALL rows of the partitions
 * p with p % G == g (its other partitions are empty) in a NEW index.  Inside a partition rows are ordered by
 * source rank, then by the source's storage order -- with contiguous row shards that is the order a single-GPU
 * index has, so a partition is scanned exactly as on one GPU (heap tie order included).  One all-gather of the K
 * partition sizes, one grouped ncclSend/ncclRecv of (codes | vectors, row ids) over NVLink.  Without a
 * communicator it returns a copy.  lb2_index_search_sharded works on the result unchanged: partitions a rank
 * does not own are empty, so every probed partition is scanned by exactly one rank. */
lb2_status lb2_index_repartition(const lb2_index* shard, lb2_index** owned_out);

#ifdef __cplusplus
}
#endif
#endif /* LANCE_B200_H_ */
