/*
 * lancedb_b200.h -- C ABI of the H100-native (sm_90a) LanceDB vector-query hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b): the entry points the Rust
 * `lancedb` crate would bind through `extern "C"` at the single place it hands a
 * vector query to lance today --
 *     rust/lancedb/src/table/query.rs:219-249   ds.scan() / scanner.nearest(..) /
 *                                                minimum_nprobes / maximum_nprobes
 *     rust/lancedb/src/table/query.rs:251-316   limit+offset, distance_range,
 *                                                use_index, refine, distance_metric
 *     rust/lancedb/src/table/query.rs:327, :121 create_plan() + execute_plan()
 * -- i.e. everything below `NativeTable::create_plan` for `AnyQuery::VectorQuery`
 * (rust/lancedb/src/table.rs:3301-3315).  INTEGRATION.md shows the Rust binding.
 *
 * Conventions
 *   - plain pointers and sizes only; no C++/torch types cross this boundary;
 *   - every function returns an lgpu_status; on failure `lgpu_last_error()`
 *     (thread-local, valid until the next call on that thread) carries the message
 *     and the status maps onto `lancedb::Error`
 *     (rust/lancedb/src/error.rs:57-130): INVALID_INPUT -> Error::InvalidInput,
 *     RUNTIME/OOM -> Error::Runtime, TIMEOUT -> Error::Timeout;
 *   - the caller owns all host buffers; inputs are borrowed for the call only,
 *     outputs are caller-allocated; the library owns device memory behind the
 *     opaque handles; index arrays are copied to HBM at open (the analogue of
 *     `prewarm_index`, rust/lancedb/src/table.rs:3283-3286);
 *   - handles are thread-safe and `lgpu_*_search*` is re-entrant (each call takes
 *     a private stream + workspace), matching `BaseTable: Send + Sync`
 *     (rust/lancedb/src/table.rs:549);
 *   - no CPU fallback exists: without a CUDA device every compute entry point
 *     fails with LGPU_RUNTIME.
 */
#ifndef LANCEDB_B200_H
#define LANCEDB_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LGPU_ABI_VERSION 2

typedef enum {
    LGPU_OK = 0,
    LGPU_INVALID_INPUT = 1,  /* lancedb::Error::InvalidInput */
    LGPU_RUNTIME = 2,        /* lancedb::Error::Runtime (CUDA failure, no device) */
    LGPU_TIMEOUT = 3,        /* lancedb::Error::Timeout */
    LGPU_OOM = 4             /* device or host allocation failure */
} lgpu_status;

/* lancedb::DistanceType, rust/lancedb/src/lib.rs:236-260 (hamming is u8-only: it has its own
 * column handle, lgpu_binary, below; rust/lancedb/src/table/query.rs:229-236) */
typedef enum { LGPU_L2 = 0, LGPU_COSINE = 1, LGPU_DOT = 2 } lgpu_metric;

typedef enum {
    LGPU_CODES_ROW_MAJOR = 0,             /* [nrows][m], rows partition-contiguous */
    LGPU_CODES_PARTITION_TRANSPOSED = 1   /* per partition [m][n_p] (lance in-memory form) */
} lgpu_codes_layout;

typedef struct lgpu_index lgpu_index;   /* an IVF_PQ index resident in HBM */
typedef struct lgpu_flat lgpu_flat;     /* a raw vector column resident in HBM */
typedef struct lgpu_binary lgpu_binary; /* a packed binary (uint8) vector column in HBM, searched by Hamming distance */
typedef struct lgpu_multivec lgpu_multivec; /* a multivector column in HBM, searched by late interaction (MaxSim) */
typedef struct lgpu_ivf_binary lgpu_ivf_binary; /* a binary IVF_FLAT index in HBM, searched by Hamming distance */

/* The arrays of one IVF_PQ index (lance v2 `IvfPq`,
 * rust/lancedb/src/table/create_index.rs:283-303, :772): IVF centroids, PQ codebook
 * (8-bit, 256 centroids per sub-vector), PQ codes and row ids grouped by partition. */
typedef struct {
    uint32_t abi_version;        /* LGPU_ABI_VERSION */
    uint32_t dim;
    uint32_t nlist;              /* IVF partitions */
    uint32_t m;                  /* PQ sub-vectors; dim % m == 0 */
    uint32_t nbits;              /* 8, or 4 (packed nibble codes, see "4-bit IVF_PQ" below) */
    int32_t  metric;             /* lgpu_metric the index was trained with */
    int32_t  codes_layout;       /* lgpu_codes_layout */
    int32_t  device;             /* CUDA device ordinal */
    uint64_t nrows;
    const float    *centroids;    /* [nlist][dim] */
    const float    *codebook;     /* [m][256][dim/m] */
    const uint64_t *part_offsets; /* [nlist+1] row offset of each partition */
    const uint8_t  *codes;        /* nrows*m bytes, layout above */
    const uint64_t *row_ids;      /* [nrows] `_rowid` of each stored row */
    const float    *vectors;      /* optional [nrows][dim] raw vectors in the same row
                                     order (enables refine_factor); NULL if absent */
} lgpu_index_desc;

/* One vector query request = lancedb::query::VectorQueryRequest
 * (rust/lancedb/src/query.rs:1066-1114) reduced to what reaches the kernels. */
typedef struct {
    uint32_t k;              /* limit + offset (table/query.rs:231); default 10 */
    uint32_t nprobes;        /* maximum_nprobes (== minimum_nprobes == 20 by default) */
    uint32_t refine_factor;  /* 0 = no refine (query.rs:1302-1332) */
    int32_t  has_lower;      /* distance_range lower bound, inclusive */
    int32_t  has_upper;      /* distance_range upper bound, exclusive */
    float    lower;
    float    upper;
    uint32_t flags;          /* reserved, 0 */
    uint32_t max_nprobes;    /* maximum_nprobes (query.rs:1250-1275): under a prefilter, queries that found fewer
                                than k rows in their `nprobes` nearest partitions are searched again over their
                                max_nprobes nearest; 0 or <= nprobes = no widening */
    uint32_t timeout_ms;     /* QueryExecutionOptions::timeout (query.rs:626-658, utils/mod.rs:328-393): the
                                host-buffer entry points return LGPU_TIMEOUT, leaving the outputs untouched,
                                when the results are not ready this many ms after the call started; 0 = none */
} lgpu_search_params;

/* ---- library ----------------------------------------------------------- */
const char *lgpu_last_error(void);
uint32_t    lgpu_abi_version(void);
int         lgpu_device_count(int *count);

/* ---- IVF_PQ (ANNIvfPartitionExec -> ANNIvfSubIndexExec -> TopK) ---------- */
int  lgpu_index_open(const lgpu_index_desc *desc, lgpu_index **out);
void lgpu_index_close(lgpu_index *ix);
/* bytes of HBM held by the index (codes + ids + centroids + codebook + vectors) */
int  lgpu_index_device_bytes(const lgpu_index *ix, uint64_t *bytes);
/* sum over a batch of the PQ code bytes its probes must scan (the roofline's
 * algorithmic bytes, SURVEY.md 8d); valid for the most recent search on the
 * calling thread */
int  lgpu_last_scanned_code_bytes(uint64_t *bytes);

/* Search a batch of B queries held in HOST memory.  queries: [B][dim] f32.
 * out_ids/out_dist: [B][k] (`_rowid` / `_distance`, ascending by
 * (_distance,_rowid)); out_count: [B] valid entries per query; unused slots are
 * UINT64_MAX / +inf.  H2D and D2H copies happen inside the call.
 * Non-finite values (DESIGN.md section 0): a NaN _distance is never returned (refine included); +-inf distances are
 * returned and ordered like any other; a partition whose coarse distance is NaN is never probed, so a query may have
 * fewer than nprobes probes.  A NaN / inf centroid, or one whose |c|^2 overflows, keeps the coarse step on the exact
 * kernels; a query whose tensor-core error band is not finite is redone by them. */
int lgpu_search(lgpu_index *ix, const float *queries, uint32_t B,
                const lgpu_search_params *params,
                uint64_t *out_ids, float *out_dist, uint32_t *out_count);

/* Asynchronous form of lgpu_search (SURVEY.md 8b "Threading": today the Python binding parks the blocking call on
 * spawn_blocking, python/src/runtime.rs:113-119).  Returns once the copies and kernels are enqueued on a private
 * stream; every buffer must stay valid (and should be page-locked for the copies to overlap) until
 * lgpu_ticket_wait returns.  Two or more tickets in flight pipeline: batch i+1's H2D overlaps batch i's kernels. */
typedef struct lgpu_ticket lgpu_ticket;
int lgpu_search_async(lgpu_index *ix, const float *queries, uint32_t B,
                      const lgpu_search_params *params,
                      uint64_t *out_ids, float *out_dist, uint32_t *out_count, lgpu_ticket **ticket);
int lgpu_ticket_poll(lgpu_ticket *ticket, int *done);   /* *done = 1 when the results are in place */
int lgpu_ticket_wait(lgpu_ticket *ticket);              /* blocks, frees the ticket, returns the call's status */

/* Single-vector search that may share a batch with concurrent callers (SURVEY.md 8b "Threading": the reference serves
 * many one-vector queries from tokio workers, each through its own plan -- rust/lancedb/src/table/query.rs:201-215).
 * Calls with identical parameters arriving within a short window (LGPU_COALESCE_US, default 50 us) are gathered by the
 * first arrival into ONE lgpu_search; every caller gets exactly the rows a solitary lgpu_search(B = 1) would return.
 * query: [dim]; out_ids / out_dist: [k]; out_count: [1]. */
int lgpu_search_coalesced(lgpu_index *ix, const float *query, const lgpu_search_params *params,
                          uint64_t *out_ids, float *out_dist, uint32_t *out_count);

/* Prefiltered search: the reference's default filter mode ("filtering will be performed
 * before the vector search", rust/lancedb/src/query.rs:489-507; the row-id allow-list the
 * scalar filter produced is what lance hands to the ANN nodes as a pre-filter [lance,
 * recalled]).  `allow` is a host bitmap over row ids: bit (r & 31) of word r >> 5 set = row
 * id r may be returned; ids >= allow_bits are excluded.  Excluded rows are dropped before the
 * top-k (and before refine), so up to k allowed rows come back from the probed partitions. */
int lgpu_search_filtered(lgpu_index *ix, const float *queries, uint32_t B,
                         const lgpu_search_params *params,
                         const uint32_t *allow, uint64_t allow_bits,
                         uint64_t *out_ids, float *out_dist, uint32_t *out_count);

/* Same, all five buffers in DEVICE memory of the index's device; enqueued on
 * `cuda_stream` (a cudaStream_t, may be 0) and NOT synchronised on return. */
int lgpu_search_device(lgpu_index *ix, const float *d_queries, uint32_t B,
                       const lgpu_search_params *params,
                       uint64_t *d_out_ids, float *d_out_dist, uint32_t *d_out_count,
                       void *cuda_stream);

/* Merge `nlists` per-rank top-k lists per query (device buffers laid out
 * [nlists][B][k], as produced by an all-gather of lgpu_search_device outputs over
 * partition-sharded indexes) into the global top-k by (_distance,_rowid). */
int lgpu_merge_topk_device(int device, uint32_t nlists, uint32_t B, uint32_t k,
                           const uint64_t *d_ids, const float *d_dist,
                           uint64_t *d_out_ids, float *d_out_dist, uint32_t *d_out_count,
                           void *cuda_stream);

/* ---- 4-bit IVF_PQ (lance `IvfPq` with num_bits = 4, rust/lancedb/src/table/create_index.rs:86-102, 283-303): an
 * ordinary lgpu_index_desc with nbits = 4.  m is even, dim % m == 0, dim / m is 1, 2, 4, 8, 16 or 32 and
 * m <= LGPU_PQ4_MAX_M; codebook is [m][16][dim/m]; codes are nrows * m / 2 bytes, byte j of a row holding sub-vector
 * 2j's code in bits 0-3 and sub-vector 2j+1's in bits 4-7 [lance, recalled]; LGPU_CODES_ROW_MAJOR is [nrows][m/2],
 * LGPU_CODES_PARTITION_TRANSPOSED is [m/2][n_p] per partition.  Any nbits other than 4 or 8 is LGPU_INVALID_INPUT.
 * Per query (normalised first for cosine) and probed partition p, with r = q - c_p (l2, cosine) or q (dot):
 *   1. T[i][j] (i < m, j < 16) = the 8-bit path's table entry on the 16 codewords (sub-vector L2, or 1 - dot).
 *   2. qmin = min over every T; qmax = max over i = 0 .. m-2 of (max_j T[i][j] + max_j T[i+1][j]); both folds skip
 *      NaN (an all-NaN fold is +inf / -inf) [lance, recalled].
 *   3. Q[i][j] = sat_u8(round(((T[i][j] - qmin) * 255) / (qmax - qmin))): each f32 op rounded to nearest, left to
 *      right, round half away from zero, NaN and below 0 -> 0, above 255 -> 255 [lance, recalled].
 *   4. S = sum_i Q[i][code_i], an exact integer.
 *   5. d = ((float) S * (qmax - qmin)) / 255 + qmin * (float) m, each op in f32 without FMA, in this order
 *      [lance, recalled]; cosine reports 0.5 d, dot d - (m - 1).
 * A row whose d is NaN is never returned.  Everything else -- k, nprobes, maximum_nprobes, prefilter, distance_range
 * (on d, before refine), refine_factor, timeout_ms and every search entry point -- is IVF_PQ's.
 * lgpu_debug_partition_distances serves the index; lgpu_search_sharded* and lgpu_debug_filter_bounds reject it. */
#define LGPU_PQ4_MAX_M 256        /* a slot's sum stays below 2^16 (255 x 256) */

/* ---- IVF_SQ (lance `IvfSq`, rust/lancedb/src/index/vector.rs:216-256): the same IVF partitions, each row stored as
 * dim 8-bit scalar codes instead of PQ codes.  One global range [lo, hi] (f64) quantises every component:
 *     code(v) = sat_u8(((double)v - lo) * 255.0 / (hi - lo))
 * evaluated left to right in f64, truncated toward zero, below 0 -> 0, above 255 -> 255, NaN -> 0, and 0 when lo == hi
 * (lance's scale_to_u8 [lance, recalled]).  Rows are encoded by the builder (normalised first for cosine); queries are
 * encoded on the device with the same f64 operations (after normalisation for cosine).
 *     _distance = (float) sum_i (k_i - q_i)^2
 * summed exactly in integers, then rounded to nearest f32, for l2 and cosine alike (not halved for cosine), in code
 * units; refine_factor re-ranks with exact f32 distances on desc.vectors.  dot is not supported (LGPU_INVALID_INPUT).
 * Partition assignment is find_partitions (lgpu_ivf_assign), there are no residuals.  The handle is an ordinary
 * lgpu_index: lgpu_search, _filtered, _device, _async and _coalesced serve it with the IVF_PQ semantics of k, nprobes,
 * maximum_nprobes, prefilter, distance_range (on the SQ distance, before refine), refine_factor and timeout_ms.
 * lgpu_search_sharded*, lgpu_debug_filter_bounds and lgpu_debug_partition_distances reject it. */
#define LGPU_SQ_MAX_DIM 65536     /* the exact sum stays below 2^32 */
typedef struct {
    uint32_t abi_version;         /* LGPU_ABI_VERSION */
    uint32_t dim;                 /* 1 .. LGPU_SQ_MAX_DIM */
    uint32_t nlist;
    int32_t  metric;              /* LGPU_L2 or LGPU_COSINE */
    int32_t  device;
    uint32_t reserved;            /* 0 */
    uint64_t nrows;
    double   lo, hi;              /* quantiser bounds, finite, lo <= hi */
    const float    *centroids;    /* [nlist][dim] */
    const uint64_t *part_offsets; /* [nlist+1] */
    const uint8_t  *codes;        /* [nrows][dim] row codes in partition order */
    const uint64_t *row_ids;      /* [nrows] */
    const float    *vectors;      /* optional [nrows][dim] raw vectors (refine_factor); NULL if absent */
} lgpu_ivf_sq_desc;
int lgpu_ivf_sq_open(const lgpu_ivf_sq_desc *desc, lgpu_index **out);

/* ---- IVF_RQ (lance `IvfRq`, RaBitQ with num_bits = 1; rust/lancedb/src/index/vector.rs:321-369): the same IVF
 * partitions, each row stored as one sign bit per dimension of its rotated residual plus two f32 factors.  With P the
 * f32 [dim][dim] orthogonal rotation and o = P (x - c_p) (f64, at build time): bit i = [o_i > 0] (bit i & 7 of byte
 * i >> 3, padding bits 0), add = (float) sum o_i^2, scale = (float) (-2 sum o_i^2 / sum |o_i|), both 0 when o = 0.
 * Search (every operation rounded to f32 on its own, no FMA): rq_i = dot(P row i, q) and rc_{p,i} = dot(P row i, c_p)
 * in lance's lane order (q normalised first for cosine); per probe slot q'_i = rq_i - rc_{p,i}, lo = min q',
 * delta = (max q' - lo) / 15, u_i = min(15, trunc((q'_i - lo) / delta + 0.5)) (0 when delta is 0), S = sum u_i,
 * qq = l2(rq, rc_p); per row ip = sum_i b_i u_i (exact), pc = popcount(b),
 *     y = delta * (float)(2 ip - S) + lo * (float)(2 pc - dim),   est = (add + qq) + scale * y
 * and _distance = est (l2) or 0.5 est (cosine, the scale of the exact cosine distance refine_factor reports).  The
 * estimate may be negative.  A slot with a NaN component in q' or a non-finite delta contributes no rows, and a NaN
 * estimate is never returned.  dot and num_bits != 1 are not supported (LGPU_INVALID_INPUT).  The handle is an
 * ordinary lgpu_index: lgpu_search, _filtered, _device, _async and _coalesced serve it with the IVF_PQ semantics of k,
 * nprobes, maximum_nprobes, prefilter, distance_range (on the estimate, before refine), refine_factor and timeout_ms.
 * lgpu_search_sharded*, lgpu_debug_filter_bounds and lgpu_debug_partition_distances reject it. */
#define LGPU_RQ_MAX_DIM 4096      /* P at most 64 MB; every integer above stays exact in f32 */
typedef struct {
    uint32_t abi_version;         /* LGPU_ABI_VERSION */
    uint32_t dim;                 /* 1 .. LGPU_RQ_MAX_DIM */
    uint32_t nlist;
    int32_t  metric;              /* LGPU_L2 or LGPU_COSINE */
    int32_t  device;
    uint32_t num_bits;            /* 1 */
    uint64_t nrows;
    const float    *centroids;    /* [nlist][dim] */
    const float    *rotation;     /* [dim][dim] P, row-major */
    const uint64_t *part_offsets; /* [nlist+1] */
    const uint8_t  *codes;        /* [nrows][ceil(dim / 8)] sign bits in partition order */
    const float    *add_factors;  /* [nrows] */
    const float    *scale_factors;/* [nrows] */
    const uint64_t *row_ids;      /* [nrows] */
    const float    *vectors;      /* optional [nrows][dim] raw vectors (refine_factor); NULL if absent */
} lgpu_ivf_rq_desc;
int lgpu_ivf_rq_open(const lgpu_ivf_rq_desc *desc, lgpu_index **out);

/* ---- partition-sharded search across GPUs (SURVEY.md 8e; the reference is single-process, so there is no
 * reference interface to replace -- this is what north_star adds for an index larger than one GPU's HBM).
 * One process (or thread) per GPU.  Centroids and codebook are replicated, every partition's codes and row ids
 * live on exactly one rank (non-owned partitions are empty in that rank's lgpu_index), every rank receives the
 * same query batch, and the only data-path collective is ONE ncclAllGather of [B][k] 16-byte (_rowid, _distance)
 * records per batch, merged on every rank by (_distance, _rowid).  NCCL is bound at run time (dlopen of
 * libnccl.so.2), so hosts that never shard need no NCCL.  The host distributes the unique id over whatever
 * channel it already has (the Rust crate: its RPC layer; the Python mirror: torch.distributed / a file). ---- */
#define LGPU_COMM_ID_BYTES 128
typedef struct lgpu_comm lgpu_comm;
/* rank 0: create the group's id (an ncclUniqueId), to be handed to every rank */
int  lgpu_comm_unique_id(void *id_out, size_t id_bytes);
/* every rank, collectively: join the group on CUDA device `device` */
int  lgpu_comm_init(const void *unique_id, size_t id_bytes, int rank, int world, int device, lgpu_comm **out);
void lgpu_comm_destroy(lgpu_comm *comm);
/* collective: every rank passes the same B queries (host buffers) and its own shard; every rank receives the
 * global top-k.  refine_factor must be 0. */
int  lgpu_search_sharded(lgpu_index *shard, lgpu_comm *comm, const float *queries, uint32_t B,
                         const lgpu_search_params *params,
                         uint64_t *out_ids, float *out_dist, uint32_t *out_count);
/* same with device buffers, enqueued on `cuda_stream`, not synchronised */
int  lgpu_search_sharded_device(lgpu_index *shard, lgpu_comm *comm, const float *d_queries, uint32_t B,
                                const lgpu_search_params *params,
                                uint64_t *d_out_ids, float *d_out_dist, uint32_t *d_out_count,
                                void *cuda_stream);
/* device time (ms) of the local search, the all-gather and the merge of the most recent sharded call made with
 * profiling on (lgpu_set_profiling).  times: [3] */
int  lgpu_comm_last_stage_ms(lgpu_comm *comm, float *times);

/* ---- index build passes (SURVEY.md 8f-2; reference: IVF_PQ build through lance, parameters at
 * rust/lancedb/src/table/create_index.rs:283-303, rust/lancedb/src/index/vector.rs:246-319; "GPU support in
 * building vector index", python/python/lancedb/table.py:2883-2937).  k-means training stays with the caller;
 * these are the two passes over every row, bit-consistent with the search kernels.  All pointers are HOST
 * memory; vectors are raw rows (normalised internally for LGPU_COSINE). ------------------------------- */
/* out_parts[r] = the partition find_partitions(vectors[r], nprobes = 1) returns */
int lgpu_ivf_assign(const float *centroids, uint32_t nlist, uint32_t dim, int metric,
                    const float *vectors, uint64_t n, int device, uint32_t *out_parts);
/* out_codes[r][i] (row-major [n][m]) = the codeword of sub-space i with the smallest distance-table entry
 * for row r's residual (row - centroid[parts[r]]; the row itself for LGPU_DOT); ties go to the lowest code */
int lgpu_pq_encode(const float *centroids, const float *codebook, uint32_t nlist, uint32_t dim, uint32_t m,
                   int metric, const float *vectors, const uint32_t *parts, uint64_t n, int device,
                   unsigned char *out_codes);

/* k-means TRAINING on the GPU (the Lloyd loops of the IVF_PQ build; parameters max_iterations / sample_rate at
 * rust/lancedb/src/index/vector.rs:286-297).  x: HOST [n][dim] training rows (already sampled, normalised for cosine).
 * centroids: in = initial centres (e.g. k sampled rows), out = trained centres.  Assignment is the search's own coarse
 * step (exact nearest centre), empty clusters keep their previous centre.  *inertia_out (optional) = sum of squared
 * distances of the rows to their nearest trained centre. */
int lgpu_kmeans_train(const float *x, uint64_t n, uint32_t dim, float *centroids, uint32_t k, uint32_t iters, int device,
                      double *inertia_out);
/* the 256-entry PQ codebooks of all m sub-spaces: x = HOST [n][dim] rows to quantise (residuals for l2 / cosine, raw rows
 * for dot); codebook [m][256][dim/m] in = initial codewords, out = trained */
int lgpu_pq_train(const float *x, uint64_t n, uint32_t dim, uint32_t m, float *codebook, uint32_t iters, int device);

/* ---- flat / brute force (LanceRead -> KNNVectorDistance -> TopK) ---------
 * A column of at least 4096 rows with dim a multiple of 8 is scored on the tensor cores (l2, no prefilter or
 * distance_range, B >= 8) with an exact re-score of every row inside the bf16 error band; a column holding a NaN or inf,
 * or a row whose |x|^2 overflows, has no finite band and is always served by the exact kernels, and so is any query
 * whose band is not finite.  NaN distances are never returned, +-inf ones are ordered like any other. */
int  lgpu_flat_open(const float *vectors, uint64_t nrows, uint32_t dim,
                    const uint64_t *row_ids /* NULL => 0..nrows-1 */, int device,
                    lgpu_flat **out);
void lgpu_flat_close(lgpu_flat *fl);
int  lgpu_flat_search(lgpu_flat *fl, int metric, const float *queries, uint32_t B,
                      const lgpu_search_params *params,
                      uint64_t *out_ids, float *out_dist, uint32_t *out_count);
/* flat search under a row-id allow-list (same bitmap as lgpu_search_filtered) */
int  lgpu_flat_search_filtered(lgpu_flat *fl, int metric, const float *queries, uint32_t B,
                               const lgpu_search_params *params,
                               const uint32_t *allow, uint64_t allow_bits,
                               uint64_t *out_ids, float *out_dist, uint32_t *out_count);
int  lgpu_flat_search_device(lgpu_flat *fl, int metric, const float *d_queries, uint32_t B,
                             const lgpu_search_params *params,
                             uint64_t *d_out_ids, float *d_out_dist, uint32_t *d_out_count,
                             void *cuda_stream);

/* ---- binary vectors: flat search by Hamming distance (the `is_binary` branch of
 * rust/lancedb/src/table/query.rs:229-236: fixed_size_list<uint8, nbytes> columns, distance_type("hamming")) ----
 * _distance = popcount(q XOR x) over the nbytes bytes, an integer in [0, 8 nbytes] (exact in f32; 8 nbytes <= 2^24).
 * Results are ascending by (_distance, _rowid), as on the float flat path; k, distance_range, timeout_ms, k > nrows
 * and nrows = 0 behave as there, nprobes and refine_factor are ignored.  vectors: [nrows][nbytes]; queries:
 * [B][nbytes]. */
int  lgpu_binary_open(const uint8_t *vectors, uint64_t nrows, uint32_t nbytes,
                      const uint64_t *row_ids /* NULL => 0..nrows-1 */, int device, lgpu_binary **out);
void lgpu_binary_close(lgpu_binary *bx);
int  lgpu_binary_search(lgpu_binary *bx, const uint8_t *queries, uint32_t B, const lgpu_search_params *params,
                        uint64_t *out_ids, float *out_dist, uint32_t *out_count);
/* under a row-id allow-list (same bitmap as lgpu_search_filtered) */
int  lgpu_binary_search_filtered(lgpu_binary *bx, const uint8_t *queries, uint32_t B, const lgpu_search_params *params,
                                 const uint32_t *allow, uint64_t allow_bits,
                                 uint64_t *out_ids, float *out_dist, uint32_t *out_count);
/* all five buffers in DEVICE memory, enqueued on `cuda_stream`, not synchronised */
int  lgpu_binary_search_device(lgpu_binary *bx, const uint8_t *d_queries, uint32_t B, const lgpu_search_params *params,
                               uint64_t *d_out_ids, float *d_out_dist, uint32_t *d_out_count, void *cuda_stream);

/* ---- binary IVF_FLAT (lance `IvfFlat` with distance_type("hamming"), the index LanceDB builds over
 * fixed_size_list<uint8, nbytes> columns; rust/lancedb/src/index/vector.rs:169-209): packed binary centroids and the
 * rows grouped by partition.  Search, per query: the nprobes partitions whose centroids are nearest by Hamming distance
 * (ties to the lower partition id; every partition when nprobes >= nlist), then every row of those partitions scored
 * exactly, _distance = popcount(q XOR x) as f32, ascending by (_distance, _rowid).  k, nprobes, maximum_nprobes (under
 * a prefilter), prefilter, distance_range (before the top-k) and timeout_ms behave as on lgpu_index; refine_factor is
 * accepted and changes nothing (the distances are exact; k x refine_factor is not limited).  With nprobes >= nlist the
 * result is lgpu_binary_search's.  nprobes above 2048 must cover every partition, and so must maximum_nprobes above
 * 2048 when it widens (under a prefilter).  queries: [B][nbytes]. */
typedef struct {
    uint32_t abi_version;         /* LGPU_ABI_VERSION */
    uint32_t nbytes;              /* bytes per vector, 8 nbytes <= 2^24 */
    uint32_t nlist;
    int32_t  device;
    uint64_t nrows;
    const uint8_t  *centroids;    /* [nlist][nbytes] packed bits */
    const uint64_t *part_offsets; /* [nlist+1] */
    const uint8_t  *vectors;      /* [nrows][nbytes] in partition order */
    const uint64_t *row_ids;      /* [nrows] */
} lgpu_ivf_binary_desc;
int  lgpu_ivf_binary_open(const lgpu_ivf_binary_desc *desc, lgpu_ivf_binary **out);
void lgpu_ivf_binary_close(lgpu_ivf_binary *ix);
int  lgpu_ivf_binary_search(lgpu_ivf_binary *ix, const uint8_t *queries, uint32_t B, const lgpu_search_params *params,
                            uint64_t *out_ids, float *out_dist, uint32_t *out_count);
int  lgpu_ivf_binary_search_filtered(lgpu_ivf_binary *ix, const uint8_t *queries, uint32_t B,
                                     const lgpu_search_params *params, const uint32_t *allow, uint64_t allow_bits,
                                     uint64_t *out_ids, float *out_dist, uint32_t *out_count);
int  lgpu_ivf_binary_search_device(lgpu_ivf_binary *ix, const uint8_t *d_queries, uint32_t B,
                                   const lgpu_search_params *params, uint64_t *d_out_ids, float *d_out_dist,
                                   uint32_t *d_out_count, void *cuda_stream);

/* ---- multivector columns: exact late-interaction (MaxSim) flat search (the `DataType::List` branch of
 * rust/lancedb/src/table/query.rs:180-199: list<fixed_size_list<float, dim>> columns; the query's vectors are packed
 * into ONE query, python/python/lancedb/query.py:3376-3382) ----
 * A row r holds n_r >= 0 vectors v_j, a query nq >= 1 vectors q_i, and
 *     _distance = sum_i min_j cosd(q_i, v_j),  summed over i in order in f32 from 0.0f,
 * cosd = 1 - q.v / |q| / sqrt(v.v) in lance's lane order (the flat path's cosine).  A pair whose cosd is NaN is
 * skipped by the min; a row where some q_i has no other pair -- an empty row, a zero or NaN query vector -- has a NaN
 * distance and is never returned.  Results are ascending by (_distance, _rowid); k, distance_range (on the summed
 * distance), the prefilter bitmap, timeout_ms, k > nrows and nrows = 0 behave as on the float flat path; nprobes and
 * refine_factor are ignored.
 * values: [T][dim] f32, T = offsets[nrows]; offsets: [nrows+1] u64, offsets[0] = 0, non-decreasing; row r's vectors
 * are values[offsets[r] .. offsets[r+1]).  Limits: dim <= 65536, n_r <= 2^20, T <= 2^40.
 * queries: [Tq][dim] f32, Tq = q_offsets[B]; q_offsets: [B+1] u32 HOST array (also for the device entry point: it is
 * the batch's shape), q_offsets[0] = 0, query b's vectors are queries[q_offsets[b] .. q_offsets[b+1]), 1..4096 each.
 * Columns of at least 65536 vectors, all finite and non-zero, with dim a multiple of 8, are scored on the tensor cores
 * (fp16 copies of the normalised vectors) when the call has no prefilter or distance_range: every row within a
 * rigorous error band of the k-th approximate distance is re-scored exactly, and a query whose shortlist overflows or
 * that holds a zero / non-finite vector is redone exactly, so the results are the exact ones either way.
 * lgpu_last_filter_stats after a profiled multivector call: [0] rows admitted to the shortlists, [1] rows scored
 * exactly (on the exact path: B x nrows), [2] queries redone densely after the shortlist, [3] queries. */
int  lgpu_multivec_open(const float *values, const uint64_t *offsets, uint64_t nrows, uint32_t dim,
                        const uint64_t *row_ids /* NULL => 0..nrows-1 */, int device, lgpu_multivec **out);
void lgpu_multivec_close(lgpu_multivec *mv);
int  lgpu_multivec_search(lgpu_multivec *mv, const float *queries, const uint32_t *q_offsets, uint32_t B,
                          const lgpu_search_params *params, uint64_t *out_ids, float *out_dist, uint32_t *out_count);
/* under a row-id allow-list (same bitmap as lgpu_search_filtered) */
int  lgpu_multivec_search_filtered(lgpu_multivec *mv, const float *queries, const uint32_t *q_offsets, uint32_t B,
                                   const lgpu_search_params *params, const uint32_t *allow, uint64_t allow_bits,
                                   uint64_t *out_ids, float *out_dist, uint32_t *out_count);
/* d_queries and the three outputs in DEVICE memory (q_offsets stays on the host), enqueued on `cuda_stream`, not
 * synchronised */
int  lgpu_multivec_search_device(lgpu_multivec *mv, const float *d_queries, const uint32_t *q_offsets, uint32_t B,
                                 const lgpu_search_params *params, uint64_t *d_out_ids, float *d_out_dist,
                                 uint32_t *d_out_count, void *cuda_stream);

/* ---- per-stage access (parity localisation and kernel benchmarks) -------- */
/* coarse stage only: the nprobes nearest partitions of each query and their
 * distances (host buffers, [B][nprobes]) */
int lgpu_debug_coarse(lgpu_index *ix, const float *queries, uint32_t B, uint32_t nprobes,
                      uint32_t *out_parts, float *out_dists);
/* final PQ distances of every row of partition `part` for one query (host
 * buffers; out has n_p floats) -- exercises the LUT build + code scan kernels */
int lgpu_debug_partition_distances(lgpu_index *ix, const float *query, uint32_t part,
                                   float *out);
/* the filter scan (dense mode) for B queries and their nprobes nearest partitions, instead of a search
 * result (host buffers): out_parts [B][nprobes] the probed partitions (UINT32_MAX = unused slot),
 * out_L [B][nprobes][ld] the lower bound L the scan kernel computed for row r < min(n_p, ld) of the slot's
 * partition, out_W / out_E [B] the band W, E of every query (unscaled: the exact distance lies in
 * [L - s E, L + s (W + E)], s = 0.5 for cosine, else 1), out_bad [B] 1 when the query goes to the exact path */
int lgpu_debug_filter_bounds(lgpu_index *ix, const float *queries, uint32_t B, uint32_t nprobes, uint64_t ld,
                             uint32_t *out_parts, float *out_L, float *out_W, float *out_E, uint32_t *out_bad);
/* the tensor-core shortlist GEMM alone: out[q][x] = |x|^2 - 2 bf16(Q[q]).bf16(X[x]) (host buffers,
 * out is [B][N] f32); dim must be a multiple of 8 */
int lgpu_debug_gemm(const float *queries, const float *vectors, uint32_t B, uint64_t N, uint32_t dim,
                    int device, float *out);
/* the binary tensor-core kernel alone: out[q][x] = Hamming distance of queries[q] and vectors[x] (host buffers,
 * queries [B][nbytes], vectors [N][nbytes], out [B][N] u32) */
int lgpu_debug_hamming_gemm(const uint8_t *queries, const uint8_t *vectors, uint32_t B, uint64_t N, uint32_t nbytes,
                            int device, uint32_t *out);
/* the binary IVF_FLAT scan kernel alone, every query one probe slot over one partition of N rows: out[q][x] = Hamming
 * distance of queries[q] and vectors[x] (host buffers: queries [B][nbytes], vectors [N][nbytes], out [B][N] u32;
 * B x N < 2^32) */
int lgpu_debug_ivf_hamming_scan(const uint8_t *queries, uint32_t B, const uint8_t *vectors, uint64_t N, uint32_t nbytes,
                                int device, uint32_t *out);
/* the IVF_SQ scan kernel alone, on one partition of the N rows that every query probes: out[q][x] = sum_i
 * (x_codes[x][i] - q_codes[q][i])^2, the exact u32 sum (host buffers: q_codes [B][dim], x_codes [N][dim], out [B][N];
 * dim <= 65536, B x N < 2^32) */
int lgpu_debug_sq_distances(const uint8_t *q_codes, uint32_t B, const uint8_t *x_codes, uint64_t N, uint32_t dim,
                            int device, uint32_t *out);
/* the 4-bit IVF_PQ scan kernel alone, every query one probe slot over one partition of N rows: out[q][x] = sum_i
 * tables[q][i][code_i(x)], the exact u32 sum (host buffers: tables [B][m][16] u8, codes [N][m/2] packed as in the
 * index, out [B][N]; m even, 2 <= m <= LGPU_PQ4_MAX_M, B x N < 2^32) */
int lgpu_debug_pq4_sums(const uint8_t *tables, uint32_t B, const uint8_t *codes, uint64_t N, uint32_t m, int device,
                        uint32_t *out);
/* the IVF_RQ planes and scan kernels alone, every query one probe slot over one partition of N rows: q_res [B][dim] the
 * rotated residuals q', codes [N][ceil(dim / 8)], add / scale [N]; out_est [B][N] the reported estimates (NaN where the
 * slot has no rows), out_ip [B][N] the exact ip = sum_i b_i u_i (either may be NULL; host buffers; dim <= 4096,
 * B x N < 2^32) */
int lgpu_debug_rq_distances(const float *q_res, uint32_t B, const uint8_t *codes, const float *add_factors,
                            const float *scale_factors, uint64_t N, uint32_t dim, int metric, int device,
                            float *out_est, uint32_t *out_ip);
/* the multivector tensor-core score alone: out[i][r] = the largest fp16(q_i / |q_i|) . fp16(v / |v|) (f32 accumulation)
 * over row r's vectors v, NaN for an empty row (host buffers: queries [nqv][dim], values [offsets[nrows]][dim],
 * out [nqv][nrows] f32); dim must be a multiple of 8 */
int lgpu_debug_maxsim_gemm(const float *queries, uint32_t nqv, const float *values, const uint64_t *offsets,
                           uint64_t nrows, uint32_t dim, int device, float *out);
/* the number of queries per sub-batch an lgpu_search* call of B queries and `nprobes` probes (the widest the call uses:
 * maximum_nprobes under a prefilter) on `ix` runs in under the process's LGPU_WS_BYTES: B when the batch is not split */
int lgpu_debug_sub_batch_size(lgpu_index *ix, uint32_t B, uint32_t nprobes, uint32_t *out);
/* per-stage device time (ms) of the most recent profiled lgpu_search* / lgpu_ivf_binary_search* call on this thread:
 * coarse, select-probes, group, scan, top-k, refine, total.  times: [7].  A call the workspace budget splits into
 * sub-batches reports, per stage, the sum over its sub-batches (profiling synchronises after each one); the
 * maximum_nprobes widening passes are not timed.  lgpu_last_scanned_code_bytes covers the same: the code bytes every
 * sub-batch's first pass handed to the scan (0 for a sub-batch on the small path, which has no regroup). */
int lgpu_last_stage_ms(float *times);
/* filter-scan counters of the most recent profiled lgpu_search* call on this thread, summed over the call's sub-batches
 * (each sub-batch picks its own filter mode): candidates the scanners appended and survivors re-scored exactly
 * (candidate mode only), queries sent to the exact fix-up pass, queries that went through the filter scan (a
 * sub-batch on the exact or the small path adds none).  stats: [4]
 * After lgpu_binary_search* (whole batch): [0] candidates the tensor-core list pass appended (0 on the dense paths),
 * [1] distances computed on the tensor cores (0 on the SIMT path), [2] queries redone densely after a list overflow,
 * [3] queries.  After lgpu_multivec_search*: see the multivector section above. */
int lgpu_last_filter_stats(uint64_t *stats);
/* kernels this process has launched through the library so far (eager launches and graph replays alike) */
int lgpu_kernel_launch_count(uint64_t *count);
/* switch per-stage CUDA-event timing (and the scanned-bytes counter) on/off for the
 * calling process; overrides LGPU_PROFILE.  While on, lgpu_search_device synchronises
 * the stream before returning. */
int lgpu_set_profiling(int enabled);

#ifdef __cplusplus
}
#endif
#endif
