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

/* Largest k (limit + offset) and k x refine_factor every single-GPU search serves (rust/lancedb/src/table/query.rs:231
 * passes limit + offset to the scanner unbounded).  k up to 2048 runs the shared-memory selects, above that the
 * global-memory radix select (DESIGN.md section 3).  The sharded search and lgpu_merge_topk_device keep k <= 2048. */
#define LGPU_K_MAX 65536

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
typedef struct lgpu_multivec lgpu_multivec; /* a multivector column in HBM or pinned host memory, searched by late
                                             * interaction (MaxSim) */
typedef struct lgpu_ivf_binary lgpu_ivf_binary; /* a binary IVF_FLAT index in HBM, searched by Hamming distance */

/* The arrays of one IVF_PQ index (lance v2 `IvfPq`,
 * rust/lancedb/src/table/create_index.rs:283-303, :772): IVF centroids, PQ codebook
 * (8-bit, 256 centroids per sub-vector), PQ codes and row ids grouped by partition. */
typedef struct {
    uint32_t abi_version;        /* LGPU_ABI_VERSION */
    uint32_t dim;                /* no upper limit is checked.  8-bit codes: the filter scan serves m <= 512, so
                                    dim <= 16384 (dim / m <= 32), where its band's underflow floor is argued; a wider
                                    index takes the exact scan, tested bit for bit up to dim 32768 (m 1024 and 2048) */
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
    uint32_t k;              /* limit + offset (table/query.rs:231); default 10; k and k x refine_factor at most
                                LGPU_K_MAX */
    uint32_t nprobes;        /* maximum_nprobes (== minimum_nprobes == 20 by default) */
    uint32_t refine_factor;  /* 0 = no refine (query.rs:1302-1332) */
    int32_t  has_lower;      /* distance_range lower bound, inclusive */
    int32_t  has_upper;      /* distance_range upper bound, exclusive */
    float    lower;
    float    upper;
    uint32_t ef;             /* IVF_HNSW_SQ: the search beam (query.rs:1290-1300); 0 = ceil(1.5 k).  Every other kind
                                ignores it */
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
/* bytes of HBM held by the index (codes when they are in HBM + ids + centroids + codebook, and the raw vectors when
 * they are in HBM) */
int  lgpu_index_device_bytes(const lgpu_index *ix, uint64_t *bytes);
/* Where an index keeps the raw vectors desc.vectors gave it (refine_factor).  Every float IVF open (lgpu_index_open,
 * lgpu_ivf_sq_open, lgpu_ivf_hnsw_sq_open, lgpu_ivf_rq_open) copies them into HBM when they fit with room to spare: the
 * device's free memory, once the rest of the index is in place, covers them plus the workspace budget (LGPU_WS_BYTES,
 * default 8 GiB), and they are at most LGPU_VECTORS_HBM_BYTES (read at every open; unset = no cap, 0 = never in HBM).
 * Otherwise the index copies them into pinned, mapped host memory that it owns (rows padded to a multiple of 4 floats,
 * freed by lgpu_index_close) and refine reads the k x refine_factor candidates over PCIe; results are identical.  A
 * pinned allocation that fails is LGPU_OOM.  The caller's buffer is borrowed for the open call only, either way. */
typedef enum { LGPU_VECTORS_NONE = 0, LGPU_VECTORS_HBM = 1, LGPU_VECTORS_HOST = 2 } lgpu_vectors_placement;
/* bytes of pinned host memory held by the index (nrows x round_up(dim, 4) x 4 when the raw vectors are on the host,
 * else 0) and where the raw vectors are (lgpu_vectors_placement); either output may be NULL */
int  lgpu_index_host_bytes(const lgpu_index *ix, uint64_t *bytes, int *placement);
/* sum over a batch of the PQ code bytes its probes must scan (the roofline's
 * algorithmic bytes, SURVEY.md 8d); valid for the most recent search on the
 * calling thread */
int  lgpu_last_scanned_code_bytes(uint64_t *bytes);
/* bytes of host-resident codes (lgpu_index_code_bytes) the most recent IVF search on the calling thread copied into HBM,
 * every sub-batch and maximum_nprobes pass included; counted while profiling (LGPU_PROFILE=1, lgpu_set_profiling),
 * else 0 */
int  lgpu_last_streamed_code_bytes(uint64_t *bytes);

/* Where an IVF index keeps its stored codes.  lgpu_ivf_sq_open, lgpu_ivf_rq_open and lgpu_ivf_binary_open put them in
 * HBM when they fit with room to spare: the device's free memory, once the centroids, partition arrays and per-row terms
 * are in place, covers them plus the workspace budget (LGPU_WS_BYTES), and they are at most LGPU_CODES_HBM_BYTES (read
 * at every open; unset = no cap, 0 = never in HBM).  Otherwise the index keeps them in pinned, mapped host memory that
 * it owns, in the HBM layout (IVF_SQ [nrows][dim_pad] bytes, dim_pad = dim rounded up to 64; IVF_RQ [nrows][wpr] u32,
 * wpr = dim rounded up to 256 bits; binary IVF_FLAT [nrows][nbytes_pad], nbytes_pad = nbytes rounded up to 32; padding
 * zero), and each search copies the partitions its queries probe into HBM in chunks of consecutive partitions, double
 * buffered, scanning one chunk while the next is copied; results are identical.  The per-row terms and row ids stay in
 * HBM.  Two staging buffers of the largest partition must fit the workspace budget, else the open is LGPU_OOM; a pinned
 * allocation that fails is LGPU_OOM too.  The codes are placed before the raw vectors (lgpu_index_host_bytes).
 * IVF_HNSW_SQ (its graph walk reads rows at random) and IVF_PQ (4-bit and 8-bit) keep their codes in HBM whatever the
 * cap says.  host_bytes: the pinned bytes of codes (0 in HBM); placement: LGPU_VECTORS_HBM or LGPU_VECTORS_HOST; either
 * output may be NULL.  lgpu_ivf_binary_code_bytes is the same for a binary IVF_FLAT handle. */
int  lgpu_index_code_bytes(const lgpu_index *ix, uint64_t *host_bytes, int *placement);

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
 * lgpu_search_sharded*, lgpu_debug_filter_bounds and lgpu_debug_partition_distances reject it.  The codes go to pinned
 * host memory when they do not fit in HBM (LGPU_CODES_HBM_BYTES, lgpu_index_code_bytes). */
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

/* ---- IVF_HNSW_SQ (lance `HnswSq`, python/python/tests/test_table.py:1565-1590): IVF_SQ's partitions, codes and
 * distance, plus one HNSW graph per partition over its rows.  Positions are row indices within the partition.
 * Search, per query [lance, recalled]: IVF_SQ's normalisation, coarse step and query codes; then in each probed
 * partition, with rows ordered by (d, position) and d IVF_SQ's f32 distance:
 *   - upper levels: from the partition's entry row on its top level, at each level >= 1 move to the best neighbour
 *     while it is better than the current row; the row reached starts level 0;
 *   - level 0: W = the ef' best rows seen (ef' = max(ef, kk), kk = k or k x refine_factor, ef = 0 meaning
 *     ceil(1.5 k)), W = {start}; while W holds an unexpanded row, expand the best one: evaluate each of its level-0
 *     neighbours and offer it to W;
 *   - the partition contributes R, the kk best evaluated rows (the start row included) that pass the row filter
 *     (distance_range, prefilter); traversal ignores the filter.
 * The R lists are merged by (_distance, _rowid); refine_factor, maximum_nprobes, timeout_ms and every entry point are
 * IVF_SQ's.  ef' above LGPU_HNSW_EF_MAX is LGPU_INVALID_INPUT.  lgpu_search_sharded*, lgpu_debug_filter_bounds and
 * lgpu_debug_partition_distances reject the handle.  The codes stay in HBM whatever LGPU_CODES_HBM_BYTES says. */
#define LGPU_HNSW_MAX_M 64        /* a level-0 list has at most 128 entries */
#define LGPU_HNSW_MAX_LEVEL 15
#define LGPU_HNSW_EF_MAX 2048     /* W lives in shared memory */
#define LGPU_HNSW_NONE 0xFFFFFFFFu
/* Positions are below 2^31: every IVF open refuses a partition of 2^31 rows or more. */
typedef struct {
    lgpu_ivf_sq_desc sq;          /* the IVF_SQ arrays */
    uint32_t m;                   /* 1 .. LGPU_HNSW_MAX_M: level-0 lists hold 2m entries, upper lists m */
    uint32_t reserved;            /* 0 */
    uint64_t upper_blocks;        /* rows of upper_adj */
    const uint8_t  *levels;       /* [nrows] level of each row, <= its partition's top_level */
    const uint32_t *adj0;         /* [nrows][2m] level-0 neighbour positions, LGPU_HNSW_NONE padded */
    const uint32_t *upper_index;  /* [nrows] first upper_adj block of a row with level >= 1 (level L at + L - 1) */
    const uint32_t *upper_adj;    /* [upper_blocks][m] neighbours at level L, each of level >= L, LGPU_HNSW_NONE padded */
    const uint32_t *entry;        /* [nlist] entry row of each non-empty partition; its level is top_level */
    const uint8_t  *top_level;    /* [nlist] <= LGPU_HNSW_MAX_LEVEL */
} lgpu_ivf_hnsw_sq_desc;
int lgpu_ivf_hnsw_sq_open(const lgpu_ivf_hnsw_sq_desc *desc, lgpu_index **out);

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
 * lgpu_search_sharded*, lgpu_debug_filter_bounds and lgpu_debug_partition_distances reject it.  The codes go to pinned
 * host memory when they do not fit in HBM (LGPU_CODES_HBM_BYTES, lgpu_index_code_bytes). */
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
 * global top-k.  refine_factor must be 0 and k at most 2048. */
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
/* out_parts[r] = the partition find_partitions(vectors[r], nprobes = 1) returns.  A row whose distance to every centroid
 * is NaN has no partition, and the call fails with LGPU_INVALID_INPUT: a row holding a NaN, and under LGPU_COSINE an
 * all-zero row (it has no direction: normalising it divides 0 by 0). */
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
 * distances of the rows to their nearest trained centre.  iters = 0 runs one iteration.  Every row must be finite: a row
 * holding a NaN or an infinity fails the call with LGPU_INVALID_INPUT before any device work. */
int lgpu_kmeans_train(const float *x, uint64_t n, uint32_t dim, float *centroids, uint32_t k, uint32_t iters, int device,
                      double *inertia_out);
/* the 256-entry PQ codebooks of all m sub-spaces: x = HOST [n][dim] rows to quantise (residuals for l2 / cosine, raw rows
 * for dot); codebook [m][256][dim/m] in = initial codewords, out = trained.  A codeword no row encodes to keeps its value;
 * iters = 0 runs one iteration; a row holding a NaN or an infinity fails the call with LGPU_INVALID_INPUT. */
int lgpu_pq_train(const float *x, uint64_t n, uint32_t dim, uint32_t m, float *codebook, uint32_t iters, int device);

/* ---- flat / brute force (LanceRead -> KNNVectorDistance -> TopK) ---------
 * A column of at least 4096 rows with dim a multiple of 8 is scored on the tensor cores (l2, no distance_range,
 * B >= 8, k <= 2048; a prefilter or deleted rows keep that path) with an exact re-score of every row inside the bf16
 * error band; a column holding a NaN or inf,
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
/* Append n rows (HOST [n][dim]) to the column; row_ids NULL => the positions that follow (nrows, nrows + 1, ...).
 * Afterwards the handle returns, on every entry point, exactly what lgpu_flat_open on the concatenated rows (and
 * ids) returns.  The call takes the handle alone: it waits for the calls inside it, keeps new ones out, and drains the
 * device before it moves or rewrites a buffer, so a device-route search enqueued earlier still reads what it was given.
 * Storage grows geometrically; the derived data (bf16 copy, |x|^2, norms) is computed for the new rows only. */
int  lgpu_flat_append(lgpu_flat *fl, const float *rows, uint64_t n, const uint64_t *row_ids);

/* ---- float16 columns (fixed_size_list<float16, dim>) kept as float16 in HBM: 2 bytes per element instead of the 6 an
 * f32 handle holds (f32 rows + their bf16 tensor-core copy).  Queries stay f32.  _distance is the f32 distance of the
 * query and the row's exact f32 upcast, so an fp16 handle opened on rows x16 returns exactly -- same ids, counts and
 * distance bits -- what lgpu_flat_open on x16 converted to f32 returns, on every entry point (host, _filtered,
 * _device, and as the tail of lgpu_search_unindexed[_device]), for every metric, k, distance_range, prefilter,
 * deleted rows, appends and sub-batch split.  The paths are chosen as for f32 rows; the l2 tensor-core path multiplies
 * fp16(q) by the stored rows themselves (fp16 wgmma, f32 accumulation) and re-scores its shortlist exactly, and a query
 * with a component beyond fp16's range (|q_i| >= 65520) is served by the exact kernels.
 * vectors / rows: IEEE binary16 bits, [nrows][dim] / [n][dim].  lgpu_flat_append on an fp16 handle, or
 * lgpu_flat_append_f16 on an f32 handle, fails with LGPU_INVALID_INPUT and changes nothing; every other lgpu_flat_*
 * function takes both row types. */
int  lgpu_flat_open_f16(const uint16_t *vectors, uint64_t nrows, uint32_t dim,
                        const uint64_t *row_ids /* NULL => 0..nrows-1 */, int device, lgpu_flat **out);
int  lgpu_flat_append_f16(lgpu_flat *fl, const uint16_t *rows, uint64_t n, const uint64_t *row_ids);
/* *bytes = the device memory the handle holds for its rows and their per-row data (rows, tensor-core operand, |x|^2,
 * row norms once a cosine search computed them, row ids, the live bitmap), capacity kept for appends included; the
 * per-call search workspaces (each within LGPU_WS_BYTES) are not counted.  Both row types.  A handle whose rows are in
 * host memory (lgpu_flat_host_bytes) holds only its row ids and live bitmap here. */
int  lgpu_flat_device_bytes(const lgpu_flat *fl, uint64_t *bytes);
/* Where a flat handle keeps its rows.  lgpu_flat_open and lgpu_flat_open_f16 copy them into HBM, as above, when their
 * row data -- the rows, plus the tensor-core operand and |x|^2 of a column of at least 4096 rows with dim a multiple of
 * 8 (a bf16 copy for f32 rows; fp16 rows are their own) -- is at most LGPU_FLAT_HBM_BYTES (read at every open; unset =
 * no cap, 0 = never in HBM) and the device's free memory covers it plus the workspace budget (LGPU_WS_BYTES, default
 * 8 GiB).  Otherwise the handle copies the rows into pinned host memory that it owns, [nrows][dim] in the row type
 * (freed by lgpu_flat_close), and keeps only the row ids and the live bitmap in HBM.  Every search of such a handle
 * (host, _filtered, _device, and as the tail of lgpu_search_unindexed[_device]) streams the rows through two staging
 * buffers of its workspace, within LGPU_WS_BYTES: each row crosses PCIe once per call when the workspace holds the
 * running top-k of all B queries, else once per group of queries it holds.  Results are identical to an HBM handle's
 * on the same rows -- same ids, counts and distance bits -- for every metric, k, distance_range, prefilter, deleted
 * rows and append.  A handle keeps its placement for life; lgpu_flat_append grows the pinned rows geometrically.  A
 * pinned allocation that fails is LGPU_OOM.  The caller's buffer is borrowed for the open call only, either way.
 * *bytes = the pinned host memory the handle holds (nrows x dim x the element size at open, capacity kept for appends
 * included; 0 for an HBM handle), *placement = LGPU_VECTORS_HBM or LGPU_VECTORS_HOST; either output may be NULL. */
int  lgpu_flat_host_bytes(const lgpu_flat *fl, uint64_t *bytes, int *placement);

/* ---- rows added after an index was built (the reference's unindexed fragments, searched unless fast_search is set;
 * rust/lancedb/src/table/query.rs:289-290).  `tail` holds them.  The result is the top-k by (_distance, _rowid) of
 * the union of
 *   - lgpu_search_filtered's result on the index (k x refine_factor candidates refined to k, maximum_nprobes widening
 *     under a prefilter), and
 *   - the exact flat top-k of the tail under the index's metric (lgpu_flat_search_filtered with the same k),
 * with distance_range and the allow bitmap (over row ids, NULL = no prefilter) applied to both.  k up to LGPU_K_MAX;
 * the tail must have the index's dimension and device.  The host entry point honours timeout_ms; the device entry point
 * takes every buffer, `allow` included, in DEVICE memory and is enqueued on `cuda_stream`, not synchronised.  The call
 * uses a workspace of each handle, each within LGPU_WS_BYTES, plus the two [B][k] lists it merges (DESIGN.md section 2). */
int  lgpu_search_unindexed(lgpu_index *ix, lgpu_flat *tail, const float *queries, uint32_t B,
                           const lgpu_search_params *params, const uint32_t *allow, uint64_t allow_bits,
                           uint64_t *out_ids, float *out_dist, uint32_t *out_count);
int  lgpu_search_unindexed_device(lgpu_index *ix, lgpu_flat *tail, const float *d_queries, uint32_t B,
                                  const lgpu_search_params *params, const uint32_t *d_allow, uint64_t allow_bits,
                                  uint64_t *d_out_ids, float *d_out_dist, uint32_t *d_out_count, void *cuda_stream);

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
/* Append n rows (HOST [n][nbytes]); everything else as lgpu_flat_append. */
int  lgpu_binary_append(lgpu_binary *bx, const uint8_t *rows, uint64_t n, const uint64_t *row_ids);
/* *bytes = the device memory the handle holds for its rows and their per-row data (the rows zero-padded to nbytes_pad
 * = nbytes rounded up to 32, their popcounts, the threshold sample of a handle above 65536 rows, row ids, the live
 * bitmap), capacity kept for appends included; the per-call search workspaces (each within LGPU_WS_BYTES) are not
 * counted.  A handle whose rows are in host memory (lgpu_binary_host_bytes) holds no rows or popcounts here. */
int  lgpu_binary_device_bytes(const lgpu_binary *bx, uint64_t *bytes);
/* Where a binary handle keeps its rows.  lgpu_binary_open packs them into HBM, as above, when the rows and their
 * popcounts, nrows x (nbytes_pad + 4) bytes, are at most LGPU_BINARY_HBM_BYTES (read at every open; unset = no cap,
 * 0 = never in HBM) and the device's free memory covers them plus the workspace budget (LGPU_WS_BYTES, default 8 GiB).
 * Otherwise the handle packs the rows into pinned host memory that it owns, [nrows][nbytes_pad] zero-padded (freed by
 * lgpu_binary_close), and keeps the row ids, the live bitmap and the threshold sample in HBM; the open then needs no
 * HBM that grows with nrows beyond those.  Every search of such a handle (host, _filtered, _device, and as the tail of
 * lgpu_ivf_binary_search_unindexed[_device]) streams the rows through two staging buffers of its workspace, within
 * LGPU_WS_BYTES, as lgpu_flat_host_bytes describes.  Results are identical to an HBM handle's on the same rows -- same
 * ids, counts and distance bits -- for every k, distance_range, prefilter, deleted rows and append.  A handle keeps its
 * placement for life; lgpu_binary_append grows the pinned rows geometrically.  A pinned allocation that fails is
 * LGPU_OOM.  *bytes = the pinned host memory the handle holds (nrows x nbytes_pad at open, capacity kept for appends
 * included; 0 for an HBM handle), *placement = LGPU_VECTORS_HBM or LGPU_VECTORS_HOST; either output may be NULL. */
int  lgpu_binary_host_bytes(const lgpu_binary *bx, uint64_t *bytes, int *placement);

/* ---- deleted rows (the reference's Table::delete; Lance keeps them per dataset in deletion files).  Delete the rows
 * whose ids are among row_ids (HOST [n]); *n_deleted (may be NULL) = how many of those ids were live and are now
 * deleted.  An id the handle does not hold, or already deleted, changes nothing.  Nothing is undeleted: rows appended
 * later (lgpu_*_append) are live, and an append that would give a row the id of a deleted row the handle still holds
 * fails with LGPU_INVALID_INPUT and changes nothing.
 * Every later search on the handle, on every entry point (host, _filtered, _device, _async, _coalesced, _sharded, and
 * each side of an _unindexed union), returns exactly what it would return with the allow bitmap
 * allow AND NOT deleted (with no allow bitmap: every id not deleted), so maximum_nprobes widening applies as under a
 * prefilter.  The handle keeps a device bitmap of its live row ids, one bit per id below id_bound = the largest row
 * id + 1, built by the first delete: a handle never deleted from holds none and searches as before.  Every row id of
 * the handle must be below LGPU_DELETE_ID_BOUND for a delete (and for an append after one), else LGPU_INVALID_INPUT.
 * The call takes the handle alone, as an append does, and invalidates captured CUDA graphs.  lgpu_index_delete serves
 * every float IVF kind; each function refuses a handle of another kind. */
#define LGPU_DELETE_ID_BOUND (1ull << 32)   /* the live bitmap takes at most 512 MiB */
int  lgpu_index_delete(lgpu_index *ix, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted);
int  lgpu_ivf_binary_delete(lgpu_ivf_binary *ix, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted);
int  lgpu_flat_delete(lgpu_flat *fl, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted);
int  lgpu_binary_delete(lgpu_binary *bx, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted);
int  lgpu_multivec_delete(lgpu_multivec *mv, const uint64_t *row_ids, uint64_t n, uint64_t *n_deleted);

/* ---- binary IVF_FLAT (lance `IvfFlat` with distance_type("hamming"), the index LanceDB builds over
 * fixed_size_list<uint8, nbytes> columns; rust/lancedb/src/index/vector.rs:169-209): packed binary centroids and the
 * rows grouped by partition.  Search, per query: the nprobes partitions whose centroids are nearest by Hamming distance
 * (ties to the lower partition id; every partition when nprobes >= nlist), then every row of those partitions scored
 * exactly, _distance = popcount(q XOR x) as f32, ascending by (_distance, _rowid).  k, nprobes, maximum_nprobes (under
 * a prefilter), prefilter, distance_range (before the top-k) and timeout_ms behave as on lgpu_index; refine_factor is
 * accepted and changes nothing (the distances are exact; k x refine_factor is not limited).  With nprobes >= nlist the
 * result is lgpu_binary_search's.  nprobes above 2048 must cover every partition, and so must maximum_nprobes above
 * 2048 when it widens (under a prefilter).  queries: [B][nbytes].  The packed rows go to pinned host memory when they do
 * not fit in HBM (LGPU_CODES_HBM_BYTES, lgpu_ivf_binary_code_bytes). */
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
/* where the packed rows are (LGPU_CODES_HBM_BYTES, see lgpu_index_code_bytes) */
int  lgpu_ivf_binary_code_bytes(const lgpu_ivf_binary *ix, uint64_t *host_bytes, int *placement);
int  lgpu_ivf_binary_search(lgpu_ivf_binary *ix, const uint8_t *queries, uint32_t B, const lgpu_search_params *params,
                            uint64_t *out_ids, float *out_dist, uint32_t *out_count);
int  lgpu_ivf_binary_search_filtered(lgpu_ivf_binary *ix, const uint8_t *queries, uint32_t B,
                                     const lgpu_search_params *params, const uint32_t *allow, uint64_t allow_bits,
                                     uint64_t *out_ids, float *out_dist, uint32_t *out_count);
int  lgpu_ivf_binary_search_device(lgpu_ivf_binary *ix, const uint8_t *d_queries, uint32_t B,
                                   const lgpu_search_params *params, uint64_t *d_out_ids, float *d_out_dist,
                                   uint32_t *d_out_count, void *cuda_stream);
/* lgpu_search_unindexed[_device] for a binary IVF_FLAT index and a binary tail (Hamming distance on both lists) */
int  lgpu_ivf_binary_search_unindexed(lgpu_ivf_binary *ix, lgpu_binary *tail, const uint8_t *queries, uint32_t B,
                                      const lgpu_search_params *params, const uint32_t *allow, uint64_t allow_bits,
                                      uint64_t *out_ids, float *out_dist, uint32_t *out_count);
int  lgpu_ivf_binary_search_unindexed_device(lgpu_ivf_binary *ix, lgpu_binary *tail, const uint8_t *d_queries,
                                             uint32_t B, const lgpu_search_params *params, const uint32_t *d_allow,
                                             uint64_t allow_bits, uint64_t *d_out_ids, float *d_out_dist,
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
 * (fp16 copies of the normalised vectors) when the call has no distance_range: every row within a rigorous error band
 * of the k-th approximate distance is re-scored exactly, and a query whose shortlist overflows or that holds a zero /
 * non-finite vector is redone exactly, so the results are the exact ones either way.  Under a prefilter or deleted rows
 * the k-th distance is taken over the allowed rows and only allowed rows are re-scored; with fewer than k allowed rows
 * every allowed row is.
 * lgpu_last_filter_stats after a profiled multivector call: [0] rows admitted to the shortlists, [1] rows scored
 * exactly (on the exact path: B x nrows), [2] queries redone densely after the shortlist, [3] queries. */
int  lgpu_multivec_open(const float *values, const uint64_t *offsets, uint64_t nrows, uint32_t dim,
                        const uint64_t *row_ids /* NULL => 0..nrows-1 */, int device, lgpu_multivec **out);
/* float16 multivector columns (list<fixed_size_list<float16, dim>>) kept as float16: 2 bytes per element instead of
 * the 6 an f32 handle of the tensor-core shape holds (f32 vectors + their fp16 normalised copy), or the 4 it holds
 * below it.  Queries stay f32.  _distance is the MaxSim distance of the query and the row's exact f32 upcast, so an
 * fp16 handle opened on values x16 returns exactly -- same ids, counts and distance bits -- what lgpu_multivec_open on
 * x16 converted to f32 returns, on every entry point (host, _filtered, _device), for every k, distance_range,
 * prefilter, deleted rows, row ids, sub-batch split and placement (HBM or host), and lgpu_last_filter_stats means the
 * same.  The paths are chosen as for f32 vectors; the tensor-core path multiplies fp16(q / |q|) by the stored vectors
 * themselves (fp16 wgmma, f32 accumulation), scales each similarity by 1 / |v|, and re-scores its shortlist exactly.  A
 * stored inf or NaN component, or a zero vector, sends the column to the exact path, as for f32 vectors.
 * values: IEEE binary16 bits, [T][dim].  Every other lgpu_multivec_* function takes both row types. */
int  lgpu_multivec_open_f16(const uint16_t *values, const uint64_t *offsets, uint64_t nrows, uint32_t dim,
                            const uint64_t *row_ids /* NULL => 0..nrows-1 */, int device, lgpu_multivec **out);
/* Append n rows to the column: values HOST [offsets[n]][dim] in the handle's row type (IEEE binary16 bits for
 * lgpu_multivec_append_f16), offsets HOST [n + 1] as lgpu_multivec_open takes them (offsets[0] = 0, non-decreasing,
 * rows of 0..2^20 vectors, the column at most 2^40 vectors); row_ids NULL => the positions that follow (nrows,
 * nrows + 1, ...).  Afterwards the handle returns, on every entry point, exactly what lgpu_multivec_open[_f16] on the
 * concatenated rows (and ids) returns, and takes the same route: the tensor-core route once the column holds 65536
 * vectors, all finite and non-zero (an append that first gets there builds the fp16 operand of every vector), the exact
 * route from the first appended zero or non-finite vector on.  As lgpu_flat_append: explicit ids stay explicit (ids
 * given to a handle that had none make the old rows' positions explicit); an appended id equal to a deleted id the
 * handle still holds, lgpu_multivec_append on an fp16 handle or lgpu_multivec_append_f16 on an f32 handle, and rows
 * the open would refuse, fail with LGPU_INVALID_INPUT; n = 0 changes nothing.  A refused call changes nothing.  The
 * handle keeps its placement for life: the vectors (and the operand) grow geometrically in HBM or in pinned host
 * memory, and a pinned allocation that fails is LGPU_OOM.  |v|, the row of each vector and the operand are computed
 * for the new vectors only.  The call takes the handle alone, as lgpu_flat_append does. */
int  lgpu_multivec_append(lgpu_multivec *mv, const float *values, const uint64_t *offsets, uint64_t n,
                          const uint64_t *row_ids /* NULL => the positions that follow */);
int  lgpu_multivec_append_f16(lgpu_multivec *mv, const uint16_t *values, const uint64_t *offsets, uint64_t n,
                              const uint64_t *row_ids);
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
/* *bytes = the device memory the handle holds for its vectors and their per-vector and per-row data (vectors in the
 * row type, an f32 handle's tensor-core operand, |v|, the row of each vector, offsets, row ids, the live bitmap); the
 * per-call search workspaces (each within LGPU_WS_BYTES) are not counted.  A handle whose row data is in host memory (lgpu_multivec_host_bytes)
 * holds only |v|, the row of each vector, the offsets, row ids and live bitmap here: 8 bytes per vector. */
int  lgpu_multivec_device_bytes(const lgpu_multivec *mv, uint64_t *bytes);
/* Where a multivector handle keeps its row data: the vectors in the row type, plus, for an f32 handle, the fp16
 * normalised tensor-core operand of a column of the tensor-core shape (at least 65536 vectors, fewer than 2^31, dim a
 * multiple of 8; an fp16 handle's vectors are their own operand).  lgpu_multivec_open[_f16] copies it into HBM when it
 * is at most LGPU_MULTIVEC_HBM_BYTES (read at every open; unset = no cap, 0 = never in HBM) and the device's free
 * memory covers it plus the workspace budget (LGPU_WS_BYTES, default 8 GiB).  Otherwise the handle copies the vectors
 * into pinned host memory that it owns and builds an f32 handle's operand there, both [T][dim] (freed by
 * lgpu_multivec_close).  Every search of such a handle (host, _filtered, _device) streams chunks of whole rows through
 * two staging buffers of its workspace, within LGPU_WS_BYTES: each vector crosses PCIe once per call when the workspace
 * holds the per-query state of all B queries, else once per group of queries it holds; the tensor-core route reads the
 * fp16 operand and re-scores its shortlist from the pinned vectors.  A staging buffer holds the longest row: a search
 * of a handle whose longest row does not fit twice in LGPU_WS_BYTES fails with LGPU_OOM before any device work.
 * Results are identical to an HBM handle's on the same rows -- same ids, counts and distance bits -- for every k,
 * distance_range, prefilter, deleted rows and append, and lgpu_last_filter_stats means the same.  A handle keeps its
 * placement for life; lgpu_multivec_append grows the pinned row data geometrically.  A pinned allocation that fails is
 * LGPU_OOM.  The caller's buffers are borrowed for the open call only,
 * either way.
 * *bytes = the pinned host memory the handle holds (T x dim x 4, plus T x dim x 2 for the operand, for an f32 handle; T
 * x dim x 2 for an fp16 handle; capacity kept for appends included; 0 for an HBM handle), *placement = LGPU_VECTORS_HBM or LGPU_VECTORS_HOST; either output
 * may be NULL. */
int  lgpu_multivec_host_bytes(const lgpu_multivec *mv, uint64_t *bytes, int *placement);

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
/* the same for fp16 values (IEEE binary16 bits), scored as an fp16 multivector handle scores them: out[i][r] = the
 * largest (fp16(q_i / |q_i|) . v) * fl(1 / |v|) (f32 accumulation, f32 reciprocal and product) over row r's
 * vectors v, NaN for an empty row; dim must be a multiple of 8 */
int lgpu_debug_maxsim_gemm_f16(const float *queries, uint32_t nqv, const uint16_t *values, const uint64_t *offsets,
                               uint64_t nrows, uint32_t dim, int device, float *out);
/* the refine kernel of an index whose raw vectors are on the host, alone: out[q][c] = the exact distance (lgpu_metric)
 * of queries[q] and rows[pos[q][c]], +inf where pos is UINT64_MAX -- the value refine_factor re-ranks by.  The rows are
 * copied into pinned, mapped host memory and read from there (host buffers: queries [B][dim], rows [N][dim],
 * pos [B][nc], out [B][nc]) */
int lgpu_debug_refine_host(const float *queries, uint32_t B, const float *rows, uint64_t N, uint32_t dim,
                           const uint64_t *pos, uint32_t nc, int metric, int device, float *out);
/* the number of queries per sub-batch an lgpu_search* call of B queries and `nprobes` probes (the widest the call uses:
 * maximum_nprobes under a prefilter) on `ix` runs in under the process's LGPU_WS_BYTES: B when the batch is not split */
int lgpu_debug_sub_batch_size(lgpu_index *ix, uint32_t B, uint32_t nprobes, uint32_t *out);
/* the top-k selection every search ends in, run as given: per query q < B, the k entries with the smallest
 * (_distance, id) among its candidates, ascending, into out_ids / out_dist (or out_rec), out_count[q] of them, the rest
 * padded with id UINT64_MAX and +inf.  A candidate is dropped when its distance is NaN or outside [lower, upper) (each
 * bound only when has_lower / has_upper is set), or when allow is set and its id is >= allow_bits or has bit 0 there;
 * -0 is reported as +0.  The candidates of query q:
 *   mode 0 (IVF distance segments): for each probe slot s = q * nprobes + j whose probes[s] = p < nlist, the part_n[p]
 *     values at dist + seg_off[s], row r with id row_ids[part_off[p] + r] (part_off[p] + r when row_ids is NULL) and
 *     pos part_off[p] + r.  Every such segment starts at a multiple of 4 floats and, padded to 4, lies in dist_len;
 *   mode 1 (dense rows): dense[q * row_stride + c] for c < ncols, id col_ids[c] (c when NULL), pos c;
 *   mode 2 (strided lists): c < ncols (< ncols_q[q] too when ncols_q is set) at
 *     addr = (c / inner) * outer_stride + q * row_stride + c % inner: id cand_ids[addr], value dense[addr] (or both from
 *     the 16-byte record cand_rec[addr] = {u64 id, f32 dist, u32 pad}), pos cand_pos[addr] (c when NULL); an entry with
 *     id UINT64_MAX is an unused slot.
 * out_pos (optional) receives each entry's pos (UINT64_MAX when padded), out_rec (optional) the entries as 16-byte
 * records instead of out_ids / out_dist.  A query with only[q] == 0, or every query when *gate == 0, is left untouched.
 * Every pointer is a device pointer on `device`; dist, cand_rec and out_rec are 16-byte aligned.  Enqueued on
 * cuda_stream, not synchronised (mode 0 synchronises the stream once to check the segments). */
typedef struct {
    int32_t mode;                 /* 0, 1 or 2 */
    const float *dist;            /* mode 0 */
    const uint64_t *seg_off;      /* mode 0: [B * nprobes] */
    const uint64_t *probes;       /* mode 0: [B * nprobes] */
    uint32_t nprobes, nlist;
    const uint32_t *part_n;       /* mode 0: [nlist] */
    const uint64_t *part_off;     /* mode 0: [nlist] */
    const uint64_t *row_ids;      /* mode 0: optional */
    const float *dense;           /* mode 1, mode 2 without cand_rec */
    uint64_t ncols, row_stride;
    uint64_t inner, outer_stride; /* mode 2: inner >= 1 */
    const uint64_t *col_ids;      /* mode 1: optional [ncols] */
    const uint64_t *cand_ids;     /* mode 2 without cand_rec */
    const uint64_t *cand_pos;     /* mode 2: optional */
    const uint32_t *ncols_q;      /* mode 2: optional [B] */
    const void *cand_rec;         /* mode 2: optional */
    uint32_t B, k;                /* 1 <= k <= 2048 (lgpu_debug_select_large: 2048 < k <= LGPU_K_MAX) */
    int32_t has_lower, has_upper;
    float lower, upper;
    uint64_t *out_ids;            /* [B][k] */
    float *out_dist;              /* [B][k] */
    uint32_t *out_count;          /* [B] */
    void *out_rec;                /* optional [B][k] */
    uint64_t *out_pos;            /* optional [B][k] */
    const uint32_t *only;         /* optional [B] */
    const uint32_t *gate;         /* optional [1] */
    const uint32_t *allow;        /* optional bitmap: bit i & 31 of word i >> 5 */
    uint64_t allow_bits;
    uint64_t dist_len;            /* mode 0: floats in dist */
} lgpu_debug_select_args;
int lgpu_debug_select(const lgpu_debug_select_args *a, int device, void *cuda_stream);
/* the same selection for 2048 < k <= LGPU_K_MAX (the global-memory radix select the searches run above k = 2048), same
 * arguments and results.  Allocates its scratch and synchronises cuda_stream before returning. */
int lgpu_debug_select_large(const lgpu_debug_select_args *a, int device, void *cuda_stream);
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
 * [3] queries.  After lgpu_flat_search* (whole batch): [1] distances computed on the tensor cores (0 on the exact
 * path), [3] queries, [0] = [2] = 0.  After lgpu_multivec_search*: see the multivector section above. */
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
