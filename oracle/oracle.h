/*
 * oracle.h -- CPU restatement of the LanceDB vector-query hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is product code: only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may load this library, and only as the checker / the timed
 * CPU baseline.  The product path (lancedb_b200/) never links or calls it.
 *
 * PARITY STATUS: "IVF_PQ parity unpinned".  The arithmetic of the reference
 * lives in the un-vendored lance crates (lance-format/lance tag
 * v11.0.0-beta.19, commit 3128c0024427cb5bf8c04d492893ae45e78b0511, pinned in
 * Cargo.toml:16-29 and Cargo.lock:4817-4819,5109-5111,
 * 5234-5236).  That source is not part of the reference tree, so every
 * function below restates the *published algorithm*
 * as recalled ("[lance, recalled]") and is anchored on the reference's own
 * call sites (rust/lancedb/src/table/query.rs:219-327) and on the flat-path
 * numeric pins the reference's tests hold (see tests/test_oracle_pins.py):
 *   python/python/lancedb/table.py:3595-3603   L2 squared: 5.220000, 23.089996
 *   python/python/lancedb/query.py:1563-1571   cosine: 0.000000, 0.000944
 *   python/python/lancedb/query.py:1364-1370   tie-break (_distance, _rowid)
 *   python/python/tests/test_query.py:993-1014 cosine == numpy formula (1e-6)
 * No reference test pins an IVF_PQ distance, row-id list or recall value.
 */
#ifndef LANCEDB_B200_ORACLE_H
#define LANCEDB_B200_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { ORC_L2 = 0, ORC_COSINE = 1, ORC_DOT = 2 };

/* ---- lance-linalg distance kernels [lance, recalled] -------------------- */
float orc_l2_f32(const float *x, const float *y, size_t d);
float orc_dot_f32(const float *x, const float *y, size_t d);
float orc_norm_l2_f32(const float *x, size_t d);
float orc_cosine_f32(const float *x, const float *y, size_t d);
/* distance as the flat KNN operator reports it for `metric` */
float orc_distance_f32(int metric, const float *x, const float *y, size_t d);
/* x / ||x||  (query normalisation for cosine IVF search) */
void orc_normalize_f32(const float *x, size_t d, float *out);
/* the PQ sub-vector kernels: l2_once<f32x8>/<f32x16> tree reduce, else l2() */
float orc_l2_subvec(const float *x, const float *y, size_t dsub);

/* ---- IVF_PQ index container (plain arrays; same arrays the GPU gets) ---- */
typedef struct {
    uint32_t dim;
    uint32_t nlist;
    uint32_t m;               /* sub-vectors; 8-bit codes, 256 centroids each */
    int      metric;          /* ORC_L2 / ORC_COSINE / ORC_DOT */
    uint64_t nrows;
    const float    *centroids;    /* [nlist][dim] */
    const float    *codebook;     /* [m][256][dim/m] */
    const uint64_t *part_offsets; /* [nlist+1] row offsets, partition-contiguous */
    const uint8_t  *codes_t;      /* per partition p: [m][n_p] (transposed) at byte
                                     offset part_offsets[p]*m */
    const uint64_t *row_ids;      /* [nrows] in partition order */
    const float    *vectors;      /* optional [nrows][dim] in partition order (refine) */
} orc_index;

typedef struct {
    uint32_t k;              /* limit + offset */
    uint32_t nprobes;
    uint32_t refine_factor;  /* 0 = none */
    int      has_lower, has_upper;
    float    lower, upper;   /* distance range [lower, upper) */
    /* prefilter (rust/lancedb/src/query.rs:489-507, the default filter mode): row-id allow-list as a
     * bitmap, bit r of word r/32 = row id r may be returned; ids >= allow_bits are excluded.
     * NULL = no filter.  Rows are dropped before the top-k, so k allowed rows come back if the probed
     * partitions hold that many. */
    const uint32_t *allow;
    uint64_t allow_bits;
    /* maximum_nprobes (rust/lancedb/src/query.rs:1250-1275); 0 or <= nprobes = no widening.  Only consulted
     * under a prefilter. */
    uint32_t max_nprobes;
} orc_params;

/* IvfModel::find_partitions [lance, recalled]: all-centroid distances, then the
 * nprobes smallest by (distance, partition id).  q must already be normalised
 * for cosine.  all_dists (optional) receives the nlist distances. */
void orc_find_partitions(const orc_index *ix, const float *q, uint32_t nprobes,
                         uint32_t *out_parts, float *out_dists, float *all_dists);

/* build_distance_table_l2 / _dot [lance, recalled]: lut[m][256] */
void orc_build_lut(const orc_index *ix, const float *resid_or_query, float *lut);

/* compute_pq_distance, 8-bit [lance, recalled]: dists[j] = sum_i lut[i][codes_t[i*n+j]]
 * accumulated sequentially in i, f32. */
void orc_pq_scan(const float *lut, const uint8_t *codes_t, size_t n, uint32_t m,
                 float *dists);

/* Whole path for a batch; nthreads worker threads over queries.
 * out_ids/out_dist: [B][k], out_count: [B].  Unused slots: id = UINT64_MAX,
 * dist = +inf.  Returns 0, a negative error for invalid arguments, or 1 when
 * allocation fails. */
int orc_ivfpq_search(const orc_index *ix, const float *queries, uint32_t B,
                     const orc_params *p, uint64_t *out_ids, float *out_dist,
                     uint32_t *out_count, int nthreads);

/* Debug / per-stage access for parity localisation: the final PQ distances of
 * one (query, partition) pair, length n_p. q is the raw query. */
void orc_partition_distances(const orc_index *ix, const float *q, uint32_t part,
                             float *dists);

/* Index-build passes [lance, recalled]: IVF assignment = find_partitions with nprobes 1 per row
 * (rows normalised first for cosine); ProductQuantizer::transform = per sub-vector the codeword with the
 * smallest distance-table entry (residual row - centroid for L2/cosine, the row for dot), ties to the
 * lowest code.  vectors are raw rows; out_codes is row-major [n][m]. */
void orc_ivf_assign(const orc_index *ix, const float *vectors, uint64_t n, uint32_t *out_parts);
void orc_pq_encode(const orc_index *ix, const float *vectors, const uint32_t *parts, uint64_t n,
                   uint8_t *out_codes);

/* Flat KNN (KNNVectorDistance + TopK by (_distance,_rowid)). row_ids may be
 * NULL (then 0..n-1). */
int orc_flat_search(const float *vectors, uint64_t n, uint32_t dim,
                    const uint64_t *row_ids, int metric, const float *queries,
                    uint32_t B, const orc_params *p, uint64_t *out_ids,
                    float *out_dist, uint32_t *out_count, int nthreads);

/* ---- the result contract every oracle shares (DESIGN.md section 0) ----- */
/* The row filter: a NaN distance is dropped (FilterExec: _distance IS NOT NULL), then distance_range [lower, upper)
 * and the allow bitmap. */
static inline int orc_keep(const orc_params *p, uint64_t id, float d)
{
    if (d != d) return 0;
    if (p->has_lower && !(d >= p->lower)) return 0;
    if (p->has_upper && !(d < p->upper)) return 0;
    return !p->allow || (id < p->allow_bits && ((p->allow[id >> 5] >> (id & 31)) & 1u));
}

/* A candidate row; pos is its index in the row order (refine reads the raw vector there). */
typedef struct { float d; uint64_t id; uint64_t pos; } orc_cand;

/* The cap best candidates by (distance ASC, row id ASC), a NaN distance after every number. */
typedef struct { orc_cand *a; uint32_t n, cap; } orc_topk;
void orc_topk_offer(orc_topk *h, float d, uint64_t id, uint64_t pos);
/* Drops NaN distances, sorts, and writes p->k slots (unused: UINT64_MAX / +inf) and the count. */
void orc_topk_emit(const orc_params *p, orc_topk *h, uint64_t *ids, float *dist, uint32_t *count);

/* The indices of the nprobes smallest of d[0..n) by (distance, index), NaN last, and their distances (out_d may be
 * NULL). */
void orc_nearest(const float *d, uint32_t n, uint32_t nprobes, uint32_t *out_idx, float *out_d);

/* Runs fn(ctx, lo, hi) over min(nthreads, n) contiguous ranges of [0, n) on worker threads (inline when a thread
 * cannot be started).  Nonzero when allocation fails or a range returns nonzero. */
int orc_parallel(uint64_t n, int nthreads, int (*fn)(void *ctx, uint64_t lo, uint64_t hi), void *ctx);

/* ---- one IVF search for every index kind --------------------------------
 * Per query: prepare, the coarse order, widening, top-k, refine and emit are the driver's (orc_ivf_search); a kind
 * supplies its query preparation, its coarse step and the distances of one partition's rows. */
typedef struct orc_ivf_kind orc_ivf_kind;
struct orc_ivf_kind {
    const orc_index *ix;     /* nlist, part_offsets, row_ids; metric, dim and vectors (NULL: no refine) for refine */
    size_t query_bytes;      /* one raw query */
    size_t state_bytes;      /* one prepared query; a float kind's starts with the query the coarse step takes */
    void (*prepare)(const orc_ivf_kind *k, const void *q, void *state);
    /* the nprobes nearest partitions by (coarse distance, partition id) and their coarse distances */
    void (*coarse)(const orc_ivf_kind *k, const void *state, uint32_t nprobes, uint32_t *parts, float *dists);
    /* the distances of partition part's rows, in row order */
    void (*partition)(const orc_ivf_kind *k, void *state, uint32_t part, float *dists);
};
int orc_ivf_search(const orc_ivf_kind *k, const void *queries, uint32_t B, const orc_params *p, uint64_t *out_ids,
                   float *out_dist, uint32_t *out_count, int nthreads);
/* The float kinds' prepare prefix (the query, normalised for cosine) and their coarse step (orc_find_partitions). */
void orc_ivf_query_f32(const orc_ivf_kind *k, const void *q, void *state);
void orc_ivf_coarse_f32(const orc_ivf_kind *k, const void *state, uint32_t nprobes, uint32_t *parts, float *dists);

/* popcount(q XOR x) over nbytes bytes (tests/hamming_oracle.c) */
uint32_t orc_hamming_row(const uint8_t *q, const uint8_t *x, uint32_t nbytes);

#ifdef __cplusplus
}
#endif
#endif
