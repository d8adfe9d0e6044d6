/*
 * oracle.c -- CPU restatement of the LanceDB vector-query hot path (see oracle.h).
 *
 * TEST INFRASTRUCTURE ONLY -- never linked or called by the product path.
 * PARITY STATUS: IVF_PQ parity UNPINNED (no golden vector exists in the
 * reference); flat-path arithmetic is pinned by the reference's doctests.
 *
 * Must be compiled with -ffp-contract=off: Rust never contracts a*b+c into an
 * FMA, so neither may this file (the GPU kernels use __fmul_rn/__fadd_rn for
 * the same reason).
 *
 * Every function cites what it follows.  "[lance, recalled]" = the un-vendored
 * lance crate at tag v11.0.0-beta.19 (Cargo.toml:16-29), restated from its
 * published source as recalled; call sites in the reference are
 * rust/lancedb/src/table/query.rs:236-238 (scanner.nearest), :245-248
 * (nprobes), :311-316 (refine, metric), :327 (create_plan).
 */
#include "oracle.h"

#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

#define LANES 16

/* ------------------------------------------------------------------------ */
/* lance-linalg distance/l2.rs::l2_scalar::<f32,f32,16> [lance, recalled]:
 * 16 lane accumulators over chunks_exact(16); remainder summed sequentially
 * into `s`; result = s + (((0+sums[0])+sums[1])+...+sums[15]).             */
float orc_l2_f32(const float *x, const float *y, size_t d)
{
    size_t nchunk = d / LANES, rem0 = nchunk * LANES;
    float s = 0.0f;
    for (size_t i = rem0; i < d; i++) {
        float diff = x[i] - y[i];
        s = s + diff * diff;
    }
    float sums[LANES];
    for (int l = 0; l < LANES; l++) sums[l] = 0.0f;
    for (size_t c = 0; c < nchunk; c++) {
        const float *xc = x + c * LANES, *yc = y + c * LANES;
        for (int l = 0; l < LANES; l++) {
            float diff = xc[l] - yc[l];
            sums[l] = sums[l] + diff * diff;
        }
    }
    float t = 0.0f;
    for (int l = 0; l < LANES; l++) t = t + sums[l];
    return s + t;
}

/* lance-linalg distance/dot.rs::dot_scalar::<f32,f32,16> [lance, recalled] */
float orc_dot_f32(const float *x, const float *y, size_t d)
{
    size_t nchunk = d / LANES, rem0 = nchunk * LANES;
    float s = 0.0f;
    for (size_t i = rem0; i < d; i++) s = s + x[i] * y[i];
    float sums[LANES];
    for (int l = 0; l < LANES; l++) sums[l] = 0.0f;
    for (size_t c = 0; c < nchunk; c++) {
        const float *xc = x + c * LANES, *yc = y + c * LANES;
        for (int l = 0; l < LANES; l++) sums[l] = sums[l] + xc[l] * yc[l];
    }
    float t = 0.0f;
    for (int l = 0; l < LANES; l++) t = t + sums[l];
    return s + t;
}

/* lance-linalg distance/norm_l2.rs [lance, recalled]: sqrt(dot(x,x)) */
float orc_norm_l2_f32(const float *x, size_t d)
{
    return sqrtf(orc_dot_f32(x, x, d));
}

/* lance-linalg distance/cosine.rs::cosine_scalar [lance, recalled]:
 * 1 - xy / x_norm / sqrt(yy); pinned by the doctest at
 * python/python/lancedb/query.py:1563-1571 and test_query.py:993-1014.      */
float orc_cosine_f32(const float *x, const float *y, size_t d)
{
    float x_norm = orc_norm_l2_f32(x, d);
    float yy = orc_dot_f32(y, y, d);
    float xy = orc_dot_f32(x, y, d);
    return 1.0f - xy / x_norm / sqrtf(yy);
}

/* rust/lancedb/src/lib.rs:236-260 (DistanceType): L2 is squared euclidean,
 * cosine = 1 - cos, dot = 1 - x.y [lance, recalled]                         */
float orc_distance_f32(int metric, const float *x, const float *y, size_t d)
{
    switch (metric) {
    case ORC_COSINE: return orc_cosine_f32(x, y, d);
    case ORC_DOT:    return 1.0f - orc_dot_f32(x, y, d);
    default:         return orc_l2_f32(x, y, d);
    }
}

/* lance-linalg normalize [lance, recalled]: x / norm_l2(x) */
void orc_normalize_f32(const float *x, size_t d, float *out)
{
    float n = orc_norm_l2_f32(x, d);
    for (size_t i = 0; i < d; i++) out[i] = x[i] / n;
}

/* lance-linalg L2::l2_batch for f32 dispatches on the dimension
 * [lance, recalled]: 8 -> l2_once::<f32x8,8>, 16 -> l2_once::<f32x16,16>,
 * otherwise l2().  l2_once = ((x-y)*(x-y)).reduce_sum(), and the AVX2
 * (target-cpu=haswell, .cargo/config.toml:44) f32x8
 * reduce_sum is permute2f128+add, permute(14)+add, hadd:
 *   ((s0+s4)+(s2+s6)) + ((s1+s5)+(s3+s7)).
 * f32x16 on AVX2 is two f32x8 halves added lane-wise first.                 */
static inline float reduce_sum_x8(const float *s)
{
    float t0 = s[0] + s[4], t1 = s[1] + s[5], t2 = s[2] + s[6], t3 = s[3] + s[7];
    float u0 = t0 + t2, u1 = t1 + t3;
    return u0 + u1;
}

float orc_l2_subvec(const float *x, const float *y, size_t dsub)
{
    if (dsub == 8) {
        float s[8];
        for (int i = 0; i < 8; i++) { float d = x[i] - y[i]; s[i] = d * d; }
        return reduce_sum_x8(s);
    }
    if (dsub == 16) {
        float s[16], h[8];
        for (int i = 0; i < 16; i++) { float d = x[i] - y[i]; s[i] = d * d; }
        for (int i = 0; i < 8; i++) h[i] = s[i] + s[i + 8];
        return reduce_sum_x8(h);
    }
    return orc_l2_f32(x, y, dsub);
}

/* ------------------------------------------------------------------------ */
/* (distance, id) ordering: `_distance ASC, _rowid ASC`, the tie-break the
 * reference pins for TopK at python/python/lancedb/query.py:1366-1368.      */
typedef struct { float d; uint64_t id; uint64_t pos; } cand_t;

static inline int cand_less(const cand_t *a, const cand_t *b)
{
    if (a->d < b->d) return 1;
    if (a->d > b->d) return 0;
    return a->id < b->id;
}

/* bounded max-heap of the k smallest (lance-index flat/index.rs keeps a
 * BinaryHeap of k with strict `<` [lance, recalled]; partitions here are in
 * ascending row-id scan order, so "first seen wins a tie" == smaller row id) */
typedef struct { cand_t *a; uint32_t n, cap; } heap_t;

static void heap_sift_up(heap_t *h, uint32_t i)
{
    while (i > 0) {
        uint32_t p = (i - 1) / 2;
        if (cand_less(&h->a[p], &h->a[i])) {
            cand_t t = h->a[p]; h->a[p] = h->a[i]; h->a[i] = t; i = p;
        } else break;
    }
}

static void heap_sift_down(heap_t *h, uint32_t i)
{
    for (;;) {
        uint32_t l = 2 * i + 1, r = l + 1, m = i;
        if (l < h->n && cand_less(&h->a[m], &h->a[l])) m = l;
        if (r < h->n && cand_less(&h->a[m], &h->a[r])) m = r;
        if (m == i) break;
        cand_t t = h->a[m]; h->a[m] = h->a[i]; h->a[i] = t; i = m;
    }
}

static inline void heap_offer(heap_t *h, float d, uint64_t id, uint64_t pos)
{
    if (h->cap == 0) return;
    cand_t c = { d, id, pos };
    if (h->n < h->cap) {
        h->a[h->n] = c; heap_sift_up(h, h->n); h->n++;
    } else if (cand_less(&c, &h->a[0])) {
        h->a[0] = c; heap_sift_down(h, 0);
    }
}

static int cand_cmp(const void *pa, const void *pb)
{
    const cand_t *a = (const cand_t *)pa, *b = (const cand_t *)pb;
    if (cand_less(a, b)) return -1;
    if (cand_less(b, a)) return 1;
    return 0;
}

static inline int allowed(const orc_params *p, uint64_t id)
{
    if (!p->allow) return 1;
    return id < p->allow_bits && ((p->allow[id >> 5] >> (id & 31)) & 1u);
}

static inline int in_range(const orc_params *p, float d)
{
    if (d != d) return 0;                      /* FilterExec: _distance IS NOT NULL */
    if (p->has_lower && !(d >= p->lower)) return 0;
    if (p->has_upper && !(d < p->upper)) return 0;
    return 1;
}

/* ------------------------------------------------------------------------ */
static float coarse_distance(const orc_index *ix, const float *q, const float *c)
{
    /* IvfModel::find_partitions [lance, recalled]: L2 for l2 and for cosine
     * (query and centroids are normalised), dot_distance = 1 - x.y for dot.  */
    if (ix->metric == ORC_DOT) return 1.0f - orc_dot_f32(q, c, ix->dim);
    return orc_l2_f32(q, c, ix->dim);
}

void orc_find_partitions(const orc_index *ix, const float *q, uint32_t nprobes,
                         uint32_t *out_parts, float *out_dists, float *all_dists)
{
    uint32_t nlist = ix->nlist;
    if (nprobes > nlist) nprobes = nlist;
    cand_t *c = (cand_t *)malloc(sizeof(cand_t) * (nlist ? nlist : 1));
    for (uint32_t p = 0; p < nlist; p++) {
        c[p].d = coarse_distance(ix, q, ix->centroids + (size_t)p * ix->dim);
        c[p].id = p; c[p].pos = p;
        if (all_dists) all_dists[p] = c[p].d;
    }
    /* sort_to_indices(dists, limit = nprobes): ascending; ties by partition id */
    qsort(c, nlist, sizeof(cand_t), cand_cmp);
    for (uint32_t j = 0; j < nprobes; j++) {
        out_parts[j] = (uint32_t)c[j].id;
        if (out_dists) out_dists[j] = c[j].d;
    }
    free(c);
}

void orc_build_lut(const orc_index *ix, const float *rq, float *lut)
{
    uint32_t m = ix->m, dsub = ix->dim / m;
    for (uint32_t i = 0; i < m; i++) {
        const float *sub = rq + (size_t)i * dsub;
        const float *cb = ix->codebook + (size_t)i * 256 * dsub;
        float *row = lut + (size_t)i * 256;
        if (ix->metric == ORC_DOT) {
            /* build_distance_table_dot: dot_distance_batch = 1 - x.y per sub-vector */
            for (int j = 0; j < 256; j++)
                row[j] = 1.0f - orc_dot_f32(sub, cb + (size_t)j * dsub, dsub);
        } else {
            /* build_distance_table_l2: l2_distance_batch(sub_vec, centroids, dsub) */
            for (int j = 0; j < 256; j++)
                row[j] = orc_l2_subvec(sub, cb + (size_t)j * dsub, dsub);
        }
    }
}

void orc_pq_scan(const float *lut, const uint8_t *codes_t, size_t n, uint32_t m,
                 float *dists)
{
    for (size_t j = 0; j < n; j++) dists[j] = 0.0f;
    for (uint32_t i = 0; i < m; i++) {
        const float *row = lut + (size_t)i * 256;
        const uint8_t *c = codes_t + (size_t)i * n;
        for (size_t j = 0; j < n; j++) dists[j] = dists[j] + row[c[j]];
    }
}

/* metric post-processing of the accumulated table sums [lance, recalled]:
 * cosine: index holds normalised vectors, L2^2 = 2(1-cos) => distance = L2^2/2;
 * dot: sum_i (1 - x_i.y_i) = m - x.y => distance = sum - (m - 1).            */
static inline float finish_pq(const orc_index *ix, float acc)
{
    if (ix->metric == ORC_COSINE) return acc * 0.5f;
    if (ix->metric == ORC_DOT) return acc - (float)(ix->m - 1);
    return acc;
}

static void partition_distances(const orc_index *ix, const float *qn, uint32_t part,
                                float *resid, float *lut, float *dists)
{
    size_t off = ix->part_offsets[part], n = ix->part_offsets[part + 1] - off;
    const float *rq = qn;
    if (ix->metric != ORC_DOT) {
        /* residual query for L2/cosine (PQ is trained on residuals) */
        const float *c = ix->centroids + (size_t)part * ix->dim;
        for (uint32_t t = 0; t < ix->dim; t++) resid[t] = qn[t] - c[t];
        rq = resid;
    }
    orc_build_lut(ix, rq, lut);
    orc_pq_scan(lut, ix->codes_t + off * ix->m, n, ix->m, dists);
    for (size_t j = 0; j < n; j++) dists[j] = finish_pq(ix, dists[j]);
}

void orc_partition_distances(const orc_index *ix, const float *q, uint32_t part,
                             float *dists)
{
    float *qn = (float *)malloc(sizeof(float) * ix->dim * 2);
    float *lut = (float *)malloc(sizeof(float) * ix->m * 256);
    if (ix->metric == ORC_COSINE) orc_normalize_f32(q, ix->dim, qn);
    else memcpy(qn, q, sizeof(float) * ix->dim);
    partition_distances(ix, qn, part, qn + ix->dim, lut, dists);
    free(qn); free(lut);
}

/* ------------------------------------------------------------------------ */
typedef struct {
    const orc_index *ix;
    const float *queries;
    uint32_t B, q0, q1;
    const orc_params *p;
    uint64_t *out_ids; float *out_dist; uint32_t *out_count;
    size_t max_part;
} ivf_job;

static void emit(const orc_params *p, heap_t *h, uint64_t *ids, float *dist,
                 uint32_t *count)
{
    qsort(h->a, h->n, sizeof(cand_t), cand_cmp);
    uint32_t n = h->n < p->k ? h->n : p->k;
    for (uint32_t j = 0; j < p->k; j++) {
        ids[j] = j < n ? h->a[j].id : UINT64_MAX;
        dist[j] = j < n ? h->a[j].d : INFINITY;
    }
    *count = n;
}

static void *ivf_worker(void *arg)
{
    ivf_job *job = (ivf_job *)arg;
    const orc_index *ix = job->ix;
    const orc_params *p = job->p;
    uint32_t dim = ix->dim, nprobes = p->nprobes < ix->nlist ? p->nprobes : ix->nlist;
    /* maximum_nprobes (rust/lancedb/src/query.rs:1250-1275): "the excess partitions will only be searched if
     * the initial search does not return enough results ... useful when there is a narrow filter".  Restated as:
     * under a prefilter, a query whose minimum_nprobes partitions yield fewer than k rows is searched again
     * over its maximum_nprobes nearest partitions. */
    uint32_t nprobes_max = nprobes;
    if (p->allow && p->max_nprobes > nprobes) nprobes_max = p->max_nprobes < ix->nlist ? p->max_nprobes : ix->nlist;
    uint32_t kk = p->refine_factor ? p->k * p->refine_factor : p->k;
    float *qn = (float *)malloc(sizeof(float) * dim * 2);
    float *resid = qn + dim;
    float *lut = (float *)malloc(sizeof(float) * ix->m * 256);
    float *dists = (float *)malloc(sizeof(float) * (job->max_part ? job->max_part : 1));
    uint32_t *parts = (uint32_t *)malloc(sizeof(uint32_t) * (nprobes_max ? nprobes_max : 1));
    heap_t h; h.a = (cand_t *)malloc(sizeof(cand_t) * (kk ? kk : 1)); h.cap = kk;

    for (uint32_t qi = job->q0; qi < job->q1; qi++) {
        const float *q = job->queries + (size_t)qi * dim;
        if (ix->metric == ORC_COSINE) orc_normalize_f32(q, dim, qn);
        else memcpy(qn, q, sizeof(float) * dim);
        for (uint32_t np_use = nprobes;;) {
            orc_find_partitions(ix, qn, np_use, parts, NULL, NULL);
            h.n = 0;
            for (uint32_t j = 0; j < np_use; j++) {
                uint32_t part = parts[j];
                size_t off = ix->part_offsets[part], n = ix->part_offsets[part + 1] - off;
                if (n == 0) continue;
                partition_distances(ix, qn, part, resid, lut, dists);
                for (size_t r = 0; r < n; r++)
                    if (in_range(p, dists[r]) && allowed(p, ix->row_ids[off + r]))
                        heap_offer(&h, dists[r], ix->row_ids[off + r], off + r);
            }
            if (np_use >= nprobes_max || h.n >= p->k) break;
            np_use = nprobes_max;
        }
        if (p->refine_factor && ix->vectors) {
            /* refine (rust/lancedb/src/query.rs:1302-1332): exact distance of the
             * k*refine_factor ANN candidates on the raw vectors, re-sort, keep k */
            for (uint32_t c = 0; c < h.n; c++)
                h.a[c].d = orc_distance_f32(ix->metric, q, ix->vectors + h.a[c].pos * dim, dim);
        }
        emit(p, &h, job->out_ids + (size_t)qi * p->k, job->out_dist + (size_t)qi * p->k,
             job->out_count + qi);
    }
    free(qn); free(lut); free(dists); free(parts); free(h.a);
    return NULL;
}

int orc_ivfpq_search(const orc_index *ix, const float *queries, uint32_t B,
                     const orc_params *p, uint64_t *out_ids, float *out_dist,
                     uint32_t *out_count, int nthreads)
{
    if (!ix || !p || ix->m == 0 || ix->dim % ix->m) return -1;
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > B) nthreads = B ? (int)B : 1;
    size_t max_part = 0;
    for (uint32_t i = 0; i < ix->nlist; i++) {
        size_t n = ix->part_offsets[i + 1] - ix->part_offsets[i];
        if (n > max_part) max_part = n;
    }
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * nthreads);
    ivf_job *jobs = (ivf_job *)malloc(sizeof(ivf_job) * nthreads);
    for (int t = 0; t < nthreads; t++) {
        ivf_job j = { ix, queries, B, (uint32_t)((uint64_t)B * t / nthreads),
                      (uint32_t)((uint64_t)B * (t + 1) / nthreads), p,
                      out_ids, out_dist, out_count, max_part };
        jobs[t] = j;
        if (nthreads == 1) ivf_worker(&jobs[t]);
        else pthread_create(&th[t], NULL, ivf_worker, &jobs[t]);
    }
    if (nthreads > 1) for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
    free(th); free(jobs);
    return 0;
}

/* ------------------------------------------------------------------------ */
void orc_ivf_assign(const orc_index *ix, const float *vectors, uint64_t n, uint32_t *out_parts)
{
    float *qn = (float *)malloc(sizeof(float) * ix->dim);
    for (uint64_t r = 0; r < n; r++) {
        const float *x = vectors + r * ix->dim;
        if (ix->metric == ORC_COSINE) orc_normalize_f32(x, ix->dim, qn);
        else memcpy(qn, x, sizeof(float) * ix->dim);
        orc_find_partitions(ix, qn, 1, out_parts + r, NULL, NULL);
    }
    free(qn);
}

void orc_pq_encode(const orc_index *ix, const float *vectors, const uint32_t *parts, uint64_t n,
                   uint8_t *out_codes)
{
    uint32_t dim = ix->dim, m = ix->m, dsub = dim / m;
    float *qn = (float *)malloc(sizeof(float) * dim * 2);
    float *res = qn + dim;
    for (uint64_t r = 0; r < n; r++) {
        const float *x = vectors + r * dim;
        if (ix->metric == ORC_COSINE) orc_normalize_f32(x, dim, qn);
        else memcpy(qn, x, sizeof(float) * dim);
        const float *rq = qn;
        if (ix->metric != ORC_DOT) {
            const float *c = ix->centroids + (size_t)parts[r] * dim;
            for (uint32_t t = 0; t < dim; t++) res[t] = qn[t] - c[t];
            rq = res;
        }
        for (uint32_t i = 0; i < m; i++) {
            const float *sub = rq + (size_t)i * dsub;
            const float *cb = ix->codebook + (size_t)i * 256 * dsub;
            float best = 0.0f; int best_c = 0;
            for (int j = 0; j < 256; j++) {
                float d = ix->metric == ORC_DOT ? 1.0f - orc_dot_f32(sub, cb + (size_t)j * dsub, dsub)
                                                : orc_l2_subvec(sub, cb + (size_t)j * dsub, dsub);
                if (j == 0 || d < best) { best = d; best_c = j; }
            }
            out_codes[r * m + i] = (uint8_t)best_c;
        }
    }
    free(qn);
}

/* ------------------------------------------------------------------------ */
typedef struct {
    const float *vectors; uint64_t n; uint32_t dim; const uint64_t *row_ids; int metric;
    const float *queries; uint32_t q0, q1; const orc_params *p;
    uint64_t *out_ids; float *out_dist; uint32_t *out_count;
} flat_job;

/* KNNVectorDistance + SortExec TopK(_distance ASC, _rowid ASC) + FilterExec
 * (_distance IS NOT NULL): python/python/lancedb/query.py:1364-1370           */
static void *flat_worker(void *arg)
{
    flat_job *job = (flat_job *)arg;
    const orc_params *p = job->p;
    heap_t h; h.a = (cand_t *)malloc(sizeof(cand_t) * (p->k ? p->k : 1)); h.cap = p->k;
    for (uint32_t qi = job->q0; qi < job->q1; qi++) {
        const float *q = job->queries + (size_t)qi * job->dim;
        h.n = 0;
        for (uint64_t r = 0; r < job->n; r++) {
            float d = orc_distance_f32(job->metric, q, job->vectors + r * job->dim, job->dim);
            uint64_t id = job->row_ids ? job->row_ids[r] : r;
            if (in_range(p, d) && allowed(p, id)) heap_offer(&h, d, id, r);
        }
        emit(p, &h, job->out_ids + (size_t)qi * p->k, job->out_dist + (size_t)qi * p->k,
             job->out_count + qi);
    }
    free(h.a);
    return NULL;
}

int orc_flat_search(const float *vectors, uint64_t n, uint32_t dim,
                    const uint64_t *row_ids, int metric, const float *queries,
                    uint32_t B, const orc_params *p, uint64_t *out_ids,
                    float *out_dist, uint32_t *out_count, int nthreads)
{
    if (!p) return -1;
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > B) nthreads = B ? (int)B : 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * nthreads);
    flat_job *jobs = (flat_job *)malloc(sizeof(flat_job) * nthreads);
    for (int t = 0; t < nthreads; t++) {
        flat_job j = { vectors, n, dim, row_ids, metric, queries,
                       (uint32_t)((uint64_t)B * t / nthreads),
                       (uint32_t)((uint64_t)B * (t + 1) / nthreads), p,
                       out_ids, out_dist, out_count };
        jobs[t] = j;
        if (nthreads == 1) flat_worker(&jobs[t]);
        else pthread_create(&th[t], NULL, flat_worker, &jobs[t]);
    }
    if (nthreads > 1) for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
    free(th); free(jobs);
    return 0;
}
