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
 * reference pins for TopK at python/python/lancedb/query.py:1366-1368.
 * A NaN distance sorts after every number (ties by id), so the order stays a
 * strict weak order whatever the data holds; +-inf are ordinary values.     */
static inline int cand_less(const orc_cand *a, const orc_cand *b)
{
    const int an = a->d != a->d, bn = b->d != b->d;
    if (an != bn) return bn;
    if (a->d < b->d) return 1;
    if (a->d > b->d) return 0;
    return a->id < b->id;
}

static int cand_cmp(const void *pa, const void *pb)
{
    const orc_cand *a = (const orc_cand *)pa, *b = (const orc_cand *)pb;
    if (cand_less(a, b)) return -1;
    if (cand_less(b, a)) return 1;
    return 0;
}

/* bounded max-heap of the k smallest (lance-index flat/index.rs keeps a
 * BinaryHeap of k with strict `<` [lance, recalled]; partitions here are in
 * ascending row-id scan order, so "first seen wins a tie" == smaller row id) */
static void heap_sift_up(orc_topk *h, uint32_t i)
{
    while (i > 0) {
        uint32_t p = (i - 1) / 2;
        if (cand_less(&h->a[p], &h->a[i])) {
            orc_cand t = h->a[p]; h->a[p] = h->a[i]; h->a[i] = t; i = p;
        } else break;
    }
}

static void heap_sift_down(orc_topk *h, uint32_t i)
{
    for (;;) {
        uint32_t l = 2 * i + 1, r = l + 1, m = i;
        if (l < h->n && cand_less(&h->a[m], &h->a[l])) m = l;
        if (r < h->n && cand_less(&h->a[m], &h->a[r])) m = r;
        if (m == i) break;
        orc_cand t = h->a[m]; h->a[m] = h->a[i]; h->a[i] = t; i = m;
    }
}

void orc_topk_offer(orc_topk *h, float d, uint64_t id, uint64_t pos)
{
    if (h->cap == 0) return;
    orc_cand c = { d, id, pos };
    if (h->n < h->cap) {
        h->a[h->n] = c; heap_sift_up(h, h->n); h->n++;
    } else if (cand_less(&c, &h->a[0])) {
        h->a[0] = c; heap_sift_down(h, 0);
    }
}

/* a NaN distance is never returned (FilterExec: _distance IS NOT NULL); the
 * row filter has dropped them already, only refine's exact distances can
 * still be NaN here */
void orc_topk_emit(const orc_params *p, orc_topk *h, uint64_t *ids, float *dist, uint32_t *count)
{
    uint32_t kept = 0;
    for (uint32_t j = 0; j < h->n; j++)
        if (h->a[j].d == h->a[j].d) h->a[kept++] = h->a[j];
    h->n = kept;
    qsort(h->a, h->n, sizeof(orc_cand), cand_cmp);
    uint32_t n = h->n < p->k ? h->n : p->k;
    for (uint32_t j = 0; j < p->k; j++) {
        ids[j] = j < n ? h->a[j].id : UINT64_MAX;
        dist[j] = j < n ? h->a[j].d : INFINITY;
    }
    *count = n;
}

void orc_nearest(const float *d, uint32_t n, uint32_t nprobes, uint32_t *out_idx, float *out_d)
{
    if (nprobes > n) nprobes = n;
    orc_cand *c = (orc_cand *)malloc(sizeof(orc_cand) * (n ? n : 1));
    if (!c) return;
    for (uint32_t i = 0; i < n; i++) { c[i].d = d[i]; c[i].id = i; c[i].pos = i; }
    qsort(c, n, sizeof(orc_cand), cand_cmp);
    for (uint32_t j = 0; j < nprobes; j++) {
        out_idx[j] = (uint32_t)c[j].id;
        if (out_d) out_d[j] = c[j].d;
    }
    free(c);
}

typedef struct {
    int (*fn)(void *, uint64_t, uint64_t);
    void *ctx;
    uint64_t lo, hi;
    int rc, threaded;
} span_t;

static void *span_run(void *arg)
{
    span_t *s = (span_t *)arg;
    s->rc = s->fn(s->ctx, s->lo, s->hi);
    return NULL;
}

int orc_parallel(uint64_t n, int nthreads, int (*fn)(void *ctx, uint64_t lo, uint64_t hi), void *ctx)
{
    if (nthreads < 1) nthreads = 1;
    if ((uint64_t)nthreads > n) nthreads = n ? (int)n : 1;
    span_t *s = (span_t *)calloc((size_t)nthreads, sizeof(span_t));
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    if (!s || !th) { free(s); free(th); return 1; }
    for (int t = 0; t < nthreads; t++) {
        span_t x = { fn, ctx, n * t / nthreads, n * (t + 1) / nthreads, 0, 0 };
        s[t] = x;
    }
    for (int t = 1; t < nthreads; t++) {
        s[t].threaded = pthread_create(&th[t], NULL, span_run, &s[t]) == 0;
        if (!s[t].threaded) span_run(&s[t]);
    }
    span_run(&s[0]);
    int rc = 0;
    for (int t = 0; t < nthreads; t++) {
        if (s[t].threaded) pthread_join(th[t], NULL);
        rc |= s[t].rc;
    }
    free(s); free(th);
    return rc;
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
    if (nlist == 0) return;
    float *d = all_dists ? all_dists : (float *)malloc(sizeof(float) * nlist);
    if (!d) return;
    for (uint32_t p = 0; p < nlist; p++)
        d[p] = coarse_distance(ix, q, ix->centroids + (size_t)p * ix->dim);
    /* sort_to_indices(dists, limit = nprobes): ascending; ties by partition id; NaN distances last (the
     * search never probes them: DESIGN.md section 0, rule c) */
    orc_nearest(d, nlist, nprobes, out_parts, out_dists);
    if (!all_dists) free(d);
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
void orc_ivf_query_f32(const orc_ivf_kind *k, const void *q, void *state)
{
    const orc_index *ix = k->ix;
    if (ix->metric == ORC_COSINE) orc_normalize_f32((const float *)q, ix->dim, (float *)state);
    else memcpy(state, q, sizeof(float) * ix->dim);
}

void orc_ivf_coarse_f32(const orc_ivf_kind *k, const void *state, uint32_t nprobes, uint32_t *parts, float *dists)
{
    orc_find_partitions(k->ix, (const float *)state, nprobes, parts, dists, NULL);
}

typedef struct {
    const orc_ivf_kind *k;
    const uint8_t *queries;
    const orc_params *p;
    uint64_t *out_ids; float *out_dist; uint32_t *out_count;
    size_t max_part;
} ivf_run;

static int ivf_range(void *arg, uint64_t q0, uint64_t q1)
{
    const ivf_run *run = (const ivf_run *)arg;
    const orc_ivf_kind *k = run->k;
    const orc_index *ix = k->ix;
    const orc_params *p = run->p;
    uint32_t nprobes = p->nprobes < ix->nlist ? p->nprobes : ix->nlist;
    /* maximum_nprobes (rust/lancedb/src/query.rs:1250-1275): "the excess partitions will only be searched if
     * the initial search does not return enough results ... useful when there is a narrow filter".  Restated as:
     * under a prefilter, a query whose minimum_nprobes partitions yield fewer than k rows is searched again
     * over its maximum_nprobes nearest partitions. */
    uint32_t nprobes_max = nprobes;
    if (p->allow && p->max_nprobes > nprobes) nprobes_max = p->max_nprobes < ix->nlist ? p->max_nprobes : ix->nlist;
    uint32_t kk = p->refine_factor ? p->k * p->refine_factor : p->k;
    void *state = malloc(k->state_bytes ? k->state_bytes : 1);
    float *dists = (float *)malloc(sizeof(float) * (run->max_part ? run->max_part : 1));
    uint32_t *parts = (uint32_t *)malloc(sizeof(uint32_t) * (nprobes_max ? nprobes_max : 1));
    float *pd = (float *)malloc(sizeof(float) * (nprobes_max ? nprobes_max : 1));
    orc_topk h = { (orc_cand *)malloc(sizeof(orc_cand) * (kk ? kk : 1)), 0, kk };
    const int err = !state || !dists || !parts || !pd || !h.a;

    for (uint64_t qi = q0; qi < q1 && !err; qi++) {
        const void *q = run->queries + qi * k->query_bytes;
        k->prepare(k, q, state);
        k->coarse(k, state, nprobes_max, parts, pd);
        for (uint32_t np_use = nprobes;;) {
            h.n = 0;
            for (uint32_t j = 0; j < np_use; j++) {
                if (pd[j] != pd[j]) continue;              /* a NaN coarse distance is never probed */
                uint32_t part = parts[j];
                size_t off = ix->part_offsets[part], n = ix->part_offsets[part + 1] - off;
                if (n == 0) continue;
                k->partition(k, state, part, dists);
                for (size_t r = 0; r < n; r++)
                    if (orc_keep(p, ix->row_ids[off + r], dists[r]))
                        orc_topk_offer(&h, dists[r], ix->row_ids[off + r], off + r);
            }
            if (np_use >= nprobes_max || h.n >= p->k) break;
            np_use = nprobes_max;
        }
        if (p->refine_factor && ix->vectors) {
            /* refine (rust/lancedb/src/query.rs:1302-1332): exact distance of the
             * k*refine_factor ANN candidates on the raw vectors, re-sort, keep k */
            for (uint32_t c = 0; c < h.n; c++)
                h.a[c].d = orc_distance_f32(ix->metric, (const float *)q, ix->vectors + h.a[c].pos * ix->dim, ix->dim);
        }
        orc_topk_emit(p, &h, run->out_ids + qi * p->k, run->out_dist + qi * p->k, run->out_count + qi);
    }
    free(state); free(dists); free(parts); free(pd); free(h.a);
    return err;
}

int orc_ivf_search(const orc_ivf_kind *k, const void *queries, uint32_t B, const orc_params *p, uint64_t *out_ids,
                   float *out_dist, uint32_t *out_count, int nthreads)
{
    size_t max_part = 0;
    for (uint32_t i = 0; i < k->ix->nlist; i++) {
        size_t n = k->ix->part_offsets[i + 1] - k->ix->part_offsets[i];
        if (n > max_part) max_part = n;
    }
    ivf_run run = { k, (const uint8_t *)queries, p, out_ids, out_dist, out_count, max_part };
    return orc_parallel(B, nthreads, ivf_range, &run);
}

/* IVF_PQ, 8-bit: state = the query (normalised for cosine), the residual, the table */
static void pq_partition(const orc_ivf_kind *k, void *state, uint32_t part, float *dists)
{
    float *qn = (float *)state;
    partition_distances(k->ix, qn, part, qn + k->ix->dim, qn + 2 * k->ix->dim, dists);
}

int orc_ivfpq_search(const orc_index *ix, const float *queries, uint32_t B,
                     const orc_params *p, uint64_t *out_ids, float *out_dist,
                     uint32_t *out_count, int nthreads)
{
    if (!ix || !p || ix->m == 0 || ix->dim % ix->m) return -1;
    const orc_ivf_kind k = { ix, sizeof(float) * ix->dim, sizeof(float) * (2 * ix->dim + (size_t)ix->m * 256),
                             orc_ivf_query_f32, orc_ivf_coarse_f32, pq_partition };
    return orc_ivf_search(&k, queries, B, p, out_ids, out_dist, out_count, nthreads);
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
    const float *queries; const orc_params *p;
    uint64_t *out_ids; float *out_dist; uint32_t *out_count;
} flat_run;

/* KNNVectorDistance + SortExec TopK(_distance ASC, _rowid ASC) + FilterExec
 * (_distance IS NOT NULL): python/python/lancedb/query.py:1364-1370           */
static int flat_range(void *arg, uint64_t q0, uint64_t q1)
{
    const flat_run *run = (const flat_run *)arg;
    const orc_params *p = run->p;
    orc_topk h = { (orc_cand *)malloc(sizeof(orc_cand) * (p->k ? p->k : 1)), 0, p->k };
    if (!h.a) return 1;
    for (uint64_t qi = q0; qi < q1; qi++) {
        const float *q = run->queries + qi * run->dim;
        h.n = 0;
        for (uint64_t r = 0; r < run->n; r++) {
            float d = orc_distance_f32(run->metric, q, run->vectors + r * run->dim, run->dim);
            uint64_t id = run->row_ids ? run->row_ids[r] : r;
            if (orc_keep(p, id, d)) orc_topk_offer(&h, d, id, r);
        }
        orc_topk_emit(p, &h, run->out_ids + qi * p->k, run->out_dist + qi * p->k, run->out_count + qi);
    }
    free(h.a);
    return 0;
}

int orc_flat_search(const float *vectors, uint64_t n, uint32_t dim,
                    const uint64_t *row_ids, int metric, const float *queries,
                    uint32_t B, const orc_params *p, uint64_t *out_ids,
                    float *out_dist, uint32_t *out_count, int nthreads)
{
    if (!p) return -1;
    flat_run run = { vectors, n, dim, row_ids, metric, queries, p, out_ids, out_dist, out_count };
    return orc_parallel(B, nthreads, flat_range, &run);
}
