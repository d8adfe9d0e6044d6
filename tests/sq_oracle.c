/* sq_oracle.c -- CPU oracle of IVF_SQ search: the lgpu_ivf_sq_open / lgpu_search semantics.
 *
 * Per query (normalised first for cosine, orc_normalize_f32): the nprobes nearest partitions by
 * orc_find_partitions (a partition whose centroid distance is NaN is not probed, as the GPU's coarse step leaves
 * such slots unused); the query's codes q_i = sat_u8(((double)v - lo) * 255 / (hi - lo)) (left to right in f64,
 * truncated toward zero, NaN -> 0, all 0 when lo == hi); and for every row of a probed partition
 *     _distance = (float) sum_i (k_i - q_i)^2,
 * the sum exact in integers, one rounding to nearest f32.  distance_range [lower, upper) on that distance and the
 * row-id allow bitmap drop rows before the top-k; maximum_nprobes (under a prefilter) searches a query again over its
 * max_nprobes nearest partitions when it found fewer than k rows; refine_factor keeps the k * refine_factor best and
 * re-ranks them by orc_distance_f32 on the raw query and the raw vectors.  Results ascend by (_distance, _rowid);
 * unused slots are UINT64_MAX / +inf.  Worker threads split the queries.  The NumPy mirror is tests/sq_oracle.py. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

uint8_t orc_sq_code(float v, double lo, double hi)
{
    if (!(hi != lo)) return 0;
    const double t = ((double)v - lo) * 255.0 / (hi - lo);
    if (!(t > 0.0)) return 0;                  /* negative, zero, NaN */
    if (t >= 255.0) return 255;
    return (uint8_t)t;                         /* truncation toward zero */
}

void orc_sq_encode(const float *x, uint64_t n, double lo, double hi, uint8_t *out)
{
    for (uint64_t i = 0; i < n; i++) out[i] = orc_sq_code(x[i], lo, hi);
}

float orc_sq_distance(const uint8_t *a, const uint8_t *b, uint32_t dim)
{
    uint64_t s = 0;
    for (uint32_t i = 0; i < dim; i++) {
        const int64_t d = (int64_t)a[i] - (int64_t)b[i];
        s += (uint64_t)(d * d);
    }
    return (float)s;
}

typedef struct { float d; uint64_t id, pos; } cand;

static int cand_cmp(const void *a, const void *b)
{
    const cand *x = (const cand *)a, *y = (const cand *)b;
    const int xn = x->d != x->d, yn = y->d != y->d;   /* NaN after every number: a strict weak order */
    if (xn != yn) return xn ? 1 : -1;
    if (x->d < y->d) return -1;
    if (x->d > y->d) return 1;
    return x->id < y->id ? -1 : (x->id > y->id ? 1 : 0);
}

static int keep_row(const orc_params *p, uint64_t id, float d)
{
    if (p->allow && (id >= p->allow_bits || !((p->allow[id >> 5] >> (id & 31)) & 1u))) return 0;
    if (p->has_lower && !(d >= p->lower)) return 0;
    if (p->has_upper && !(d < p->upper)) return 0;
    return 1;
}

typedef struct {
    const orc_index *ix;       /* dim, nlist, metric, centroids, part_offsets, row_ids, vectors (codebook unused) */
    const uint8_t *codes;      /* [nrows][dim] */
    double lo, hi;
    const float *queries;
    uint32_t q0, q1;
    const orc_params *p;
    uint64_t *out_ids; float *out_dist; uint32_t *out_count;
    int err;
} job;

static void *worker(void *arg)
{
    job *j = (job *)arg;
    const orc_index *ix = j->ix;
    const orc_params *p = j->p;
    const uint32_t dim = ix->dim, nlist = ix->nlist;
    const uint32_t nprobes = p->nprobes < nlist ? p->nprobes : nlist;
    uint32_t nprobes_max = nprobes;
    if (p->allow && p->max_nprobes > nprobes) nprobes_max = p->max_nprobes < nlist ? p->max_nprobes : nlist;
    const uint32_t kk = p->refine_factor ? p->k * p->refine_factor : p->k;
    float *qn = (float *)malloc(sizeof(float) * (dim ? dim : 1));
    uint8_t *qc = (uint8_t *)malloc(dim ? dim : 1);
    uint32_t *parts = (uint32_t *)malloc(sizeof(uint32_t) * (nlist ? nlist : 1));
    float *pd = (float *)malloc(sizeof(float) * (nlist ? nlist : 1));
    cand *c = (cand *)malloc(sizeof(cand) * (ix->nrows ? ix->nrows : 1));
    if (!qn || !qc || !parts || !pd || !c) { j->err = 1; goto done; }
    for (uint32_t qi = j->q0; qi < j->q1; qi++) {
        const float *q = j->queries + (size_t)qi * dim;
        if (ix->metric == ORC_COSINE) orc_normalize_f32(q, dim, qn);
        else memcpy(qn, q, sizeof(float) * dim);
        orc_sq_encode(qn, dim, j->lo, j->hi, qc);
        uint64_t nc = 0;
        for (uint32_t np_use = nprobes;;) {
            orc_find_partitions(ix, qn, np_use, parts, pd, NULL);
            nc = 0;
            for (uint32_t s = 0; s < np_use; s++) {
                if (pd[s] != pd[s]) continue;
                const uint64_t a = ix->part_offsets[parts[s]], b = ix->part_offsets[parts[s] + 1];
                for (uint64_t r = a; r < b; r++) {
                    const float d = orc_sq_distance(j->codes + r * dim, qc, dim);
                    if (keep_row(p, ix->row_ids[r], d)) { c[nc].d = d; c[nc].id = ix->row_ids[r]; c[nc].pos = r; nc++; }
                }
            }
            if (np_use >= nprobes_max || nc >= p->k) break;
            np_use = nprobes_max;
        }
        qsort(c, nc, sizeof(cand), cand_cmp);
        if (nc > kk) nc = kk;
        if (p->refine_factor && ix->vectors) {
            uint64_t kept = 0;                     /* a NaN exact distance is never returned */
            for (uint64_t i = 0; i < nc; i++) {
                c[kept] = c[i];
                c[kept].d = orc_distance_f32(ix->metric, q, ix->vectors + c[i].pos * dim, dim);
                if (c[kept].d == c[kept].d) kept++;
            }
            nc = kept;
            qsort(c, nc, sizeof(cand), cand_cmp);
        }
        const uint32_t cnt = (uint32_t)(nc < p->k ? nc : p->k);
        for (uint32_t i = 0; i < p->k; i++) {
            j->out_ids[(size_t)qi * p->k + i] = i < cnt ? c[i].id : UINT64_MAX;
            j->out_dist[(size_t)qi * p->k + i] = i < cnt ? c[i].d : INFINITY;
        }
        j->out_count[qi] = cnt;
    }
done:
    free(qn); free(qc); free(parts); free(pd); free(c);
    return NULL;
}

/* ix: the IVF arrays (codebook and codes_t unused); codes [nrows][dim] row codes in partition order */
int orc_sq_search(const orc_index *ix, const uint8_t *codes, double lo, double hi, const float *queries, uint32_t B,
                  const orc_params *p, uint64_t *out_ids, float *out_dist, uint32_t *out_count, int nthreads)
{
    if (!ix || !p || p->k == 0 || ix->dim == 0) return 1;
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > B) nthreads = B ? (int)B : 1;
    job *js = (job *)calloc((size_t)nthreads, sizeof(job));
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    if (!js || !th) { free(js); free(th); return 1; }
    for (int t = 0; t < nthreads; t++) {
        job x = { ix, codes, lo, hi, queries, (uint32_t)((uint64_t)B * t / nthreads),
                  (uint32_t)((uint64_t)B * (t + 1) / nthreads), p, out_ids, out_dist, out_count, 0 };
        js[t] = x;
        if (pthread_create(&th[t], NULL, worker, &js[t]) != 0) { worker(&js[t]); th[t] = 0; }
    }
    int rc = 0;
    for (int t = 0; t < nthreads; t++) {
        if (th[t]) pthread_join(th[t], NULL);
        rc |= js[t].err;
    }
    free(js);
    free(th);
    return rc;
}
