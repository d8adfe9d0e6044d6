/* rq_oracle.c -- CPU oracle of IVF_RQ search: the lgpu_ivf_rq_open / lgpu_search semantics.
 *
 * Per query (normalised first for cosine, orc_normalize_f32): the nprobes nearest partitions by orc_find_partitions (a
 * partition whose centroid distance is NaN is not probed); the rotated query rq_i = orc_dot_f32(P row i, q) and, per
 * probed partition p, q'_i = rq_i - rc_{p,i} (rc_{p,i} = orc_dot_f32(P row i, c_p)), its 4-bit grid
 *     lo = min q', delta = (max q' - lo) / 15, u_i = min(15, trunc((q'_i - lo) / delta + 0.5)), S = sum u_i,
 * qq = orc_l2_f32(rq, rc_p), and for every row of p, with ip = sum_i b_i u_i and pc = popcount(b),
 *     y = delta * (float)(2 ip - S) + lo * (float)(2 pc - dim),   est = (add + qq) + scale * y,
 * each operation rounded to f32 on its own (this file is built with -ffp-contract=off); _distance = est (l2) or 0.5 est
 * (cosine).  -0 orders below +0 in min and max.  A NaN component of q' makes lo, hi and delta NaN; a slot whose delta is not finite contributes no rows
 * (u is 0 then, as when delta is 0), and a NaN estimate is dropped like a NULL _distance.  distance_range [lower,
 * upper) on the estimate and the row-id allow bitmap drop rows before the top-k; maximum_nprobes (under a prefilter)
 * searches a query again over its max_nprobes nearest partitions when it found fewer than k rows; refine_factor keeps
 * the k * refine_factor best and re-ranks them by orc_distance_f32 on the raw query and the raw vectors.  Results
 * ascend by (_distance, _rowid); unused slots are UINT64_MAX / +inf.  Worker threads split the queries.  The NumPy
 * mirror is tests/rq_oracle.py. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

/* out[v][i] = orc_dot_f32(P row i, x[v]) */
void orc_rq_rotate(const float *P, const float *x, uint64_t n, uint32_t dim, float *out)
{
    for (uint64_t v = 0; v < n; v++)
        for (uint32_t i = 0; i < dim; i++) out[v * dim + i] = orc_dot_f32(P + (size_t)i * dim, x + v * dim, dim);
}

/* one probe slot: u [dim], grid[0..2] = lo, delta, qq, *S */
void orc_rq_slot(const float *rq, const float *rc, uint32_t dim, float *qp, uint8_t *u, float *grid, uint32_t *S)
{
    float lo = INFINITY, hi = -INFINITY;
    int nan = 0;
    for (uint32_t i = 0; i < dim; i++) {
        const float d = rq[i] - rc[i];
        qp[i] = d;
        if (d != d) nan = 1;
        else {                                  /* -0 orders below +0, so the extremes do not depend on the order */
            if (d < lo || (d == lo && signbit(d))) lo = d;
            if (d > hi || (d == hi && !signbit(d))) hi = d;
        }
    }
    if (nan) lo = hi = NAN;
    const float delta = (hi - lo) / 15.0f;
    const int ongrid = delta > 0.0f && isfinite(delta);
    uint32_t s = 0;
    for (uint32_t i = 0; i < dim; i++) {
        uint32_t c = 0;
        if (ongrid) {
            const float f = (qp[i] - lo) / delta + 0.5f;
            c = (uint32_t)f;
            if (c > 15) c = 15;
        }
        u[i] = (uint8_t)c;
        s += c;
    }
    grid[0] = lo; grid[1] = delta; grid[2] = orc_l2_f32(rq, rc, dim);
    *S = s;
}

/* the reported distance of one row (code [ceil(dim / 8)] bytes, LSB first) in a slot */
float orc_rq_estimate(const uint8_t *code, float add, float scale, const uint8_t *u, const float *grid, uint32_t S,
                      uint32_t dim, int metric)
{
    int64_t ip = 0, pc = 0;
    for (uint32_t i = 0; i < dim; i++) {
        const int b = (code[i >> 3] >> (i & 7)) & 1;
        ip += b * u[i];
        pc += b;
    }
    const float t1 = grid[1] * (float)(2 * ip - (int64_t)S);
    const float t2 = grid[0] * (float)(2 * pc - (int64_t)dim);
    const float y = t1 + t2;
    const float a = add + grid[2];
    const float sy = scale * y;
    float est = a + sy;
    if (metric == ORC_COSINE) est = 0.5f * est;
    return isfinite(grid[1]) ? est : NAN;
}

typedef struct { float d; uint64_t id, pos; } cand;

static int cand_cmp(const void *a, const void *b)
{
    const cand *x = (const cand *)a, *y = (const cand *)b;
    if (x->d < y->d) return -1;
    if (x->d > y->d) return 1;
    return x->id < y->id ? -1 : (x->id > y->id ? 1 : 0);
}

static int keep_row(const orc_params *p, uint64_t id, float d)
{
    if (d != d) return 0;
    if (p->allow && (id >= p->allow_bits || !((p->allow[id >> 5] >> (id & 31)) & 1u))) return 0;
    if (p->has_lower && !(d >= p->lower)) return 0;
    if (p->has_upper && !(d < p->upper)) return 0;
    return 1;
}

typedef struct {
    const orc_index *ix;       /* dim, nlist, metric, centroids, part_offsets, row_ids, vectors (codebook unused) */
    const float *P, *rc;       /* [dim][dim], [nlist][dim] */
    const uint8_t *codes;      /* [nrows][ceil(dim / 8)] */
    const float *add, *scale;
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
    const uint32_t dim = ix->dim, nlist = ix->nlist, nb = (dim + 7) / 8;
    const uint32_t nprobes = p->nprobes < nlist ? p->nprobes : nlist;
    uint32_t nprobes_max = nprobes;
    if (p->allow && p->max_nprobes > nprobes) nprobes_max = p->max_nprobes < nlist ? p->max_nprobes : nlist;
    const uint32_t kk = p->refine_factor ? p->k * p->refine_factor : p->k;
    float *qn = (float *)malloc(sizeof(float) * dim), *rq = (float *)malloc(sizeof(float) * dim);
    float *qp = (float *)malloc(sizeof(float) * dim);
    uint8_t *u = (uint8_t *)malloc(dim);
    uint32_t *parts = (uint32_t *)malloc(sizeof(uint32_t) * nlist);
    float *pd = (float *)malloc(sizeof(float) * nlist);
    cand *c = (cand *)malloc(sizeof(cand) * (ix->nrows ? ix->nrows : 1));
    if (!qn || !rq || !qp || !u || !parts || !pd || !c) { j->err = 1; goto done; }
    for (uint32_t qi = j->q0; qi < j->q1; qi++) {
        const float *q = j->queries + (size_t)qi * dim;
        if (ix->metric == ORC_COSINE) orc_normalize_f32(q, dim, qn);
        else memcpy(qn, q, sizeof(float) * dim);
        orc_rq_rotate(j->P, qn, 1, dim, rq);
        uint64_t nc = 0;
        for (uint32_t np_use = nprobes;;) {
            orc_find_partitions(ix, qn, np_use, parts, pd, NULL);
            nc = 0;
            for (uint32_t s = 0; s < np_use; s++) {
                if (pd[s] != pd[s]) continue;
                const uint64_t a = ix->part_offsets[parts[s]], b = ix->part_offsets[parts[s] + 1];
                if (a == b) continue;
                float grid[3];
                uint32_t S;
                orc_rq_slot(rq, j->rc + (size_t)parts[s] * dim, dim, qp, u, grid, &S);
                if (!isfinite(grid[1])) continue;
                for (uint64_t r = a; r < b; r++) {
                    const float d = orc_rq_estimate(j->codes + r * nb, j->add[r], j->scale[r], u, grid, S, dim,
                                                    ix->metric);
                    if (keep_row(p, ix->row_ids[r], d)) { c[nc].d = d; c[nc].id = ix->row_ids[r]; c[nc].pos = r; nc++; }
                }
            }
            if (np_use >= nprobes_max || nc >= p->k) break;
            np_use = nprobes_max;
        }
        qsort(c, nc, sizeof(cand), cand_cmp);
        if (nc > kk) nc = kk;
        if (p->refine_factor && ix->vectors) {
            for (uint64_t i = 0; i < nc; i++) c[i].d = orc_distance_f32(ix->metric, q, ix->vectors + c[i].pos * dim, dim);
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
    free(qn); free(rq); free(qp); free(u); free(parts); free(pd); free(c);
    return NULL;
}

/* ix: the IVF arrays (codebook and codes_t unused); P [dim][dim]; codes [nrows][ceil(dim / 8)], add / scale [nrows]
 * in partition order */
int orc_rq_search(const orc_index *ix, const float *P, const uint8_t *codes, const float *add, const float *scale,
                  const float *queries, uint32_t B, const orc_params *p, uint64_t *out_ids, float *out_dist,
                  uint32_t *out_count, int nthreads)
{
    if (!ix || !p || p->k == 0 || ix->dim == 0 || ix->nlist == 0) return 1;
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > B) nthreads = B ? (int)B : 1;
    float *rc = (float *)malloc(sizeof(float) * ix->nlist * ix->dim);
    job *js = (job *)calloc((size_t)nthreads, sizeof(job));
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    if (!rc || !js || !th) { free(rc); free(js); free(th); return 1; }
    orc_rq_rotate(P, ix->centroids, ix->nlist, ix->dim, rc);
    for (int t = 0; t < nthreads; t++) {
        job x = { ix, P, rc, codes, add, scale, queries, (uint32_t)((uint64_t)B * t / nthreads),
                  (uint32_t)((uint64_t)B * (t + 1) / nthreads), p, out_ids, out_dist, out_count, 0 };
        js[t] = x;
        if (pthread_create(&th[t], NULL, worker, &js[t]) != 0) { worker(&js[t]); th[t] = 0; }
    }
    int rc_ = 0;
    for (int t = 0; t < nthreads; t++) {
        if (th[t]) pthread_join(th[t], NULL);
        rc_ |= js[t].err;
    }
    free(rc);
    free(js);
    free(th);
    return rc_;
}
