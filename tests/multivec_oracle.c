/* multivec_oracle.c -- CPU oracle of multivector (late-interaction, MaxSim) flat search: the lgpu_multivec_*
 * semantics.
 *
 * A row r holds vectors v_0..v_{n_r-1}, a query q_0..q_{nq-1}.  _distance(q, r) = sum_i min_j cosd(q_i, v_j), the sum
 * over i in order in f32 from 0.0f, cosd = orc_cosine_f32 (the float oracle's lance cosine, oracle/oracle.c, built
 * into this library from that source).  A NaN cosd is skipped by the min; a q_i with no other pair makes the row's
 * distance NaN, and NaN distances are never returned (as the flat path's FilterExec `_distance IS NOT NULL`).
 * orc_params' distance range [lower, upper) and row-id allow bitmap drop rows before the top-k; results ascend by
 * (_distance, _rowid); unused slots are UINT64_MAX / +inf.  Worker threads split the rows.  The NumPy mirror is
 * tests/multivec_oracle.py. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

/* the MaxSim distance of one (query, row) pair */
static float maxsim_distance(const float *q, uint32_t nq, const float *v, uint64_t nr, uint32_t dim)
{
    float s = 0.0f;
    for (uint32_t i = 0; i < nq; i++) {
        float m = NAN;
        for (uint64_t j = 0; j < nr; j++) {
            const float c = orc_cosine_f32(q + (size_t)i * dim, v + j * dim, dim);
            if (c < m || m != m) m = c;                  /* a NaN c never replaces a number */
        }
        s = s + m;
    }
    return s;
}

typedef struct {
    const float *values, *queries;
    const uint64_t *offsets;
    const uint32_t *q_off;
    uint32_t dim, B;
    uint64_t r0, r1, nrows;
    float *out;                 /* [B][nrows] */
} job;

static void *dist_worker(void *arg)
{
    job *j = (job *)arg;
    for (uint64_t r = j->r0; r < j->r1; r++) {
        const float *v = j->values + j->offsets[r] * j->dim;
        const uint64_t nr = j->offsets[r + 1] - j->offsets[r];
        for (uint32_t b = 0; b < j->B; b++)
            j->out[(size_t)b * j->nrows + r] =
                maxsim_distance(j->queries + (size_t)j->q_off[b] * j->dim, j->q_off[b + 1] - j->q_off[b], v, nr, j->dim);
    }
    return NULL;
}

/* out[b][r] = _distance(query b, row r).  values [offsets[nrows]][dim], queries [q_off[B]][dim]. */
int orc_multivec_distances(const float *values, const uint64_t *offsets, uint64_t nrows, uint32_t dim,
                           const float *queries, const uint32_t *q_off, uint32_t B, float *out, int nthreads)
{
    if (nthreads < 1) nthreads = 1;
    if ((uint64_t)nthreads > nrows) nthreads = nrows ? (int)nrows : 1;
    job *js = (job *)calloc((size_t)nthreads, sizeof(job));
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    if (!js || !th) { free(js); free(th); return 1; }
    for (int t = 0; t < nthreads; t++) {
        job p = { values, queries, offsets, q_off, dim, B, nrows * t / nthreads, nrows * (t + 1) / nthreads, nrows, out };
        js[t] = p;
        if (pthread_create(&th[t], NULL, dist_worker, &js[t]) != 0) { dist_worker(&js[t]); th[t] = 0; }
    }
    for (int t = 0; t < nthreads; t++)
        if (th[t]) pthread_join(th[t], NULL);
    free(js);
    free(th);
    return 0;
}

typedef struct { float d; uint64_t id; } cand;

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

/* flat MaxSim search: p->k results per query (k, has_lower/has_upper, allow/allow_bits are used) */
int orc_multivec_search(const float *values, const uint64_t *offsets, uint64_t nrows, uint32_t dim,
                        const uint64_t *row_ids, const float *queries, const uint32_t *q_off, uint32_t B,
                        const orc_params *p, uint64_t *out_ids, float *out_dist, uint32_t *out_count, int nthreads)
{
    if (!p || p->k == 0 || dim == 0) return 1;
    const size_t nd = (size_t)B * nrows;
    float *d = (float *)malloc((nd ? nd : 1) * sizeof(float));
    cand *c = (cand *)malloc((nrows ? nrows : 1) * sizeof(cand));
    if (!d || !c) { free(d); free(c); return 1; }
    int rc = orc_multivec_distances(values, offsets, nrows, dim, queries, q_off, B, d, nthreads);
    for (uint32_t b = 0; b < B && rc == 0; b++) {
        uint64_t nc = 0;
        for (uint64_t r = 0; r < nrows; r++) {
            const uint64_t id = row_ids ? row_ids[r] : r;
            const float x = d[(size_t)b * nrows + r];
            if (keep_row(p, id, x)) { c[nc].d = x; c[nc].id = id; nc++; }
        }
        qsort(c, nc, sizeof(cand), cand_cmp);
        const uint32_t cnt = (uint32_t)(nc < p->k ? nc : p->k);
        for (uint32_t i = 0; i < p->k; i++) {
            out_ids[(size_t)b * p->k + i] = i < cnt ? c[i].id : UINT64_MAX;
            out_dist[(size_t)b * p->k + i] = i < cnt ? c[i].d : INFINITY;
        }
        out_count[b] = cnt;
    }
    free(d);
    free(c);
    return rc;
}
